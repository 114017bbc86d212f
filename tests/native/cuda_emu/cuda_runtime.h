// A miniature CUDA execution model on host threads -- TEST INFRASTRUCTURE ONLY.
//
// tests/native/build_emu.py compiles the UNMODIFIED product sources (bellman_b200/csrc/*.cu) with
// g++ against this header instead of the CUDA toolkit's <cuda_runtime.h>, after rewriting the two
// pieces of CUDA syntax a host compiler cannot parse (`kernel<<<grid, block, shmem, stream>>>(args)`
// and `extern __shared__ T name[]`).  Every CUDA thread of a block is a user-level fiber,
// __syncthreads() is a barrier between the fibers, warp shuffles exchange through a per-warp
// buffer, "device memory" is the heap, streams and events are synchronous.  Blocks run one after
// another on the calling thread.  This executes the host orchestration and the kernels' index logic of the
// whole MSM / NTT / prover pipeline on a CPU at tiny sizes (tests/test_emulated_pipeline.py); it
// says nothing about what nvcc generates, about memory-model races, or about speed -- the GPU
// parity tests remain the gate.  Nothing in the product build includes this file, and the
// library built from it is never loaded outside tests/.
#pragma once
#include <ucontext.h>

#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <mutex>
#include <type_traits>
#include <utility>
#include <vector>

// ---- qualifiers -------------------------------------------------------------------------------
#define __global__
#define __device__
#define __host__
#define __constant__
#define __forceinline__ inline
#define __noinline__
#define __launch_bounds__(...)
#define __shared__ static

// ---- vector types -----------------------------------------------------------------------------
struct uint3 { unsigned x, y, z; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{x, y, z, w}; }
struct dim3 {
    unsigned x, y, z;
    dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};

// ---- runtime API (synchronous) ----------------------------------------------------------------
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2 };
typedef struct bb_emu_stream* cudaStream_t;
typedef struct bb_emu_event* cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
struct cudaDeviceProp { int multiProcessorCount; char name[64]; };

inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "emulated CUDA error"; }
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int) { p->multiProcessorCount = 2; std::strcpy(p->name, "host-thread emulation"); return cudaSuccess; }
inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
// fresh "device memory" is filled with a poison pattern: real cudaMalloc memory holds whatever the
// previous owner left, so a kernel that relies on zero-initialised buffers must fail here too
inline cudaError_t cudaMalloc(void** p, size_t n) {
    const size_t bytes = (n + 255) & ~size_t(255);
    *p = std::aligned_alloc(256, bytes ? bytes : 256);
    if (!*p) return cudaErrorMemoryAllocation;
    std::memset(*p, 0xCD, bytes ? bytes : 256);
    return cudaSuccess;
}
template <class T> inline cudaError_t cudaMalloc(T** p, size_t n) { return cudaMalloc((void**)p, n); }
inline cudaError_t cudaFree(void* p) { std::free(p); return cudaSuccess; }
inline cudaError_t cudaMallocHost(void** p, size_t n) { return cudaMalloc(p, n); }
inline cudaError_t cudaFreeHost(void* p) { std::free(p); return cudaSuccess; }
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { if (n) std::memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { if (n) std::memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = nullptr) { if (n) std::memset(d, v, n); return cudaSuccess; }
inline cudaError_t cudaMemset2DAsync(void* d, size_t pitch, int v, size_t width, size_t height, cudaStream_t = nullptr) {
    for (size_t r = 0; r < height; r++) std::memset((char*)d + r * pitch, v, width);
    return cudaSuccess;
}
inline cudaError_t cudaMemcpy2DAsync(void* d, size_t dpitch, const void* s, size_t spitch, size_t width, size_t height, cudaMemcpyKind, cudaStream_t = nullptr) {
    for (size_t r = 0; r < height; r++) std::memmove((char*)d + r * dpitch, (const char*)s + r * spitch, width);
    return cudaSuccess;
}
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = (cudaStream_t)std::malloc(8); return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithPriority(cudaStream_t* s, unsigned f, int) { return cudaStreamCreateWithFlags(s, f); }
inline cudaError_t cudaDeviceGetStreamPriorityRange(int* lo, int* hi) { *lo = 0; *hi = -5; return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t s) { std::free(s); return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
enum { cudaEventBlockingSync = 1 };
inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = (cudaEvent_t)std::malloc(8); return cudaSuccess; }
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { return cudaEventCreate(e); }
inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return cudaSuccess; }
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventDestroy(cudaEvent_t e) { std::free(e); return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0.f; return cudaSuccess; }
template <class K> inline cudaError_t cudaFuncSetAttribute(K, int, int) { return cudaSuccess; }

// ---- execution model --------------------------------------------------------------------------
// Kernels without barriers: the threads of a block run one after another on the calling thread.
// Cooperative kernels (__syncthreads / warp shuffles, classified by build_emu.py from the source
// text): every CUDA thread of the block is a user-level fiber (ucontext) on the calling thread; a
// barrier yields to the scheduler, which resumes the fibers round-robin once the barrier's
// generation has advanced.  Deterministic, no OS threads, blocks run one after another.
namespace bb_emu {

struct Barrier {
    unsigned expected = 0, arrived = 0, gen = 0;
    void reset(unsigned n) { expected = n; arrived = 0; }
    inline void wait();
    void drop() {                                   // a thread that returned no longer takes part
        expected--;
        if (expected > 0 && arrived >= expected) { arrived = 0; gen++; }
    }
};

struct Block {
    Barrier bar;
    Barrier warp[32];
    unsigned xchg[1024];
};

struct Fiber {
    ucontext_t ctx;
    bool done = false;
    Barrier* wait_bar = nullptr;
    unsigned wait_gen = 0;
};

struct Idx { unsigned x, y, z; };

struct State {
    Block* block = nullptr;            // non-null while a cooperative kernel runs
    void* dyn_shared = nullptr;
    Fiber* cur = nullptr;
    ucontext_t sched;
    void (*call)(void*) = nullptr;
    void* obj = nullptr;
    std::vector<void*> stacks;
    std::mutex launch_mu;
};
inline State& state() { static State s; return s; }
inline void* dyn_shared() { return state().dyn_shared; }
constexpr size_t STACK_BYTES = 256 * 1024;

}  // namespace bb_emu

inline thread_local bb_emu::Idx threadIdx, blockIdx, blockDim, gridDim;
inline thread_local unsigned bb_emu_tid = 0;          // linear thread index inside the block

namespace bb_emu {

inline void Barrier::wait() {
    if (++arrived >= expected) { arrived = 0; gen++; return; }
    State& S = state();
    Fiber* f = S.cur;
    f->wait_bar = this;
    f->wait_gen = gen;
    swapcontext(&f->ctx, &S.sched);                 // resumed only after gen has advanced
    f->wait_bar = nullptr;
}

inline void fiber_entry() {
    State& S = state();
    S.call(S.obj);
    Fiber* f = S.cur;
    f->done = true;
    S.block->bar.drop();
    S.block->warp[bb_emu_tid >> 5].drop();
    swapcontext(&f->ctx, &S.sched);                 // never resumed
}

template <class Fn>
void launch(bool cooperative, dim3 grid, dim3 block, size_t shmem, cudaStream_t, Fn&& fn) {
    State& S = state();
    std::lock_guard<std::mutex> serial(S.launch_mu);           // one kernel at a time
    const unsigned nt = block.x * block.y * block.z;
    if (nt == 0 || nt > 1024 || (size_t)grid.x * grid.y * grid.z == 0) return;
    const size_t sh_bytes = ((shmem ? shmem : 16) + 127) & ~size_t(127);
    void* sh = std::aligned_alloc(128, sh_bytes);
    std::memset(sh, 0xCD, sh_bytes);                  // shared memory starts uninitialised on the device
    S.dyn_shared = sh;
    blockDim = {block.x, block.y, block.z};
    gridDim = {grid.x, grid.y, grid.z};
    auto set_thread = [&](unsigned t) {
        bb_emu_tid = t;
        threadIdx = {t % block.x, (t / block.x) % block.y, t / (block.x * block.y)};
    };
    Block blk;
    std::vector<Fiber> fib;
    if (cooperative) {
        fib.resize(nt);
        while (S.stacks.size() < nt) S.stacks.push_back(std::aligned_alloc(4096, STACK_BYTES));
        S.call = [](void* o) { (*static_cast<typename std::remove_reference<Fn>::type*>(o))(); };
        S.obj = (void*)&fn;
        S.block = &blk;
    }
    static const bool blocks_reversed = std::getenv("BB_EMU_ORDER") != nullptr;   // blocks must be independent too
    for (unsigned bzi = 0; bzi < grid.z; bzi++)
        for (unsigned byi = 0; byi < grid.y; byi++)
            for (unsigned bxi = 0; bxi < grid.x; bxi++) {
                const unsigned bx = blocks_reversed ? grid.x - 1 - bxi : bxi, by = blocks_reversed ? grid.y - 1 - byi : byi,
                               bz = blocks_reversed ? grid.z - 1 - bzi : bzi;
                blockIdx = {bx, by, bz};
                if (!cooperative) {
                    static const bool rev = std::getenv("BB_EMU_ORDER") != nullptr;
                    for (unsigned t = 0; t < nt; t++) { set_thread(rev ? nt - 1 - t : t); fn(); }
                    continue;
                }
                blk.bar.reset(nt);
                for (unsigned w = 0; w * 32 < nt; w++) blk.warp[w].reset(nt - w * 32 < 32 ? nt - w * 32 : 32);
                for (unsigned t = 0; t < nt; t++) {
                    Fiber& f = fib[t];
                    f.done = false; f.wait_bar = nullptr;
                    getcontext(&f.ctx);
                    f.ctx.uc_stack.ss_sp = S.stacks[t];
                    f.ctx.uc_stack.ss_size = STACK_BYTES;
                    f.ctx.uc_link = nullptr;
                    makecontext(&f.ctx, (void (*)())fiber_entry, 0);
                }
                // BB_EMU_ORDER=reverse|random: resume the fibers in another order between barriers; the
                // results of a correctly synchronised kernel cannot depend on it
                static const int order_mode = [] { const char* e = std::getenv("BB_EMU_ORDER"); return !e ? 0 : e[0] == 'r' && e[1] == 'e' ? 1 : 2; }();
                std::vector<unsigned> order(nt);
                for (unsigned t = 0; t < nt; t++) order[t] = order_mode == 1 ? nt - 1 - t : t;
                if (order_mode == 2) {
                    uint64_t x = 0x9E3779B97F4A7C15ull * (bx + 1) + by * 7919 + bz;
                    for (unsigned t = nt - 1; t > 0; t--) {
                        x = x * 6364136223846793005ull + 1442695040888963407ull;
                        std::swap(order[t], order[(unsigned)((x >> 33) % (t + 1))]);
                    }
                }
                unsigned remaining = nt;
                while (remaining) {
                    bool progress = false;
                    for (unsigned oi = 0; oi < nt; oi++) {
                        const unsigned t = order[oi];
                        Fiber& f = fib[t];
                        if (f.done || (f.wait_bar && f.wait_bar->gen == f.wait_gen)) continue;
                        set_thread(t);
                        S.cur = &f;
                        swapcontext(&S.sched, &f.ctx);
                        progress = true;
                        if (f.done) remaining--;
                    }
                    if (!progress) { std::fprintf(stderr, "cuda_emu: barrier deadlock (divergent __syncthreads?)\n"); std::abort(); }
                }
            }
    S.block = nullptr;
    S.cur = nullptr;
    S.dyn_shared = nullptr;
    std::free(sh);
}

}  // namespace bb_emu

inline void bb_emu_need_block(const char* what) {
    if (!bb_emu::state().block) { std::fprintf(stderr, "cuda_emu: %s in a kernel build_emu.py classified as barrier-free\n", what); std::abort(); }
}

// ---- device builtins --------------------------------------------------------------------------
inline void __syncthreads() { bb_emu_need_block("__syncthreads"); bb_emu::state().block->bar.wait(); }
inline unsigned __shfl_up_sync(unsigned, unsigned v, unsigned d) {
    bb_emu_need_block("__shfl_up_sync");
    bb_emu::Block* b = bb_emu::state().block;
    const unsigned t = bb_emu_tid, lane = t & 31;
    b->xchg[t] = v;
    b->warp[t >> 5].wait();
    unsigned r = lane >= d ? b->xchg[t - d] : v;
    b->warp[t >> 5].wait();
    return r;
}
inline unsigned atomicAdd(unsigned* p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
inline unsigned atomicOr(unsigned* p, unsigned v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
inline unsigned atomicMin(unsigned* p, unsigned v) {
    unsigned old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
    while (old > v && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
    return old;
}
template <class T> inline T __ldg(const T* p) { return *p; }
inline int __popcll(unsigned long long v) { return __builtin_popcountll(v); }
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline int __ffs(int v) { return __builtin_ffs(v); }
// threads run one after another here: each one is alone in its "converged group"
inline unsigned __activemask() { return 1u << (bb_emu_tid & 31u); }
inline unsigned __brev(unsigned v) {
    v = ((v >> 1) & 0x55555555u) | ((v & 0x55555555u) << 1);
    v = ((v >> 2) & 0x33333333u) | ((v & 0x33333333u) << 2);
    v = ((v >> 4) & 0x0f0f0f0fu) | ((v & 0x0f0f0f0fu) << 4);
    return __builtin_bswap32(v);
}
