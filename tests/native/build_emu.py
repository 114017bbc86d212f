"""Builds libbellman_b200_emu.so: the product sources compiled for host threads against
tests/native/cuda_emu/cuda_runtime.h (see that header).  TEST INFRASTRUCTURE ONLY.

The product sources are not modified: copies are rewritten textually where a host compiler cannot
parse CUDA syntax --
    kernel<<<grid, block, shmem, stream>>>(args);   ->  bb_emu::launch(grid, block, shmem, stream, [&] { kernel(args); });
    extern __shared__ T name[];                     ->  T* name = (T*)bb_emu::dyn_shared();
"""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
CSRC = os.path.join(ROOT, "bellman_b200", "csrc")
# the translation units libbellman_b200.so links, in the Makefile's order
SOURCES = re.search(r"^SRCS\s*:=(.*)$", open(os.path.join(CSRC, "Makefile")).read(), re.M).group(1).split()

_KERNEL = re.compile(r"([A-Za-z_]\w*(?:<[^<>();]*>)?)<<<")


def _matching(text, start, open_ch, close_ch):
    depth = 0
    for i in range(start, len(text)):
        if text[i] == open_ch:
            depth += 1
        elif text[i] == close_ch:
            depth -= 1
            if depth == 0:
                return i
    raise ValueError("unbalanced")


_BARRIER = re.compile(r"__syncthreads|__shfl_\w+_sync|__syncwarp")


def _strip_comments(text):
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    return re.sub(r"//[^\n]*", " ", text)


def _function_bodies(text):
    """(name, body) of every function definition `name(params) {`; params may nest parentheses
    one level.  Used only to classify kernels as cooperative or barrier-free."""
    text = _strip_comments(text)
    for m in re.finditer(r"\b([A-Za-z_]\w*)\s*\(((?:[^(){};]|\([^(){};]*\))*)\)\s*(?:const\s*)?\{", text):
        if m.group(1) in ("if", "for", "while", "switch", "catch", "__launch_bounds__"):
            continue
        end = _matching(text, m.end() - 1, "{", "}")
        yield m.group(1), text[m.end():end]


def cooperative_functions(text):
    bodies = list(_function_bodies(text))
    coop = {name for name, body in bodies if _BARRIER.search(body)}
    changed = True
    while changed:                                   # helpers that call a cooperative helper
        changed = False
        for name, body in bodies:
            if name not in coop and any(re.search(r"\b%s\s*(?:<[^;{}()]*>)?\s*\(" % re.escape(c), body) for c in coop):
                coop.add(name)
                changed = True
    return coop


def rewrite(text):
    coop = cooperative_functions(text)
    out, pos, count = [], 0, 0
    while True:
        m = _KERNEL.search(text, pos)
        if not m:
            out.append(text[pos:])
            break
        cfg_end = text.index(">>>", m.end())
        assert text[cfg_end + 3] == "(", text[m.start():cfg_end + 20]
        args_end = _matching(text, cfg_end + 3, "(", ")")
        assert text[args_end + 1] == ";", text[m.start():args_end + 2]
        out.append(text[pos:m.start()])
        kname = m.group(1).split("<")[0]
        is_coop = kname in coop or kname == "kernel"        # `kernel`: a launch through a function parameter
        out.append("bb_emu::launch(%s, %s, [&] { %s(%s); });" % ("true" if is_coop else "false", text[m.end():cfg_end], m.group(1),
                                                                 text[cfg_end + 4:args_end]))
        pos = args_end + 2
        count += 1
    text = "".join(out)
    text = re.sub(r"extern\s+__shared__\s+(\w+)\s+(\w+)\[\];", r"\1* \2 = (\1*)bb_emu::dyn_shared();", text)
    assert "<<<" not in text and "extern __shared__" not in text
    return text, count, sorted(coop)


def build(out_dir, extra_flags=(), emulate_ptx=True):
    """emulate_ptx=False compiles the kernels over mp.cuh's HOST arithmetic path (64-bit CIOS) instead of
    the modelled PTX carry chains: the same pipeline over the other implementation of the field."""
    os.makedirs(out_dir, exist_ok=True)
    objs, launches, procs = [], 0, []
    for name in SOURCES:
        src, n, _ = rewrite(open(os.path.join(CSRC, name)).read())
        launches += n
        cpp = os.path.join(out_dir, name.replace(".cu", "_emu.cpp"))
        with open(cpp, "w") as f:
            f.write(src)
        obj = cpp.replace(".cpp", ".o")
        cmd = ["g++", "-O2", "-std=c++20", "-fPIC", "-pthread", "-w", *(["-DBB_EMULATE_PTX"] if emulate_ptx else []), *extra_flags,
               "-I", os.path.join(ROOT, "tests", "native", "cuda_emu"), "-I", CSRC, "-c", cpp, "-o", obj]
        procs.append((cmd, subprocess.Popen(cmd)))          # the translation units compile side by side
        objs.append(obj)
    for cmd, proc in procs:
        if proc.wait() != 0:
            raise subprocess.CalledProcessError(proc.returncode, cmd)
    lib = os.path.join(out_dir, "libbellman_b200_emu.so")
    subprocess.run(["g++", "-shared", "-pthread", *extra_flags, "-o", lib, *objs], check=True)
    return lib, launches


if __name__ == "__main__":
    for name in SOURCES:
        print(name, "cooperative:", rewrite(open(os.path.join(CSRC, name)).read())[2])
    lib, n = build(sys.argv[1] if len(sys.argv) > 1 else "/tmp/bb_emu")
    print(lib, "kernel launch sites rewritten:", n)
