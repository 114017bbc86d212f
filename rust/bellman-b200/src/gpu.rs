//! Safe layer over `bellman_b200_sys`.  Every item cites the bellman item it stands for
//! (paths relative to the bellman source tree).
use std::any::Any;
use std::ffi::{CStr, CString};
use std::io;
use std::marker::PhantomData;
use std::os::raw::c_void;
use std::ptr;
use std::sync::Arc;

use bellman::groth16::{Parameters, Proof, VerifyingKey};
use bellman::{Circuit, ConstraintSystem, Index, LinearCombination, SynthesisError, VerificationError, Variable};
use bellman_b200_sys::*;
use bls12_381::{Bls12, G1Affine, G1Projective, G2Affine, G2Projective, Scalar};
use ff::{Field, PrimeField};
use group::{prime::PrimeCurveAffine, Curve, UncompressedEncoding};
use rand_core::{CryptoRng, RngCore};

fn last_error() -> String {
    unsafe { CStr::from_ptr(bb_last_error()).to_string_lossy().into_owned() }
}

/// bb_status -> SynthesisError (src/lib.rs:304-319)
fn status(rc: i32) -> Result<(), SynthesisError> {
    match rc {
        BB_OK => Ok(()),
        BB_ERR_POLYNOMIAL_DEGREE_TOO_LARGE => Err(SynthesisError::PolynomialDegreeTooLarge),
        BB_ERR_UNEXPECTED_IDENTITY => Err(SynthesisError::UnexpectedIdentity),
        BB_ERR_IO_UNEXPECTED_EOF => Err(io::Error::new(io::ErrorKind::UnexpectedEof, "expected more bases from source").into()),
        BB_ERR_UNCONSTRAINED_VARIABLE => Err(SynthesisError::UnconstrainedVariable),
        BB_ERR_DENSITY_MISMATCH => panic!("assertion failed: query_size == exponents.len()"), // the assert! of multiexp.rs:324-329
        _ => Err(io::Error::new(io::ErrorKind::Other, last_error()).into()),
    }
}

/// multicore::Worker (src/multicore.rs:21-92): one CUDA device.
pub struct GpuWorker { pub(crate) ctx: *mut bb_ctx }
unsafe impl Send for GpuWorker {}
unsafe impl Sync for GpuWorker {}

impl GpuWorker {
    /// Worker::new().  Fails when no CUDA device is usable: there is no CPU fallback.
    pub fn new(device: i32) -> Result<Self, SynthesisError> {
        let mut ctx = ptr::null_mut();
        status(unsafe { bb_ctx_create(device, &mut ctx) })?;
        Ok(GpuWorker { ctx })
    }
    pub fn set_option(&self, key: &str, value: i64) -> Result<(), SynthesisError> {
        let k = CString::new(key).unwrap();
        status(unsafe { bb_ctx_set_option(self.ctx, k.as_ptr(), value as _) })
    }
}
impl Drop for GpuWorker {
    fn drop(&mut self) { unsafe { bb_ctx_destroy(self.ctx) } }
}

/// Coordinates of an affine point in the ABI's form: little-endian Montgomery limbs, identity = zeros.
/// The uncompressed ZCash encoding is big-endian canonical; bb_fp_convert turns canonical limbs into
/// Montgomery ones, so no private layout of the bls12_381 crate is relied on.
pub trait B200Affine: PrimeCurveAffine + UncompressedEncoding {
    const GROUP: i32;
    const WORDS: usize;          // u64 limbs per point: 12 (G1) / 24 (G2)
    /// order of the 48-byte coordinates inside the uncompressed encoding -> ABI order
    const COORD_ORDER: &'static [usize];
    fn to_b200(&self, out: &mut [u64]) {
        if bool::from(self.is_identity()) { out.iter_mut().for_each(|w| *w = 0); return; }
        let enc = self.to_uncompressed();
        let bytes = enc.as_ref();
        for (k, &src) in Self::COORD_ORDER.iter().enumerate() {
            let be = &bytes[48 * src..48 * (src + 1)];
            for limb in 0..6 {
                let mut w = 0u64;
                for b in 0..8 { w |= (be[47 - (8 * limb + b)] as u64) << (8 * b); }
                out[6 * k + limb] = w;
            }
        }
        // (the three flag bits of byte 0 are clear in the uncompressed encoding of a non-identity point)
        unsafe { bb_fp_convert(out.as_mut_ptr() as *mut c_void, Self::WORDS / 6, 1) };
    }
    fn from_b200(words: &[u64]) -> Self {
        if words.iter().all(|w| *w == 0) { return Self::identity(); }
        let mut w = words.to_vec();
        unsafe { bb_fp_convert(w.as_mut_ptr() as *mut c_void, Self::WORDS / 6, 0) };
        let mut enc = Self::Uncompressed::default();
        {
            let bytes = enc.as_mut();
            for (k, &dst) in Self::COORD_ORDER.iter().enumerate() {
                for limb in 0..6 {
                    for b in 0..8 { bytes[48 * dst + 47 - (8 * limb + b)] = (w[6 * k + limb] >> (8 * b)) as u8; }
                }
            }
        }
        Option::from(Self::from_uncompressed_unchecked(&enc)).expect("device returned a valid encoding")
    }
}
impl B200Affine for G1Affine { const GROUP: i32 = BB_G1; const WORDS: usize = 12; const COORD_ORDER: &'static [usize] = &[0, 1]; }
// uncompressed G2: x.c1 | x.c0 | y.c1 | y.c0; ABI: x.c0 | x.c1 | y.c0 | y.c1
impl B200Affine for G2Affine { const GROUP: i32 = BB_G2; const WORDS: usize = 24; const COORD_ORDER: &'static [usize] = &[1, 0, 3, 2]; }

/// Device-resident `Arc<Vec<G::Affine>>` (groth16/src/lib.rs:227-243), uploaded once per key.
pub struct GpuBases<A: B200Affine> { pub(crate) handle: *mut bb_bases, _a: PhantomData<A> }
unsafe impl<A: B200Affine> Send for GpuBases<A> {}
unsafe impl<A: B200Affine> Sync for GpuBases<A> {}

impl<A: B200Affine> GpuBases<A> {
    pub fn upload(worker: &GpuWorker, points: &[A]) -> Result<Self, SynthesisError> {
        let mut flat = vec![0u64; points.len() * A::WORDS];
        for (p, out) in points.iter().zip(flat.chunks_mut(A::WORDS)) { p.to_b200(out); }
        let mut handle = ptr::null_mut();
        status(unsafe { bb_bases_upload(worker.ctx, A::GROUP, flat.as_ptr() as *const c_void, points.len(), 0, points.len(), &mut handle) })?;
        Ok(GpuBases { handle, _a: PhantomData })
    }
}
impl<A: B200Affine> Drop for GpuBases<A> {
    fn drop(&mut self) { unsafe { bb_bases_free(self.handle) } }
}

/// `DensityTracker { bv: BitVec }` / `FullDensity` (src/multiexp.rs:88-157) as the ABI wants it:
/// raw LSB-first words and the length in bits; `FullDensity` is (null, 0).
pub trait DensityWords { fn raw_words(&self) -> (*const u64, usize); }
pub struct FullDensity;
impl DensityWords for FullDensity { fn raw_words(&self) -> (*const u64, usize) { (ptr::null(), 0) } }
impl DensityWords for bitvec::vec::BitVec<usize, bitvec::order::Lsb0> {
    fn raw_words(&self) -> (*const u64, usize) { (self.as_raw_slice().as_ptr() as *const u64, self.len()) }   // 64-bit targets
}

/// `Waiter<Result<G, SynthesisError>>` (src/multicore.rs:94-118)
pub struct GpuWaiter<A: B200Affine> { job: *mut bb_msm_job, _keep: (Arc<dyn Any + Send + Sync>, Arc<dyn Any + Send + Sync>), _a: PhantomData<A> }

impl<A: B200Affine> GpuWaiter<A> {
    /// Waiter::wait (src/multicore.rs:98-108): blocks on the job's CUDA stream, folds, returns the point.
    pub fn wait(self) -> Result<A::Curve, SynthesisError> {
        let mut out = vec![0u64; A::WORDS];
        status(unsafe { bb_msm_wait(self.job, out.as_mut_ptr() as *mut c_void) })?;
        Ok(A::from_b200(&out).to_curve())
    }
}

/// Drop-in for `bellman::multiexp::multiexp` (src/multiexp.rs:305-332).  `exponents` are the canonical
/// little-endian integers `Exponent::Bits` wraps (`to_le_bits`, :179); zero and one need no special
/// casing, the kernels classify them (`Exponent::Zero` / `Exponent::One`, :172-182).
pub fn multiexp<A, D>(pool: &GpuWorker, bases: (Arc<GpuBases<A>>, usize), density_map: &D, exponents: Arc<Vec<[u64; 4]>>) -> GpuWaiter<A>
where A: B200Affine + 'static, D: DensityWords {
    let (words, len) = density_map.raw_words();
    let mut job = ptr::null_mut();
    let rc = unsafe {
        bb_msm_async(pool.ctx, bases.0.handle, bases.1, words, len, exponents.as_ptr() as *const c_void, exponents.len(),
                     BB_FORM_CANONICAL, &mut job)
    };
    assert_eq!(rc, BB_OK, "{}", last_error());                 // argument errors only; run-time errors surface in wait()
    GpuWaiter { job, _keep: (bases.0, exponents), _a: PhantomData }
}

/// EvaluationDomain::{fft, ifft, coset_fft, icoset_fft} (src/domain.rs:81-125) in place on `coeffs`
/// (length 2^log_n, the in-memory `Scalar`s are passed through their canonical representation).
pub fn ntt(pool: &GpuWorker, coeffs: &mut [Scalar], log_n: u32, mode: i32) -> Result<(), SynthesisError> {
    assert_eq!(coeffs.len(), 1usize << log_n);
    let mut flat: Vec<[u8; 32]> = coeffs.iter().map(|s| s.to_repr()).collect();
    status(unsafe { bb_ntt(pool.ctx, flat.as_mut_ptr() as *mut c_void, log_n, mode, BB_FORM_CANONICAL) })?;
    for (c, r) in coeffs.iter_mut().zip(flat.iter()) { *c = Option::from(Scalar::from_repr(*r)).expect("canonical output"); }
    Ok(())
}

/// Device-resident `groth16::Parameters` (groth16/src/lib.rs:222-244).
pub struct GpuParameters { pub(crate) ctx: *mut bb_ctx, pub(crate) handle: *mut bb_crs }
unsafe impl Send for GpuParameters {}
unsafe impl Sync for GpuParameters {}

impl GpuParameters {
    pub fn upload(worker: &GpuWorker, p: &Parameters<Bls12>) -> Result<Self, SynthesisError> {
        fn flat<A: B200Affine>(v: &[A]) -> Vec<u64> {
            let mut f = vec![0u64; v.len() * A::WORDS];
            for (p, out) in v.iter().zip(f.chunks_mut(A::WORDS)) { p.to_b200(out); }
            f
        }
        let (alpha, beta1, delta1) = (flat(&[p.vk.alpha_g1]), flat(&[p.vk.beta_g1]), flat(&[p.vk.delta_g1]));
        let (beta2, delta2) = (flat(&[p.vk.beta_g2]), flat(&[p.vk.delta_g2]));
        let (h, l, a, b1, b2) = (flat(&p.h[..]), flat(&p.l[..]), flat(&p.a[..]), flat(&p.b_g1[..]), flat(&p.b_g2[..]));
        let desc = bb_crs_desc {
            alpha_g1: alpha.as_ptr() as _, beta_g1: beta1.as_ptr() as _, delta_g1: delta1.as_ptr() as _,
            beta_g2: beta2.as_ptr() as _, delta_g2: delta2.as_ptr() as _,
            h: h.as_ptr() as _, h_len: p.h.len(), l: l.as_ptr() as _, l_len: p.l.len(), a: a.as_ptr() as _, a_len: p.a.len(),
            b_g1: b1.as_ptr() as _, b_g1_len: p.b_g1.len(), b_g2: b2.as_ptr() as _, b_g2_len: p.b_g2.len(),
            shard_index: 0, shard_count: 1,
        };
        let mut handle = ptr::null_mut();
        status(unsafe { bb_crs_create(worker.ctx, &desc, &mut handle) })?;
        Ok(GpuParameters { ctx: worker.ctx, handle })
    }
}
impl Drop for GpuParameters {
    fn drop(&mut self) { unsafe { bb_crs_destroy(self.handle) } }
}

/// The io::Error `Parameters::read` / `VerifyingKey::read` (groth16/src/lib.rs:158-218, 289-398) return for a status of
/// bb_params_read / bb_vk_read: InvalidData with the reference's text ("invalid G1", "invalid G2", "point at infinity"),
/// UnexpectedEof, or Other for a back-end failure (its message)
fn params_read_error(rc: i32, rep: &bb_params_report) -> io::Error {
    match rc {
        BB_ERR_IO_INVALID_DATA => {
            let g2 = [BB_PARAMS_BETA_G2, BB_PARAMS_GAMMA_G2, BB_PARAMS_DELTA_G2, BB_PARAMS_B_G2].contains(&rep.section);
            let msg = if rep.why == BB_READ_IDENTITY as i32 { "point at infinity" } else if g2 { "invalid G2" } else { "invalid G1" };
            io::Error::new(io::ErrorKind::InvalidData, msg)
        }
        BB_ERR_IO_UNEXPECTED_EOF => io::Error::new(io::ErrorKind::UnexpectedEof, "failed to fill whole buffer"),
        _ => io::Error::new(io::ErrorKind::Other, last_error()),
    }
}

impl GpuParameters {
    /// `Parameters::read(bytes, checked)` on the device: the file is decoded and checked there, straight into the resident
    /// key (bb_params_read), with no `Parameters<Bls12>` on the host.  Same acceptance rules and the same first error as the
    /// reference.  A caller that also needs the host `VerifyingKey` reads it with `VerifyingKey::read` from the same bytes.
    pub fn read(worker: &GpuWorker, bytes: &[u8], checked: bool) -> io::Result<GpuParameters> {
        let (mut handle, mut rep) = (ptr::null_mut(), bb_params_report::default());
        let rc = unsafe {
            bb_params_read(worker.ctx, bytes.as_ptr() as _, bytes.len(), 0, checked as i32, &mut handle, ptr::null_mut(), &mut rep)
        };
        if rc != BB_OK { return Err(params_read_error(rc, &rep)); }
        Ok(GpuParameters { ctx: worker.ctx, handle })
    }
}

/// What `ProvingAssignment` holds when synthesis is done (groth16/src/prover.rs:57-71,193-215); the fields
/// are private upstream, so the `b200` feature exposes them to this module (`pub(crate)` in-tree).
pub struct WitnessView<'a> {
    pub a: &'a [Scalar], pub b: &'a [Scalar], pub c: &'a [Scalar],
    pub input_assignment: &'a [Scalar], pub aux_assignment: &'a [Scalar],
    pub a_aux_density: &'a bitvec::vec::BitVec<usize, bitvec::order::Lsb0>,
    pub b_input_density: &'a bitvec::vec::BitVec<usize, bitvec::order::Lsb0>,
    pub b_aux_density: &'a bitvec::vec::BitVec<usize, bitvec::order::Lsb0>,
}

impl<'a> WitnessView<'a> {
    fn as_ffi(&self) -> bb_witness {
        const _: () = assert!(std::mem::size_of::<Scalar>() == 32);
        bb_witness {
            a: self.a.as_ptr() as _, b: self.b.as_ptr() as _, c: self.c.as_ptr() as _, n_constraints: self.a.len(),
            input_assignment: self.input_assignment.as_ptr() as _, n_inputs: self.input_assignment.len(),
            aux_assignment: self.aux_assignment.as_ptr() as _, n_aux: self.aux_assignment.len(),
            a_aux_density: self.a_aux_density.as_raw_slice().as_ptr() as _,
            b_input_density: self.b_input_density.as_raw_slice().as_ptr() as _,
            b_aux_density: self.b_aux_density.as_raw_slice().as_ptr() as _,
            on_device: 0,
        }
    }
}

impl GpuParameters {
    /// Once per key (a key serves many proofs): proves `w` with every MSM form of the back-end on this device and
    /// leaves the key configured for the fastest form whose partial sums are byte-identical to the default form's
    /// (`bb_groth16_autotune`).  Returns the index chosen and the milliseconds measured per form.
    pub fn autotune(&mut self, w: &WitnessView, reps: i32) -> Result<(usize, Vec<f64>), SynthesisError> {
        let n = unsafe { bb_tuning_count() } as usize;
        let mut ms = vec![0f64; n];
        let mut chosen = 0i32;
        let wit = w.as_ffi();
        status(unsafe { bb_groth16_autotune(self.ctx, self.handle, &wit, reps, &mut chosen, ms.as_mut_ptr()) })?;
        Ok((chosen as usize, ms))
    }
}

/// The constraint system on the device (bb_r1cs_*): the A, B, C matrices of a circuit kept in HBM beside the key, so that
/// a proof needs only the witness -- `ProvingAssignment::enforce` (groth16/src/prover.rs:105-145) is never run.
pub struct GpuR1cs { pub(crate) ctx: *mut bb_ctx, pub(crate) handle: *mut bb_r1cs, n_inputs: usize, n_aux: usize }
unsafe impl Send for GpuR1cs {}
unsafe impl Sync for GpuR1cs {}

/// Records what `KeypairAssembly` records (generator.rs:43-155), by constraint: each row's terms as the circuit pushed
/// them, unmerged.  The witness closures are not called.

struct R1csRecorder { n_inputs: usize, n_aux: usize, rows: usize, m: [(Vec<u64>, Vec<Index>, Vec<Scalar>); 3] }
impl ConstraintSystem<Scalar> for R1csRecorder {
    type Root = Self;
    fn alloc<F, A, AR>(&mut self, _: A, _: F) -> Result<Variable, SynthesisError>
    where F: FnOnce() -> Result<Scalar, SynthesisError>, A: FnOnce() -> AR, AR: Into<String> {
        self.n_aux += 1;
        Ok(Variable::new_unchecked(Index::Aux(self.n_aux - 1)))
    }
    fn alloc_input<F, A, AR>(&mut self, _: A, _: F) -> Result<Variable, SynthesisError>
    where F: FnOnce() -> Result<Scalar, SynthesisError>, A: FnOnce() -> AR, AR: Into<String> {
        self.n_inputs += 1;
        Ok(Variable::new_unchecked(Index::Input(self.n_inputs - 1)))
    }
    fn enforce<A, AR, LA, LB, LC>(&mut self, _: A, a: LA, b: LB, c: LC)
    where A: FnOnce() -> AR, AR: Into<String>, LA: FnOnce(LinearCombination<Scalar>) -> LinearCombination<Scalar>,
          LB: FnOnce(LinearCombination<Scalar>) -> LinearCombination<Scalar>, LC: FnOnce(LinearCombination<Scalar>) -> LinearCombination<Scalar> {
        let lcs = [a(LinearCombination::zero()), b(LinearCombination::zero()), c(LinearCombination::zero())];
        for (lc, m) in lcs.iter().zip(self.m.iter_mut()) {
            for (v, coeff) in lc.as_ref() {
                m.1.push(v.get_unchecked());
                m.2.push(*coeff);
            }
            m.0.push(m.1.len() as u64);
        }
        self.rows += 1;
    }
    fn push_namespace<NR, N>(&mut self, _: N) where NR: Into<String>, N: FnOnce() -> NR {}
    fn pop_namespace(&mut self) {}
    fn get_root(&mut self) -> &mut Self::Root { self }
}

/// Runs the `alloc` / `alloc_input` closures of a circuit and never the `enforce` closures: the witness alone.
#[derive(Default)]
pub struct WitnessCS { pub input_assignment: Vec<Scalar>, pub aux_assignment: Vec<Scalar> }

impl ConstraintSystem<Scalar> for WitnessCS {
    type Root = Self;
    fn alloc<F, A, AR>(&mut self, _: A, f: F) -> Result<Variable, SynthesisError>
    where F: FnOnce() -> Result<Scalar, SynthesisError>, A: FnOnce() -> AR, AR: Into<String> {
        self.aux_assignment.push(f()?);
        Ok(Variable::new_unchecked(Index::Aux(self.aux_assignment.len() - 1)))
    }
    fn alloc_input<F, A, AR>(&mut self, _: A, f: F) -> Result<Variable, SynthesisError>
    where F: FnOnce() -> Result<Scalar, SynthesisError>, A: FnOnce() -> AR, AR: Into<String> {
        self.input_assignment.push(f()?);
        Ok(Variable::new_unchecked(Index::Input(self.input_assignment.len() - 1)))
    }
    fn enforce<A, AR, LA, LB, LC>(&mut self, _: A, _: LA, _: LB, _: LC)
    where A: FnOnce() -> AR, AR: Into<String>, LA: FnOnce(LinearCombination<Scalar>) -> LinearCombination<Scalar>,
          LB: FnOnce(LinearCombination<Scalar>) -> LinearCombination<Scalar>, LC: FnOnce(LinearCombination<Scalar>) -> LinearCombination<Scalar> {}
    fn push_namespace<NR, N>(&mut self, _: N) where NR: Into<String>, N: FnOnce() -> NR {}
    fn pop_namespace(&mut self) {}
    fn get_root(&mut self) -> &mut Self::Root { self }
}

impl GpuR1cs {
    /// Synthesises `circuit` once for its shape (after `alloc_input(ONE)`, as prover.rs:204-206 and generator.rs:188 do)
    /// and uploads the matrices.  The input rows are appended by the library.  The shape must not depend on witness
    /// values -- which R1CS already requires, since the key is made from one synthesis too.
    pub fn synthesize<C: Circuit<Scalar>>(worker: &GpuWorker, circuit: C) -> Result<Self, SynthesisError> {
        let mut cs = R1csRecorder { n_inputs: 0, n_aux: 0, rows: 0, m: Default::default() };
        for m in cs.m.iter_mut() { m.0.push(0); }
        cs.alloc_input(|| "", || Ok(Scalar::one()))?;
        circuit.synthesize(&mut cs)?;
        let (ni, na) = (cs.n_inputs, cs.n_aux);
        // variables as the ABI numbers them: inputs first, then aux (an index too large for u32 is left to bb_r1cs_create)
        let vars: Vec<Vec<u32>> = cs.m.iter()
            .map(|m| m.1.iter().map(|v| match v { Index::Input(i) => *i as u32, Index::Aux(i) => (ni + i).min(u32::MAX as usize) as u32 }).collect())
            .collect();
        let mat = |k: usize| bb_r1cs_matrix {
            row_offsets: cs.m[k].0.as_ptr(), vars: vars[k].as_ptr(), coeffs: cs.m[k].2.as_ptr() as *const c_void,   // Scalar = Montgomery limbs
        };
        let desc = bb_r1cs_desc { a: mat(0), b: mat(1), c: mat(2), n_constraints: cs.rows, n_inputs: ni, n_aux: na };
        let mut handle = ptr::null_mut();
        status(unsafe { bb_r1cs_create(worker.ctx, &desc, &mut handle) })?;
        Ok(GpuR1cs { ctx: worker.ctx, handle, n_inputs: ni, n_aux: na })
    }

    /// `TestConstraintSystem::which_is_unsatisfied` (src/gadgets/test/mod.rs:254-267) on the device (bb_r1cs_check): the
    /// index of the first constraint with <A_k,z> <B_k,z> != <C_k,z> for the witness `WitnessCS` collects (input 0 = ONE
    /// included), or None.  Constraints have no names here; the index is the enforce order.
    pub fn which_is_unsatisfied(&self, input_assignment: &[Scalar], aux_assignment: &[Scalar]) -> Result<Option<usize>, SynthesisError> {
        let (mut first, mut count) = (0usize, 0usize);
        status(unsafe {
            bb_r1cs_check(self.ctx, self.handle, input_assignment.as_ptr() as _, input_assignment.len(), aux_assignment.as_ptr() as _,
                          aux_assignment.len(), 0, &mut first, &mut count, ptr::null_mut())
        })?;
        Ok(if first == usize::MAX { None } else { Some(first) })
    }

    /// `TestConstraintSystem::is_satisfied` (src/gadgets/test/mod.rs:269-272) on the device
    pub fn is_satisfied(&self, input_assignment: &[Scalar], aux_assignment: &[Scalar]) -> Result<bool, SynthesisError> {
        Ok(self.which_is_unsatisfied(input_assignment, aux_assignment)?.is_none())
    }
}
impl Drop for GpuR1cs {
    fn drop(&mut self) { unsafe { bb_r1cs_destroy(self.handle) } }
}

/// `groth16::create_proof` (groth16/src/prover.rs:182-360) with the constraint system on the device: synthesis runs only
/// the witness closures (`WitnessCS`); a, b, c and the densities are computed from `r1cs` on the device.  The same bytes
/// as `create_proof_b200` on the `ProvingAssignment` bellman's synthesis would build.
pub fn create_proof_r1cs_b200<C: Circuit<Scalar>>(circuit: C, r1cs: &GpuR1cs, crs: &GpuParameters, r: Scalar, s: Scalar)
    -> Result<Proof<Bls12>, SynthesisError> {
    let mut cs = WitnessCS::default();
    cs.alloc_input(|| "", || Ok(Scalar::one()))?;
    circuit.synthesize(&mut cs)?;
    assert_eq!((cs.input_assignment.len(), cs.aux_assignment.len()), (r1cs.n_inputs, r1cs.n_aux), "the circuit's shape changed");
    let mut bytes = [0u8; 192];
    status(unsafe {
        bb_groth16_prove_r1cs(crs.ctx, crs.handle, r1cs.handle, cs.input_assignment.as_ptr() as _, cs.input_assignment.len(),
                              cs.aux_assignment.as_ptr() as _, cs.aux_assignment.len(), 0, r.to_repr().as_ptr(), s.to_repr().as_ptr(),
                              bytes.as_mut_ptr())
    })?;
    Proof::read(&bytes[..]).map_err(Into::into)
}

/// One rank's part of a proof from the witness on a sharded key (bb_groth16_prove_r1cs_begin): `begin` uploads the witness
/// once and, for every polynomial whose bit is set in `own` (1 = a, 2 = b, 4 = c), evaluates its matrix straight into
/// `d_evals[i]` (m Fr, device) and takes it through ifft + coset_fft, ahead of this shard's seven witness MSMs.  After
/// `bb_h_coset_evals_wait` and the broadcast of the owners' vectors, `end` runs the last transform, the h MSM and the
/// waits and returns the 960-byte partial sums for `bb_groth16_finalize`.  `d_evals = None` (own = 0) runs the whole H
/// pipeline on this rank; `end(None)` finishes it.
pub struct GpuR1csProof { handle: *mut bb_prove }
unsafe impl Send for GpuR1csProof {}

impl GpuR1cs {
    /// # Safety
    /// `input_assignment` and `aux_assignment` must stay alive and unchanged until the returned state is ended or
    /// dropped: the library reads them asynchronously.  Every `d_evals[i]` with bit `1 << i` set in `own`, and all three
    /// given to `end`, must be device allocations of m Fr (m = the next power of two >= the constraints), 16-byte
    /// aligned, of this worker's device, not read or written by anything else until `bb_h_coset_evals_wait` returns (an
    /// owned one) or `end` returns; the library writes the owned ones and overwrites the first one given to `end`.
    pub unsafe fn begin(&self, crs: &GpuParameters, input_assignment: &[Scalar], aux_assignment: &[Scalar], own: u32,
                 d_evals: Option<[*mut c_void; 3]>) -> Result<GpuR1csProof, SynthesisError> {
        let mut handle = ptr::null_mut();
        let evals = d_evals.as_ref().map_or(ptr::null(), |e| e.as_ptr());
        status(unsafe {
            bb_groth16_prove_r1cs_begin(crs.ctx, crs.handle, self.handle, input_assignment.as_ptr() as _, input_assignment.len(),
                                        aux_assignment.as_ptr() as _, aux_assignment.len(), 0, own, evals, &mut handle)
        })?;
        Ok(GpuR1csProof { handle })
    }
}

impl GpuR1csProof {
    /// # Safety
    /// The three vectors must be valid as `GpuR1cs::begin` requires.
    pub unsafe fn end(mut self, d_evals: Option<[*const c_void; 3]>) -> Result<[u8; 960], SynthesisError> {
        let mut partials = [0u8; 960];
        let [a, b, c] = d_evals.unwrap_or([ptr::null(); 3]);
        let handle = std::mem::replace(&mut self.handle, ptr::null_mut());
        status(unsafe { bb_groth16_prove_end(handle, a, b, c, partials.as_mut_ptr()) })?;     // frees the state, also on an error
        Ok(partials)
    }
}
impl Drop for GpuR1csProof {
    fn drop(&mut self) {                                       // never ended: drain and free (with vectors or without, one is refused)
        if !self.handle.is_null() {
            let mut partials = [0u8; 960];
            unsafe { bb_groth16_prove_end(self.handle, ptr::null(), ptr::null(), ptr::null(), partials.as_mut_ptr()) };
        }
    }
}

/// Drop-in for the body of `groth16::create_proof` after synthesis (groth16/src/prover.rs:217-360).
/// `Scalar` is `[u64; 4]` in Montgomery form (R = 2^256), which is BB_FORM_MONTGOMERY byte for byte; the
/// cast below is version-pinned (`bls12_381 = "=0.8.0"`) because `#[repr(transparent)]` is not promised.
pub fn create_proof_b200(w: &WitnessView, crs: &GpuParameters, r: Scalar, s: Scalar) -> Result<Proof<Bls12>, SynthesisError> {
    let wit = w.as_ffi();
    let mut bytes = [0u8; 192];
    status(unsafe { bb_groth16_prove(crs.ctx, crs.handle, &wit, r.to_repr().as_ptr(), s.to_repr().as_ptr(), bytes.as_mut_ptr()) })?;
    Proof::read(&bytes[..]).map_err(Into::into)               // the same 192 bytes Proof::write emits (lib.rs:39-45)
}

/// `create_proof_b200` for many witnesses of ONE circuit in one call (bb_groth16_prove_batch): one result per item, each
/// exactly what `create_proof_b200` returns for that item alone.  `Err` only when the call itself was refused (witnesses of
/// different shapes, a sharded key).
pub fn create_proof_batch_b200(ws: &[WitnessView], crs: &GpuParameters, rs: &[Scalar], ss: &[Scalar])
    -> Result<Vec<Result<Proof<Bls12>, SynthesisError>>, SynthesisError> {
    assert!(rs.len() == ws.len() && ss.len() == ws.len(), "one r and one s per witness");
    let wit: Vec<_> = ws.iter().map(|w| w.as_ffi()).collect();
    batch_results(ws.len(), rs, ss, |r, s, proofs, st| unsafe {
        bb_groth16_prove_batch(crs.ctx, crs.handle, wit.as_ptr(), ws.len(), r, s, proofs, st)
    })
}

/// `create_proof_r1cs_b200` for many circuits of one shape (bb_groth16_prove_r1cs_batch): every circuit is synthesised
/// with `WitnessCS` and the witnesses are proved in one call; one result per circuit.
pub fn create_proof_r1cs_batch_b200<C: Circuit<Scalar>>(circuits: Vec<C>, r1cs: &GpuR1cs, crs: &GpuParameters, rs: &[Scalar], ss: &[Scalar])
    -> Result<Vec<Result<Proof<Bls12>, SynthesisError>>, SynthesisError> {
    let count = circuits.len();
    assert!(rs.len() == count && ss.len() == count, "one r and one s per circuit");
    let (mut inputs, mut aux) = (Vec::with_capacity(count * r1cs.n_inputs), Vec::with_capacity(count * r1cs.n_aux));
    for circuit in circuits {
        let mut cs = WitnessCS::default();
        cs.alloc_input(|| "", || Ok(Scalar::one()))?;
        circuit.synthesize(&mut cs)?;
        assert_eq!((cs.input_assignment.len(), cs.aux_assignment.len()), (r1cs.n_inputs, r1cs.n_aux), "the circuit's shape changed");
        inputs.extend(cs.input_assignment);
        aux.extend(cs.aux_assignment);
    }
    batch_results(count, rs, ss, |r, s, proofs, st| unsafe {
        bb_groth16_prove_r1cs_batch(crs.ctx, crs.handle, r1cs.handle, inputs.as_ptr() as _, r1cs.n_inputs, aux.as_ptr() as _, r1cs.n_aux,
                                    count, 0, r, s, proofs, st)
    })
}

/// the per-item statuses and 192-byte records of a batch call -> one `Result` per item
fn batch_results(count: usize, rs: &[Scalar], ss: &[Scalar], call: impl FnOnce(*const u8, *const u8, *mut u8, *mut i32) -> i32)
    -> Result<Vec<Result<Proof<Bls12>, SynthesisError>>, SynthesisError> {
    let r: Vec<u8> = rs.iter().flat_map(|v| v.to_repr()).collect();
    let s: Vec<u8> = ss.iter().flat_map(|v| v.to_repr()).collect();
    let mut bytes = vec![0u8; 192 * count];
    let mut st = vec![0i32; count];
    status(call(r.as_ptr(), s.as_ptr(), bytes.as_mut_ptr(), st.as_mut_ptr()))?;
    Ok(st.iter().zip(bytes.chunks(192))
        .map(|(&rc, b)| status(rc).and_then(|_| Proof::read(b).map_err(Into::into)))
        .collect())
}

/// `PreparedVerifyingKey` (groth16/src/lib.rs:400-409, verifier.rs:11-21): the verifying key resident on the device.
pub struct GpuVerifyingKey { pub(crate) ctx: *mut bb_ctx, pub(crate) handle: *mut bb_vk, pub(crate) ic_len: usize }
unsafe impl Send for GpuVerifyingKey {}
unsafe impl Sync for GpuVerifyingKey {}

fn flat<A: B200Affine>(v: &[A]) -> Vec<u64> {
    let mut f = vec![0u64; v.len() * A::WORDS];
    for (p, out) in v.iter().zip(f.chunks_mut(A::WORDS)) { p.to_b200(out); }
    f
}

/// bb_status of the verifier -> VerificationError (src/lib.rs:353-358); other statuses are back-end failures
fn verification_status(rc: i32) -> Result<(), VerificationError> {
    match rc {
        BB_OK => Ok(()),
        BB_ERR_INVALID_VERIFYING_KEY => Err(VerificationError::InvalidVerifyingKey),
        BB_ERR_INVALID_PROOF => Err(VerificationError::InvalidProof),
        _ => panic!("bellman_b200 verifier failed: {}", last_error()),
    }
}

impl GpuVerifyingKey {
    /// prepare_verifying_key (verifier.rs:11-21)
    pub fn prepare(worker: &GpuWorker, vk: &VerifyingKey<Bls12>) -> Result<Self, SynthesisError> {
        let (alpha, beta, gamma, delta) = (flat(&[vk.alpha_g1]), flat(&[vk.beta_g2]), flat(&[vk.gamma_g2]), flat(&[vk.delta_g2]));
        let ic = flat(&vk.ic[..]);
        let desc = bb_vk_desc {
            alpha_g1: alpha.as_ptr() as _, beta_g2: beta.as_ptr() as _, gamma_g2: gamma.as_ptr() as _, delta_g2: delta.as_ptr() as _,
            ic: ic.as_ptr() as _, ic_len: vk.ic.len(),
        };
        let mut handle = ptr::null_mut();
        status(unsafe { bb_vk_prepare(worker.ctx, &desc, &mut handle) })?;
        Ok(GpuVerifyingKey { ctx: worker.ctx, handle, ic_len: vk.ic.len() })
    }
}
impl GpuVerifyingKey {
    /// `VerifyingKey::read(bytes)` + prepare_verifying_key on the device (bb_vk_read), and the bytes it consumed
    /// (868 + 96 |ic|); a Parameters file starts with its VerifyingKey
    pub fn read(worker: &GpuWorker, bytes: &[u8]) -> io::Result<(GpuVerifyingKey, usize)> {
        let (mut handle, mut rep) = (ptr::null_mut(), bb_params_report::default());
        let rc = unsafe { bb_vk_read(worker.ctx, bytes.as_ptr() as _, bytes.len(), 0, &mut handle, &mut rep) };
        if rc != BB_OK { return Err(params_read_error(rc, &rep)); }
        Ok((GpuVerifyingKey { ctx: worker.ctx, handle, ic_len: rep.len[0] }, rep.consumed))
    }
}
impl Drop for GpuVerifyingKey {
    fn drop(&mut self) { unsafe { bb_vk_destroy(self.handle) } }
}

/// Drop-in for `groth16::verify_proof` (verifier.rs:23-58).
pub fn verify_proof_b200(pvk: &GpuVerifyingKey, proof: &Proof<Bls12>, public_inputs: &[Scalar]) -> Result<(), VerificationError> {
    let (a, b, c) = (flat(&[proof.a]), flat(&[proof.b]), flat(&[proof.c]));
    verification_status(unsafe {
        bb_groth16_verify(pvk.ctx, pvk.handle, a.as_ptr() as _, b.as_ptr() as _, c.as_ptr() as _, public_inputs.as_ptr() as _,
                          public_inputs.len())
    })
}

/// Drop-in for `batch::Verifier::verify` (verifier/batch.rs:100-173) over queued `(proof, inputs)` items: the random
/// z_i come from `rng` (non-zero, batch.rs:124-129) and are passed canonical; all items must have as many inputs as the key
/// expects, otherwise InvalidVerifyingKey, before any device work.
pub fn batch_verify_b200<R: RngCore + CryptoRng>(worker: &GpuWorker, vk: &GpuVerifyingKey, items: &[(Proof<Bls12>, Vec<Scalar>)],
                                                 mut rng: R) -> Result<(), VerificationError> {
    let n_inputs = items.first().map_or(0, |(_, x)| x.len());
    if items.iter().any(|(_, x)| x.len() != n_inputs) { return Err(VerificationError::InvalidVerifyingKey); }
    let (mut a, mut b, mut c) = (Vec::with_capacity(items.len() * 12), Vec::with_capacity(items.len() * 24), Vec::with_capacity(items.len() * 12));
    let mut inputs: Vec<Scalar> = Vec::with_capacity(items.len() * n_inputs);
    let mut z: Vec<u8> = Vec::with_capacity(items.len() * 32);
    for (proof, x) in items {
        a.extend(flat(&[proof.a]));
        b.extend(flat(&[proof.b]));
        c.extend(flat(&[proof.c]));
        inputs.extend_from_slice(x);
        let zi = loop { let v = Scalar::random(&mut rng); if !bool::from(v.is_zero()) { break v; } };
        z.extend_from_slice(zi.to_repr().as_ref());
    }
    let batch = bb_proof_batch {
        a: a.as_ptr() as _, b: b.as_ptr() as _, c: c.as_ptr() as _, n: items.len(),
        inputs: inputs.as_ptr() as _, n_inputs, on_device: 0,
    };
    verification_status(unsafe { bb_groth16_verify_batch(worker.ctx, vk.handle, &batch, z.as_ptr() as _) })
}

/// bellman's io::Error of `Proof::read` (groth16/src/lib.rs:47-99) for a non-zero bb_proofs_read status byte
fn read_error(st: u8) -> io::Error {
    let msg = if st & 15 == BB_READ_IDENTITY { "point at infinity" } else if st >> 4 == 2 { "invalid G2" } else { "invalid G1" };
    io::Error::new(io::ErrorKind::InvalidData, msg)
}

fn whole_proofs(len: usize, stride: usize) -> usize {
    if len < BB_PROOF_BYTES { 0 } else { 1 + (len - BB_PROOF_BYTES) / stride }
}

/// Drop-in for `Proof::read` (groth16/src/lib.rs:47-99) over a batch, decoded on the device: proof i is the 192 bytes at
/// `bytes[i * stride..]` (stride 0 = 192; e.g. 384 for Sapling spend descriptions sliced at the proof's offset 128), for
/// every whole record.  Errors are the `InvalidData` io::Errors Proof::read returns ("invalid G1", "invalid G2",
/// "point at infinity").
pub fn read_proofs_b200(worker: &GpuWorker, bytes: &[u8], stride: usize) -> Vec<io::Result<Proof<Bls12>>> {
    let stride = if stride == 0 { BB_PROOF_BYTES } else { stride };
    assert!(stride >= BB_PROOF_BYTES, "a proof record is at least {} bytes", BB_PROOF_BYTES);
    let n = whole_proofs(bytes.len(), stride);
    let (mut a, mut b, mut c) = (vec![0u64; n * 12], vec![0u64; n * 24], vec![0u64; n * 12]);
    let mut st = vec![0u8; n];
    let mut n_invalid = 0usize;
    let input = bb_proof_bytes { bytes: bytes.as_ptr() as _, n, stride, on_device: 0 };
    let rc = unsafe {
        bb_proofs_read(worker.ctx, &input, a.as_mut_ptr() as _, b.as_mut_ptr() as _, c.as_mut_ptr() as _, 0, st.as_mut_ptr(), &mut n_invalid)
    };
    if rc != BB_OK { panic!("bellman_b200 bb_proofs_read failed: {}", last_error()); }
    (0..n).map(|i| {
        if st[i] != 0 { return Err(read_error(st[i])); }
        Ok(Proof { a: G1Affine::from_b200(&a[12 * i..12 * (i + 1)]), b: G2Affine::from_b200(&b[24 * i..24 * (i + 1)]),
                   c: G1Affine::from_b200(&c[12 * i..12 * (i + 1)]) })
    }).collect()
}

/// What `batch_verify_bytes_b200` fails with: a proof that does not read (its index and the io::Error of `Proof::read`),
/// or the `VerificationError` of the batch.
#[derive(Debug)]
pub enum BytesBatchError { Read { index: usize, error: io::Error }, Verification(VerificationError) }

/// A device buffer of the context's allocator, freed on drop.
struct DeviceBuf { ctx: *mut bb_ctx, p: *mut c_void }
impl DeviceBuf {
    fn new(ctx: *mut bb_ctx, bytes: usize) -> Self {
        let mut p = ptr::null_mut();
        if unsafe { bb_device_alloc(ctx, bytes.max(16), &mut p) } != BB_OK { panic!("bellman_b200 device allocation failed: {}", last_error()); }
        DeviceBuf { ctx, p }
    }
}
impl Drop for DeviceBuf {
    fn drop(&mut self) { unsafe { bb_device_free(self.ctx, self.p); } }
}

/// `batch::Verifier::verify` over items queued as `Proof::write` bytes: one bb_proofs_read decodes every proof into device
/// buffers and the batch verifier runs on them there, so the points never return to the host.  A proof that does not read
/// is reported before any pairing work -- a bellman caller's `Proof::read` fails before the proof could be queued; only
/// the first 192 bytes of each item are read, and a shorter item fails as `read_exact` does.  Otherwise the result is that
/// of `batch_verify_b200`.
pub fn batch_verify_bytes_b200<R: RngCore + CryptoRng>(worker: &GpuWorker, vk: &GpuVerifyingKey, items: &[(&[u8], Vec<Scalar>)],
                                                       mut rng: R) -> Result<(), BytesBatchError> {
    let n = items.len();
    let mut bytes = Vec::with_capacity(n * BB_PROOF_BYTES);
    for (index, (b, _)) in items.iter().enumerate() {
        if b.len() < BB_PROOF_BYTES {
            return Err(BytesBatchError::Read { index, error: io::Error::new(io::ErrorKind::UnexpectedEof, "failed to fill whole buffer") });
        }
        bytes.extend_from_slice(&b[..BB_PROOF_BYTES]);
    }
    let (d_a, d_b, d_c) = (DeviceBuf::new(worker.ctx, n * 96), DeviceBuf::new(worker.ctx, n * 192), DeviceBuf::new(worker.ctx, n * 96));
    let mut st = vec![0u8; n];
    let mut n_invalid = 0usize;
    let input = bb_proof_bytes { bytes: bytes.as_ptr() as _, n, stride: BB_PROOF_BYTES, on_device: 0 };
    let rc = unsafe { bb_proofs_read(worker.ctx, &input, d_a.p, d_b.p, d_c.p, 1, st.as_mut_ptr(), &mut n_invalid) };
    if rc != BB_OK { panic!("bellman_b200 bb_proofs_read failed: {}", last_error()); }
    if let Some(index) = st.iter().position(|&s| s != 0) {
        return Err(BytesBatchError::Read { index, error: read_error(st[index]) });
    }
    let n_inputs = items.first().map_or(0, |(_, x)| x.len());
    if items.iter().any(|(_, x)| x.len() != n_inputs) { return Err(BytesBatchError::Verification(VerificationError::InvalidVerifyingKey)); }
    let mut inputs: Vec<Scalar> = Vec::with_capacity(n * n_inputs);
    let mut z: Vec<u8> = Vec::with_capacity(n * 32);
    for (_, x) in items {
        inputs.extend_from_slice(x);
        let zi = loop { let v = Scalar::random(&mut rng); if !bool::from(v.is_zero()) { break v; } };
        z.extend_from_slice(zi.to_repr().as_ref());
    }
    let d_x = DeviceBuf::new(worker.ctx, inputs.len() * 32);
    if !inputs.is_empty() && unsafe { bb_device_upload(worker.ctx, d_x.p, inputs.as_ptr() as _, inputs.len() * 32) } != BB_OK {
        panic!("bellman_b200 upload failed: {}", last_error());
    }
    let batch = bb_proof_batch { a: d_a.p, b: d_b.p, c: d_c.p, n, inputs: d_x.p, n_inputs, on_device: 1 };
    verification_status(unsafe { bb_groth16_verify_batch(worker.ctx, vk.handle, &batch, z.as_ptr() as _) })
        .map_err(BytesBatchError::Verification)
}

/// verify_single's key check for one item (batch.rs:57-65 -> verifier.rs:28-30)
fn input_count(pvk: &GpuVerifyingKey, x: &[Scalar]) -> Result<(), VerificationError> {
    if x.len() + 1 == pvk.ic_len { Ok(()) } else { Err(VerificationError::InvalidVerifyingKey) }
}

/// The n x L input matrix of the items, with zero rows for the items of a wrong input count (their verdicts are not used).
fn each_inputs<'a>(pvk: &GpuVerifyingKey, xs: impl Iterator<Item = &'a Vec<Scalar>>, n: usize) -> Vec<Scalar> {
    let l = pvk.ic_len - 1;
    let mut inputs = vec![Scalar::from(0u64); n * l];
    for (i, x) in xs.enumerate() {
        if x.len() == l { inputs[i * l..(i + 1) * l].copy_from_slice(x); }
    }
    inputs
}

/// bb_groth16_verify_each: one verdict byte per proof of the batch, 0 = valid
fn each_verdicts(pvk: &GpuVerifyingKey, batch: &bb_proof_batch) -> Vec<u8> {
    let mut verdicts = vec![0u8; batch.n];
    let mut n_invalid = 0usize;
    let rc = unsafe { bb_groth16_verify_each(pvk.ctx, pvk.handle, batch, verdicts.as_mut_ptr(), &mut n_invalid) };
    if rc != BB_OK { panic!("bellman_b200 bb_groth16_verify_each failed: {}", last_error()); }
    verdicts
}

/// `Item::verify_single` (verifier/batch.rs:57-65), i.e. `verify_proof`, for every item in one device call: the fallback
/// that finds the bad proofs of a batch `batch_verify_b200` rejected.  One result per item, in order: InvalidVerifyingKey
/// for an item whose input count does not match the key (the other items are still verified), InvalidProof for an item
/// whose equation fails.
pub fn verify_each_b200(pvk: &GpuVerifyingKey, items: &[(Proof<Bls12>, Vec<Scalar>)]) -> Vec<Result<(), VerificationError>> {
    let n = items.len();
    let mut out: Vec<Result<(), VerificationError>> = items.iter().map(|(_, x)| input_count(pvk, x)).collect();
    if n == 0 || pvk.ic_len == 0 { return out; }
    let (mut a, mut b, mut c) = (Vec::with_capacity(n * 12), Vec::with_capacity(n * 24), Vec::with_capacity(n * 12));
    for (proof, _) in items {
        a.extend(flat(&[proof.a]));
        b.extend(flat(&[proof.b]));
        c.extend(flat(&[proof.c]));
    }
    let inputs = each_inputs(pvk, items.iter().map(|(_, x)| x), n);
    let batch = bb_proof_batch {
        a: a.as_ptr() as _, b: b.as_ptr() as _, c: c.as_ptr() as _, n,
        inputs: inputs.as_ptr() as _, n_inputs: pvk.ic_len - 1, on_device: 0,
    };
    for (r, v) in out.iter_mut().zip(each_verdicts(pvk, &batch)) {
        if r.is_ok() && v != 0 { *r = Err(VerificationError::InvalidProof); }
    }
    out
}

/// `verify_each_b200` over items given as `Proof::write` bytes: one bb_proofs_read decodes every proof into device buffers
/// and bb_groth16_verify_each runs on them there.  One result per item, in order: `Read` (its index and the io::Error of
/// `Proof::read`; a shorter item fails as `read_exact` does) for a proof that does not read, otherwise what
/// `verify_each_b200` gives for it.
pub fn verify_each_bytes_b200(worker: &GpuWorker, pvk: &GpuVerifyingKey, items: &[(&[u8], Vec<Scalar>)]) -> Vec<Result<(), BytesBatchError>> {
    let n = items.len();
    let mut bytes = Vec::with_capacity(n * BB_PROOF_BYTES);
    for (b, _) in items {
        if b.len() < BB_PROOF_BYTES { bytes.extend_from_slice(&[0u8; BB_PROOF_BYTES]); } else { bytes.extend_from_slice(&b[..BB_PROOF_BYTES]); }
    }
    let (d_a, d_b, d_c) = (DeviceBuf::new(worker.ctx, n * 96), DeviceBuf::new(worker.ctx, n * 192), DeviceBuf::new(worker.ctx, n * 96));
    let mut st = vec![0u8; n];
    let mut n_invalid = 0usize;
    let input = bb_proof_bytes { bytes: bytes.as_ptr() as _, n, stride: BB_PROOF_BYTES, on_device: 0 };
    let rc = unsafe { bb_proofs_read(worker.ctx, &input, d_a.p, d_b.p, d_c.p, 1, st.as_mut_ptr(), &mut n_invalid) };
    if rc != BB_OK { panic!("bellman_b200 bb_proofs_read failed: {}", last_error()); }
    let mut out: Vec<Result<(), BytesBatchError>> = items.iter().enumerate().map(|(index, (b, x))| {
        if b.len() < BB_PROOF_BYTES {
            Err(BytesBatchError::Read { index, error: io::Error::new(io::ErrorKind::UnexpectedEof, "failed to fill whole buffer") })
        } else if st[index] != 0 {
            Err(BytesBatchError::Read { index, error: read_error(st[index]) })
        } else {
            input_count(pvk, x).map_err(BytesBatchError::Verification)
        }
    }).collect();
    if n == 0 || pvk.ic_len == 0 { return out; }
    let inputs = each_inputs(pvk, items.iter().map(|(_, x)| x), n);
    let d_x = DeviceBuf::new(worker.ctx, inputs.len() * 32);
    if !inputs.is_empty() && unsafe { bb_device_upload(worker.ctx, d_x.p, inputs.as_ptr() as _, inputs.len() * 32) } != BB_OK {
        panic!("bellman_b200 upload failed: {}", last_error());
    }
    let batch = bb_proof_batch { a: d_a.p, b: d_b.p, c: d_c.p, n, inputs: d_x.p, n_inputs: pvk.ic_len - 1, on_device: 1 };
    for (r, v) in out.iter_mut().zip(each_verdicts(pvk, &batch)) {
        if r.is_ok() && v != 0 { *r = Err(BytesBatchError::Verification(VerificationError::InvalidProof)); }
    }
    out
}

#[allow(dead_code)]
fn _projective_types_are_what_wait_returns(_: G1Projective, _: G2Projective) {}

impl GpuParameters {
    /// `generate_parameters(circuit, g1, g2, alpha, beta, gamma, delta, tau)` (groth16/src/generator.rs:159-507) for the
    /// circuit whose constraint system `r1cs` holds, computed on the device (bb_groth16_generate): the same points, element
    /// for element, as a resident key and its prepared verifying key.  Nothing but the toxic waste crosses the bus; the
    /// library wipes its copies of it.  Errors as the reference: UnexpectedIdentity for gamma or delta zero,
    /// UnconstrainedVariable.
    #[allow(clippy::too_many_arguments)]
    pub fn generate(worker: &GpuWorker, r1cs: &GpuR1cs, g1: G1Projective, g2: G2Projective, alpha: Scalar, beta: Scalar, gamma: Scalar,
                    delta: Scalar, tau: Scalar) -> Result<(GpuParameters, GpuVerifyingKey), SynthesisError> {
        let (mut p1, mut p2) = (vec![0u64; G1Affine::WORDS], vec![0u64; G2Affine::WORDS]);
        g1.to_affine().to_b200(&mut p1);
        g2.to_affine().to_b200(&mut p2);
        let mut toxic = bb_toxic {
            g1: p1.as_ptr() as _, g2: p2.as_ptr() as _, alpha: alpha.to_repr(), beta: beta.to_repr(), gamma: gamma.to_repr(),
            delta: delta.to_repr(), tau: tau.to_repr(),
        };
        let res = generate_impl(worker, r1cs, &toxic);
        for k in [&mut toxic.alpha, &mut toxic.beta, &mut toxic.gamma, &mut toxic.delta, &mut toxic.tau] {
            for b in k.iter_mut() { unsafe { ptr::write_volatile(b, 0) } }
        }
        res
    }

    /// `Parameters::write` (groth16/src/lib.rs:258-287) of this resident key, encoded on the device (bb_params_write): the
    /// bytes the reference writes for the same key.  `vk` is this key's prepared verifying key (it holds gamma_g2 and ic).
    pub fn write<W: io::Write>(&self, vk: &GpuVerifyingKey, writer: W) -> io::Result<()> { self.write_impl(vk, false, writer) }

    /// `VerifyingKey::write` (groth16/src/lib.rs:143-156) of this key's verifying key
    pub fn write_verifying_key<W: io::Write>(&self, vk: &GpuVerifyingKey, writer: W) -> io::Result<()> { self.write_impl(vk, true, writer) }

    fn write_impl<W: io::Write>(&self, vk: &GpuVerifyingKey, vk_only: bool, mut writer: W) -> io::Result<()> {
        let mut len = 0usize;
        let rc = unsafe { bb_params_write(self.ctx, self.handle, vk.handle, vk_only as i32, ptr::null_mut(), 0, 0, &mut len) };
        if rc != BB_OK { return Err(io::Error::new(io::ErrorKind::Other, last_error())); }
        let mut buf = vec![0u8; len];
        let rc = unsafe { bb_params_write(self.ctx, self.handle, vk.handle, vk_only as i32, buf.as_mut_ptr() as _, len, 0, &mut len) };
        if rc != BB_OK { return Err(io::Error::new(io::ErrorKind::Other, last_error())); }
        writer.write_all(&buf)
    }
}

fn generate_impl(worker: &GpuWorker, r1cs: &GpuR1cs, toxic: *const bb_toxic) -> Result<(GpuParameters, GpuVerifyingKey), SynthesisError> {
    let (mut crs, mut vk, mut rep) = (ptr::null_mut(), ptr::null_mut(), bb_generate_report::default());
    status(unsafe { bb_groth16_generate(worker.ctx, r1cs.handle, toxic, &mut crs, &mut vk, &mut rep) })?;
    Ok((GpuParameters { ctx: worker.ctx, handle: crs }, GpuVerifyingKey { ctx: worker.ctx, handle: vk, ic_len: rep.len[0] }))
}

/// `generate_random_parameters` (groth16/src/generator.rs:21-40) on the device: the library draws the toxic waste and the
/// generators from the operating system (getrandom), and none of them leaves it.
pub fn generate_random_parameters_b200(worker: &GpuWorker, r1cs: &GpuR1cs) -> Result<(GpuParameters, GpuVerifyingKey), SynthesisError> {
    generate_impl(worker, r1cs, ptr::null())
}
