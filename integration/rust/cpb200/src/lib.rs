//! `cpb200` -- ark-crypto-primitives traits over the H100 library (`include/cpb200.h`).
//!
//! SOURCE ONLY (not compiled in this repository: the image has no Rust toolchain).  It shows exactly what a
//! maintainer binds: the raw `extern "C"` block mirrors `include/cpb200.h`; the wrappers implement
//! `CRHScheme` / `TwoToOneCRHScheme` (R/crh/mod.rs:18-51) for Poseidon and a `GpuMerkleTree` with the
//! reference's public method set (R/merkle_tree/mod.rs:397-533).  `ark-crypto-primitives` itself forbids
//! `unsafe` (R/lib.rs:9), hence a sibling crate.
use ark_crypto_primitives::crh::{CRHScheme, TwoToOneCRHScheme};
use ark_crypto_primitives::sponge::poseidon::PoseidonConfig;
use ark_crypto_primitives::Error;
use ark_ff::{BigInt, Fp256, MontBackend, MontConfig, PrimeField};
use ark_std::{borrow::Borrow, marker::PhantomData, rand::Rng, sync::Arc};
use std::os::raw::{c_char, c_int};

#[allow(non_camel_case_types)]
#[repr(C)]
pub struct cpb_poseidon_ctx {
    _private: [u8; 0],
}

extern "C" {
    fn cpb_last_error() -> *const c_char;
    fn cpb_poseidon_ctx_create(field_id: c_int, rate: c_int, capacity: c_int, full_rounds: c_int, partial_rounds: c_int,
                               alpha: u64, ark: *const u64, mds: *const u64, device: c_int, out: *mut *mut cpb_poseidon_ctx) -> c_int;
    fn cpb_poseidon_ctx_destroy(ctx: *mut cpb_poseidon_ctx);
    fn cpb_poseidon_crh_batch(ctx: *mut cpb_poseidon_ctx, input: *const u64, len: usize, out: *mut u64, n: usize) -> c_int;
    fn cpb_poseidon_compress_batch(ctx: *mut cpb_poseidon_ctx, pairs: *const u64, out: *mut u64, n: usize) -> c_int;
    fn cpb_merkle_poseidon_build(leaf: *mut cpb_poseidon_ctx, node: *mut cpb_poseidon_ctx, leaves: *const u64, leaf_len: usize,
                                 n: usize, leaf_nodes: *mut u64, non_leaf_nodes: *mut u64) -> c_int;
    // inputs of different lengths (ABI v4): input i = values[offsets[i] .. offsets[i+1])
    fn cpb_poseidon_crh_ragged_batch(ctx: *mut cpb_poseidon_ctx, values: *const u64, offsets: *const u64, out: *mut u64, n: usize) -> c_int;
    fn cpb_merkle_poseidon_build_ragged(leaf: *mut cpb_poseidon_ctx, node: *mut cpb_poseidon_ctx, values: *const u64, offsets: *const u64,
                                        n: usize, leaf_nodes: *mut u64, non_leaf_nodes: *mut u64) -> c_int;
    // k x MerkleTree::update / check_update on host arrays in place (ABI v5); asserted_root and applied may be null
    fn cpb_merkle_poseidon_update(leaf: *mut cpb_poseidon_ctx, node: *mut cpb_poseidon_ctx, leaf_nodes: *mut u64, non_leaf_nodes: *mut u64,
                                  n: usize, indexes: *const u64, new_leaves: *const u64, leaf_len: usize, k: usize,
                                  asserted_root: *const u64, applied: *mut c_int) -> c_int;
    // page-lock a `Vec<Fr>`'s storage once so the host-pointer calls copy at full PCIe rate (ABI v3)
    fn cpb_host_register(ptr: *mut core::ffi::c_void, bytes: usize) -> c_int;
    fn cpb_host_unregister(ptr: *mut core::ffi::c_void) -> c_int;
    // one process, several GPUs (ABI v3): peer-memory root exchange fused into the last kernel, or ncclCommInitAll + ncclAllGather
    fn cpb_multi_create(ndev: c_int, devices: *const c_int, out: *mut *mut cpb_multi) -> c_int;
    fn cpb_multi_destroy(m: *mut cpb_multi);
    fn cpb_multi_uses_nccl(m: *const cpb_multi) -> c_int;
    fn cpb_merkle_poseidon_build_multi(m: *mut cpb_multi, leaf_ctxs: *const *mut cpb_poseidon_ctx, node_ctxs: *const *mut cpb_poseidon_ctx,
                                       leaves: *const u64, leaf_len: usize, n: usize, leaf_nodes: *mut u64, non_leaf_nodes: *mut u64) -> c_int;
}

#[allow(non_camel_case_types)]
#[repr(C)]
pub struct cpb_multi {
    _private: [u8; 0],
}

const CPB_OK: c_int = 0;
const CPB_BAD_LENGTH: c_int = 1;
const CPB_NOT_POW2: c_int = 3;
#[allow(dead_code)]
const CPB_NCCL_ERROR: c_int = 9;      // surfaces as Err(CpbError(9, ..)) through `check`

#[derive(Debug)]
pub struct CpbError(pub c_int, pub String);
impl core::fmt::Display for CpbError {
    fn fmt(&self, f: &mut core::fmt::Formatter<'_>) -> core::fmt::Result {
        write!(f, "cpb200 status {}: {}", self.0, self.1)
    }
}
impl ark_std::error::Error for CpbError {}

fn check(status: c_int) -> Result<(), Error> {
    match status {
        CPB_OK => Ok(()),
        // the reference panics on these (R/crh/pedersen/mod.rs:82-89, R/merkle_tree/mod.rs:430-433); so does the shim
        CPB_BAD_LENGTH => panic!("incorrect input length"),
        CPB_NOT_POW2 => panic!("`leaves.len() should be power of two and greater than one"),
        s => {
            let msg = unsafe { std::ffi::CStr::from_ptr(cpb_last_error()) }.to_string_lossy().into_owned();
            Err(Box::new(CpbError(s, msg)))
        },
    }
}

/// Fields the library has kernels for.  The ABI element is the memory image of `Fp256<MontBackend<_, 4>>`:
/// `BigInt<4>` little-endian limbs in Montgomery form, so conversion is a copy of `.0 .0`.
pub trait GpuField: PrimeField {
    const FIELD_ID: c_int;
    fn mont_limbs(&self) -> [u64; 4];
    fn from_mont_limbs(limbs: [u64; 4]) -> Self;
}
macro_rules! gpu_field {
    ($cfg:ty, $id:expr) => {
        impl GpuField for Fp256<MontBackend<$cfg, 4>> {
            const FIELD_ID: c_int = $id;
            fn mont_limbs(&self) -> [u64; 4] { (self.0).0 }
            fn from_mont_limbs(limbs: [u64; 4]) -> Self { Self::new_unchecked(BigInt::new(limbs)) }   // already Montgomery
        }
    };
}
gpu_field!(ark_bls12_381::FrConfig, 0);
gpu_field!(ark_bn254::FrConfig, 1);
gpu_field!(ark_ed_on_bls12_381::FrConfig, 2);
// ark_ed_on_bls12_381::Fq is ark_bls12_381::Fr (the Jubjub base field): already covered by id 0.

fn flatten<F: GpuField>(xs: &[F]) -> Vec<u64> { xs.iter().flat_map(|x| x.mont_limbs()).collect() }
fn unflatten<F: GpuField>(l: &[u64]) -> Vec<F> { l.chunks_exact(4).map(|c| F::from_mont_limbs([c[0], c[1], c[2], c[3]])).collect() }
/// `Some(len)` when every input has the same length (the uniform calls), `None` when they differ (the ragged calls).
fn common_len<T: AsRef<[F]>, F>(inputs: &[T]) -> Option<usize> {
    let len = inputs.first().map_or(0, |i| i.as_ref().len());
    inputs.iter().all(|i| i.as_ref().len() == len).then_some(len)
}
/// The ragged layout of the ABI: the inputs' elements back to back and the n + 1 prefix sums of their lengths.
fn offsets<T: AsRef<[F]>, F>(inputs: &[T]) -> Vec<u64> {
    let mut off = Vec::with_capacity(inputs.len() + 1);
    off.push(0u64);
    for i in inputs {
        off.push(off[off.len() - 1] + i.as_ref().len() as u64);
    }
    off
}

struct Ctx(*mut cpb_poseidon_ctx);
unsafe impl Send for Ctx {}
unsafe impl Sync for Ctx {}          // the library serialises host-pointer calls per context
impl Drop for Ctx {
    fn drop(&mut self) { unsafe { cpb_poseidon_ctx_destroy(self.0) } }
}

/// `PoseidonConfig<F>` plus the device context built from it (`Parameters: Clone + Sync`, R/crh/mod.rs:21).
#[derive(Clone)]
pub struct GpuPoseidonParams<F: GpuField> {
    pub config: PoseidonConfig<F>,
    ctx: Arc<Ctx>,
}
impl<F: GpuField> GpuPoseidonParams<F> {
    pub fn new(config: PoseidonConfig<F>, device: i32) -> Result<Self, Error> {
        let ark: Vec<u64> = config.ark.iter().flat_map(|r| flatten(r)).collect();
        let mds: Vec<u64> = config.mds.iter().flat_map(|r| flatten(r)).collect();
        let mut raw = core::ptr::null_mut();
        check(unsafe {
            cpb_poseidon_ctx_create(F::FIELD_ID, config.rate as c_int, config.capacity as c_int, config.full_rounds as c_int,
                                    config.partial_rounds as c_int, config.alpha, ark.as_ptr(), mds.as_ptr(), device, &mut raw)
        })?;
        Ok(Self { config, ctx: Arc::new(Ctx(raw)) })
    }
}

/// `crh::poseidon::CRH` (R/crh/poseidon/mod.rs:15-41) on the GPU.
pub struct GpuPoseidonCRH<F>(PhantomData<F>);
impl<F: GpuField> GpuPoseidonCRH<F> {
    /// n inputs, one call: equal lengths take the uniform kernel, different lengths the ragged call (each input hashed at
    /// its own length, as `CRH::evaluate` does).
    pub fn evaluate_batch(p: &GpuPoseidonParams<F>, inputs: &[&[F]]) -> Result<Vec<F>, Error> {
        let flat: Vec<u64> = inputs.iter().flat_map(|i| flatten(i)).collect();
        let mut out = vec![0u64; 4 * inputs.len()];
        match common_len::<_, F>(inputs) {
            Some(len) => check(unsafe { cpb_poseidon_crh_batch(p.ctx.0, flat.as_ptr(), len, out.as_mut_ptr(), inputs.len()) })?,
            None => {
                let off = offsets::<_, F>(inputs);
                check(unsafe { cpb_poseidon_crh_ragged_batch(p.ctx.0, flat.as_ptr(), off.as_ptr(), out.as_mut_ptr(), inputs.len()) })?
            },
        }
        Ok(unflatten(&out))
    }
}
impl<F: GpuField + ark_crypto_primitives::sponge::Absorb> CRHScheme for GpuPoseidonCRH<F> {
    type Input = [F];
    type Output = F;
    type Parameters = GpuPoseidonParams<F>;
    fn setup<R: Rng>(_: &mut R) -> Result<Self::Parameters, Error> { unimplemented!() }        // as the reference, mod.rs:24-28
    fn evaluate<T: Borrow<Self::Input>>(p: &Self::Parameters, input: T) -> Result<F, Error> {
        Ok(Self::evaluate_batch(p, &[input.borrow()])?[0])                                     // correct; prefer the batch call
    }
}

/// `crh::poseidon::TwoToOneCRH` (mod.rs:43-80); `evaluate` is an alias of `compress` (:58-64).
pub struct GpuPoseidonTwoToOneCRH<F>(PhantomData<F>);
impl<F: GpuField> GpuPoseidonTwoToOneCRH<F> {
    pub fn compress_batch(p: &GpuPoseidonParams<F>, pairs: &[(F, F)]) -> Result<Vec<F>, Error> {
        let flat: Vec<u64> = pairs.iter().flat_map(|(l, r)| [l.mont_limbs(), r.mont_limbs()].concat()).collect();
        let mut out = vec![0u64; 4 * pairs.len()];
        check(unsafe { cpb_poseidon_compress_batch(p.ctx.0, flat.as_ptr(), out.as_mut_ptr(), pairs.len()) })?;
        Ok(unflatten(&out))
    }
}
impl<F: GpuField + ark_crypto_primitives::sponge::Absorb> TwoToOneCRHScheme for GpuPoseidonTwoToOneCRH<F> {
    type Input = F;
    type Output = F;
    type Parameters = GpuPoseidonParams<F>;
    fn setup<R: Rng>(_: &mut R) -> Result<Self::Parameters, Error> { unimplemented!() }
    fn evaluate<T: Borrow<F>>(p: &Self::Parameters, l: T, r: T) -> Result<F, Error> { Self::compress(p, l, r) }
    fn compress<T: Borrow<F>>(p: &Self::Parameters, l: T, r: T) -> Result<F, Error> {
        Ok(Self::compress_batch(p, &[(*l.borrow(), *r.borrow())])?[0])
    }
}

/// `MerkleTree<FieldMTConfig>` (R/merkle_tree/tests/mod.rs:198-206) built on the GPU: the ABI returns the reference's
/// own two arrays (R/merkle_tree/mod.rs:383-395), so proofs are the reference's index arithmetic (mod.rs:547-575)
/// and `Path<P>` (public fields, mod.rs:146-152) verifies with the reference's `Path::verify`.
pub struct GpuMerkleTree<F: GpuField> {
    pub leaf_nodes: Vec<F>,
    pub non_leaf_nodes: Vec<F>,
    height: usize,
}
impl<F: GpuField> GpuMerkleTree<F> {
    /// `MerkleTree::new` hashes each leaf at its own length (R/merkle_tree/mod.rs:411-422): leaves of different lengths take
    /// the ragged build, equal lengths the uniform one.
    pub fn new(leaf: &GpuPoseidonParams<F>, two_to_one: &GpuPoseidonParams<F>, leaves: &[Vec<F>]) -> Result<Self, Error> {
        let n = leaves.len();
        let flat: Vec<u64> = leaves.iter().flat_map(|l| flatten(l)).collect();
        let (mut ln, mut nn) = (vec![0u64; 4 * n], vec![0u64; 4 * n.saturating_sub(1)]);
        check(unsafe {
            match common_len::<_, F>(leaves) {
                Some(leaf_len) => cpb_merkle_poseidon_build(leaf.ctx.0, two_to_one.ctx.0, flat.as_ptr(), leaf_len, n, ln.as_mut_ptr(),
                                                            nn.as_mut_ptr()),
                None => {
                    let off = offsets::<_, F>(leaves);
                    cpb_merkle_poseidon_build_ragged(leaf.ctx.0, two_to_one.ctx.0, flat.as_ptr(), off.as_ptr(), n, ln.as_mut_ptr(),
                                                     nn.as_mut_ptr())
                },
            }
        })?;
        Ok(Self { leaf_nodes: unflatten(&ln), non_leaf_nodes: unflatten(&nn), height: n.trailing_zeros() as usize + 1 })
    }
    pub fn root(&self) -> F { self.non_leaf_nodes[0] }
    pub fn height(&self) -> usize { self.height }
    /// authentication path of leaf `index`, root side first (compute_auth_path, mod.rs:548-573)
    pub fn auth_path(&self, index: usize) -> Vec<F> {
        let mut cur = (index + self.leaf_nodes.len() - 2) >> 1;
        let mut path = Vec::with_capacity(self.height - 2);
        while cur != 0 {
            path.push(self.non_leaf_nodes[if cur % 2 == 1 { cur + 1 } else { cur - 1 }]);
            cur = (cur - 1) >> 1;
        }
        path.reverse();
        path
    }
    /// k x `MerkleTree::update` (R/merkle_tree/mod.rs:690-701) in one call: the touched nodes of every level are hashed on the GPU,
    /// and only they and the siblings they read cross PCIe.  A repeated index takes its last leaf; new leaves of one length.
    pub fn update_batch(&mut self, leaf: &GpuPoseidonParams<F>, two_to_one: &GpuPoseidonParams<F>, indexes: &[usize],
                        new_leaves: &[Vec<F>]) -> Result<(), Error> {
        self.update_impl(leaf, two_to_one, indexes, new_leaves, None).map(|_| ())
    }
    pub fn update(&mut self, leaf: &GpuPoseidonParams<F>, two_to_one: &GpuPoseidonParams<F>, index: usize, new_leaf: &[F]) -> Result<(), Error> {
        self.update_batch(leaf, two_to_one, &[index], &[new_leaf.to_vec()])
    }
    /// `MerkleTree::check_update` (mod.rs:706-725) for all k at once: the tree changes only when the new root equals
    /// `asserted_new_root`; returns whether it did.
    pub fn check_update_batch(&mut self, leaf: &GpuPoseidonParams<F>, two_to_one: &GpuPoseidonParams<F>, indexes: &[usize],
                              new_leaves: &[Vec<F>], asserted_new_root: &F) -> Result<bool, Error> {
        self.update_impl(leaf, two_to_one, indexes, new_leaves, Some(asserted_new_root))
    }
    pub fn check_update(&mut self, leaf: &GpuPoseidonParams<F>, two_to_one: &GpuPoseidonParams<F>, index: usize, new_leaf: &[F],
                        asserted_new_root: &F) -> Result<bool, Error> {
        self.check_update_batch(leaf, two_to_one, &[index], &[new_leaf.to_vec()], asserted_new_root)
    }
    fn update_impl(&mut self, leaf: &GpuPoseidonParams<F>, two_to_one: &GpuPoseidonParams<F>, indexes: &[usize], new_leaves: &[Vec<F>],
                   asserted_new_root: Option<&F>) -> Result<bool, Error> {
        assert_eq!(indexes.len(), new_leaves.len(), "one new leaf per index");
        let leaf_len = common_len::<_, F>(new_leaves).expect("an update batch takes new leaves of one length");
        let idx: Vec<u64> = indexes.iter().map(|&i| i as u64).collect();
        let flat: Vec<u64> = new_leaves.iter().flat_map(|l| flatten(l)).collect();
        let (mut ln, mut nn) = (flatten(&self.leaf_nodes), flatten(&self.non_leaf_nodes));
        let root = asserted_new_root.map(|r| r.mont_limbs());
        let mut applied: c_int = 0;
        check(unsafe {
            cpb_merkle_poseidon_update(leaf.ctx.0, two_to_one.ctx.0, ln.as_mut_ptr(), nn.as_mut_ptr(), self.leaf_nodes.len(), idx.as_ptr(),
                                       flat.as_ptr(), leaf_len, idx.len(), root.as_ref().map_or(core::ptr::null(), |r| r.as_ptr()), &mut applied)
        })?;
        if applied != 0 {
            self.leaf_nodes = unflatten(&ln);
            self.non_leaf_nodes = unflatten(&nn);
        }
        Ok(applied != 0)
    }
}

/// `MerkleTree::new` (R/merkle_tree/mod.rs:411-422) on ALL the GPUs of a group driven by this process: the leaves are sharded
/// contiguously over the devices, every device builds its subtree, the subtree roots are exchanged once (inside the last
/// kernel over NVLink peer memory, or by one `ncclAllGather`) and the result is the reference's two arrays, exactly as from
/// one GPU.  `params[d]` are contexts of the SAME `PoseidonConfig` created on `devices[d]`.
pub struct GpuGroup {
    raw: *mut cpb_multi,
    ndev: usize,
}
unsafe impl Send for GpuGroup {}
unsafe impl Sync for GpuGroup {}
impl GpuGroup {
    pub fn new(devices: &[i32]) -> Result<Self, Error> {
        let mut raw = core::ptr::null_mut();
        check(unsafe { cpb_multi_create(devices.len() as c_int, devices.as_ptr(), &mut raw) })?;
        Ok(Self { raw, ndev: devices.len() })
    }
    pub fn uses_nccl(&self) -> bool { unsafe { cpb_multi_uses_nccl(self.raw) != 0 } }
    pub fn merkle_tree<F: GpuField>(&self, leaf: &[GpuPoseidonParams<F>], two_to_one: &[GpuPoseidonParams<F>], leaves: &[Vec<F>])
        -> Result<GpuMerkleTree<F>, Error> {
        assert!(leaf.len() == self.ndev && two_to_one.len() == self.ndev, "one context per device");
        let n = leaves.len();
        // the sharded build takes one leaf length; leaves of different lengths would be hashed wrongly, so refuse them
        let leaf_len = common_len::<_, F>(leaves).expect("the multi-GPU build needs leaves of equal length; use GpuMerkleTree::new for others");
        let mut flat: Vec<u64> = leaves.iter().flat_map(|l| flatten(l)).collect();
        let (mut ln, mut nn) = (vec![0u64; 4 * n], vec![0u64; 4 * n.saturating_sub(1)]);
        let lc: Vec<*mut cpb_poseidon_ctx> = leaf.iter().map(|p| p.ctx.0).collect();
        let nc: Vec<*mut cpb_poseidon_ctx> = two_to_one.iter().map(|p| p.ctx.0).collect();
        // optional: pin the big buffers for the duration of the call (pageable memory works, at about half the PCIe rate)
        unsafe { cpb_host_register(flat.as_mut_ptr() as *mut _, flat.len() * 8) };
        let st = unsafe { cpb_merkle_poseidon_build_multi(self.raw, lc.as_ptr(), nc.as_ptr(), flat.as_ptr(), leaf_len, n, ln.as_mut_ptr(), nn.as_mut_ptr()) };
        unsafe { cpb_host_unregister(flat.as_mut_ptr() as *mut _) };
        check(st)?;
        Ok(GpuMerkleTree { leaf_nodes: unflatten(&ln), non_leaf_nodes: unflatten(&nn), height: n.trailing_zeros() as usize + 1 })
    }
}
impl Drop for GpuGroup {
    fn drop(&mut self) { unsafe { cpb_multi_destroy(self.raw) } }
}

// ------------------------------------------------------------------------------------------------------------------
// Pedersen CRH / commitment over Jubjub (`ark_ed_on_bls12_381::EdwardsProjective`, curve id 0 of the library).
// ------------------------------------------------------------------------------------------------------------------
pub mod pedersen {
    use super::{check, GpuField};
    use ark_crypto_primitives::commitment::{pedersen as ref_comm, CommitmentScheme};
    use ark_crypto_primitives::crh::{pedersen as ref_crh, CRHScheme};
    use ark_crypto_primitives::Error;
    use ark_ec::CurveGroup;
    use ark_ed_on_bls12_381::{EdwardsAffine, EdwardsProjective, Fq};
    use ark_ff::{BigInteger, PrimeField};
    use ark_std::{borrow::Borrow, marker::PhantomData, rand::Rng, sync::Arc};
    use std::os::raw::c_int;

    #[allow(non_camel_case_types)]
    #[repr(C)]
    pub struct cpb_pedersen_ctx {
        _private: [u8; 0],
    }
    extern "C" {
        fn cpb_pedersen_ctx_create(curve_id: c_int, window_size: c_int, num_windows: c_int, generators_xy: *const u64, n_rand: usize,
                                   rand_generators_xy: *const u64, device: c_int, out: *mut *mut cpb_pedersen_ctx) -> c_int;
        fn cpb_pedersen_ctx_destroy(ctx: *mut cpb_pedersen_ctx);
        fn cpb_pedersen_crh_batch(ctx: *mut cpb_pedersen_ctx, input: *const u8, len: usize, stride: usize, out_xy: *mut u64, n: usize) -> c_int;
        fn cpb_pedersen_commit_batch(ctx: *mut cpb_pedersen_ctx, input: *const u8, len: usize, stride: usize, randomness_le32: *const u8,
                                     out_xy: *mut u64, n: usize) -> c_int;
        fn cpb_merkle_pedersen_build(leaf: *mut cpb_pedersen_ctx, node: *mut cpb_pedersen_ctx, leaves: *const u8, leaf_len: usize, n: usize,
                                     leaf_nodes_xy: *mut u64, non_leaf_nodes_xy: *mut u64) -> c_int;
        // k x MerkleTree::update / check_update of a byte tree on host arrays in place; asserted_root_xy and applied may be null
        fn cpb_merkle_pedersen_update(leaf: *mut cpb_pedersen_ctx, node: *mut cpb_pedersen_ctx, leaf_nodes_xy: *mut u64,
                                      non_leaf_nodes_xy: *mut u64, n: usize, indexes: *const u64, new_leaves: *const u8, leaf_len: usize,
                                      k: usize, asserted_root_xy: *const u64, applied: *mut c_int) -> c_int;
    }

    struct Ctx(*mut cpb_pedersen_ctx);
    unsafe impl Send for Ctx {}
    unsafe impl Sync for Ctx {}
    impl Drop for Ctx {
        fn drop(&mut self) { unsafe { cpb_pedersen_ctx_destroy(self.0) } }
    }

    fn xy(points: &[EdwardsProjective]) -> Vec<u64> {
        // Parameters.generators holds projective points (R/crh/pedersen/mod.rs:28-31); the ABI takes affine x, y limbs
        EdwardsProjective::normalize_batch(points).iter().flat_map(|p| [p.x.mont_limbs(), p.y.mont_limbs()].concat()).collect()
    }
    fn points(limbs: &[u64]) -> Vec<EdwardsAffine> {
        limbs.chunks_exact(8)
            .map(|c| EdwardsAffine::new_unchecked(Fq::from_mont_limbs([c[0], c[1], c[2], c[3]]), Fq::from_mont_limbs([c[4], c[5], c[6], c[7]])))
            .collect()
    }

    /// `pedersen::Parameters<C>` (+ the commitment's `randomness_generator`) and the device tables built from them.
    #[derive(Clone)]
    pub struct GpuPedersenParams {
        pub generators: Vec<Vec<EdwardsProjective>>,
        pub randomness_generator: Vec<EdwardsProjective>,
        ctx: Arc<Ctx>,
    }
    impl GpuPedersenParams {
        pub fn from_crh<W: ref_crh::Window>(p: &ref_crh::Parameters<EdwardsProjective>, device: i32) -> Result<Self, Error> {
            Self::build::<W>(p.generators.clone(), Vec::new(), device)
        }
        pub fn from_commitment<W: ref_crh::Window>(p: &ref_comm::Parameters<EdwardsProjective>, device: i32) -> Result<Self, Error> {
            Self::build::<W>(p.generators.clone(), p.randomness_generator.clone(), device)
        }
        fn build<W: ref_crh::Window>(generators: Vec<Vec<EdwardsProjective>>, randomness_generator: Vec<EdwardsProjective>, device: i32)
                                     -> Result<Self, Error> {
            let flat: Vec<EdwardsProjective> = generators.iter().flatten().cloned().collect();
            let (g, r) = (xy(&flat), xy(&randomness_generator));
            let mut raw = core::ptr::null_mut();
            check(unsafe {
                cpb_pedersen_ctx_create(0, W::WINDOW_SIZE as c_int, W::NUM_WINDOWS as c_int, g.as_ptr(), randomness_generator.len(),
                                        if r.is_empty() { core::ptr::null() } else { r.as_ptr() }, device, &mut raw)
            })?;
            Ok(Self { generators, randomness_generator, ctx: Arc::new(Ctx(raw)) })
        }
    }

    /// `crh::pedersen::CRH<EdwardsProjective, W>` (R/crh/pedersen/mod.rs:58-130).
    pub struct GpuPedersenCRH<W>(PhantomData<W>);
    impl<W: ref_crh::Window> GpuPedersenCRH<W> {
        /// n inputs of `len` bytes each, contiguous.
        pub fn evaluate_batch(p: &GpuPedersenParams, inputs: &[u8], len: usize) -> Result<Vec<EdwardsAffine>, Error> {
            let n = if len == 0 { 0 } else { inputs.len() / len };
            let mut out = vec![0u64; 8 * n];
            check(unsafe { cpb_pedersen_crh_batch(p.ctx.0, inputs.as_ptr(), len, len, out.as_mut_ptr(), n) })?;
            Ok(points(&out))
        }
    }
    impl<W: ref_crh::Window> CRHScheme for GpuPedersenCRH<W> {
        type Input = [u8];
        type Output = EdwardsAffine;
        type Parameters = GpuPedersenParams;
        fn setup<R: Rng>(rng: &mut R) -> Result<Self::Parameters, Error> {
            GpuPedersenParams::from_crh::<W>(&ref_crh::CRH::<EdwardsProjective, W>::setup(rng)?, 0)
        }
        fn evaluate<T: Borrow<[u8]>>(p: &Self::Parameters, input: T) -> Result<EdwardsAffine, Error> {
            let input = input.borrow();
            let mut out = [0u64; 8];
            check(unsafe { cpb_pedersen_crh_batch(p.ctx.0, input.as_ptr(), input.len(), input.len(), out.as_mut_ptr(), 1) })?;
            Ok(points(&out)[0])
        }
    }

    fn affine_limbs(points: &[EdwardsAffine]) -> Vec<u64> {
        points.iter().flat_map(|p| [p.x.mont_limbs(), p.y.mont_limbs()].concat()).collect()
    }

    /// `MerkleTree<JubJubMerkleTreeParams>` (R/merkle_tree/tests/mod.rs:19-33: byte leaves, pedersen::CRH leaf hash,
    /// ByteDigestConverter, pedersen::TwoToOneCRH inner nodes) built and updated on the GPU.  The ABI returns the reference's own two
    /// arrays (R/merkle_tree/mod.rs:383-395) of affine points, so proofs are the reference's index arithmetic.
    pub struct GpuPedersenMerkleTree {
        pub leaf_nodes: Vec<EdwardsAffine>,
        pub non_leaf_nodes: Vec<EdwardsAffine>,
        height: usize,
    }
    impl GpuPedersenMerkleTree {
        /// `MerkleTree::new` over leaves of one byte length (Pedersen zero-pads, R/crh/pedersen/mod.rs:94-99).
        pub fn new(leaf: &GpuPedersenParams, two_to_one: &GpuPedersenParams, leaves: &[Vec<u8>]) -> Result<Self, Error> {
            let n = leaves.len();
            let leaf_len = leaves.first().map_or(0, |l| l.len());
            assert!(leaves.iter().all(|l| l.len() == leaf_len), "leaves of one length");
            let flat: Vec<u8> = leaves.concat();
            let (mut ln, mut nn) = (vec![0u64; 8 * n], vec![0u64; 8 * n.saturating_sub(1)]);
            check(unsafe { cpb_merkle_pedersen_build(leaf.ctx.0, two_to_one.ctx.0, flat.as_ptr(), leaf_len, n, ln.as_mut_ptr(), nn.as_mut_ptr()) })?;
            Ok(Self { leaf_nodes: points(&ln), non_leaf_nodes: points(&nn), height: n.trailing_zeros() as usize + 1 })
        }
        pub fn root(&self) -> EdwardsAffine { self.non_leaf_nodes[0] }
        pub fn height(&self) -> usize { self.height }
        /// k x `MerkleTree::update` (R/merkle_tree/mod.rs:690-701) in one call: the new leaves and the touched nodes of every level
        /// are hashed on the GPU, and only those nodes and the siblings they read cross PCIe.  A repeated index takes its last leaf;
        /// new leaves of one length.
        pub fn update_batch(&mut self, leaf: &GpuPedersenParams, two_to_one: &GpuPedersenParams, indexes: &[usize], new_leaves: &[Vec<u8>])
                            -> Result<(), Error> {
            self.update_impl(leaf, two_to_one, indexes, new_leaves, None).map(|_| ())
        }
        pub fn update(&mut self, leaf: &GpuPedersenParams, two_to_one: &GpuPedersenParams, index: usize, new_leaf: &[u8]) -> Result<(), Error> {
            self.update_batch(leaf, two_to_one, &[index], &[new_leaf.to_vec()])
        }
        /// `MerkleTree::check_update` (mod.rs:706-725) for all k at once: the tree changes only when the new root equals
        /// `asserted_new_root`; returns whether it did.
        pub fn check_update_batch(&mut self, leaf: &GpuPedersenParams, two_to_one: &GpuPedersenParams, indexes: &[usize],
                                  new_leaves: &[Vec<u8>], asserted_new_root: &EdwardsAffine) -> Result<bool, Error> {
            self.update_impl(leaf, two_to_one, indexes, new_leaves, Some(asserted_new_root))
        }
        pub fn check_update(&mut self, leaf: &GpuPedersenParams, two_to_one: &GpuPedersenParams, index: usize, new_leaf: &[u8],
                            asserted_new_root: &EdwardsAffine) -> Result<bool, Error> {
            self.check_update_batch(leaf, two_to_one, &[index], &[new_leaf.to_vec()], asserted_new_root)
        }
        fn update_impl(&mut self, leaf: &GpuPedersenParams, two_to_one: &GpuPedersenParams, indexes: &[usize], new_leaves: &[Vec<u8>],
                       asserted_new_root: Option<&EdwardsAffine>) -> Result<bool, Error> {
            assert_eq!(indexes.len(), new_leaves.len(), "one new leaf per index");
            let leaf_len = new_leaves.first().map_or(0, |l| l.len());
            assert!(new_leaves.iter().all(|l| l.len() == leaf_len), "an update batch takes new leaves of one length");
            let idx: Vec<u64> = indexes.iter().map(|&i| i as u64).collect();
            let flat: Vec<u8> = new_leaves.concat();
            let (mut ln, mut nn) = (affine_limbs(&self.leaf_nodes), affine_limbs(&self.non_leaf_nodes));
            let root = asserted_new_root.map(|r| affine_limbs(&[*r]));
            let mut applied: c_int = 0;
            check(unsafe {
                cpb_merkle_pedersen_update(leaf.ctx.0, two_to_one.ctx.0, ln.as_mut_ptr(), nn.as_mut_ptr(), self.leaf_nodes.len(), idx.as_ptr(),
                                           flat.as_ptr(), leaf_len, idx.len(), root.as_ref().map_or(core::ptr::null(), |r| r.as_ptr()),
                                           &mut applied)
            })?;
            if applied != 0 {
                self.leaf_nodes = points(&ln);
                self.non_leaf_nodes = points(&nn);
            }
            Ok(applied != 0)
        }
    }

    /// `commitment::pedersen::Commitment<EdwardsProjective, W>` (R/commitment/pedersen/mod.rs:38-106).
    pub struct GpuPedersenCommitment<W>(PhantomData<W>);
    impl<W: ref_crh::Window> CommitmentScheme for GpuPedersenCommitment<W> {
        type Parameters = GpuPedersenParams;
        type Randomness = ref_comm::Randomness<EdwardsProjective>;
        type Output = EdwardsAffine;
        fn setup<R: Rng>(rng: &mut R) -> Result<Self::Parameters, Error> {
            GpuPedersenParams::from_commitment::<W>(&ref_comm::Commitment::<EdwardsProjective, W>::setup(rng)?, 0)
        }
        fn commit(p: &Self::Parameters, input: &[u8], randomness: &Self::Randomness) -> Result<EdwardsAffine, Error> {
            let r = randomness.0.into_bigint().to_bytes_le();          // the bits R/commitment/pedersen/mod.rs:93 iterates, 32 bytes
            let mut out = [0u64; 8];
            check(unsafe { cpb_pedersen_commit_batch(p.ctx.0, input.as_ptr(), input.len(), input.len(), r.as_ptr(), out.as_mut_ptr(), 1) })?;
            Ok(points(&out)[0])
        }
    }
}

/// `signature::schnorr::Schnorr<EdwardsProjective, Blake2s256>` and `encryption::elgamal::ElGamal<EdwardsProjective>` over Jubjub
/// (R/signature/schnorr/mod.rs, R/encryption/elgamal/mod.rs) on `cpb_te_base_ctx`.  SOURCE ONLY, like the rest of this crate.
/// Keys and signatures are the reference's own types, so a key pair or signature made here verifies with the reference and
/// the other way round.  Signing is not constant time (secret scalars select table entries by value), as the reference's.
pub mod signature {
    use super::{check, GpuField};
    use ark_crypto_primitives::encryption::{elgamal as ref_eg, AsymmetricEncryptionScheme};
    use ark_crypto_primitives::signature::{schnorr as ref_sig, SignatureScheme};
    use ark_crypto_primitives::Error;
    use ark_ec::AffineRepr;
    use ark_ed_on_bls12_381::{EdwardsAffine, EdwardsProjective, Fq, Fr};
    use ark_std::{rand::Rng, sync::Arc, UniformRand};
    use blake2::Blake2s256;
    use std::os::raw::c_int;

    #[allow(non_camel_case_types)]
    #[repr(C)]
    pub struct cpb_te_base_ctx {
        _private: [u8; 0],
    }
    extern "C" {
        fn cpb_te_base_ctx_create(curve_id: c_int, generator_xy: *const u64, device: c_int, out: *mut *mut cpb_te_base_ctx) -> c_int;
        fn cpb_te_base_ctx_destroy(ctx: *mut cpb_te_base_ctx);
        fn cpb_te_base_mul_batch(ctx: *mut cpb_te_base_ctx, scalars: *const u64, out_xy: *mut u64, n: usize) -> c_int;
        fn cpb_schnorr_sign_batch(ctx: *mut cpb_te_base_ctx, salt: *const u8, sks: *const u64, nonces: *const u64, msgs: *const u8,
                                  msg_offsets: *const u64, sigs_out: *mut u64, signed_out: *mut u8, n: usize) -> c_int;
        fn cpb_schnorr_verify_batch(ctx: *mut cpb_te_base_ctx, salt: *const u8, pks_xy: *const u64, msgs: *const u8, msg_offsets: *const u64,
                                    sigs: *const u64, ok_out: *mut u8, n: usize) -> c_int;
        fn cpb_schnorr_randomize_public_key_batch(ctx: *mut cpb_te_base_ctx, pks_xy: *const u64, randomness: *const u8, len: usize,
                                                  stride: usize, out_xy: *mut u64, n: usize) -> c_int;
        fn cpb_schnorr_randomize_signature_batch(ctx: *mut cpb_te_base_ctx, sigs: *const u64, randomness: *const u8, len: usize,
                                                 stride: usize, sigs_out: *mut u64, n: usize) -> c_int;
        fn cpb_elgamal_encrypt_batch(ctx: *mut cpb_te_base_ctx, pks_xy: *const u64, msgs_xy: *const u64, rands: *const u64,
                                     ciphertexts_out: *mut u64, n: usize) -> c_int;
        fn cpb_elgamal_decrypt_batch(ctx: *mut cpb_te_base_ctx, sks: *const u64, ciphertexts: *const u64, msgs_out: *mut u64, n: usize) -> c_int;
    }

    struct Ctx(*mut cpb_te_base_ctx);
    unsafe impl Send for Ctx {}
    unsafe impl Sync for Ctx {}
    impl Drop for Ctx {
        fn drop(&mut self) { unsafe { cpb_te_base_ctx_destroy(self.0) } }
    }

    fn xy(p: &EdwardsAffine) -> [u64; 8] {
        let (x, y) = p.xy().unwrap_or((Fq::from(0u64), Fq::from(1u64)));     // the identity is (0, 1)
        let mut out = [0u64; 8];
        out[..4].copy_from_slice(&x.mont_limbs());
        out[4..].copy_from_slice(&y.mont_limbs());
        out
    }
    fn point(l: &[u64]) -> EdwardsAffine {
        EdwardsAffine::new_unchecked(Fq::from_mont_limbs([l[0], l[1], l[2], l[3]]), Fq::from_mont_limbs([l[4], l[5], l[6], l[7]]))
    }

    /// A generator and its device tables (`cpb_te_base_ctx`).
    #[derive(Clone)]
    pub struct GpuBase {
        pub generator: EdwardsAffine,
        ctx: Arc<Ctx>,
    }
    impl GpuBase {
        pub fn new(generator: EdwardsAffine, device: i32) -> Result<Self, Error> {
            let g = xy(&generator);
            let mut raw = core::ptr::null_mut();
            check(unsafe { cpb_te_base_ctx_create(0, g.as_ptr(), device, &mut raw) })?;
            Ok(Self { generator, ctx: Arc::new(Ctx(raw)) })
        }
        fn mul(&self, s: &Fr) -> Result<EdwardsAffine, Error> {
            let mut out = [0u64; 8];
            check(unsafe { cpb_te_base_mul_batch(self.ctx.0, s.mont_limbs().as_ptr(), out.as_mut_ptr(), 1) })?;
            Ok(point(&out))
        }
    }

    /// `schnorr::Parameters` + device tables.
    #[derive(Clone)]
    pub struct GpuSchnorrParams {
        pub base: GpuBase,
        pub salt: [u8; 32],
    }
    impl GpuSchnorrParams {
        pub fn from_reference(p: &ref_sig::Parameters<EdwardsProjective, Blake2s256>, device: i32) -> Result<Self, Error> {
            Ok(Self { base: GpuBase::new(p.generator, device)?, salt: p.salt })
        }
    }

    fn sig_limbs(s: &ref_sig::Signature<EdwardsProjective>) -> [u64; 8] {
        let mut out = [0u64; 8];
        out[..4].copy_from_slice(&s.prover_response.mont_limbs());
        out[4..].copy_from_slice(&s.verifier_challenge.mont_limbs());
        out
    }
    fn sig_from(l: &[u64]) -> ref_sig::Signature<EdwardsProjective> {
        ref_sig::Signature {
            prover_response: Fr::from_mont_limbs([l[0], l[1], l[2], l[3]]),
            verifier_challenge: Fr::from_mont_limbs([l[4], l[5], l[6], l[7]]),
        }
    }

    pub struct GpuSchnorr;
    impl GpuSchnorr {
        /// Many messages at once: one verification per (pk, message, signature), one device call.
        pub fn verify_batch(pp: &GpuSchnorrParams, pks: &[EdwardsAffine], messages: &[&[u8]], sigs: &[ref_sig::Signature<EdwardsProjective>])
                            -> Result<Vec<bool>, Error> {
            let n = pks.len();
            assert!(messages.len() == n && sigs.len() == n);
            let pk: Vec<u64> = pks.iter().flat_map(xy).collect();
            let sg: Vec<u64> = sigs.iter().flat_map(sig_limbs).collect();
            let mut values: Vec<u8> = messages.concat();
            values.push(0);
            let mut off = vec![0u64];
            for m in messages {
                off.push(off[off.len() - 1] + m.len() as u64);
            }
            let mut ok = vec![0u8; n];
            check(unsafe {
                cpb_schnorr_verify_batch(pp.base.ctx.0, pp.salt.as_ptr(), pk.as_ptr(), values.as_ptr(), off.as_ptr(), sg.as_ptr(), ok.as_mut_ptr(), n)
            })?;
            Ok(ok.into_iter().map(|b| b != 0).collect())
        }
    }
    impl SignatureScheme for GpuSchnorr {
        type Parameters = GpuSchnorrParams;
        type PublicKey = EdwardsAffine;
        type SecretKey = ref_sig::SecretKey<EdwardsProjective>;
        type Signature = ref_sig::Signature<EdwardsProjective>;

        fn setup<R: Rng>(rng: &mut R) -> Result<Self::Parameters, Error> {
            GpuSchnorrParams::from_reference(&ref_sig::Schnorr::<EdwardsProjective, Blake2s256>::setup(rng)?, 0)
        }
        fn keygen<R: Rng>(pp: &Self::Parameters, rng: &mut R) -> Result<(Self::PublicKey, Self::SecretKey), Error> {
            let sk = Fr::rand(rng);
            Ok((pp.base.mul(&sk)?, ref_sig::SecretKey(sk)))
        }
        /// mod.rs:80-115: draw a nonce, one device call, redraw while the challenge is not a field element.
        fn sign<R: Rng>(pp: &Self::Parameters, sk: &Self::SecretKey, message: &[u8], rng: &mut R) -> Result<Self::Signature, Error> {
            let off = [0u64, message.len() as u64];
            let mut values = message.to_vec();
            values.push(0);
            loop {
                let k = Fr::rand(rng);
                let (mut sig, mut signed) = ([0u64; 8], 0u8);
                check(unsafe {
                    cpb_schnorr_sign_batch(pp.base.ctx.0, pp.salt.as_ptr(), sk.0.mont_limbs().as_ptr(), k.mont_limbs().as_ptr(), values.as_ptr(),
                                           off.as_ptr(), sig.as_mut_ptr(), &mut signed, 1)
                })?;
                if signed != 0 {
                    return Ok(sig_from(&sig));
                }
            }
        }
        fn verify(pp: &Self::Parameters, pk: &Self::PublicKey, message: &[u8], signature: &Self::Signature) -> Result<bool, Error> {
            Ok(GpuSchnorr::verify_batch(pp, &[*pk], &[message], core::slice::from_ref(signature))?[0])
        }
        fn randomize_public_key(pp: &Self::Parameters, public_key: &Self::PublicKey, randomness: &[u8]) -> Result<Self::PublicKey, Error> {
            let (pk, mut out) = (xy(public_key), [0u64; 8]);
            check(unsafe {
                cpb_schnorr_randomize_public_key_batch(pp.base.ctx.0, pk.as_ptr(), randomness.as_ptr(), randomness.len(), randomness.len(),
                                                       out.as_mut_ptr(), 1)
            })?;
            Ok(point(&out))
        }
        fn randomize_signature(pp: &Self::Parameters, signature: &Self::Signature, randomness: &[u8]) -> Result<Self::Signature, Error> {
            let (sg, mut out) = (sig_limbs(signature), [0u64; 8]);
            check(unsafe {
                cpb_schnorr_randomize_signature_batch(pp.base.ctx.0, sg.as_ptr(), randomness.as_ptr(), randomness.len(), randomness.len(),
                                                      out.as_mut_ptr(), 1)
            })?;
            Ok(sig_from(&out))
        }
    }

    /// `encryption::elgamal::ElGamal<EdwardsProjective>` (R/encryption/elgamal/mod.rs:34-101).
    pub struct GpuElGamal;
    impl AsymmetricEncryptionScheme for GpuElGamal {
        type Parameters = GpuBase;
        type PublicKey = EdwardsAffine;
        type SecretKey = ref_eg::SecretKey<EdwardsProjective>;
        type Randomness = ref_eg::Randomness<EdwardsProjective>;
        type Plaintext = EdwardsAffine;
        type Ciphertext = (EdwardsAffine, EdwardsAffine);

        fn setup<R: Rng>(rng: &mut R) -> Result<Self::Parameters, Error> {
            GpuBase::new(ref_eg::ElGamal::<EdwardsProjective>::setup(rng)?.generator, 0)
        }
        fn keygen<R: Rng>(pp: &Self::Parameters, rng: &mut R) -> Result<(Self::PublicKey, Self::SecretKey), Error> {
            let sk = Fr::rand(rng);
            Ok((pp.mul(&sk)?, ref_eg::SecretKey(sk)))
        }
        fn encrypt(pp: &Self::Parameters, pk: &Self::PublicKey, message: &Self::Plaintext, r: &Self::Randomness) -> Result<Self::Ciphertext, Error> {
            let (p, m, mut out) = (xy(pk), xy(message), [0u64; 16]);
            check(unsafe { cpb_elgamal_encrypt_batch(pp.ctx.0, p.as_ptr(), m.as_ptr(), r.0.mont_limbs().as_ptr(), out.as_mut_ptr(), 1) })?;
            Ok((point(&out[..8]), point(&out[8..])))
        }
        fn decrypt(pp: &Self::Parameters, sk: &Self::SecretKey, ciphertext: &Self::Ciphertext) -> Result<Self::Plaintext, Error> {
            let mut ct = [0u64; 16];
            ct[..8].copy_from_slice(&xy(&ciphertext.0));
            ct[8..].copy_from_slice(&xy(&ciphertext.1));
            let mut out = [0u64; 8];
            check(unsafe { cpb_elgamal_decrypt_batch(pp.ctx.0, sk.0.mont_limbs().as_ptr(), ct.as_ptr(), out.as_mut_ptr(), 1) })?;
            Ok(point(&out))
        }
    }
}
