//! `ark-b200`: H100 (sm_90a) backend for the two data-parallel hot paths of arkworks-rs/algebra.
//!
//! * MSM — `B200<C>` wraps any `SWCurveConfig` whose base field is a 4- or 6-limb `Fp` and overrides the one hook
//!   the reference provides for specialised back-ends, `SWCurveConfig::msm`
//!   (ec/src/models/short_weierstrass/mod.rs:111-119; `impl VariableBaseMSM for Projective<P>` forwards to it,
//!   group.rs:650-657).  Every other overridable item of the trait — constants, `mul_by_a`, `add_b`, the subgroup check,
//!   `clear_cofactor`, `mul_projective` / `mul_affine` (GLV for BLS12-381) and the three serialization hooks (zkcrypto wire
//!   format for BLS12-381, curves/bls12_381/src/curves/g1.rs:96-156) — is forwarded to `C`, so `Affine<B200<C>>` behaves and
//!   serializes exactly like `Affine<C>`.  The MSM uses every GPU of the node (`b200_msm_sw_g1_multi`).
//! * NTT — `B200Radix2Domain<F>` wraps `Radix2EvaluationDomain<F>` and implements `EvaluationDomain<F>`
//!   (poly/src/domain/mod.rs:31-329); `fft_in_place` / `ifft_in_place` resize exactly like radix2/mod.rs:140-153,
//!   then hand the limb slice to the GPU when `T == F` (`b200_ntt_fr`) or when `T` is G1 `Projective` of BLS12-381 or BN254
//!   (or of `B200<..>` of them) whose scalar field is `F` (`b200_ntt_g1`, FFTs over group elements as in poly/src/test.rs:57,
//!   e.g. an SRS to its Lagrange basis), and fall back to the inner CPU domain for any other `DomainCoeff` (G2 included).
//!
//! Data crosses the FFI as arkworks' in-memory Montgomery limbs (no serialization): `Fp<MontBackend<_,N>,N>` is
//! `BigInt<N>([u64; N])` + a ZST, `Affine<P>` is `{x, y, infinity: ()}` with the identity stored as (0,0).
//! These are `repr(Rust)`, so the slice casts below are guarded by size/offset assertions evaluated once.
use ark_ec::short_weierstrass::{Affine, Projective, SWCurveConfig};
use ark_ec::CurveConfig;
use ark_ff::{FftField, PrimeField};
use ark_poly::{domain::DomainCoeff, EvaluationDomain, Radix2EvaluationDomain};
use ark_serialize::{CanonicalDeserialize, CanonicalSerialize, Compress, SerializationError, Validate};
use ark_std::io::{Read, Write};
use ark_std::marker::PhantomData;

pub mod ffi;

/// Curves the CUDA library has kernels for.
pub trait B200Curve: SWCurveConfig {
    const CURVE_ID: core::ffi::c_int;
    /// u64 limbs of the base field
    const N: usize;
}
impl B200Curve for ark_bls12_381::g1::Config { const CURVE_ID: core::ffi::c_int = ffi::B200_CURVE_BLS12_381; const N: usize = 6; }
impl B200Curve for ark_bn254::g1::Config { const CURVE_ID: core::ffi::c_int = ffi::B200_CURVE_BN254; const N: usize = 4; }
/// G2 of BLS12-381: coordinates in Fq2 = 2 x 6 limbs (QuadExtField { c0, c1 }), N counts u64 per coordinate.
impl B200Curve for ark_bls12_381::g2::Config { const CURVE_ID: core::ffi::c_int = ffi::B200_CURVE_BLS12_381_G2; const N: usize = 12; }

#[inline]
fn to_inner<C: B200Curve>(p: &Affine<B200<C>>) -> Affine<C> {
    // same coordinates, same ZeroFlag = (): the identity stays (0, 0)
    Affine::<C>::new_unchecked(p.x, p.y)
}
#[inline]
fn from_inner<C: B200Curve>(p: Affine<C>) -> Affine<B200<C>> {
    Affine::<B200<C>>::new_unchecked(p.x, p.y)
}
#[inline]
fn proj_to_inner<C: B200Curve>(p: &Projective<B200<C>>) -> Projective<C> {
    Projective::<C>::new_unchecked(p.x, p.y, p.z)
}
#[inline]
fn proj_from_inner<C: B200Curve>(p: Projective<C>) -> Projective<B200<C>> {
    Projective::<B200<C>>::new_unchecked(p.x, p.y, p.z)
}

/// `B200<C>`: same curve as `C`, MSM on the GPU.
#[derive(Clone, Copy, Debug, Default, PartialEq, Eq)]
pub struct B200<C>(PhantomData<C>);

impl<C: B200Curve> CurveConfig for B200<C> {
    type BaseField = C::BaseField;
    type ScalarField = C::ScalarField;
    const COFACTOR: &'static [u64] = C::COFACTOR;
    const COFACTOR_INV: Self::ScalarField = C::COFACTOR_INV;
}

impl<C: B200Curve> SWCurveConfig for B200<C> {
    const COEFF_A: Self::BaseField = C::COEFF_A;
    const COEFF_B: Self::BaseField = C::COEFF_B;
    const GENERATOR: Affine<Self> = Affine::new_unchecked(C::GENERATOR.x, C::GENERATOR.y);
    type ZeroFlag = ();

    #[inline(always)]
    fn mul_by_a(elem: Self::BaseField) -> Self::BaseField { C::mul_by_a(elem) }
    #[inline(always)]
    fn add_b(elem: Self::BaseField) -> Self::BaseField { C::add_b(elem) }
    fn is_in_correct_subgroup_assuming_on_curve(item: &Affine<Self>) -> bool {
        C::is_in_correct_subgroup_assuming_on_curve(&to_inner::<C>(item))
    }
    fn clear_cofactor(item: &Affine<Self>) -> Affine<Self> { from_inner::<C>(C::clear_cofactor(&to_inner::<C>(item))) }
    fn mul_projective(base: &Projective<Self>, scalar: &[u64]) -> Projective<Self> {
        proj_from_inner::<C>(C::mul_projective(&proj_to_inner::<C>(base), scalar))
    }
    fn mul_affine(base: &Affine<Self>, scalar: &[u64]) -> Projective<Self> {
        proj_from_inner::<C>(C::mul_affine(&to_inner::<C>(base), scalar))
    }
    fn serialize_with_mode<W: Write>(item: &Affine<Self>, writer: W, compress: Compress) -> Result<(), SerializationError> {
        C::serialize_with_mode(&to_inner::<C>(item), writer, compress)
    }
    fn deserialize_with_mode<R: Read>(reader: R, compress: Compress, validate: Validate) -> Result<Affine<Self>, SerializationError> {
        C::deserialize_with_mode(reader, compress, validate).map(from_inner::<C>)
    }
    fn serialized_size(compress: Compress) -> usize { C::serialized_size(compress) }

    /// The plugin hook.  Length mismatch -> `Err(min_len)` exactly like the default body (variable_base/mod.rs:73-77).
    fn msm(bases: &[Affine<Self>], scalars: &[Self::ScalarField]) -> Result<Projective<Self>, usize> {
        if bases.len() != scalars.len() {
            return Err(bases.len().min(scalars.len()));
        }
        Ok(msm_raw::<C, Self>(bases, scalars))
    }
}

/// Free-function form for callers that hold `ark_bls12_381::G1Affine` slices (no type change needed).
pub fn msm_b200<C: B200Curve>(bases: &[Affine<C>], scalars: &[C::ScalarField]) -> Result<Projective<C>, usize> {
    if bases.len() != scalars.len() {
        return Err(bases.len().min(scalars.len()));
    }
    Ok(msm_raw::<C, C>(bases, scalars))
}

fn msm_raw<C: B200Curve, P: SWCurveConfig<BaseField = C::BaseField, ScalarField = C::ScalarField>>(
    bases: &[Affine<P>],
    scalars: &[P::ScalarField],
) -> Projective<P> {
    let n = bases.len();
    layout_checks::<C, P>();
    let mut out = [0u64; 36];   // 3 coordinates x N <= 12 limbs
    // One process drives every GPU of the node: the pairs are sharded by contiguous chunk, the partial sums are added on
    // device 0.  Small inputs stay on one device (a second device costs more in launch latency than it saves).
    let ngpus = if n >= (1 << 22) { unsafe { ffi::b200_device_count() }.max(1) } else { 1 };
    // SAFETY: layout_checks() proved Affine<P> == [u64; 2N] (x then y) and ScalarField == [u64; 4], Montgomery form.
    let rc = unsafe {
        ffi::b200_msm_sw_g1_multi(C::CURVE_ID, ngpus, bases.as_ptr() as *const u64, scalars.as_ptr() as *const u64, n, out.as_mut_ptr())
    };
    ffi::check(rc);
    let limb = |k: usize| -> P::BaseField {
        // new_unchecked keeps the Montgomery limbs as they are (ff/src/fields/models/fp/mod.rs:117-121)
        let mut v = P::BaseField::default();
        unsafe { core::ptr::copy_nonoverlapping(out.as_ptr().add(k * C::N), &mut v as *mut _ as *mut u64, C::N) };
        v
    };
    Projective::<P>::new_unchecked(limb(0), limb(1), limb(2))
}

fn layout_checks<C: B200Curve, P: SWCurveConfig>() {
    use core::mem::{align_of, size_of};
    assert_eq!(size_of::<P::BaseField>(), 8 * C::N);
    assert_eq!(size_of::<P::ScalarField>(), 32);
    assert_eq!(size_of::<Affine<P>>(), 16 * C::N);
    assert_eq!(align_of::<Affine<P>>(), 8);
    let probe = Affine::<P>::identity();
    let base = &probe as *const _ as usize;
    assert_eq!(&probe.x as *const _ as usize - base, 0, "Affine.x must be at offset 0");
    assert_eq!(&probe.y as *const _ as usize - base, 8 * C::N, "Affine.y must follow x");
}

/// Scalar fields the NTT kernels exist for.
pub trait B200FftField: FftField + PrimeField {
    const FIELD_ID: core::ffi::c_int;
}
impl B200FftField for ark_bls12_381::Fr { const FIELD_ID: core::ffi::c_int = ffi::B200_FIELD_BLS12_381_FR; }
impl B200FftField for ark_bn254::Fr { const FIELD_ID: core::ffi::c_int = ffi::B200_FIELD_BN254_FR; }

#[derive(Copy, Clone, Hash, Eq, PartialEq, Debug, CanonicalSerialize, CanonicalDeserialize)]
pub struct B200Radix2Domain<F: B200FftField>(pub Radix2EvaluationDomain<F>);

impl<F: B200FftField> B200Radix2Domain<F> {
    fn gpu<T: DomainCoeff<F>>(&self, x: &mut [T], inverse: bool) -> bool {
        let off = self.0.coset_offset();
        let offp = if off.is_one() { core::ptr::null() } else { &off as *const F as *const u64 };
        // Rust has no specialisation and T is not 'static: compare type names + sizes to detect T == F or a G1 point type.
        let rc = if core::any::type_name::<T>() == core::any::type_name::<F>() && core::mem::size_of::<T>() == 32 {
            unsafe { ffi::b200_ntt_fr(F::FIELD_ID, x.as_mut_ptr() as *mut u64, self.0.log_size_of_group, inverse as i32, offp) }
        } else if let Some(curve) = g1_point_curve::<F, T>() {
            unsafe { ffi::b200_ntt_g1(curve, x.as_mut_ptr() as *mut u64, self.0.log_size_of_group, inverse as i32, offp) }
        } else {
            return false;
        };
        ffi::check(rc);
        true
    }
}

/// The curve id when `T` is `Projective` of a G1 the library has point-FFT kernels for (directly or through `B200<..>`) and its
/// scalar field is `F`; the point layout (x, y, z, each N Montgomery limbs) is asserted before the slice is handed over.
fn g1_point_curve<F: B200FftField, T>() -> Option<core::ffi::c_int> {
    fn is<C: B200Curve, F: B200FftField, T>() -> bool {
        use core::any::type_name;
        let named = type_name::<T>() == type_name::<Projective<C>>() || type_name::<T>() == type_name::<Projective<B200<C>>>();
        if !named || type_name::<C::ScalarField>() != type_name::<F>() {
            return false;
        }
        projective_layout_checks::<C>();
        core::mem::size_of::<T>() == 24 * C::N
    }
    if is::<ark_bls12_381::g1::Config, F, T>() {
        Some(ffi::B200_CURVE_BLS12_381)
    } else if is::<ark_bn254::g1::Config, F, T>() {
        Some(ffi::B200_CURVE_BN254)
    } else {
        None
    }
}

fn projective_layout_checks<C: B200Curve>() {
    use core::mem::size_of;
    assert_eq!(size_of::<Projective<C>>(), 24 * C::N);
    assert_eq!(size_of::<Projective<B200<C>>>(), 24 * C::N);
    let probe = Projective::<C>::default();
    let base = &probe as *const _ as usize;
    assert_eq!(&probe.x as *const _ as usize - base, 0, "Projective.x must be at offset 0");
    assert_eq!(&probe.y as *const _ as usize - base, 8 * C::N, "Projective.y must follow x");
    assert_eq!(&probe.z as *const _ as usize - base, 16 * C::N, "Projective.z must follow y");
}

impl<F: B200FftField> EvaluationDomain<F> for B200Radix2Domain<F> {
    type Elements = <Radix2EvaluationDomain<F> as EvaluationDomain<F>>::Elements;
    fn new(num_coeffs: usize) -> Option<Self> { Radix2EvaluationDomain::new(num_coeffs).map(Self) }
    fn get_coset(&self, offset: F) -> Option<Self> { self.0.get_coset(offset).map(Self) }
    fn compute_size_of_domain(num_coeffs: usize) -> Option<usize> { Radix2EvaluationDomain::<F>::compute_size_of_domain(num_coeffs) }
    fn size(&self) -> usize { self.0.size() }
    fn log_size_of_group(&self) -> u64 { self.0.log_size_of_group() }
    fn size_inv(&self) -> F { self.0.size_inv() }
    fn group_gen(&self) -> F { self.0.group_gen() }
    fn group_gen_inv(&self) -> F { self.0.group_gen_inv() }
    fn coset_offset(&self) -> F { self.0.coset_offset() }
    fn coset_offset_inv(&self) -> F { self.0.coset_offset_inv() }
    fn coset_offset_pow_size(&self) -> F { self.0.coset_offset_pow_size() }
    fn elements(&self) -> Self::Elements { self.0.elements() }

    fn fft_in_place<T: DomainCoeff<F>>(&self, coeffs: &mut Vec<T>) {
        // same resize as radix2/mod.rs:140-147 (the degree-aware route computes the same values)
        coeffs.resize(self.size(), T::zero());
        if !self.gpu(coeffs.as_mut_slice(), false) {
            self.0.fft_in_place(coeffs)
        }
    }
    fn ifft_in_place<T: DomainCoeff<F>>(&self, evals: &mut Vec<T>) {
        evals.resize(self.size(), T::zero());
        if !self.gpu(evals.as_mut_slice(), true) {
            self.0.ifft_in_place(evals)
        }
    }
}

/// Bases kept in HBM across MSM calls (an SRS), sharded over every GPU: `b200_bases_upload` / `b200_msm_bases`.
pub struct ResidentBases<C: B200Curve> {
    handle: *mut ffi::b200_bases_t,
    len: usize,
    _c: PhantomData<C>,
}
impl<C: B200Curve> ResidentBases<C> {
    pub fn upload(bases: &[Affine<C>]) -> Self {
        layout_checks::<C, C>();
        let mut handle = core::ptr::null_mut();
        let ngpus = unsafe { ffi::b200_device_count() }.max(1);
        ffi::check(unsafe { ffi::b200_bases_upload(C::CURVE_ID, ngpus, bases.as_ptr() as *const u64, bases.len(), &mut handle) });
        Self { handle, len: bases.len(), _c: PhantomData }
    }
    /// `VariableBaseMSM::msm` against the resident bases: `Err(min_len)` on a length mismatch (variable_base/mod.rs:73-77).
    pub fn msm(&self, scalars: &[C::ScalarField]) -> Result<Projective<C>, usize> {
        if scalars.len() != self.len {
            return Err(scalars.len().min(self.len));
        }
        let mut out = [0u64; 36];
        ffi::check(unsafe {
            ffi::b200_msm_bases(self.handle, ffi::B200_SCALARS_FR_MONT, scalars.as_ptr() as *const core::ffi::c_void, scalars.len(), out.as_mut_ptr())
        });
        let limb = |k: usize| -> C::BaseField {
            let mut v = C::BaseField::default();
            unsafe { core::ptr::copy_nonoverlapping(out.as_ptr().add(k * C::N), &mut v as *mut _ as *mut u64, C::N) };
            v
        };
        Ok(Projective::<C>::new_unchecked(limb(0), limb(1), limb(2)))
    }
}
impl<C: B200Curve> Drop for ResidentBases<C> {
    fn drop(&mut self) {
        unsafe { ffi::b200_bases_free(self.handle) };
    }
}

/// Bucket slice `slice` of `slices` of the MSM over inputs that every caller holds in full (an SRS replicated on every GPU,
/// one process or thread per device): the `slices` results add up to `msm_b200`.  `b200_set_msm_bucket_slice` + the
/// streaming entry points, which run on the calling thread's current device.
pub fn msm_bucket_slice_b200<C: B200Curve>(bases: &[Affine<C>], scalars: &[C::ScalarField], slice: usize, slices: usize) -> Result<Projective<C>, usize> {
    if bases.len() != scalars.len() {
        return Err(bases.len().min(scalars.len()));
    }
    ffi::check(unsafe { ffi::b200_set_msm_bucket_slice(slice as i32, slices as i32) });
    let out = msm_chunks_b200::<C>(bases, scalars, bases.len().max(1));
    ffi::check(unsafe { ffi::b200_set_msm_bucket_slice(0, 1) });
    Ok(out)
}

/// `VariableBaseMSM::msm_chunks` (variable_base/mod.rs:119-150) on the streaming entry points: every chunk of `step` pairs is
/// pushed (H2D under the previous chunk's arithmetic), one bucket reduction at the end.
pub fn msm_chunks_b200<C: B200Curve>(bases: &[Affine<C>], scalars: &[C::ScalarField], step: usize) -> Projective<C> {
    assert!(scalars.len() <= bases.len());   // same precondition as the reference
    layout_checks::<C, C>();
    let bases = &bases[bases.len() - scalars.len()..];   // `skip(bases.len() - scalars.len())`
    let mut s = core::ptr::null_mut();
    ffi::check(unsafe { ffi::b200_msm_stream_begin(C::CURVE_ID, ffi::B200_SCALARS_FR_MONT, scalars.len(), step.max(1), &mut s) });
    for (b, k) in bases.chunks(step.max(1)).zip(scalars.chunks(step.max(1))) {
        ffi::check(unsafe { ffi::b200_msm_stream_push(s, b.as_ptr() as *const u64, k.as_ptr() as *const core::ffi::c_void, b.len()) });
    }
    let mut out = [0u64; 36];
    ffi::check(unsafe { ffi::b200_msm_stream_finish(s, out.as_mut_ptr()) });
    let limb = |k: usize| -> C::BaseField {
        let mut v = C::BaseField::default();
        unsafe { core::ptr::copy_nonoverlapping(out.as_ptr().add(k * C::N), &mut v as *mut _ as *mut u64, C::N) };
        v
    };
    Projective::<C>::new_unchecked(limb(0), limb(1), limb(2))
}
