/*
 * algebra_b200.h — C ABI of the H100-native (sm_90a) backend for the arkworks-rs/algebra hot path
 * (variable-base MSM over short-Weierstrass G1, radix-2 NTT over the scalar field).
 *
 * This is the boundary a Rust backend crate binds with `extern "C"` (see INTEGRATION.md).  Plain
 * pointers and sizes only; no torch / CUDA types in any signature (streams travel as void*).
 *
 * Data layout = arkworks' in-memory layout (NOT ark-serialize bytes):
 *   Fp<MontBackend<_,N>,N>  = N little-endian u64 limbs, Montgomery form (R = 2^(64N)), value < p
 *                             (ff/src/fields/models/fp/mod.rs:107-115, ff/src/biginteger/mod.rs:34)
 *   Affine<P>               = x limbs, then y limbs; the identity is (0,0) when ZeroFlag = ()
 *                             (ec/src/models/short_weierstrass/affine.rs:30-37,91-104)
 *   Projective<P>           = x, y, z limbs (Jacobian); z == 0 is the identity and is returned as
 *                             (R, R, 0) like `Projective::zero()` (group.rs:142-158)
 * N = 6 for BLS12-381 Fq, 4 for BLS12-381 Fr / BN254 Fq / BN254 Fr.
 *
 * Every function returns 0 on success, a negative B200_E* code on argument errors and a positive
 * cudaError_t value on CUDA failures; b200_last_error() gives the message.  All entry points are
 * thread-safe (per-device context behind a mutex).  There is no CPU fallback: without a CUDA device
 * every compute entry point fails with a CUDA error.
 */
#ifndef ALGEBRA_B200_H
#define ALGEBRA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* group ids                      reference parameters                                         */
#define B200_CURVE_BLS12_381 0 /* G1: curves/bls12_381/src/curves/g1.rs:28-95                  */
#define B200_CURVE_BN254 1     /* G1: curves/bn254/src/curves/g1.rs:16-90                      */
#define B200_CURVE_BLS12_381_G2 2 /* G2: curves/bls12_381/src/curves/g2.rs:54; coordinates in Fq2 = (c0, c1), each 6 u64
                                   * (ff/src/fields/models/quadratic_extension.rs:105-113), i.e. "N" = 12 u64 per coordinate */
/* scalar-field ids for the NTT */
#define B200_FIELD_BLS12_381_FR 0 /* curves/bls12_381/src/fields/fr.rs, TWO_ADICITY = 32        */
#define B200_FIELD_BN254_FR 1     /* curves/bn254/src/fields/fr.rs,     TWO_ADICITY = 28        */

#define B200_EINVAL (-1)      /* bad id / null pointer                                          */
#define B200_ETOOLARGE (-2)   /* log_n > TWO_ADICITY: Radix2EvaluationDomain::new returns None  */
#define B200_ENOMEM (-3)

const char *b200_version(void);
const char *b200_last_error(void);

/* ---------------------------------------------------------------------------------------------
 * MSM — replaces the body of `SWCurveConfig::msm` (ec/src/models/short_weierstrass/mod.rs:111-119),
 * i.e. `VariableBaseMSM::msm_unchecked` (ec/src/scalar_mul/variable_base/mod.rs:59-64) for
 * Projective<P>: sum_i scalars[i] * bases[i] over the first n pairs.  The caller does the
 * `bases.len() == scalars.len()` check and maps a mismatch to Err(min_len) (:73-77).
 *   bases   n x 2N u64  (affine, Montgomery)        scalars  n x 4 u64 (Fr, Montgomery)
 *   out_xyz 3N u64      (Jacobian, Montgomery)
 * The result is the same group element the reference computes (limb-identical after into_affine()).
 * --------------------------------------------------------------------------------------------- */
int b200_msm_sw_g1(int curve, const uint64_t *bases, const uint64_t *scalars, size_t n, uint64_t *out_xyz);

/* Same, operands already resident in device memory of the current device (bases can be uploaded once
 * and reused, the analogue of holding `&[G1Affine]` across calls); out_xyz is a HOST pointer.
 * `stream` is a cudaStream_t passed as void* (NULL = default stream).  Synchronises before returning. */
int b200_msm_sw_g1_dev(int curve, const void *d_bases, const void *d_scalars, size_t n, uint64_t *out_xyz,
                       void *stream);

/* The rest of the VariableBaseMSM surface (ec/src/scalar_mul/variable_base/mod.rs:80-115), which the reference does NOT route
 * through the SWCurveConfig::msm hook: scalars given as canonical BigInt<4> (`msm_bigint`) or as small unsigned integers
 * (`msm_u1` = bool bytes use U8, `msm_u8`, `msm_u16`, `msm_u32`, `msm_u64`).  Small kinds use ceil(bits/c) windows only.
 *   scalars: n elements of 32 B (FR_MONT, BIGINT) or 1/2/4/8 B (U8..U64)                                                  */
#define B200_SCALARS_FR_MONT 0
#define B200_SCALARS_BIGINT 1
#define B200_SCALARS_U8 2
#define B200_SCALARS_U16 3
#define B200_SCALARS_U32 4
#define B200_SCALARS_U64 5
int b200_msm_sw_g1_scalars(int curve, int scalar_kind, const uint64_t *bases, const void *scalars, size_t n, uint64_t *out_xyz);
int b200_msm_sw_g1_scalars_dev(int curve, int scalar_kind, const void *d_bases, const void *d_scalars, size_t n, uint64_t *out_xyz,
                               void *stream);

/* G2 of BLS12-381 through the same pipeline (SWCurveConfig::msm hook of g2::Config, same file:line as above): affine points are
 * x.c0, x.c1, y.c0, y.c1 (24 u64), the result is a Jacobian point over Fq2 (36 u64).  b200_g1_sum / b200_g1_into_affine accept
 * B200_CURVE_BLS12_381_G2 as well (36 -> 24 u64). */
int b200_msm_sw_g2(const uint64_t *bases, const uint64_t *scalars, size_t n, uint64_t *out_xyz);
int b200_msm_sw_g2_dev(const void *d_bases, const void *d_scalars, size_t n, uint64_t *out_xyz, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Multi-GPU and resident-bases entry points: ONE process, one host thread + two streams per device, no torch, no NCCL —
 * the partial sums come back to the host as 3N u64 each and are added on device 0 (Projective::add_assign).  This is what a
 * Rust caller of `SWCurveConfig::msm` (ec/src/models/short_weierstrass/mod.rs:111-119) binds to use every GPU of the node.
 *   ngpus   1 .. b200_device_count(); the n pairs are split into ngpus contiguous shards
 * Host buffers may be pinned or pageable: pageable memory is staged through a per-device ring of pinned buffers filled by
 * several host threads, so the PCIe copy of one slice overlaps the memcpy of the next.
 * --------------------------------------------------------------------------------------------- */
int b200_device_count(void);
int b200_msm_sw_g1_multi(int curve, int ngpus, const uint64_t *bases, const uint64_t *scalars, size_t n, uint64_t *out_xyz);
/* Bases uploaded once and kept in HBM (sharded over ngpus devices), the analogue of holding `&[G1Affine]` (an SRS) across
 * calls; b200_msm_bases then moves only the scalars (n <= the handle's size; the first n bases are used, like msm_unchecked). */
typedef struct b200_bases b200_bases_t;
int b200_bases_upload(int curve, int ngpus, const uint64_t *bases, size_t n, b200_bases_t **handle);
int b200_msm_bases(const b200_bases_t *handle, int scalar_kind, const void *scalars, size_t n, uint64_t *out_xyz);
int b200_bases_free(b200_bases_t *handle);

/* Streaming MSM — `VariableBaseMSM::msm_chunks` (ec/src/scalar_mul/variable_base/mod.rs:119-150) and `ChunkedPippenger`
 * (stream_pippenger.rs:10-66) without a full reduce per chunk: every pushed chunk is copied (H2D of chunk k+1 under the
 * arithmetic of chunk k), digit-sorted and accumulated into ONE set of buckets; the bucket reduction and window combine run
 * once in finish.  n_total_hint (0 = unknown -> max_chunk) picks the window; every push must have n <= max_chunk.
 * finish and abort release the handle. */
typedef struct b200_msm_stream b200_msm_stream_t;
int b200_msm_stream_begin(int curve, int scalar_kind, size_t n_total_hint, size_t max_chunk, b200_msm_stream_t **stream);
int b200_msm_stream_push(b200_msm_stream_t *stream, const uint64_t *bases, const void *scalars, size_t n);
int b200_msm_stream_finish(b200_msm_stream_t *stream, uint64_t *out_xyz);
int b200_msm_stream_abort(b200_msm_stream_t *stream);

/* Pippenger window size c used by subsequent MSM calls on this thread's device: 0 = automatic.
 * (The reference's rule is ln_without_floats(n)+2, ec/src/scalar_mul/variable_base/mod.rs:445-449; any c
 * yields the same group element.)  b200_msm_window_for(n) reports what "automatic" picks. */
int b200_set_msm_window(int c);
int b200_msm_window_for(int curve, size_t n);
/* Number of batched-affine pre-reduction levels run between the sort and the XYZZ accumulation (each level halves the
 * bucket runs with affine additions sharing one inversion per batch): 0 = off, -1 = automatic.  Result-neutral. */
int b200_set_msm_affine_levels(int levels);
/* Bucket slicing, the second way an MSM shards (the first: input chunks, b200_msm_sw_g1_multi).  After
 * b200_set_msm_bucket_slice(s, S) the single-device MSM entry points called on this thread accumulate and reduce only the
 * buckets [nb*s/S, nb*(s+1)/S) of every Pippenger window (window_sums, variable_base/mod.rs:456-487, restricted to a bucket
 * range), so the S results over the SAME bases and scalars add up (b200_g1_sum) to the complete msm.  Every phase after the
 * digit extraction shrinks by 1/S, including the per-bucket reduction that input-chunk sharding repeats on every device:
 * the better split when the inputs are already resident (replicated) on every GPU.  (0, 1) = whole MSM, the default.
 * The multi-device and resident-bases entry points ignore the setting. */
int b200_set_msm_bucket_slice(int slice, int slices);

/* sum of k Jacobian points (k x 3N u64, host) -> out_xyz: the local "reduce" after the multi-GPU
 * all-gather of per-rank partial sums (Projective::add_assign, group.rs:450-538). */
int b200_g1_sum(int curve, const uint64_t *points_xyz, size_t k, uint64_t *out_xyz);
/* Jacobian -> affine (affine.rs:374-396): 3N u64 in, 2N u64 out; identity -> (0,0). */
int b200_g1_into_affine(int curve, const uint64_t *xyz, uint64_t *out_xy);

/* ---------------------------------------------------------------------------------------------
 * NTT — replaces Radix2EvaluationDomain::{fft_in_place, ifft_in_place} after their resize step
 * (poly/src/domain/radix2/mod.rs:140-153; fft.rs:74-88): natural order in, natural order out,
 *   forward: out[i] = sum_j in[j] * (h * g^i)^j          inverse: the exact inverse incl. 1/n,
 * g = get_root_of_unity(2^log_n) (ff/src/fields/fft_friendly.rs:66-82), h = coset offset.
 *   data          2^log_n x 4 u64 (Montgomery Fr), transformed in place
 *   coset_offset  NULL (h = 1) or 4 u64 Montgomery limbs of h (domain.coset_offset())
 * Returns B200_ETOOLARGE when log_n > TWO_ADICITY (where Radix2EvaluationDomain::new gives None).
 * --------------------------------------------------------------------------------------------- */
int b200_ntt_fr(int field, uint64_t *data, uint32_t log_n, int inverse, const uint64_t *coset_offset);
/* Same with the resize of `fft_in_place` (radix2/mod.rs:140-147) folded in: `in` holds len_in <= 2^log_n elements (longer inputs
 * are truncated), only those cross PCIe, the zero padding is produced on the device; `out` receives all 2^log_n results (may be
 * `in` if it has the room).  This is the transfer-side half of the reference's degree-aware route (fft.rs:29-71); its arithmetic
 * half saves no multiplications on this kernel (a butterfly with a zero upper input still needs its twiddle product). */
int b200_ntt_fr_padded(int field, const uint64_t *in, size_t len_in, uint64_t *out, uint32_t log_n, int inverse, const uint64_t *coset_offset);
/* device-resident variant: d_data is a device pointer; coset_offset stays a host pointer. */
int b200_ntt_fr_dev(int field, void *d_data, uint32_t log_n, int inverse, const uint64_t *coset_offset,
                    void *stream);
/* FFT over G1 points — Radix2EvaluationDomain::{fft_in_place, ifft_in_place} with T = Projective<g1::Config>
 * (T: DomainCoeff<Fr>, poly/src/domain/mod.rs:332-361) after the resize step: the same transform as b200_ntt_fr with the
 * scalars replaced by points,
 *   forward: out[i] = sum_j (h * g^i)^j * P_j          inverse: the exact inverse incl. 1/n,
 * over the domain of the curve's scalar field Fr (B200_CURVE_BLS12_381 -> B200_FIELD_BLS12_381_FR, B200_CURVE_BN254 ->
 * B200_FIELD_BN254_FR: the same number).
 *   points        2^log_n x 3N u64 (Jacobian x, y, z, Montgomery), transformed in place; any point with z = 0 is the identity,
 *                 and every identity in the output is written as (R, R, 0)
 *   coset_offset  NULL (h = 1) or 4 u64 Montgomery limbs of h
 * Outputs are the reference's group elements; their Jacobian limbs may differ (compare after into_affine).
 * B200_ETOOLARGE past TWO_ADICITY, B200_EINVAL for a null pointer, an unknown curve or B200_CURVE_BLS12_381_G2 (no launch).
 * The host entry stages through pinned buffers (pinned or pageable `points`); the _dev entry takes a device pointer and is
 * ordered on `stream` (coset_offset stays a host pointer). */
int b200_ntt_g1(int curve, uint64_t *points, uint32_t log_n, int inverse, const uint64_t *coset_offset);
int b200_ntt_g1_dev(int curve, void *d_points, uint32_t log_n, int inverse, const uint64_t *coset_offset, void *stream);
/* Dense polynomial product over the scalar field, device-resident end to end: the body of
 * `impl Mul<&DensePolynomial<F>> for &DensePolynomial<F>` (poly/src/polynomial/univariate/dense.rs:641-656) —
 * domain of size n = next_pow2(la + lb - 1), fft(a), fft(b), `self_evals *= &other_evals`
 * (poly/src/evaluations/univariate/mod.rs), interpolate (ifft) — with the three vectors staying in HBM between the steps.
 *   a, b   la / lb coefficients (x 4 u64, Montgomery), la, lb >= 1      out   n x 4 u64 (the caller trims leading zeros
 *   like DensePolynomial::from_coefficients_vec); b200_poly_mul_size gives n (0 if past TWO_ADICITY).              */
size_t b200_poly_mul_size(int field, size_t la, size_t lb);
int b200_poly_mul_fr(int field, const uint64_t *a, size_t la, const uint64_t *b, size_t lb, uint64_t *out);
int b200_poly_mul_fr_dev(int field, const void *d_a, size_t la, const void *d_b, size_t lb, void *d_out, void *stream);
/* drop cached twiddle tables of the current device and return the scratch retained by its default memory pool */
int b200_clear_cache(void);

/* ---------------------------------------------------------------------------------------------
 * Synthetic-input generators for benchmarks and large-size property tests (device-resident).
 *   b200_gen_bases_dev:   P_i = b_i * G for a splitmix64 stream b_i (seeded), written as affine
 *                         Montgomery points to d_bases (n x 2N u64) and b_i to d_b (n u64, may be
 *                         NULL) — so the exact MSM answer is (sum s_i*b_i mod r) * G.
 *   b200_gen_scalars_dev: n uniform Fr elements (rejection sampling like Fp::rand,
 *                         ff/src/fields/models/fp/mod.rs:521-548), interpreted as Montgomery limbs.
 * --------------------------------------------------------------------------------------------- */
int b200_gen_bases_dev(int curve, uint64_t seed, size_t n, void *d_bases, void *d_b, void *stream);
int b200_gen_scalars_dev(int field, uint64_t seed, size_t n, void *d_scalars, void *stream);

/* Fixed-base batch multiplication and batch normalisation — the data-parallel steps that PRODUCE MSM bases (SRS powers):
 *   b200_g1_batch_mul_dev        out[i] = scalars[i] * base   (BatchMulPreprocessing::batch_mul, ec/src/scalar_mul/mod.rs:156-245;
 *                                8-bit fixed-base windows + batch inversion); base_xy: HOST, affine 2N u64; d_scalars n x 4 u64
 *                                (Fr Montgomery); d_out_xy n x 2N u64 affine, identity = (0,0)
 *   b200_g1_normalize_batch_dev  Projective::normalize_batch (ec/src/models/short_weierstrass/group.rs:302-319): n x 3N -> n x 2N */
int b200_g1_batch_mul_dev(int curve, const uint64_t *base_xy, const void *d_scalars, size_t n, void *d_out_xy, void *stream);
int b200_g1_normalize_batch_dev(int curve, const void *d_xyz, size_t n, void *d_out_xy, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Element-wise primitive kernels (parity tests and the field micro-benchmark, cf.
 * bench-templates/src/macros/field.rs:69-155).  Device pointers; 1 thread per element.
 *   b200_fp_op_dev  field: 0 BLS Fq, 1 BLS Fr, 2 BN254 Fq, 3 BN254 Fr, 4 BLS Fq2 (12 u64 per element: c0 | c1; ops 6/7 undefined)
 *                   op: 0 mul 1 add 2 sub 3 square 4 double 5 neg 6 into_bigint 7 from_bigint 8 inverse
 *   b200_ec_op_dev  op: 0 bucket+=affine 1 bucket-=affine 2 bucket+=bucket 3 bucket.double
 *                       4 bucket->jacobian 5 jacobian->affine 6 jacobian+=jacobian 7 jacobian.double
 *                   (bucket = XYZZ, 4N u64; jacobian 3N; affine 2N)
 *   reps > 1 re-applies the op to its own output (micro-benchmark mode).
 * --------------------------------------------------------------------------------------------- */
int b200_fp_op_dev(int field, int op, const void *d_a, const void *d_b, void *d_out, size_t n, int reps, void *stream);
int b200_ec_op_dev(int curve, int op, const void *d_a, const void *d_b, void *d_out, size_t n, void *stream);

/* per-phase device timings (ms) of the last MSM on this thread: [digits+histogram, scan, scatter,
 * bucket accumulate, bucket reduce, window combine, total]; and the window / counts it used. */
int b200_msm_last_timings(float *ms7, int *c, int *windows, unsigned long long *bucket_adds);
/* kernel launches issued by this library since load (for bench.py's gpu_launches) */
unsigned long long b200_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* ALGEBRA_B200_H */
