//! Raw bindings of include/algebra_b200.h (what `bindgen` would emit for the entry points used here).
#![allow(non_camel_case_types)]
use core::ffi::{c_char, c_int, c_void};

pub const B200_CURVE_BLS12_381: c_int = 0;
pub const B200_CURVE_BN254: c_int = 1;
pub const B200_CURVE_BLS12_381_G2: c_int = 2;
pub const B200_SCALARS_FR_MONT: c_int = 0;
pub const B200_SCALARS_BIGINT: c_int = 1;

/// opaque handles of include/algebra_b200.h
#[repr(C)] pub struct b200_bases_t { _p: [u8; 0] }
#[repr(C)] pub struct b200_msm_stream_t { _p: [u8; 0] }
pub const B200_FIELD_BLS12_381_FR: c_int = 0;
pub const B200_FIELD_BN254_FR: c_int = 1;

extern "C" {
    pub fn b200_last_error() -> *const c_char;
    pub fn b200_msm_sw_g1(curve: c_int, bases: *const u64, scalars: *const u64, n: usize, out_xyz: *mut u64) -> c_int;
    pub fn b200_msm_sw_g1_dev(curve: c_int, d_bases: *const c_void, d_scalars: *const c_void, n: usize,
                              out_xyz: *mut u64, stream: *mut c_void) -> c_int;
    pub fn b200_device_count() -> c_int;
    pub fn b200_set_msm_bucket_slice(slice: c_int, slices: c_int) -> c_int;
    pub fn b200_msm_sw_g1_multi(curve: c_int, ngpus: c_int, bases: *const u64, scalars: *const u64, n: usize, out_xyz: *mut u64) -> c_int;
    pub fn b200_bases_upload(curve: c_int, ngpus: c_int, bases: *const u64, n: usize, handle: *mut *mut b200_bases_t) -> c_int;
    pub fn b200_msm_bases(handle: *const b200_bases_t, scalar_kind: c_int, scalars: *const c_void, n: usize, out_xyz: *mut u64) -> c_int;
    pub fn b200_bases_free(handle: *mut b200_bases_t) -> c_int;
    pub fn b200_msm_stream_begin(curve: c_int, scalar_kind: c_int, n_total_hint: usize, max_chunk: usize, stream: *mut *mut b200_msm_stream_t) -> c_int;
    pub fn b200_msm_stream_push(stream: *mut b200_msm_stream_t, bases: *const u64, scalars: *const c_void, n: usize) -> c_int;
    pub fn b200_msm_stream_finish(stream: *mut b200_msm_stream_t, out_xyz: *mut u64) -> c_int;
    pub fn b200_msm_stream_abort(stream: *mut b200_msm_stream_t) -> c_int;
    pub fn b200_ntt_fr(field: c_int, data: *mut u64, log_n: u32, inverse: c_int, coset_offset: *const u64) -> c_int;
    pub fn b200_ntt_g1(curve: c_int, points: *mut u64, log_n: u32, inverse: c_int, coset_offset: *const u64) -> c_int;
    pub fn b200_ntt_g1_dev(curve: c_int, d_points: *mut c_void, log_n: u32, inverse: c_int, coset_offset: *const u64,
                           stream: *mut c_void) -> c_int;
    pub fn b200_g1_sum(curve: c_int, points_xyz: *const u64, k: usize, out_xyz: *mut u64) -> c_int;
}

pub(crate) fn check(rc: c_int) {
    if rc != 0 {
        // fft_in_place returns () and SWCurveConfig::msm's Err is reserved for length mismatch, so a CUDA failure
        // cannot be propagated through the reference's trait signatures: panic (release profile is panic = abort).
        let msg = unsafe { core::ffi::CStr::from_ptr(b200_last_error()) };
        panic!("algebra_b200 failed with code {rc}: {}", msg.to_string_lossy());
    }
}
