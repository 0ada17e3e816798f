// algebra_b200.hpp — C++ host-side mirror of the two reference interfaces on the hot path, header-only over the C ABI
// (include/algebra_b200.h).  The reference's toolchain (Rust) is absent from this image, so the host side above the ABI
// is C++ here; the Rust crate a maintainer would add is rust/ark-b200 (see INTEGRATION.md).  Names, argument meaning and
// error behaviour follow the reference:
//   ab200::VariableBaseMSM<Curve>::msm / msm_unchecked      ec/src/scalar_mul/variable_base/mod.rs:59-77
//   ab200::Radix2EvaluationDomain<Field>                    poly/src/domain/radix2/mod.rs:22-153
// Field elements are arkworks' in-memory Montgomery limbs (std::array<uint64_t, N>).  Host-side domain parameters are
// computed with the same Fp code the kernels use (algebra_b200/csrc/fp.cuh compiles for the host).
#pragma once
#include <array>
#include <cstdint>
#include <optional>
#include <stdexcept>
#include <string>
#include <variant>
#include <vector>

#include "../algebra_b200/csrc/fp.cuh"
#include "algebra_b200.h"

namespace ab200 {

struct Bls12_381G1 {
    static constexpr int ID = B200_CURVE_BLS12_381, N = 6;
    using BaseParams = BlsFq;
    using ScalarParams = BlsFr;
    static constexpr int FIELD_ID = B200_FIELD_BLS12_381_FR;
};
struct Bn254G1 {
    static constexpr int ID = B200_CURVE_BN254, N = 4;
    using BaseParams = BnFq;
    using ScalarParams = BnFr;
    static constexpr int FIELD_ID = B200_FIELD_BN254_FR;
};

// G2 of BLS12-381: coordinates in Fq2 = (c0, c1), 12 u64 per coordinate (curves/bls12_381/src/curves/g2.rs:54)
struct Bls12_381G2 {
    static constexpr int ID = B200_CURVE_BLS12_381_G2, N = 12;
    using BaseParams = BlsFq;   // Fq2 one = (Fq one, 0)
    using ScalarParams = BlsFr;
    static constexpr int FIELD_ID = B200_FIELD_BLS12_381_FR;
};

struct B200Error : std::runtime_error {
    int code;
    B200Error(int c) : std::runtime_error(std::string("algebra_b200: ") + b200_last_error()), code(c) {}
};
inline void check(int rc) {
    if (rc != 0) throw B200Error(rc);
}

using Fr = std::array<uint64_t, 4>;
template <class Curve> using Fq = std::array<uint64_t, Curve::N>;
template <class Curve> struct Affine { Fq<Curve> x, y; };          // identity = (0,0)   (affine.rs:91-104)
template <class Curve> struct Projective { Fq<Curve> x, y, z; };   // identity: z = 0     (group.rs:142-158)

// Result<Projective, usize>: Err(min_len) on a length mismatch (variable_base/mod.rs:73-77)
template <class Curve> using MsmResult = std::variant<Projective<Curve>, size_t>;

template <class Curve> struct VariableBaseMSM {
    static Projective<Curve> msm_unchecked(const std::vector<Affine<Curve>> &bases, const std::vector<Fr> &scalars) {
        const size_t n = bases.size() < scalars.size() ? bases.size() : scalars.size();   // truncates (:59-64)
        Projective<Curve> out{};
        check(b200_msm_sw_g1(Curve::ID, reinterpret_cast<const uint64_t *>(bases.data()),
                             reinterpret_cast<const uint64_t *>(scalars.data()), n, reinterpret_cast<uint64_t *>(&out)));
        return out;
    }
    static MsmResult<Curve> msm(const std::vector<Affine<Curve>> &bases, const std::vector<Fr> &scalars) {
        if (bases.size() != scalars.size()) return bases.size() < scalars.size() ? bases.size() : scalars.size();
        return msm_unchecked(bases, scalars);
    }
    // the same hook on `ngpus` devices of the node, driven from this one process (b200_msm_sw_g1_multi); ngpus = 0: all of them
    static Projective<Curve> msm_unchecked_multi(const std::vector<Affine<Curve>> &bases, const std::vector<Fr> &scalars, int ngpus = 0) {
        const size_t n = bases.size() < scalars.size() ? bases.size() : scalars.size();
        Projective<Curve> out{};
        check(b200_msm_sw_g1_multi(Curve::ID, ngpus > 0 ? ngpus : b200_device_count(), reinterpret_cast<const uint64_t *>(bases.data()),
                                   reinterpret_cast<const uint64_t *>(scalars.data()), n, reinterpret_cast<uint64_t *>(&out)));
        return out;
    }
    // bucket slice `slice` of `slices` of the msm over these (replicated) inputs: the `slices` results add up to msm_unchecked
    // (b200_set_msm_bucket_slice; one caller per GPU, e.g. one rank per device, then b200_g1_sum over the gathered points)
    static Projective<Curve> msm_bucket_slice(const std::vector<Affine<Curve>> &bases, const std::vector<Fr> &scalars, int slice, int slices) {
        check(b200_set_msm_bucket_slice(slice, slices));
        Projective<Curve> out{};
        const size_t n = bases.size() < scalars.size() ? bases.size() : scalars.size();
        const int rc = b200_msm_sw_g1(Curve::ID, reinterpret_cast<const uint64_t *>(bases.data()), reinterpret_cast<const uint64_t *>(scalars.data()), n,
                                      reinterpret_cast<uint64_t *>(&out));
        b200_set_msm_bucket_slice(0, 1);
        check(rc);
        return out;
    }
    // VariableBaseMSM::msm_chunks (variable_base/mod.rs:119-150) on the streaming entry points: `step` pairs per push, one reduction
    static Projective<Curve> msm_chunks(const std::vector<Affine<Curve>> &bases, const std::vector<Fr> &scalars, size_t step) {
        if (scalars.size() > bases.size()) throw std::invalid_argument("scalars_stream.len() <= bases_stream.len()");
        const size_t ns = scalars.size(), skip = bases.size() - ns;   // `skip(bases.len() - scalars.len())`
        Projective<Curve> out{};
        if (ns == 0) return msm_unchecked({}, {});
        if (step == 0) step = ns;
        b200_msm_stream_t *st = nullptr;
        check(b200_msm_stream_begin(Curve::ID, B200_SCALARS_FR_MONT, ns, step < ns ? step : ns, &st));
        for (size_t lo = 0; lo < ns; lo += step) {
            const size_t cnt = lo + step <= ns ? step : ns - lo;
            const int rc = b200_msm_stream_push(st, reinterpret_cast<const uint64_t *>(bases.data() + skip + lo), scalars.data() + lo, cnt);
            if (rc) { b200_msm_stream_abort(st); throw B200Error(rc); }
        }
        check(b200_msm_stream_finish(st, reinterpret_cast<uint64_t *>(&out)));
        return out;
    }
    static Affine<Curve> into_affine(const Projective<Curve> &p) {
        Affine<Curve> a{};
        check(b200_g1_into_affine(Curve::ID, reinterpret_cast<const uint64_t *>(&p), reinterpret_cast<uint64_t *>(&a)));
        return a;
    }
};

// Bases kept in HBM across MSM calls (an SRS), sharded over `ngpus` devices: b200_bases_upload / b200_msm_bases / b200_bases_free
template <class Curve> class ResidentBases {
    b200_bases_t *h_ = nullptr;
    size_t n_ = 0;

  public:
    explicit ResidentBases(const std::vector<Affine<Curve>> &bases, int ngpus = 0) : n_(bases.size()) {
        check(b200_bases_upload(Curve::ID, ngpus > 0 ? ngpus : b200_device_count(), reinterpret_cast<const uint64_t *>(bases.data()), bases.size(), &h_));
    }
    ResidentBases(const ResidentBases &) = delete;
    ResidentBases &operator=(const ResidentBases &) = delete;
    ~ResidentBases() { b200_bases_free(h_); }
    MsmResult<Curve> msm(const std::vector<Fr> &scalars) const {
        if (scalars.size() != n_) return scalars.size() < n_ ? scalars.size() : n_;
        Projective<Curve> out{};
        check(b200_msm_bases(h_, B200_SCALARS_FR_MONT, scalars.data(), scalars.size(), reinterpret_cast<uint64_t *>(&out)));
        return out;
    }
};

template <class Curve> class Radix2EvaluationDomain {
    using P = typename Curve::ScalarParams;
    using F = Fp<P>;
    static Fr pack(const uint32_t *l) {
        Fr r;
        for (int i = 0; i < 4; i++) r[i] = (uint64_t)l[2 * i] | ((uint64_t)l[2 * i + 1] << 32);
        return r;
    }
    static void unpack(uint32_t *l, const Fr &v) {
        for (int i = 0; i < 4; i++) { l[2 * i] = (uint32_t)v[i]; l[2 * i + 1] = (uint32_t)(v[i] >> 32); }
    }

  public:
    uint64_t size = 1;
    uint32_t log_size_of_group = 0;
    Fr size_as_field_element{}, size_inv{}, group_gen{}, group_gen_inv{}, offset{}, offset_inv{}, offset_pow_size{};

    // Radix2EvaluationDomain::new (radix2/mod.rs:55-83): None when log2(size) > TWO_ADICITY
    static std::optional<Radix2EvaluationDomain> make(size_t num_coeffs) {
        Radix2EvaluationDomain d;
        uint64_t size = 1;
        uint32_t lg = 0;
        while (size < num_coeffs) { size <<= 1; lg++; }
        if ((int)lg > P::TWO_ADICITY) return std::nullopt;
        d.size = size;
        d.log_size_of_group = lg;
        uint32_t g[8], t[8], one[8];
        for (int i = 0; i < 8; i++) g[i] = P::TWO_ADIC_ROOT(i);            // get_root_of_unity (fft_friendly.rs:66-82)
        for (int i = (int)lg; i < P::TWO_ADICITY; i++) F::sqr(g, g);
        d.group_gen = pack(g);
        F::inv(t, g);
        d.group_gen_inv = pack(t);
        uint32_t nn[8] = {(uint32_t)size, (uint32_t)(size >> 32), 0, 0, 0, 0, 0, 0};
        F::to_mont(nn, nn);
        d.size_as_field_element = pack(nn);
        F::inv(t, nn);
        d.size_inv = pack(t);
        F::set_one(one);
        d.offset = d.offset_inv = d.offset_pow_size = pack(one);
        return d;
    }
    // get_coset (radix2/mod.rs:85-92): None when the offset has no inverse
    std::optional<Radix2EvaluationDomain> get_coset(const Fr &off) const {
        uint32_t o[8], t[8];
        unpack(o, off);
        if (limbs_is_zero<8>(o)) return std::nullopt;
        Radix2EvaluationDomain d = *this;
        d.offset = off;
        F::inv(t, o);
        d.offset_inv = pack(t);
        F::pow_u64(t, o, size);
        d.offset_pow_size = pack(t);
        return d;
    }
    Fr element(uint64_t i) const {   // offset * g^i (domain/mod.rs:274-280)
        uint32_t g[8], o[8];
        unpack(g, group_gen);
        unpack(o, offset);
        F::pow_u64(g, g, i);
        F::mul(g, g, o);
        return pack(g);
    }
    bool offset_is_one() const {
        uint32_t o[8], one[8];
        unpack(o, offset);
        F::set_one(one);
        return limbs_eq<8>(o, one);
    }
    // fft_in_place / ifft_in_place: `coeffs.resize(size, zero)` then transform (radix2/mod.rs:140-153)
    void fft_in_place(std::vector<Fr> &coeffs) const { run(coeffs, 0); }
    void ifft_in_place(std::vector<Fr> &evals) const { run(evals, 1); }
    std::vector<Fr> fft(std::vector<Fr> coeffs) const { run(coeffs, 0); return coeffs; }
    std::vector<Fr> ifft(std::vector<Fr> evals) const { run(evals, 1); return evals; }
    // T = Projective<Curve> (G1 point coefficients, DomainCoeff for Projective, poly/src/domain/mod.rs:332-361): resized with
    // the identity, transformed by b200_ntt_g1; G2 is refused with B200_EINVAL
    void fft_in_place(std::vector<Projective<Curve>> &coeffs) const { run_points(coeffs, 0); }
    void ifft_in_place(std::vector<Projective<Curve>> &evals) const { run_points(evals, 1); }
    std::vector<Projective<Curve>> fft(std::vector<Projective<Curve>> coeffs) const { run_points(coeffs, 0); return coeffs; }
    std::vector<Projective<Curve>> ifft(std::vector<Projective<Curve>> evals) const { run_points(evals, 1); return evals; }

  private:
    static Projective<Curve> point_zero() {   // Projective::zero() = (1, 1, 0), Montgomery (group.rs:142-158)
        using PB = typename Curve::BaseParams;
        Projective<Curve> p{};
        uint32_t one[PB::L];
        Fp<PB>::set_one(one);
        for (int i = 0; i < PB::L / 2; i++) p.x[i] = p.y[i] = (uint64_t)one[2 * i] | ((uint64_t)one[2 * i + 1] << 32);
        return p;
    }
    void run_points(std::vector<Projective<Curve>> &v, int inverse) const {
        v.resize(size, point_zero());
        check(b200_ntt_g1(Curve::ID, reinterpret_cast<uint64_t *>(v.data()), log_size_of_group, inverse, offset_is_one() ? nullptr : offset.data()));
    }
    void run(std::vector<Fr> &v, int inverse) const {
        v.resize(size, Fr{0, 0, 0, 0});
        check(b200_ntt_fr(Curve::FIELD_ID, reinterpret_cast<uint64_t *>(v.data()), log_size_of_group, inverse,
                          offset_is_one() ? nullptr : offset.data()));
    }
};

}  // namespace ab200
