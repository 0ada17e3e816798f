/*
 * point_fft_oracle.c — CPU restatement of Radix2EvaluationDomain::{fft_in_place, ifft_in_place} with T = Projective<g1::Config>
 * (poly/src/domain/radix2/fft.rs:74-88 and :190-349 with T: DomainCoeff<F>, poly/src/domain/mod.rs:332-361), plus a batch of
 * scalar multiples k_i * G.
 *
 * TEST INFRASTRUCTURE ONLY, like oracle/ark_oracle.c, whose field, Jacobian and parallel-for code it reuses unchanged by
 * including it; tests/point_oracle.py compiles this file with the oracle's flags into a temporary directory.
 *
 * T *= F is `MulAssign<F> for Projective` -> mul_bigint(F::into_bigint()), whose default body is double-and-add over the
 * canonical bits, most significant first (ec/src/models/short_weierstrass/mod.rs mul_projective, BitIteratorBE without leading
 * zeros).  Points are n x 3N u64 (x, y, z Jacobian, Montgomery); z == 0 is the identity whatever x and y hold.
 */
#include "../oracle/ark_oracle.c"

/* p <- k * p, k canonical (4 u64 little-endian) */
static void jac_mul_bigint(const field_t *f, jac_t *p, const u64 *k) {
    jac_t acc; jac_set_zero(f, &acc);
    int top = 255;
    while (top >= 0 && !((k[top / 64] >> (top % 64)) & 1)) top--;
    for (int i = top; i >= 0; i--) {
        jac_dbl(f, &acc);
        if ((k[i / 64] >> (i % 64)) & 1) jac_add(f, &acc, p);
    }
    *p = acc;
}
/* p <- s * p, s a Montgomery Fr element */
static void jac_mul_fr(const curve_t *cv, jac_t *p, const u64 *s_mont) {
    u64 k[4]; memcpy(k, s_mont, 32); fp_into_bigint(cv->fr, k);
    jac_mul_bigint(cv->fq, p, k);
}
static void load_jac(int N, jac_t *p, const u64 *src) { memcpy(p->x, src, 8 * N); memcpy(p->y, src + N, 8 * N); memcpy(p->z, src + 2 * N, 8 * N); }
static void store_jac(int N, u64 *dst, const jac_t *p) { memcpy(dst, p->x, 8 * N); memcpy(dst + N, p->y, 8 * N); memcpy(dst + 2 * N, p->z, 8 * N); }

typedef struct { curve_t cv; u64 *x; const u64 *roots; size_t gap, step; const u64 *g, *c; } pbf_ctx;

static void pbf_io_range(size_t tlo, size_t thi, void *vp) { /* butterfly_fn_io, fft.rs:190-198: neg = lo - hi; lo += hi; hi = neg * w */
    pbf_ctx *c = vp; int N = c->cv.N; const field_t *f = c->cv.fq; size_t gap = c->gap;
    for (size_t t = tlo; t < thi; t++) {
        size_t c0 = (t / gap) * 2 * gap, j = t % gap;
        u64 *plo = c->x + 3 * N * (c0 + j), *phi = plo + 3 * N * gap;
        jac_t lo, hi, neg;
        load_jac(N, &lo, plo); load_jac(N, &hi, phi);
        neg = hi; fp_neg(f, neg.y); jac_add(f, &neg, &lo);
        jac_add(f, &lo, &hi);
        jac_mul_fr(&c->cv, &neg, c->roots + 4 * (j * c->step));
        store_jac(N, plo, &lo); store_jac(N, phi, &neg);
    }
}
static void pbf_oi_range(size_t tlo, size_t thi, void *vp) { /* butterfly_fn_oi, fft.rs:201-210: hi *= w; neg = lo - hi; lo += hi */
    pbf_ctx *c = vp; int N = c->cv.N; const field_t *f = c->cv.fq; size_t gap = c->gap;
    for (size_t t = tlo; t < thi; t++) {
        size_t c0 = (t / gap) * 2 * gap, j = t % gap;
        u64 *plo = c->x + 3 * N * (c0 + j), *phi = plo + 3 * N * gap;
        jac_t lo, hi, neg;
        load_jac(N, &lo, plo); load_jac(N, &hi, phi);
        jac_mul_fr(&c->cv, &hi, c->roots + 4 * (j * c->step));
        neg = hi; fp_neg(f, neg.y); jac_add(f, &neg, &lo);
        jac_add(f, &lo, &hi);
        store_jac(N, plo, &lo); store_jac(N, phi, &neg);
    }
}
/* distribute_powers_and_mul_by_const (poly/src/domain/mod.rs:119-148): x[i] *= c * g^i */
static void pdist_range(size_t lo, size_t hi, void *vp) {
    pbf_ctx *c = vp; int N = c->cv.N; const field_t *fr = c->cv.fr;
    u64 e[1] = {lo}, pw[MAXN];
    fp_pow(fr, pw, c->g, e, 1); fp_mul(fr, pw, c->c);
    for (size_t i = lo; i < hi; i++) {
        jac_t p; load_jac(N, &p, c->x + 3 * N * i);
        jac_mul_fr(&c->cv, &p, pw);
        store_jac(N, c->x + 3 * N * i, &p);
        fp_mul(fr, pw, c->g);
    }
}
static void pderange(int N, u64 *x, int log_len) { /* fft.rs:373-380 */
    size_t n = (size_t)1 << log_len;
    for (u64 idx = 1; idx + 1 < n; idx++) {
        u64 r = bitrev64(idx, log_len);
        if (idx < r) { jac_t a, b; load_jac(N, &a, x + 3 * N * idx); load_jac(N, &b, x + 3 * N * r); store_jac(N, x + 3 * N * idx, &b); store_jac(N, x + 3 * N * r, &a); }
    }
}

/* curve: 0 = BLS12-381 G1, 1 = BN254 G1.  pts: 2^log_n x 3N u64, transformed in place.  offset: NULL or 4 Montgomery Fr limbs. */
int ark_fft_g1(int curve, u64 *pts, unsigned log_n, int inverse, const u64 *offset, int threads) {
    pbf_ctx c;
    if (get_curve(curve, &c.cv)) return 1;
    const int field = curve == 0 ? 1 : 3;
    const field_t *fr = c.cv.fr;
    int s; u64 w[4]; fr_params(field, &s, w);
    if ((int)log_n > s) return 2;
    if (threads < 1) threads = 1;
    const size_t n = (size_t)1 << log_n, half = n / 2;
    const int N = c.cv.N;
    u64 g[4]; get_root_of_unity(fr, log_n, s, w, g);
    if (inverse) fp_inv(fr, g);
    const int coset = offset && !eq(offset, fr->R, 4);
    u64 *roots = roots_of_unity(fr, g, half, threads);   /* [1, w, .., w^(n/2-1)], fft.rs:125-153 */
    c.x = pts; c.roots = roots;
    if (!inverse) {                                        /* in_order_fft_in_place, fft.rs:74-79 */
        if (coset) { c.g = offset; c.c = fr->R; par_for(n, threads, 16, pdist_range, &c); }
        for (size_t gap = half; gap > 0; gap /= 2) {       /* io_helper, fft.rs:252-295 */
            c.gap = gap; c.step = n / (2 * gap);
            par_for(half, threads, 16, pbf_io_range, &c);
        }
        pderange(N, pts, log_n);
    } else {                                               /* in_order_ifft_in_place, fft.rs:81-88 */
        pderange(N, pts, log_n);
        for (size_t gap = 1; gap < n; gap *= 2) {          /* oi_helper, fft.rs:297-349 */
            c.gap = gap; c.step = n / (2 * gap);
            par_for(half, threads, 16, pbf_oi_range, &c);
        }
        u64 ninv[4] = {n, 0, 0, 0}; fp_from_bigint(fr, ninv); fp_inv(fr, ninv);
        u64 oinv[4]; memcpy(oinv, fr->R, 32);
        if (coset) { memcpy(oinv, offset, 32); fp_inv(fr, oinv); }
        c.g = oinv; c.c = ninv;
        par_for(n, threads, 16, pdist_range, &c);
    }
    free(roots);
    return 0;
}

/* out_affine[i] = into_affine(k_i * B) for an affine base B (2N u64) and Montgomery Fr scalars k_i (4 u64 each) */
typedef struct { curve_t cv; const u64 *base, *scalars; u64 *out; } pmul_ctx;
static void pmul_range(size_t lo, size_t hi, void *vp) {
    pmul_ctx *c = vp; int N = c->cv.N; const field_t *f = c->cv.fq;
    for (size_t i = lo; i < hi; i++) {
        jac_t p; jac_set_zero(f, &p);
        if (!(is_zero(c->base, N) && is_zero(c->base + N, N))) { memcpy(p.x, c->base, 8 * N); memcpy(p.y, c->base + N, 8 * N); memcpy(p.z, f->R, 8 * N); }
        jac_mul_fr(&c->cv, &p, c->scalars + 4 * i);
        jac_to_affine(f, c->out + 2 * N * i, c->out + 2 * N * i + N, &p);
    }
}
int ark_g1_mul_batch(int curve, const u64 *base_affine, const u64 *scalars, size_t n, u64 *out_affine, int threads) {
    pmul_ctx c;
    if (get_curve(curve, &c.cv)) return 1;
    c.base = base_affine; c.scalars = scalars; c.out = out_affine;
    par_for(n, threads < 1 ? 1 : threads, 64, pmul_range, &c);
    return 0;
}
