// msm_common.cuh — shared declarations of the MSM translation units: curve traits, window geometry, bucket I/O helpers and the
// launcher interfaces.  The kernels are templates over the curve; each (kernel group, curve) pair is instantiated in its own
// small .cu file (msm_inst_*.cu) so that the library builds in parallel, and msm.cu (host driver) only sees the launchers.
#pragma once
#include "common.cuh"
#include "ec.cuh"

namespace ab200 {


// Curve traits: F = operations class of the coordinate field (Fp<P> for G1, Fp2<P> for G2), Fr = scalar-field parameter pack.
// (The Montgomery rows stay unrolled rather than in a real loop: the unrolled rows let ptxas interleave six carry chains.)
struct CurveBls {
    using F = Fp<BlsFq>;
    using Fr = BlsFr;
    static constexpr int SCALAR_BITS = 255;  // Fr::MODULUS_BIT_SIZE (variable_base/mod.rs:451)
    static constexpr bool AUTO_LEVELS = true;
    static constexpr int LEVEL_CAP = 4;      // automatic mode: at most this many batched-affine levels
    static constexpr int PAIR_MINB = 4;      // resident blocks per SM the pair-add kernels are compiled for (128 registers)
};
struct CurveBn {
    using F = Fp<BnFq>;
    using Fr = BnFr;
    static constexpr int SCALAR_BITS = 254;
    // 8-limb coordinates: the affine additions are 2.2x cheaper in multiplies but move almost as many bytes, so at most 3 levels
    static constexpr bool AUTO_LEVELS = true;
    static constexpr int LEVEL_CAP = 3;
    static constexpr int PAIR_MINB = 4;
};
// G2 of BLS12-381: coordinates in Fq2 (curves/bls12_381/src/curves/g2.rs:54), same scalar field
struct CurveBlsG2 {
    using F = Fp2<BlsFq>;
    using Fr = BlsFr;
    static constexpr int SCALAR_BITS = 255;
    static constexpr bool AUTO_LEVELS = true;
    static constexpr int LEVEL_CAP = 4;
    static constexpr int PAIR_MINB = 2;      // 24-word coordinates: 255 registers, two blocks per SM
};

struct MsmGeom {
    int c, W, top_bits;          // window bits, number of windows, bits in the top window
    uint32_t nb;                 // buckets of this slice per non-top window (whole window: 2^(c-1))
    uint32_t nb_top;             // buckets of this slice in the top window  (whole window: 2^top_bits)
    uint32_t total_buckets;      // (W-1)*nb + nb_top
    uint32_t off, off_top;       // first bucket of the slice inside a non-top / the top window (0 for the whole window)
};

// Bucket slice `slice` of `slices`: every window keeps the contiguous range [nbw*slice/slices, nbw*(slice+1)/slices) of its
// buckets (bucket j of a window has weight j+1, so a slice's sums carry `off` as an extra chunk offset in the reduction) and
// the slices' results add up to the complete MSM.  A window with fewer buckets than slices is given whole to slice 0.
inline MsmGeom make_geom(int c, int scalar_bits, int slice = 0, int slices = 1) {
    MsmGeom g;
    g.c = c;
    g.W = (scalar_bits + c - 1) / c;  // digits_count (:452)
    g.top_bits = scalar_bits - (g.W - 1) * c;
    const uint32_t full = 1u << (c - 1), full_top = 1u << g.top_bits;
    auto cut = [&](uint32_t nbw, int i) -> uint32_t {
        if (nbw < (uint32_t)slices) return i == 0 ? 0u : nbw;
        return (uint32_t)((uint64_t)nbw * (uint64_t)i / (uint64_t)slices);
    };
    g.off = cut(full, slice);
    g.nb = cut(full, slice + 1) - g.off;
    g.off_top = cut(full_top, slice);
    g.nb_top = cut(full_top, slice + 1) - g.off_top;
    g.total_buckets = (uint32_t)(g.W - 1) * g.nb + g.nb_top;
    return g;
}

static constexpr uint32_t kNoBucket = 0xffffffffu;
static constexpr uint32_t kFixupSmall = 16;

// ---- bucket sort of a chunk's entries (msm_sort.cu) ----
// The digit pass writes every (window, scalar) digit once, window-major: digits[w * nk + i] = rel | sign << 31, where rel is
// the bucket inside the window's slice, or kNoDigit (zero digit, or a bucket outside the slice).  Per window the buckets are
// cut into G <= kSortGroups groups of 2^gs consecutive buckets and the entries are counted per group; the groups are then
// joined into bins of consecutive groups, planned from those counts so that a bin holds at most kSortCap entries (whenever
// no group holds more than kSortCap / 2) and spans at most kSortSpan buckets.  One pass partitions the window's entries by
// bin; a second sorts every bin by bucket in shared memory and writes `sorted` and `offsets` coalesced.
static constexpr uint32_t kNoDigit = 0xffffffffu;
static constexpr uint32_t kSortGroups = 8192;   // count groups per window at most
static constexpr uint32_t kSortCap = 24576;     // entries a bin sorts in shared memory
static constexpr uint32_t kSortSpan = 2048;     // buckets of a bin at most
static constexpr uint32_t kSortBins = 8192;     // bins per window at most

struct MsmSortWin {
    uint32_t gs;    // a group is 2^gs buckets
    uint32_t G;     // groups of the window
    uint32_t gpb;   // groups a bin may join: gpb << gs == kSortSpan
};
__host__ __device__ inline MsmSortWin sort_window(uint32_t nbw) {   // nbw: buckets of the window (<= 2^23)
    MsmSortWin s;
    s.gs = 0;
    while ((((uint64_t)nbw + (1ull << s.gs) - 1) >> s.gs) > kSortGroups) s.gs++;
    s.G = (uint32_t)(((uint64_t)nbw + (1ull << s.gs) - 1) >> s.gs);
    s.gpb = kSortSpan >> s.gs;   // gs <= 10, so gpb >= 2
    return s;
}
// Bin of group g whose first entry is at `start` (window-relative): bins are the runs of groups sharing both start / h and
// g / gpb.  So a bin holds at most h - 1 + (largest group) entries and spans at most gpb groups, and the bin index never
// decreases with g.  A window has sort_bin_of(start of group G-1, G-1) + 1 <= total / h + (G-1) / gpb + 1 bins.
__host__ __device__ inline uint32_t sort_bin_of(uint32_t start, uint32_t g, uint32_t h, uint32_t gpb) { return start / h + g / gpb; }
// bin height h of a window from its entry total and its largest group: bins of at most kSortCap entries while the largest
// group holds less than kSortCap / 2, never shorter than kSortCap / 2 (larger groups overflow into the unstaged path of the
// bin sort), and never more than kSortBins bins
__host__ __device__ inline uint32_t sort_bin_height(uint32_t total, uint32_t max_group, uint32_t G, uint32_t gpb) {
    uint32_t h = max_group < kSortCap / 2 ? kSortCap + 1 - max_group : kSortCap / 2;
    const uint32_t room = kSortBins - 1 - (G ? (G - 1) / gpb : 0);   // >= kSortBins / 2
    const uint32_t h_min = (uint32_t)(((uint64_t)total + room - 1) / room);
    return h > h_min ? h : h_min;
}
// upper bound on the bins of a window with nbw buckets and at most nk entries (the grid of the bin sort)
inline uint32_t sort_max_bins(size_t nk, uint32_t nbw) {
    const MsmSortWin s = sort_window(nbw);
    const uint64_t b = (uint64_t)nk / (kSortCap / 2) + (s.G ? (s.G - 1) / s.gpb : 0) + 1;
    return (uint32_t)(b < kSortBins ? b : kSortBins);
}

// device scratch of the sort (msm_sort.cu), per window w: group counts, group -> bin, bin start / first group / fill cursor
struct MsmSortPlan {
    uint32_t *gcount;    // [W][kSortGroups], zeroed before the count pass
    uint16_t *gbin;      // [W][kSortGroups]
    uint32_t *bstart;    // [W][kSortBins + 1]: first entry of bin k (window-relative); [nbins] = the window's total
    uint32_t *bgroup;    // [W][kSortBins + 1]: first group of bin k; [nbins] = G
    uint32_t *bcur;      // [W][kSortBins]: fill cursor of the partition pass
    uint32_t *nbins;     // [W]
    uint32_t *wbase;     // [W + 1]: entries of the chunk before window w (wbase[W] = all of them)
    static size_t bytes(int W) { return (size_t)W * (kSortGroups * 6 + (kSortBins + 1) * 8 + kSortBins * 4 + 4) + ((size_t)W + 1) * 4 + 64; }
    void carve(void *p, int W) {
        char *q = (char *)p;
        gcount = (uint32_t *)q; q += (size_t)W * kSortGroups * 4;
        bstart = (uint32_t *)q; q += (size_t)W * (kSortBins + 1) * 4;
        bgroup = (uint32_t *)q; q += (size_t)W * (kSortBins + 1) * 4;
        bcur = (uint32_t *)q; q += (size_t)W * kSortBins * 4;
        nbins = (uint32_t *)q; q += (size_t)W * 4;
        wbase = (uint32_t *)q; q += ((size_t)W + 1) * 4;
        gbin = (uint16_t *)q;
    }
};
// count the digits of every window per group (plan.gcount must be zero)
int msm_sort_count(const uint32_t *digits, size_t nk, const MsmGeom &g, const MsmSortPlan &plan, cudaStream_t st);
// plan the bins of every window; writes plan.* and offsets[total_buckets] (the chunk's entry count)
int msm_sort_plan(const MsmGeom &g, const MsmSortPlan &plan, uint32_t *offsets, cudaStream_t st);
// partition every window into its bins (through `part`, nk entries of 8 bytes) and sort the bins: writes sorted and offsets
int msm_sort_scatter(const uint32_t *digits, size_t nk, const MsmGeom &g, const MsmSortPlan &plan, uint2 *part, uint32_t *offsets, uint32_t *sorted,
                     cudaStream_t st);

template <int L> __device__ __forceinline__ void load_xyzz(Xyzz<L> &b, const uint32_t *p) {
    load_limbs<L>(b.x, p);
    load_limbs<L>(b.y, p + L);
    load_limbs<L>(b.zz, p + 2 * L);
    load_limbs<L>(b.zzz, p + 3 * L);
}
template <int L> __device__ __forceinline__ void store_xyzz(uint32_t *p, const Xyzz<L> &b) {
    store_limbs<L>(p, b.x);
    store_limbs<L>(p + L, b.y);
    store_limbs<L>(p + 2 * L, b.zz);
    store_limbs<L>(p + 3 * L, b.zzz);
}

// ---- launchers (definitions: msm_k_pair.cuh / msm_k_acc.cuh / msm_k_red.cuh; instantiations: msm_inst_*.cu) ----
template <class C> struct MsmPairLaunch {
    // one batched-affine level over the buckets [0, nbg) (first: the inputs are the bases, gathered through the sorted indices `src`)
    static int run(bool first, const uint32_t *bases, const uint32_t *src, const uint32_t *offsets_out, const uint32_t *pairmap, uint32_t nbg,
                   uint32_t batch, size_t out_cap, uint32_t *out, cudaStream_t st);
};
template <class C> struct MsmAccLaunch {
    // signed digits of every window, window-major (digits: g.W * nk words)
    static int digits(const void *scalars, int kind, size_t nk, MsmGeom g, uint32_t *digits, cudaStream_t st);
    static int occupancy(bool direct);   // resident 128-thread blocks per SM of the accumulate kernel
    // XYZZ accumulation + both fix-up kernels
    static int accumulate(bool direct, const uint32_t *pts, const uint32_t *sorted_idx, const uint32_t *offs, uint32_t nbk, uint32_t T,
                          uint32_t num_tasks, uint32_t *dst, uint32_t *head, uint32_t *tail, uint32_t *head_bucket, uint32_t *tail_bucket,
                          cudaStream_t st);
    static int merge(uint32_t *buckets, const uint32_t *extra, uint32_t nb, cudaStream_t st);
};
template <class C> struct MsmRedLaunch {
    // partials: W * chunks buckets of scratch; partials2: W * 32
    static int reduce(const uint32_t *buckets, MsmGeom g, int log_m, uint32_t chunks, uint32_t *partials, uint32_t *partials2, uint32_t *window_sums,
                      cudaStream_t st);
    static int combine(const uint32_t *window_sums, int W, int c, uint32_t *out, cudaStream_t st);
    static int sum_or_affine(bool to_affine, const uint32_t *d_in, size_t k, uint32_t *d_out, cudaStream_t st);
};

}  // namespace ab200
