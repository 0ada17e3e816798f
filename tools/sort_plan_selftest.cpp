// Host-side exerciser of the bin planning of the MSM bucket sort (algebra_b200/csrc/msm_common.cuh: sort_window,
// sort_bin_height, sort_bin_of), walked exactly as msm_sort_plan_kernel walks it.  Test tool (tests/test_gpu_msm_sort.py):
// not part of the product library.
// Build: g++ -std=c++17 -fpermissive -w -x c++ -I/usr/local/cuda/include -shared -fPIC (device intrinsics stay uninstantiated).
#include <algorithm>
#include <vector>

#include "../algebra_b200/csrc/msm_common.cuh"

using namespace ab200;

extern "C" void selftest_sort_consts(unsigned out[4]) {
    out[0] = kSortGroups; out[1] = kSortCap; out[2] = kSortSpan; out[3] = kSortBins;
}

// counts[0..nbw): entries per bucket of one window; nk: the chunk size the bin-sort grid is sized for.
// Out: info = {gs, G, gpb, h, max_group, nbins, grid bins (sort_max_bins)}; per bin k < nbins: bucket range [blo[k], bhi[k]),
// entry range [est[k], est[k] + ecnt[k]).  Returns nbins.
extern "C" unsigned selftest_sort_plan(const unsigned *counts, unsigned nbw, unsigned long long nk, unsigned info[7], unsigned *blo,
                                       unsigned *bhi, unsigned *est, unsigned *ecnt) {
    const MsmSortWin s = sort_window(nbw);
    std::vector<uint32_t> gc(s.G, 0);
    for (uint32_t b = 0; b < nbw; b++) gc[b >> s.gs] += counts[b];
    uint32_t total = 0, mx = 0;
    for (uint32_t v : gc) { total += v; mx = std::max(mx, v); }
    const uint32_t h = sort_bin_height(total, mx, s.G, s.gpb);
    std::vector<uint32_t> bstart(kSortBins + 1, 0), bgroup(kSortBins + 1, 0);
    uint32_t nbins = 0, start = 0, prev = 0xffffffffu;
    for (uint32_t g = 0; g < s.G; g++) {
        const uint32_t k = sort_bin_of(start, g, h, s.gpb);
        for (uint32_t kk = prev + 1; kk <= k; kk++) { bstart[kk] = start; bgroup[kk] = g; }
        if (g == s.G - 1) { bstart[k + 1] = total; bgroup[k + 1] = s.G; nbins = k + 1; }
        prev = k;
        start += gc[g];
    }
    for (uint32_t k = 0; k < nbins; k++) {
        blo[k] = bgroup[k] << s.gs;
        bhi[k] = std::min(bgroup[k + 1] << s.gs, nbw);
        est[k] = bstart[k];
        ecnt[k] = bstart[k + 1] - bstart[k];
    }
    info[0] = s.gs; info[1] = s.G; info[2] = s.gpb; info[3] = h; info[4] = mx; info[5] = nbins; info[6] = sort_max_bins(nk, nbw);
    return nbins;
}
