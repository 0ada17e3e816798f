// GPU driver of the C++ host mirror's point FFT (Radix2EvaluationDomain<Curve>::fft / ifft on std::vector<Projective<Curve>>):
//   point_ntt_mirror <curve 0|1> <num_coeffs> <in.bin> <out.bin>
// reads num_coeffs Jacobian points (3N u64 each), writes fft(points) then ifft(fft(points)), size points each; the domain is
// the smallest one that holds num_coeffs, so the mirror pads with the identity.  tests/test_gpu_point_ntt.py checks the output.
#include <cstdio>
#include <cstdlib>
#include "../../include/algebra_b200.hpp"
using namespace ab200;

template <class C> static int run(size_t m, const char *in, const char *out) {
    std::vector<Projective<C>> pts(m);
    FILE *f = fopen(in, "rb");
    if (!f || fread(pts.data(), sizeof(Projective<C>), m, f) != m) return 2;
    fclose(f);
    auto dom = Radix2EvaluationDomain<C>::make(m).value();
    auto fwd = dom.fft(pts);
    auto back = dom.ifft(fwd);
    f = fopen(out, "wb");
    if (!f) return 3;
    fwrite(fwd.data(), sizeof(Projective<C>), fwd.size(), f);
    fwrite(back.data(), sizeof(Projective<C>), back.size(), f);
    fclose(f);
    printf("size %zu\n", fwd.size());
    return 0;
}
int main(int argc, char **argv) {
    if (argc != 5) return 1;
    const size_t m = strtoull(argv[2], nullptr, 10);
    return atoi(argv[1]) == 0 ? run<Bls12_381G1>(m, argv[3], argv[4]) : run<Bn254G1>(m, argv[3], argv[4]);
}
