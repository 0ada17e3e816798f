// explicit instantiation: MsmAccLaunch<CurveBlsG2>::digits / merge (see msm_inst_acc_g2.cu)
#include "msm_k_acc.cuh"
namespace ab200 {
template int MsmAccLaunch<CurveBlsG2>::digits(const void *, int, size_t, MsmGeom, uint32_t *, cudaStream_t);
template int MsmAccLaunch<CurveBlsG2>::merge(uint32_t *, const uint32_t *, uint32_t, cudaStream_t);
}  // namespace ab200
