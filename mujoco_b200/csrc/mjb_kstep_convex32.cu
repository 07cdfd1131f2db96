// the instantiations that carry the convex narrow phase (FEAT_CONVEX, mjb_convex.h): the fused step kernel with 32
// lanes per environment and the solver chosen at run time, and the lane-per-environment validation mapping.
// GJK / EPA need far more registers than the 72 the other fused kernels are held to (7 CTAs per SM), so this unit
// trades occupancy for fewer spills: 4 CTAs per SM (DESIGN.md section 4).
#define MJB_CTAS_PER_SM 4
#define MJB_CONVEX_UNIT   // compiles the convex branch of collision() (mjb_collision.h)
#define MJB_KSTEP_INSTANCE
#include "mjb_kstep.h"
namespace mjb {
MJB_KSTEP_LAUNCHER(launch_kstep_convex32, -1, 32, FEAT_ALL | FEAT_CONVEX)

__global__ void __launch_bounds__(32) k_step_lane_convex(DModel m, Batch b, int mask, int flags) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= b.nenv) return;
  run_env(m, b, e, mask, flags, 0, 1, nullptr, 0, -1, 0xffffffffu, FEAT_ALL | FEAT_CONVEX);
}
namespace backend {
void launch_kstep_lane_convex(const DModel& dm, const Batch& b, int mask, int flags, void* stream) {
  k_step_lane_convex<<<(b.nenv + 31) / 32, 32, 0, (cudaStream_t)stream>>>(dm, b, mask, flags);
}
}  // namespace backend
}  // namespace mjb
