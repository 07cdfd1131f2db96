// the instantiations that carry spatial tendons (FEAT_SPATIAL: site paths, sphere / cylinder wrapping, pulleys and the
// tendon-armature bias, mjb_smooth.h / mjb_forward.h): the fused step kernel with 32 lanes per environment and the
// solver chosen at run time, and the lane-per-environment validation mapping.  CTAs per SM: DESIGN.md section 4.
#define MJB_CTAS_PER_SM 4
#define MJB_SPATIAL_UNIT   // compiles the spatial branch of tendon() and the tendon-armature bias
#define MJB_KSTEP_INSTANCE
#include "mjb_kstep.h"
namespace mjb {
MJB_KSTEP_LAUNCHER(launch_kstep_spatial32, -1, 32, FEAT_ALL | FEAT_SPATIAL)

__global__ void __launch_bounds__(32) k_step_lane_spatial(DModel m, Batch b, int mask, int flags) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= b.nenv) return;
  run_env(m, b, e, mask, flags, 0, 1, nullptr, 0, -1, 0xffffffffu, FEAT_ALL | FEAT_SPATIAL);
}
namespace backend {
void launch_kstep_lane_spatial(const DModel& dm, const Batch& b, int mask, int flags, void* stream) {
  k_step_lane_spatial<<<(b.nenv + 31) / 32, 32, 0, (cudaStream_t)stream>>>(dm, b, mask, flags);
}
}  // namespace backend
}  // namespace mjb
