// the instantiations that carry actuator and sensor history buffers (FEAT_HISTORY: delayed controls, delayed and
// sampled sensors, mjb_history.h / mjb_forward.h): the fused step kernel with 32 lanes per environment and the solver
// chosen at run time, the lane-per-environment validation mapping, and the Runge-Kutta phase kernel whose last phase
// runs the history part of mj_advance (sensor code that k_rk4 does not carry).  CTAs per SM: DESIGN.md section 4.
#define MJB_CTAS_PER_SM 4
#define MJB_HISTORY_UNIT   // compiles the history call sites of the pipeline (mjb_history.h)
#define MJB_KSTEP_INSTANCE
#include "mjb_kstep.h"
namespace mjb {
MJB_KSTEP_LAUNCHER(launch_kstep_history32, -1, 32, FEAT_ALL | FEAT_HISTORY)

__global__ void __launch_bounds__(32) k_step_lane_history(DModel m, Batch b, int mask, int flags) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= b.nenv) return;
  run_env(m, b, e, mask, flags, 0, 1, nullptr, 0, -1, 0xffffffffu, FEAT_ALL | FEAT_HISTORY);
}
__global__ void __launch_bounds__(32 * kWarpsPerCta) k_rk4_history(DModel m, Batch b, int phase, int flags) {
  const int e = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
  if (e >= b.nenv) return;
  run_rk4(m, b, e, phase, flags, threadIdx.x & 31, 32, FEAT_ALL | FEAT_HISTORY);
}
namespace backend {
void launch_kstep_lane_history(const DModel& dm, const Batch& b, int mask, int flags, void* stream) {
  k_step_lane_history<<<(b.nenv + 31) / 32, 32, 0, (cudaStream_t)stream>>>(dm, b, mask, flags);
}
void launch_rk4_history(const DModel& dm, const Batch& b, int phase, int flags, void* stream) {
  k_rk4_history<<<(b.nenv + kWarpsPerCta - 1) / kWarpsPerCta, 32 * kWarpsPerCta, 0, (cudaStream_t)stream>>>(dm, b, phase, flags);
}
}  // namespace backend
}  // namespace mjb
