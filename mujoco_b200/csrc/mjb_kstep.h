// Fused step kernel: declaration of the per-instantiation launchers and, when MJB_KSTEP_INSTANCE is
// defined, the kernel template plus ONE explicit instantiation.  Each instantiation lives in its own
// translation unit (mjb_kstep_*.cu) so that the build compiles them in parallel.
#pragma once
#include "mjb_stage.h"

namespace mjb {

constexpr int kWarpsPerCta = 4;

namespace backend {
void launch_kstep_pgs32(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
void launch_kstep_newton32(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
void launch_kstep_cg32(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
void launch_kstep_newton16(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
void launch_kstep_any16(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
// convex narrow phase (FEAT_ALL | FEAT_CONVEX, solver chosen at run time): fused 32-lane kernel and the lane-per-env
// validation mapping (mjb_kstep_convex32.cu)
void launch_kstep_convex32(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
void launch_kstep_lane_convex(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
// spatial tendons (FEAT_ALL | FEAT_SPATIAL, solver chosen at run time): fused 32-lane kernel and the lane-per-env
// validation mapping (mjb_kstep_spatial32.cu)
void launch_kstep_spatial32(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
void launch_kstep_lane_spatial(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
// history buffers (FEAT_ALL | FEAT_HISTORY, solver chosen at run time): fused 32-lane kernel, the lane-per-env
// validation mapping and the Runge-Kutta phase kernel, whose last phase records samples (mjb_kstep_history32.cu)
void launch_kstep_history32(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
void launch_kstep_lane_history(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
void launch_rk4_history(const DModel& dm, const Batch& b, int phase, int flags, void* stream);
// lean instantiations (FEAT = 0): models without sensors, equalities, several trees or implicitfast
void launch_kstep_pgs32_lean(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
void launch_kstep_newton32_lean(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
void launch_kstep_newton16_lean(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
// split step (PGS as its own launch): part 1 = position + velocity, part 2 = finish + check + integrate
// (mjb_stage.h run_part); the mask argument is ignored.  mjb_pgs4.cu: the solve, 4 lanes per environment.
void launch_kpart1_lean(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
void launch_kpart1(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
void launch_kpart2_lean(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
void launch_kpart2(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
// the same halves with 16 / 8 lanes per environment (2 / 4 environments per warp)
void launch_kpart1_lean16(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
void launch_kpart2_lean16(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
void launch_kpart1_lean8(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
void launch_kpart2_lean8(const DModel& dm, const Batch& b, int mask, int flags, void* stream);
int launch_pgs4(const DModel& dm, const Batch& b, int flags, void* stream);
int launch_krollout_lean(const DModel& dm, const Batch& b, int t0, int t1, int nstep, int first, int later, int layout,
                         const double* ctrl, double* state, int nstate, void* stream);   // mjb_krollout.cu
void pgs4_set_force_slots(int on);
}  // namespace backend

#if defined(MJB_KSTEP_INSTANCE) && defined(__CUDACC__)
// FUSED STEP KERNEL: one warp per environment, all pipeline stages of mj_step in one launch.
// The environment's block lives in global memory (env-major: the 32 lanes touch consecutive
// elements, one 256-byte line per 32 doubles) and is kept hot by L1/L2; occupancy, not staging, hides
// the latency of the short dependent chains (staging the whole block in shared memory caps residency at
// 3 warps/SM).  Each warp owns kSmemPerWarp doubles of
// shared memory used by the one truly serial loop, the PGS sweep (AR + sweep vectors on chip).
#ifndef MJB_CTAS_PER_SM
#define MJB_CTAS_PER_SM 7   // 28 warps/SM (needs <= 72 regs): 3696 environments per wave on the 132 SMs of an H100
#endif
#ifndef MJB_SMEM_PER_WARP
#define MJB_SMEM_PER_WARP 832
#endif
constexpr int kSmemPerWarp = MJB_SMEM_PER_WARP;    // doubles = 6.5 KB: eight sweep vectors, order + draws, and a 4-row ring for nefc <= 64 (or all of AR for nefc <= 24)
// Specialised per constraint solver (template constant propagated through Env::solver) so that each
// instantiation carries only its own solver's code and register pressure.
// NLANE = 16 maps TWO small environments onto each warp (models with <= 16 bodies and dofs leave half
// of a warp idle in every cooperative loop); the two halves synchronise with their own lane masks.
// PART = 0: stages by mask (fused step).  PART = 1 / 2: the two halves of a split step, compiled without the
// solver (no shared-memory scratch, their own register budget and a fraction of the fused kernel's code).
// Sub-warp halves (PART != 0, NLANE < 32) run few warps per SM (4096 environments = 1024 warps at 8 lanes): they
// trade the register cap that buys occupancy for a spill-free, latency-oriented allocation.
template <int SOLVER, int NLANE, int FEAT, int PART>
__global__ void __launch_bounds__(32 * kWarpsPerCta, (PART != 0 && NLANE < 32) ? (NLANE == 16 ? 4 : 2) : MJB_CTAS_PER_SM) k_step_warp(DModel m, Batch b, int mask, int flags) {
  constexpr int kPerWarp = 32 / NLANE;
  __shared__ double smem[(NLANE == 32 && PART == 0) ? kWarpsPerCta * kSmemPerWarp : 1];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  const int e = (blockIdx.x * kWarpsPerCta + w) * kPerWarp + l / NLANE;
  if (e >= b.nenv) return;
  if (NLANE == 32) {
    if (PART == 0) run_env(m, b, e, mask, flags, l, 32, smem + w * kSmemPerWarp, kSmemPerWarp, SOLVER, 0xffffffffu, FEAT);
    else run_env(m, b, e, 0, flags & ~16, l, 32, nullptr, 0, SOLVER, 0xffffffffu, FEAT, PART);
  } else {
    const unsigned lanes = ((1u << NLANE) - 1u) << ((l / NLANE) * NLANE);
    run_env(m, b, e, mask, PART ? (flags & ~16) : flags, l % NLANE, NLANE, nullptr, 0, SOLVER, lanes, FEAT, PART);
  }
}


#define MJB_KSTEP_LAUNCHER_PART(NAME, SOLVER, NLANE, FEAT, PART)                                                  \
  namespace backend {                                                                                        \
  void NAME(const DModel& dm, const Batch& b, int mask, int flags, void* stream) {                            \
    const int per_cta = kWarpsPerCta * (32 / NLANE);                                                         \
    const int grid = (b.nenv + per_cta - 1) / per_cta;                                                       \
    k_step_warp<SOLVER, NLANE, FEAT, PART><<<grid, 32 * kWarpsPerCta, 0, (cudaStream_t)stream>>>(dm, b, mask, flags);     \
  }                                                                                                          \
  }
#define MJB_KSTEP_LAUNCHER(NAME, SOLVER, NLANE, FEAT) MJB_KSTEP_LAUNCHER_PART(NAME, SOLVER, NLANE, FEAT, 0)
#if defined(MJB_STAGE_PROF) && defined(MJB_STAGE_PROF_FN)   // development aid: read (and clear) this unit's sub-stage counters
extern "C" __attribute__((visibility("default"))) int MJB_STAGE_PROF_FN(unsigned long long* out) {
  int rc = (int)cudaMemcpyFromSymbol(out, g_stage_prof, sizeof(unsigned long long) * 64);
  unsigned long long zero[64] = {0};
  cudaMemcpyToSymbol(g_stage_prof, zero, sizeof(zero));
  return rc;
}
#endif
#endif

}  // namespace mjb
