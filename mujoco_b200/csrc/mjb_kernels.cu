// CUDA backend of libmjb200 for sm_90a (H100): kernels + the mjb_backend.h implementation.
//
// This translation unit holds the backend glue (allocation, copies, streams, the small I/O kernels, the
// Runge-Kutta phase kernel, the validation mapping k_step_lane) and dispatches the fused step kernel,
// whose instantiations (solver x lanes-per-environment) are compiled in their own translation units
// (mjb_kstep.h, mjb_kstep_*.cu).  Mapping and occupancy rationale: mjb_kstep.h and DESIGN.md section 4.
// Compiled with -fmad=false: contact in/out decisions must round like the reference's C build.
#include <cuda_runtime.h>

#include <cstring>

#include <cstdio>
#include <cstdlib>
#include <string>

#include "mjb_backend.h"
#include "mjb_model.h"
#include "mjb_stage.h"
#include "mjb_kstep.h"   // kWarpsPerCta + launchers of the fused step kernel (one translation unit per instantiation)

namespace mjb {

// validation mapping: one environment per lane (same env-major storage, no cooperation)
__global__ void __launch_bounds__(32) k_step_lane(DModel m, Batch b, int mask, int flags) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= b.nenv) return;
  run_env(m, b, e, mask, flags, 0, 1, nullptr, 0);
}

// Runge-Kutta phase between forward launches: one warp per environment (coalesced env-major access)
__global__ void __launch_bounds__(32 * kWarpsPerCta) k_rk4(DModel m, Batch b, int phase, int flags) {
  const int e = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
  if (e >= b.nenv) return;
  run_rk4(m, b, e, phase, flags, threadIdx.x & 31, 32);
}

__global__ void k_pack(Batch b, int is_int, long off, long cnt, void* dense, int to_dense) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)b.nenv * cnt) return;
  run_pack(b, is_int, off, cnt, dense, to_dense, idx);
}
__global__ void k_fill_zero(Batch b, int is_int, long off, long cnt) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)b.nenv * cnt) return;
  run_fill_zero(b, is_int, off, cnt, idx);
}

__global__ void k_reset(DModel m, Batch b) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= b.nenv) return;
  Env d(m, b, e);
  reset_env(d, true);
}

// history buffers as mj_resetData leaves them (models with history buffers, after k_reset)
__global__ void k_reset_history(DModel m, Batch b) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= b.nenv) return;
  Env d(m, b, e);
  reset_history(d);
}

__global__ void k_set_control(DModel m, Batch b, const double* control, int nstep, int t, unsigned spec, int ncontrol, int skip_warned) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= b.nenv) return;
  run_set_control(m, b, e, control, nstep, t, spec, ncontrol, skip_warned != 0);
}

// control_spec == CTRL (the common case): one thread per (environment, actuator)
__global__ void k_set_ctrl_only(DModel m, Batch b, const double* control, int nstep, int t, int skip_warned) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int nu = m.sz.nu;
  if (idx >= (long)b.nenv * nu) return;
  const int e = (int)(idx / nu), k = (int)(idx - (long)e * nu);
  Env d(m, b, e);
  if (skip_warned && env_has_warning(d)) return;
  d.ctrl()[k] = control[((size_t)e * nstep + t) * nu + k];
}

// one thread per (environment, state element): consecutive threads write consecutive elements of an environment's
// state row (FULLPHYSICS = time, qpos, qvel, act)
__global__ void k_get_state(DModel m, Batch b, double* state, int nstep, int t, int nstate) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)b.nenv * nstate) return;
  const int e = (int)(idx / nstate), k = (int)(idx - (long)e * nstate);
  Env d(m, b, e);
  const int nq = m.sz.nq, nv = m.sz.nv;
  const double v = (k == 0) ? d.time()[0] : (k <= nq) ? d.qpos()[k - 1] : (k <= nq + nv) ? d.qvel()[k - 1 - nq] : d.act()[k - 1 - nq - nv];
  state[((size_t)e * nstep + t) * nstate + k] = v;
}

// k_get_state for models with history buffers: the state row ends with the history segment
__global__ void k_get_state_history(DModel m, Batch b, double* state, int nstep, int t, int nstate) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)b.nenv * nstate) return;
  const int e = (int)(idx / nstate), k = (int)(idx - (long)e * nstate);
  Env d(m, b, e);
  const int nq = m.sz.nq, nv = m.sz.nv, na = m.sz.na;
  const double v = (k == 0) ? d.time()[0] : (k <= nq) ? d.qpos()[k - 1] : (k <= nq + nv) ? d.qvel()[k - 1 - nq]
                 : (k <= nq + nv + na) ? d.act()[k - 1 - nq - nv] : d.history()[k - 1 - nq - nv - na];
  state[((size_t)e * nstep + t) * nstate + k] = v;
}

__global__ void k_get_sensor(DModel m, Batch b, double* sens, int nstep, int t, int nsens) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= b.nenv) return;
  run_get_sensor(m, b, e, sens, nstep, t, nsens);
}

// one thread per (actuator, environment): consecutive threads read consecutive environments of one actuator's row
__global__ void k_set_control_native(DModel m, Batch b, const double* ctrl, int t) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int nu = m.sz.nu;
  if (idx >= (long)b.nenv * nu) return;
  const int i = (int)(idx / b.nenv), e = (int)(idx - (long)i * b.nenv);
  Env d(m, b, e);
  d.ctrl()[i] = ctrl[((size_t)t * nu + i) * b.stride + e];
}

__global__ void k_get_state_native(DModel m, Batch b, double* state, int t, int nstate) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= b.nenv) return;
  run_get_state_native(m, b, e, state, t, nstate);
}

namespace backend {

static long g_launches = 0;

static int cuda_fail(cudaError_t e, const char* what) {
  set_error(std::string("CUDA error in ") + what + ": " + cudaGetErrorString(e));
  return -3;
}
#define CK(call, what) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return cuda_fail(e_, what); } while (0)

const char* name() { return "cuda-sm100a"; }

int init(int device) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    set_error(std::string("no usable CUDA device (") + (e != cudaSuccess ? cudaGetErrorString(e) : "device count 0") +
              "); libmjb200 has no CPU fallback");
    return -3;
  }
  if (device >= 0) CK(cudaSetDevice(device), "cudaSetDevice");
  return 0;
}

void* dev_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaMalloc(&p, bytes ? bytes : 1) != cudaSuccess) return nullptr;
  // zero-fill, then WAIT: the memset runs on the legacy default stream while every batch works on its
  // own non-blocking stream, so without this barrier it could land after (and wipe) the first upload
  if (cudaMemset(p, 0, bytes ? bytes : 1) != cudaSuccess || cudaStreamSynchronize(0) != cudaSuccess) {
    cudaFree(p);
    return nullptr;
  }
  return p;
}
void dev_free(void* p) { if (p) cudaFree(p); }
int h2d(void* dst, const void* src, size_t bytes, void* s) {
  CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, (cudaStream_t)s), "h2d");
  return 0;
}
int d2h(void* dst, const void* src, size_t bytes, void* s) {
  CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)s), "d2h");
  return 0;
}
int dev_zero(void* dst, size_t bytes, void* s) {
  CK(cudaMemsetAsync(dst, 0, bytes, (cudaStream_t)s), "memset");
  return 0;
}
void* stream_create() {
  cudaStream_t s = nullptr;
  cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
  return (void*)s;
}
void stream_destroy(void* s) { if (s) cudaStreamDestroy((cudaStream_t)s); }
int sync(void* s) {
  CK(cudaStreamSynchronize((cudaStream_t)s), "stream synchronize");
  CK(cudaGetLastError(), "kernel execution");
  return 0;
}
int stream_order(void* signaller, void* waiter) {
  cudaEvent_t ev;
  CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming), "event create");
  CK(cudaEventRecord(ev, (cudaStream_t)signaller), "event record");
  CK(cudaStreamWaitEvent((cudaStream_t)waiter, ev, 0), "stream wait");
  CK(cudaEventDestroy(ev), "event destroy");   // released once the wait has been satisfied
  return 0;
}
void* event_record(void* stream) {
  cudaEvent_t ev;
  if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) return nullptr;
  if (cudaEventRecord(ev, (cudaStream_t)stream) != cudaSuccess) { cudaEventDestroy(ev); return nullptr; }
  return (void*)ev;
}
int stream_wait_event(void* stream, void* event) {
  CK(cudaStreamWaitEvent((cudaStream_t)stream, (cudaEvent_t)event, 0), "stream wait");
  CK(cudaEventDestroy((cudaEvent_t)event), "event destroy");
  return 0;
}
int d2h_2d(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t height, void* s) {
  CK(cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, height, cudaMemcpyDeviceToHost, (cudaStream_t)s), "d2h 2d");
  return 0;
}
long launches() { return g_launches; }

static inline int nblocks(const Batch& b, int threads) { return (b.nenv + threads - 1) / threads; }

// (an empty field, e.g. ctrl of a model without actuators, launches nothing: a grid of 0 blocks is a launch error)
int launch_pack(const Batch& b, int is_int, long off, long cnt, void* dense, int to_dense, void* s) {
  const long n = (long)b.nenv * cnt;
  if (n == 0) return 0;
  k_pack<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)s>>>(b, is_int, off, cnt, dense, to_dense);
  g_launches++;
  CK(cudaPeekAtLastError(), "k_pack launch");
  return 0;
}
int launch_fill_zero(const Batch& b, int is_int, long off, long cnt, void* s) {
  const long n = (long)b.nenv * cnt;
  if (n == 0) return 0;
  k_fill_zero<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)s>>>(b, is_int, off, cnt);
  g_launches++;
  CK(cudaPeekAtLastError(), "k_fill_zero launch");
  return 0;
}

// lean kernels (FEAT = 0) when the model needs none of the optional pipeline parts (FEAT_*); a model with convex
// collision pairs, spatial tendons or history buffers is never lean, since only the FEAT_CONVEX / FEAT_SPATIAL /
// FEAT_HISTORY instantiations carry their code
static bool lean_model(const DModel& dm, const Batch& b) {
  return dm.sz.nsensor == 0 && dm.sz.neq == 0 && dm.sz.ntree == 1 && dm.opt.integrator != INT_IMPLICITFAST && !dm.sz.actfeat && !dm.sz.colbox && !dm.sz.epot && !dm.sz.ekin && !b.xfrc && !dm.sz.convex && !dm.sz.spatial && !dm.sz.nhistory;
}

// split step: position + velocity | PGS (4 lanes per environment, mjb_pgs4.cu) | finish + integrate | redo
// launch for environments whose acceleration check failed (exits at once everywhere else).
bool split_step_available(const DModel& dm, const Batch& b) {
  static int want = -1;
  if (want < 0) { const char* s = getenv("MJB_SPLIT"); want = s ? atoi(s) : 1; }
  const bool islands = dm.sz.ntree > 1 && !(dm.opt.disableflags & DSBL_ISLAND);
  return want && b.warp_per_env && b.nlane == 32 && !dm.sz.convex && !dm.sz.spatial && !dm.sz.nhistory && dm.opt.solver == SOL_PGS && !islands && dm.opt.noslip_iterations <= 0 &&
         (dm.opt.integrator == INT_EULER || dm.opt.integrator == INT_IMPLICITFAST);
}
int launch_split_step(const DModel& dm, const Batch& b, int first, int later, void* s, void* stagger) {
  const bool lean = lean_model(dm, b);
  static const int part_lanes = [] { const char* e = getenv("MJB_PART_LANES"); return e ? atoi(e) : 16; }();
  if (lean && part_lanes == 16) launch_kpart1_lean16(dm, b, 0, first, s);
  else if (lean && part_lanes == 8) launch_kpart1_lean8(dm, b, 0, first, s);
  else if (lean) launch_kpart1_lean(dm, b, 0, first, s); else launch_kpart1(dm, b, 0, first, s);
  if (stagger) { if (int rc = stream_order(s, stagger)) return rc; }   // the next group starts once this group's first half is done
  if (launch_pgs4(dm, b, later, s)) return cuda_fail(cudaGetLastError(), "PGS order table");
  if (lean && part_lanes == 16) launch_kpart2_lean16(dm, b, 0, later, s);
  else if (lean && part_lanes == 8) launch_kpart2_lean8(dm, b, 0, later, s);
  else if (lean) launch_kpart2_lean(dm, b, 0, later, s); else launch_kpart2(dm, b, 0, later, s);
  g_launches += 3;
  CK(cudaPeekAtLastError(), "split step launch");
  if (!(dm.opt.disableflags & DSBL_AUTORESET)) {
    if (lean) launch_kstep_pgs32_lean(dm, b, kMaskStep, later | 16, s); else launch_kstep_pgs32(dm, b, kMaskStep, later | 16, s);
    g_launches++;
    CK(cudaPeekAtLastError(), "redo launch");
  }
  return 0;
}

// persistent rollout (mjb_krollout.cu): eligible when the step is the lean 16-lane split step and the batch fits one
// CTA per SM.  ON by default (MJB_PERSISTENT=0 or mjb_set_debug("persistent", 0) turn it off): on H100, humanoid
// x4096, dropping the device-wide barrier - no wait for the slowest of 4096 environments at each of the three launches
// of a step - gains more than the halves of the step lose to the PGS pool's share of L1.  Bit-identical to the split
// step, which the tests compare it with.
static int g_persistent = -1;
bool rollout_persistent_available(const DModel& dm, const Batch& b, int nstep) {
  if (g_persistent < 0) { const char* e = getenv("MJB_PERSISTENT"); g_persistent = e ? atoi(e) : 1; }
  static const int part_lanes = [] { const char* e = getenv("MJB_PART_LANES"); return e ? atoi(e) : 16; }();
  return g_persistent > 0 && nstep >= 2 && part_lanes == 16 && split_step_available(dm, b) && lean_model(dm, b);
}
int launch_rollout_persistent(const DModel& dm, const Batch& b, int t0, int t1, int nstep, int first, int later, int layout,
                              const double* ctrl, double* state, int nstate, void* s) {
  const int rc = launch_krollout_lean(dm, b, t0, t1, nstep, first, later, layout, ctrl, state, nstate, s);
  if (rc == -1) return -1;   // does not fit the mapping: the caller steps launch by launch
  if (rc) return cuda_fail(cudaGetLastError(), "persistent rollout setup");
  g_launches++;
  CK(cudaPeekAtLastError(), "k_rollout launch");
  return 0;
}
int set_debug(const char* key, int value) {
  if (!strcmp(key, "pgs4_slots")) { pgs4_set_force_slots(value); return 0; }
  if (!strcmp(key, "persistent")) { g_persistent = value ? 1 : 0; return 0; }
  return -1;
}

// one split step with CUDA events around each launch (bench.py: per-kernel durations on the launching stream)
int profile_split_step(const DModel& dm, const Batch& b, void* s, float* ms) {
  cudaStream_t st = (cudaStream_t)s;
  cudaEvent_t ev[5];
  for (auto& e : ev) CK(cudaEventCreate(&e), "event create");
  const bool lean = lean_model(dm, b);
  static const int part_lanes = [] { const char* e = getenv("MJB_PART_LANES"); return e ? atoi(e) : 16; }();
  cudaEventRecord(ev[0], st);
  if (lean && part_lanes == 16) launch_kpart1_lean16(dm, b, 0, 1, s);
  else if (lean && part_lanes == 8) launch_kpart1_lean8(dm, b, 0, 1, s);
  else if (lean) launch_kpart1_lean(dm, b, 0, 1, s); else launch_kpart1(dm, b, 0, 1, s);
  cudaEventRecord(ev[1], st);
  if (launch_pgs4(dm, b, 0, s)) return cuda_fail(cudaGetLastError(), "PGS order table");
  cudaEventRecord(ev[2], st);
  if (lean && part_lanes == 16) launch_kpart2_lean16(dm, b, 0, 0, s);
  else if (lean && part_lanes == 8) launch_kpart2_lean8(dm, b, 0, 0, s);
  else if (lean) launch_kpart2_lean(dm, b, 0, 0, s); else launch_kpart2(dm, b, 0, 0, s);
  cudaEventRecord(ev[3], st);
  if (!(dm.opt.disableflags & DSBL_AUTORESET)) {
    if (lean) launch_kstep_pgs32_lean(dm, b, kMaskStep, 16, s); else launch_kstep_pgs32(dm, b, kMaskStep, 16, s);
  }
  cudaEventRecord(ev[4], st);
  g_launches += 4;
  CK(cudaStreamSynchronize(st), "profile step");
  for (int i = 0; i < 4; i++) cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]);
  for (auto& e : ev) cudaEventDestroy(e);
  return 0;
}

int launch_stages(const DModel& dm, const Batch& b, int mask, int flags, void* s) {
  if (dm.sz.nhistory) {   // history buffers: only these instantiations carry them (32 lanes or one lane per env)
    if (b.warp_per_env) launch_kstep_history32(dm, b, mask, flags, s); else launch_kstep_lane_history(dm, b, mask, flags, s);
  } else if (dm.sz.spatial) {   // spatial tendons: only these instantiations carry the tendon paths (32 lanes or one lane per env)
    if (b.warp_per_env) launch_kstep_spatial32(dm, b, mask, flags, s); else launch_kstep_lane_spatial(dm, b, mask, flags, s);
  } else if (dm.sz.convex) {   // convex collision pairs: only these instantiations carry GJK / EPA (32 lanes or one lane per env)
    if (b.warp_per_env) launch_kstep_convex32(dm, b, mask, flags, s); else launch_kstep_lane_convex(dm, b, mask, flags, s);
  } else if (b.warp_per_env) {
    // lean kernels when the model needs none of the optional pipeline parts (FEAT_*)
    const bool lean = lean_model(dm, b);
    if (b.nlane == 16) {
      if (dm.opt.solver == SOL_NEWTON) { if (lean) launch_kstep_newton16_lean(dm, b, mask, flags, s); else launch_kstep_newton16(dm, b, mask, flags, s); }
      else launch_kstep_any16(dm, b, mask, flags, s);
    } else if (dm.opt.solver == SOL_PGS) { if (lean) launch_kstep_pgs32_lean(dm, b, mask, flags, s); else launch_kstep_pgs32(dm, b, mask, flags, s); }
    else if (dm.opt.solver == SOL_NEWTON) { if (lean) launch_kstep_newton32_lean(dm, b, mask, flags, s); else launch_kstep_newton32(dm, b, mask, flags, s); }
    else launch_kstep_cg32(dm, b, mask, flags, s);
  } else {
    k_step_lane<<<nblocks(b, 32), 32, 0, (cudaStream_t)s>>>(dm, b, mask, flags);
  }
  g_launches++;
  CK(cudaPeekAtLastError(), "step kernel launch");
  return 0;
}
int launch_get_sensor(const DModel& dm, const Batch& b, double* sens, int nstep, int t, int nsens, void* s) {
  k_get_sensor<<<nblocks(b, 128), 128, 0, (cudaStream_t)s>>>(dm, b, sens, nstep, t, nsens);
  g_launches++;
  CK(cudaPeekAtLastError(), "get_sensor launch");
  return 0;
}
int launch_rk4(const DModel& dm, const Batch& b, int phase, int flags, void* s) {
  if (dm.sz.nhistory) launch_rk4_history(dm, b, phase, flags, s);   // the sensor code of mj_advance (mjb_kstep_history32.cu)
  else k_rk4<<<(b.nenv + kWarpsPerCta - 1) / kWarpsPerCta, 32 * kWarpsPerCta, 0, (cudaStream_t)s>>>(dm, b, phase, flags);
  g_launches++;
  CK(cudaPeekAtLastError(), "rk4 kernel launch");
  return 0;
}
int launch_reset(const DModel& dm, const Batch& b, void* s) {
  k_reset<<<nblocks(b, 128), 128, 0, (cudaStream_t)s>>>(dm, b);
  if (dm.sz.nhistory) k_reset_history<<<nblocks(b, 128), 128, 0, (cudaStream_t)s>>>(dm, b);
  g_launches++;
  CK(cudaPeekAtLastError(), "k_reset launch");
  return 0;
}
int launch_set_control(const DModel& dm, const Batch& b, const double* control, int nstep, int t, unsigned spec,
                       int ncontrol, void* s, bool skip_warned) {
  if (ncontrol == 0) return 0;
  if (spec == (1u << 6) && ncontrol == dm.sz.nu)
    k_set_ctrl_only<<<(unsigned)(((long)b.nenv * dm.sz.nu + 255) / 256), 256, 0, (cudaStream_t)s>>>(dm, b, control, nstep, t, skip_warned ? 1 : 0);
  else
    k_set_control<<<nblocks(b, 128), 128, 0, (cudaStream_t)s>>>(dm, b, control, nstep, t, spec, ncontrol, skip_warned ? 1 : 0);
  g_launches++;
  CK(cudaPeekAtLastError(), "k_set_control launch");
  return 0;
}
int launch_get_state(const DModel& dm, const Batch& b, double* state, int nstep, int t, int nstate, void* s) {
  if (dm.sz.nhistory) k_get_state_history<<<(unsigned)(((long)b.nenv * nstate + 255) / 256), 256, 0, (cudaStream_t)s>>>(dm, b, state, nstep, t, nstate);
  else k_get_state<<<(unsigned)(((long)b.nenv * nstate + 255) / 256), 256, 0, (cudaStream_t)s>>>(dm, b, state, nstep, t, nstate);
  g_launches++;
  CK(cudaPeekAtLastError(), "k_get_state launch");
  return 0;
}
int launch_set_control_native(const DModel& dm, const Batch& b, const double* ctrl, int t, void* s) {
  if (dm.sz.nu == 0) return 0;
  k_set_control_native<<<(unsigned)(((long)b.nenv * dm.sz.nu + 255) / 256), 256, 0, (cudaStream_t)s>>>(dm, b, ctrl, t);
  g_launches++;
  CK(cudaPeekAtLastError(), "k_set_control_native launch");
  return 0;
}
int launch_get_state_native(const DModel& dm, const Batch& b, double* state, int t, int nstate, void* s) {
  k_get_state_native<<<nblocks(b, 128), 128, 0, (cudaStream_t)s>>>(dm, b, state, t, nstate);
  g_launches++;
  CK(cudaPeekAtLastError(), "k_get_state_native launch");
  return 0;
}

}  // namespace backend
}  // namespace mjb
