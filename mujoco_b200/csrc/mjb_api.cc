// C ABI of libmjb200 (include/mjb.h): batch management, state I/O with the reference's mjtState
// signature semantics (src/engine/engine_support.c:138-315), mj_step/mj_forward on all
// environments and the batched rollout that mirrors python/mujoco/rollout.cc:67-178.
// Device work goes through mjb_backend.h (CUDA in the product; host loops only in tests/hostemu).
#include "../../include/mjb.h"

#include <cstdio>
#include <cstdlib>
#include <dlfcn.h>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include <mujoco/mjdata.h>   // the reference's own mjData (public header), for the mjData bridge

#include "mjb_backend.h"
#include "mjb_model.h"

using namespace mjb;

namespace {
enum {  // mjtState bits (include/mujoco/mjtype.h:503-517)
  ST_TIME = 1 << 0, ST_QPOS = 1 << 1, ST_QVEL = 1 << 2, ST_ACT = 1 << 3, ST_HISTORY = 1 << 4,
  ST_WARMSTART = 1 << 5, ST_CTRL = 1 << 6, ST_QFRC_APPLIED = 1 << 7, ST_XFRC_APPLIED = 1 << 8,
  ST_EQ_ACTIVE = 1 << 9, ST_MOCAP_POS = 1 << 10, ST_MOCAP_QUAT = 1 << 11, ST_USERDATA = 1 << 12,
  ST_PLUGIN = 1 << 13
};
const unsigned kSupportedState = ST_TIME | ST_QPOS | ST_QVEL | ST_ACT | ST_HISTORY | ST_WARMSTART | ST_CTRL |
                                 ST_QFRC_APPLIED | ST_XFRC_APPLIED | ST_EQ_ACTIVE | ST_MOCAP_POS | ST_MOCAP_QUAT | ST_USERDATA | ST_PLUGIN;
}  // namespace

struct mjbBatch_ {
  HostModel hm;          // host copy (pointers into hm.ib / hm.db)
  DModel dm;             // device copy (pointers into d_ib / d_db)
  int* d_ib = nullptr;
  double* d_db = nullptr;
  Batch b;               // device storage
  void* stream = nullptr;
  void* own_stream = nullptr;   // the stream created with the batch (stream == own_stream unless mjb_set_stream replaced it)
  int device = 0;
  double* io_ctrl = nullptr;    // staging for mjb_step_host
  double* io_state = nullptr;
  void* stage = nullptr;        // dense staging for field I/O
  size_t stage_bytes = 0;
  void* copy_stream = nullptr;  // device -> host copies of finished rollout chunks, overlapped with the steps that follow
  void* roll[3] = {nullptr, nullptr, nullptr};   // control / state / sensordata buffers of mjb_rollout, kept between calls
  size_t roll_bytes[3] = {0, 0, 0};
  std::vector<void*> gstreams;  // extra streams of the grouped multi-step execution (see env_groups)
};

static int fail(int code, const std::string& msg) { set_error(msg); return code; }

// mju_error / mju_warning of the reference library when it is loaded in this process (looked up once, never
// linked): the Python bindings install their handlers there (python/mujoco/errors.h:140-226)
static void route_error(const std::string& msg) {
  typedef void (*fn_t)(const char*, ...);
  static fn_t fn = (fn_t)dlsym(RTLD_DEFAULT, "mju_error");
  set_error(msg);
  if (fn) { fn("%s", msg.c_str()); return; }   // normally does not return
  fprintf(stderr, "ERROR: %s\n", msg.c_str());
  abort();
}
static void route_warning(int type, double time) {
  typedef void (*fn_t)(const char*, ...);
  static fn_t fn = (fn_t)dlsym(RTLD_DEFAULT, "mju_warning");
  static const char* text[NWARNING] = {
      "Inertia matrix is too close to singular. Check model.", "Pre-allocated contact buffer is full (nconmax of the batch).",
      "Pre-allocated constraint buffer is full (njmax of the batch).", "Nan, Inf or huge value in QPOS. The simulation is unstable.",
      "Nan, Inf or huge value in QVEL. The simulation is unstable.", "Nan, Inf or huge value in QACC. The simulation is unstable.",
      "Nan, Inf or huge value in CTRL.", "Pre-allocated visual geom buffer is full."};
  if (fn) fn("%s Time = %.4f.", text[type], time);
  else fprintf(stderr, "WARNING: %s Time = %.4f.\n", text[type], time);
}

// thread mapping for new batches: 1 = one warp per environment (default), 0 = one lane per environment
static int g_warp_per_env = 1;

// ---- layout-agnostic field movement through a dense [nenv][cnt] device staging buffer ----------
static int stage_reserve(mjbBatch* B, size_t bytes) {
  if (B->stage_bytes >= bytes) return 0;
  backend::sync(B->stream);
  backend::dev_free(B->stage);
  B->stage = backend::dev_alloc(bytes);
  B->stage_bytes = B->stage ? bytes : 0;
  return B->stage ? 0 : fail(MJB_ERR_CUDA, "device allocation failed (staging)");
}
static int field_to_host(mjbBatch* B, bool is_int, long off, long cnt, void* host) {
  const size_t bytes = (size_t)B->b.nenv * cnt * (is_int ? sizeof(int) : sizeof(double));
  if (!bytes) return 0;
  if (int rc = stage_reserve(B, bytes)) return rc;
  if (int rc = backend::launch_pack(B->b, is_int, off, cnt, B->stage, 1, B->stream)) return rc;
  if (int rc = backend::d2h(host, B->stage, bytes, B->stream)) return rc;
  return backend::sync(B->stream);
}
static int field_from_host(mjbBatch* B, bool is_int, long off, long cnt, const void* host) {
  const size_t bytes = (size_t)B->b.nenv * cnt * (is_int ? sizeof(int) : sizeof(double));
  if (!bytes) return 0;
  if (int rc = stage_reserve(B, bytes)) return rc;
  if (int rc = backend::h2d(B->stage, host, bytes, B->stream)) return rc;
  if (int rc = backend::launch_pack(B->b, is_int, off, cnt, B->stage, 0, B->stream)) return rc;
  return backend::sync(B->stream);
}
static int field_zero(mjbBatch* B, bool is_int, long off, long cnt) {
  return backend::launch_fill_zero(B->b, is_int, off, cnt, B->stream);
}

extern "C" {

const char* mjb_last_error(void) { return get_error(); }
int mjb_version(void) { return 100; }

struct mjModel_* mjb_load_model(const char* path) { return (struct mjModel_*)load_mjb(path); }
void mjb_free_model(struct mjModel_* m) { free_mjb((mjModel*)m); }
int mjb_check_model(const struct mjModel_* m) { return check_model((const mjModel*)m); }
long mjb_model_size(const struct mjModel_* m, const char* name) { return model_size((const mjModel*)m, name); }
int mjb_get_option(const struct mjModel_* m, const char* name, double* v) { return get_option((const mjModel*)m, name, v) ? MJB_ERR_ARG : 0; }
int mjb_set_option(struct mjModel_* m, const char* name, double v) { return set_option((mjModel*)m, name, v) ? MJB_ERR_ARG : 0; }

mjbBatch* mjb_make_batch(const struct mjModel_* m, int nenv, int nconmax, int njmax, int device) {
  if (!m || nenv <= 0) { set_error("mjb_make_batch: bad arguments"); return nullptr; }
  if (int rc = backend::init(device)) { (void)rc; return nullptr; }
  mjbBatch* B = new mjbBatch_();
  if (build_host_model((const mjModel*)m, nconmax, njmax, &B->hm)) { delete B; return nullptr; }   // nothing on the device yet
  const DModel& H = B->hm.dm;
  if (H.opt.solver == SOL_NEWTON) {
#ifndef MJB_HAVE_NEWTON
    set_error("unsupported: Newton solver not built");
    delete B;
    return nullptr;
#endif
  }
  if (H.sz.nu > 4 * H.sz.nv) { set_error("unsupported: nu > 4*nv"); delete B; return nullptr; }
  if (H.sz.nlim > 6 * H.sz.njmax) { set_error("njmax too small for the model's limit candidates"); delete B; return nullptr; }
  B->device = device;
  B->stream = backend::stream_create();
  B->own_stream = B->stream;
  // device copy of the model blobs, pointers rebased
  B->d_ib = (int*)backend::dev_alloc(B->hm.ib.size() * sizeof(int));
  B->d_db = (double*)backend::dev_alloc(B->hm.db.size() * sizeof(double));
  if (!B->d_ib || !B->d_db) { set_error("device allocation failed (model)"); mjb_free_batch(B); return nullptr; }
  backend::h2d(B->d_ib, B->hm.ib.data(), B->hm.ib.size() * sizeof(int), B->stream);
  backend::h2d(B->d_db, B->hm.db.data(), B->hm.db.size() * sizeof(double), B->stream);
  B->dm = H;
#define X(name) B->dm.name = B->d_ib + (H.name - B->hm.ib.data());
  MJB_MODEL_INT_FIELDS(X)
#undef X
#define X(name) B->dm.name = B->d_db + (H.name - B->hm.db.data());
  MJB_MODEL_DBL_FIELDS(X)
#undef X
  // batch storage
  Batch& b = B->b;
  b.nenv = nenv;
  b.stride = ((size_t)nenv + 31) / 32 * 32;
  b.L = make_layout(H.sz);
  b.warp_per_env = g_warp_per_env;
  // small models (<= 16 bodies and dofs) with a primal solver: two environments per warp.  PGS keeps a
  // whole warp per environment (its on-chip sweep uses warp-wide shuffles).  MJB_LANES=32|16 overrides.
  b.nlane = (H.sz.nbody <= 16 && H.sz.nv <= 16 && H.opt.solver != SOL_PGS) ? 16 : 32;
  b.xfrc = 0;
  if (const char* ls = getenv("MJB_LANES")) { const int v = atoi(ls); if (v == 16 || v == 32) b.nlane = v; }
  if (H.sz.convex) b.nlane = 32;   // the convex narrow phase is built for the 32-lane mapping only
  if (H.sz.spatial) b.nlane = 32;  // so are spatial tendons
  if (H.sz.nhistory) b.nlane = 32; // and history buffers
  b.dpitch = ((size_t)b.L.ndbl + 15) / 16 * 16;   // env-major blocks, 128-byte aligned
  b.ipitch = ((size_t)b.L.nint + 31) / 32 * 32;
  size_t nd = b.dpitch * b.stride;
  size_t ni = b.ipitch * b.stride;
  b.dbl = (double*)backend::dev_alloc(nd * sizeof(double));
  b.itg = (int*)backend::dev_alloc(ni * sizeof(int));
  if (!b.dbl || !b.itg) { set_error("device allocation failed (batch)"); mjb_free_batch(B); return nullptr; }
  backend::launch_reset(B->dm, b, B->stream);
  if (backend::sync(B->stream)) { mjb_free_batch(B); return nullptr; }
  return B;
}

void mjb_free_batch(mjbBatch* B) {
  if (!B) return;
  backend::sync(B->stream);
  for (void* gs : B->gstreams) { backend::sync(gs); backend::stream_destroy(gs); }
  backend::dev_free(B->b.dbl);
  backend::dev_free(B->b.itg);
  backend::dev_free(B->d_ib);
  backend::dev_free(B->d_db);
  backend::dev_free(B->io_ctrl);
  backend::dev_free(B->io_state);
  backend::dev_free(B->stage);
  for (void* r : B->roll) backend::dev_free(r);
  if (B->copy_stream) { backend::sync(B->copy_stream); backend::stream_destroy(B->copy_stream); }
  backend::stream_destroy(B->own_stream);
  delete B;
}

int mjb_nenv(const mjbBatch* B) { return B ? B->b.nenv : 0; }
long mjb_env_stride(const mjbBatch* B) { return B ? (long)B->b.stride : 0; }
void* mjb_stream(mjbBatch* B) { return B ? B->stream : nullptr; }

int mjb_set_stream(mjbBatch* B, void* stream) {
  if (!B) return fail(MJB_ERR_ARG, "mjb_set_stream: null batch");
  if (int rc = backend::sync(B->stream)) return rc;      // nothing of the batch is left in flight on the old stream
  B->stream = stream ? stream : B->own_stream;
  return 0;
}
long mjb_kernel_launches(const mjbBatch*) { return backend::launches(); }

int mjb_reset(mjbBatch* B) {
  if (!B) return fail(MJB_ERR_ARG, "null batch");
  if (int rc = backend::launch_reset(B->dm, B->b, B->stream)) return rc;
  return backend::sync(B->stream);
}

// ---- state vector <-> fields ---------------------------------------------------------------------
struct Seg { long off; int n; };   // field offset (elements) and count
static int state_segments(const mjbBatch* B, unsigned sig, std::vector<Seg>* segs) {
  const Sizes& S = B->hm.dm.sz;
  const Layout& L = B->b.L;
  if (sig & ~kSupportedState) return -1;
  segs->clear();
  if (sig & ST_TIME) segs->push_back({L.time, 1});
  if (sig & ST_QPOS) segs->push_back({L.qpos, S.nq});
  if (sig & ST_QVEL) segs->push_back({L.qvel, S.nv});
  if ((sig & ST_ACT) && S.na) segs->push_back({L.act, S.na});
  if ((sig & ST_HISTORY) && S.nhistory) segs->push_back({L.history, S.nhistory});
  if (sig & ST_WARMSTART) segs->push_back({L.qacc_warmstart, S.nv});
  if (sig & ST_CTRL) segs->push_back({L.ctrl, S.nu});
  if (sig & ST_QFRC_APPLIED) segs->push_back({L.qfrc_applied, S.nv});
  if (sig & ST_XFRC_APPLIED) segs->push_back({L.xfrc_applied, 6 * S.nbody});
  if ((sig & ST_EQ_ACTIVE) && S.neq) segs->push_back({L.eq_active, S.neq});   // values 0 / 1 as doubles, like mj_getState
  if ((sig & ST_MOCAP_POS) && S.nmocap) segs->push_back({L.mocap_pos, 3 * S.nmocap});
  if ((sig & ST_MOCAP_QUAT) && S.nmocap) segs->push_back({L.mocap_quat, 4 * S.nmocap});
  // USERDATA, PLUGIN: zero-sized on supported models
  return 0;
}

int mjb_state_size(const mjbBatch* B, unsigned int sig) {
  std::vector<Seg> segs;
  if (!B || state_segments(B, sig, &segs)) { set_error("mjb_state_size: unsupported state signature"); return MJB_ERR_ARG; }
  int n = 0;
  for (auto& s : segs) n += s.n;
  return n;
}

int mjb_set_state(mjbBatch* B, const double* state, unsigned int sig) {
  std::vector<Seg> segs;
  if (!B || !state || state_segments(B, sig, &segs)) return fail(MJB_ERR_ARG, "mjb_set_state: bad arguments / unsupported signature");
  if (sig & ST_XFRC_APPLIED) B->b.xfrc = 1;
  int ns = 0;
  for (auto& s : segs) ns += s.n;
  std::vector<double> tmp;
  int col = 0;
  for (auto& s : segs) {
    tmp.resize((size_t)s.n * B->b.nenv);
    for (int e = 0; e < B->b.nenv; e++)
      for (int i = 0; i < s.n; i++) tmp[(size_t)e * s.n + i] = state[(size_t)e * ns + col + i];
    if (int rc = field_from_host(B, false, s.off, s.n, tmp.data())) return rc;
    col += s.n;
  }
  return 0;
}

int mjb_get_state(mjbBatch* B, double* state, unsigned int sig) {
  std::vector<Seg> segs;
  if (!B || !state || state_segments(B, sig, &segs)) return fail(MJB_ERR_ARG, "mjb_get_state: bad arguments / unsupported signature");
  int ns = 0;
  for (auto& s : segs) ns += s.n;
  std::vector<double> tmp;
  int col = 0;
  for (auto& s : segs) {
    tmp.resize((size_t)s.n * B->b.nenv);
    if (int rc = field_to_host(B, false, s.off, s.n, tmp.data())) return rc;
    for (int e = 0; e < B->b.nenv; e++)
      for (int i = 0; i < s.n; i++) state[(size_t)e * ns + col + i] = tmp[(size_t)e * s.n + i];
    col += s.n;
  }
  return 0;
}

// ---- stepping --------------------------------------------------------------------------------------
// one mj_step of every environment.  skip_warned: rollout rule (environments carrying a warning do
// not step).  Euler: all four stages in ONE fused launch.  RK4 (mj_RungeKutta): forward + acceleration
// check, then three (phase, forward) pairs and the final combination = 8 launches.
static int run_step_on(mjbBatch* B, const Batch& b, void* stream, bool skip_warned, void* stagger = nullptr) {
  const int first = 1 | (skip_warned ? 2 : 0), later = skip_warned ? 4 : 0;
  const int sub = later | 8;   // RK4 sub-steps: mj_forwardSkip(.., skipsensor = 1)
  if (B->hm.dm.opt.integrator == INT_RK4) {
    int rc = backend::launch_stages(B->dm, b, 0x7 | 32, first, stream);
    for (int phase = 1; phase <= 3 && !rc; phase++) {
      rc = backend::launch_rk4(B->dm, b, phase, later, stream);
      if (!rc) rc = backend::launch_stages(B->dm, b, 0x17, sub, stream);
    }
    if (!rc) rc = backend::launch_rk4(B->dm, b, 4, later, stream);
    return rc;
  }
  if (backend::split_step_available(B->dm, b)) return backend::launch_split_step(B->dm, b, first, later, stream, stagger);
  return backend::launch_stages(B->dm, b, 0xF, first, stream);
}
static int run_step(mjbBatch* B, bool skip_warned) { return run_step_on(B, B->b, B->stream, skip_warned); }

// Optional grouped execution of MULTI-step calls (MJB_GROUPS=n, default 1 = off): the batch is cut into
// contiguous env groups, each advanced through all steps on its own stream.  It does not pay off on humanoid x4096
// (PGS), because every group still waits for ITS slowest environment each step and the per-step maximum over 1024
// environments is almost the maximum over 4096.  Kept (bit-identical results, tests/test_groups.py) as
// the scaffold for a finer-grained scheme; calls that return after ONE step always use a single launch.
struct EnvGroup { Batch b; long e0; void* stream; };
static std::vector<EnvGroup> env_groups(mjbBatch* B, int nstep) {
  static int want = -1;
  if (want < 0) { const char* s = getenv("MJB_GROUPS"); want = s ? atoi(s) : 1; if (want < 1) want = 1; }
  int G = want;
  const int nenv = B->b.nenv;
  if (nstep < 2 || nenv < 64 * G) G = 1;
  std::vector<EnvGroup> out;
  const int per = ((nenv + G - 1) / G + 15) / 16 * 16;   // whole CTAs (4, 8 or 16 envs) per group
  for (int g = 0, e0 = 0; e0 < nenv; g++, e0 += per) {
    EnvGroup v{B->b, e0, B->stream};
    v.b.nenv = (e0 + per <= nenv) ? per : nenv - e0;
    v.b.dbl = B->b.dbl + (size_t)e0 * B->b.dpitch;
    v.b.itg = B->b.itg + (size_t)e0 * B->b.ipitch;
    if (g > 0) {
      while ((int)B->gstreams.size() < g) B->gstreams.push_back(backend::stream_create());
      v.stream = B->gstreams[g - 1];
    }
    out.push_back(v);
  }
  return out;
}
static int groups_fork(mjbBatch* B, std::vector<EnvGroup>& gs) {
  for (size_t g = 1; g < gs.size(); g++) if (int rc = backend::stream_order(B->stream, gs[g].stream)) return rc;
  return 0;
}
static int groups_join(mjbBatch* B, std::vector<EnvGroup>& gs) {
  for (size_t g = 1; g < gs.size(); g++) if (int rc = backend::stream_order(gs[g].stream, B->stream)) return rc;
  return 0;
}

int mjb_forward(mjbBatch* B) {
  if (!B) return fail(MJB_ERR_ARG, "null batch");
  if (int rc = backend::launch_stages(B->dm, B->b, 0x17, 0, B->stream)) return rc;   // stages 0,1,2 + dual finish
  return backend::sync(B->stream);
}

int mjb_step(mjbBatch* B, int nstep) {
  if (!B || nstep < 0) return fail(MJB_ERR_ARG, "mjb_step: bad arguments");
  std::vector<EnvGroup> gs = env_groups(B, nstep);
  if (int rc = groups_fork(B, gs)) return rc;
  for (int t = 0; t < nstep; t++)
    for (size_t g = 0; g < gs.size(); g++)
      if (int rc = run_step_on(B, gs[g].b, gs[g].stream, false, (t == 0 && g + 1 < gs.size()) ? gs[g + 1].stream : nullptr)) return rc;
  if (int rc = groups_join(B, gs)) return rc;
  return backend::sync(B->stream);
}

int mjb_run_stages(mjbBatch* B, int first, int last) {
  if (!B || first < 0 || last > 4 || first > last) return fail(MJB_ERR_ARG, "mjb_run_stages: bad range");
  int mask = 0;
  for (int s = first; s <= last; s++) mask |= 1 << s;
  if (int rc = backend::launch_stages(B->dm, B->b, mask, 1, B->stream)) return rc;
  return backend::sync(B->stream);
}

int mjb_set_debug(const char* key, int value) {
  if (!key || backend::set_debug(key, value)) return fail(MJB_ERR_ARG, "mjb_set_debug: unknown key");
  return 0;
}

int mjb_step_profile(mjbBatch* B, float* ms4) {
  if (!B || !ms4) return fail(MJB_ERR_ARG, "mjb_step_profile: bad arguments");
  if (!backend::split_step_available(B->dm, B->b)) return fail(MJB_ERR_UNSUPPORTED, "mjb_step_profile: this batch steps with the fused kernel (one launch)");
  return backend::profile_split_step(B->dm, B->b, B->stream, ms4);
}

int mjb_rollout(mjbBatch* B, int nstep, unsigned int control_spec, const double* state0,
                const double* warmstart0, const double* control, double* state, double* sensordata) {
  if (!B || nstep < 0 || !state0) return fail(MJB_ERR_ARG, "mjb_rollout: bad arguments");
  const int nsens = B->hm.dm.sz.nsensordata;
  if (sensordata && !nsens) return fail(MJB_ERR_ARG, "mjb_rollout: the model has no sensors (nsensordata == 0)");
  const unsigned full = ST_TIME | ST_QPOS | ST_QVEL | ST_ACT | ST_HISTORY | ST_PLUGIN;
  std::vector<Seg> csegs;
  const unsigned user_inputs = ST_CTRL | ST_QFRC_APPLIED | ST_XFRC_APPLIED | ST_EQ_ACTIVE | ST_MOCAP_POS | ST_MOCAP_QUAT;
  if (control && ((control_spec & ~user_inputs) || state_segments(B, control_spec, &csegs)))
    return fail(MJB_ERR_ARG, "mjb_rollout: control_spec may hold CTRL, QFRC_APPLIED, XFRC_APPLIED, EQ_ACTIVE, MOCAP_POS, MOCAP_QUAT only");
  const int nenv = B->b.nenv, nv = B->hm.dm.sz.nv;
  const int nstate = mjb_state_size(B, full);
  int ncontrol = 0;
  for (auto& s : csegs) ncontrol += s.n;
  // defaults for unspecified user inputs, initial state, warmstart, warning counters
  {
    if (!(control_spec & ST_CTRL) || !control) { if (int rc = field_zero(B, false, B->b.L.ctrl, B->hm.dm.sz.nu)) return rc; }
    if (!(control_spec & ST_QFRC_APPLIED) || !control) { if (int rc = field_zero(B, false, B->b.L.qfrc_applied, nv)) return rc; }
    if ((control_spec & ST_XFRC_APPLIED) && control) B->b.xfrc = 1;
    else if (B->b.xfrc) { if (int rc = field_zero(B, false, B->b.L.xfrc_applied, 6 * B->hm.dm.sz.nbody)) return rc; }
    if (B->hm.dm.sz.neq && (!(control_spec & ST_EQ_ACTIVE) || !control)) {   // rollout.cc:110-114
      const int neq = B->hm.dm.sz.neq;
      std::vector<double> ea((size_t)nenv * neq);
      for (int e = 0; e < nenv; e++) for (int i = 0; i < neq; i++) ea[(size_t)e * neq + i] = B->hm.dm.eq_active0[i];
      field_from_host(B, false, B->b.L.eq_active, neq, ea.data());
    }
    const Sizes& S = B->hm.dm.sz;
    if (S.nmocap) {   // unspecified mocap inputs come from the model (rollout.cc:98-109)
      const DModel& hm = B->hm.dm;
      std::vector<double> mp((size_t)nenv * 3 * S.nmocap), mq((size_t)nenv * 4 * S.nmocap);
      for (int e = 0; e < nenv; e++)
        for (int i = 0; i < S.nbody; i++) {
          const int id = hm.body_mocapid[i];
          if (id < 0) continue;
          for (int k = 0; k < 3; k++) mp[((size_t)e * S.nmocap + id) * 3 + k] = hm.body_pos[3 * i + k];
          for (int k = 0; k < 4; k++) mq[((size_t)e * S.nmocap + id) * 4 + k] = hm.body_quat[4 * i + k];
        }
      if (!(control_spec & ST_MOCAP_POS) || !control) field_from_host(B, false, B->b.L.mocap_pos, 3 * S.nmocap, mp.data());
      if (!(control_spec & ST_MOCAP_QUAT) || !control) field_from_host(B, false, B->b.L.mocap_quat, 4 * S.nmocap, mq.data());
    }
    if (int rc = field_zero(B, true, B->b.L.warning, NWARNING)) return rc;
    if (int rc = mjb_set_state(B, state0, full)) return rc;
    if (warmstart0) {
      if (int rc = mjb_set_state(B, warmstart0, ST_WARMSTART)) return rc;
    } else {
      if (int rc = field_zero(B, false, B->b.L.qacc_warmstart, nv)) return rc;
    }
  }
  double* d_control = nullptr;
  double* d_state = nullptr;
  const size_t cbytes = (size_t)nenv * nstep * ncontrol * sizeof(double);
  const size_t sbytes = (size_t)nenv * nstep * nstate * sizeof(double);
  // device-side images of the caller's arrays: kept in the batch and grown on demand (an allocation per call costs
  // more than the copies of a short rollout)
  auto reserve = [&](int k, size_t bytes) -> double* {
    if (B->roll_bytes[k] < bytes) {
      backend::sync(B->stream);
      backend::dev_free(B->roll[k]);
      B->roll[k] = backend::dev_alloc(bytes);
      B->roll_bytes[k] = B->roll[k] ? bytes : 0;
    }
    return (double*)B->roll[k];
  };
  if (control && ncontrol && nstep) {
    d_control = reserve(0, cbytes);
    if (!d_control) return fail(MJB_ERR_CUDA, "device allocation failed (control)");
    backend::h2d(d_control, control, cbytes, B->stream);
  }
  if (state && nstep) {
    d_state = reserve(1, sbytes);
    if (!d_state) return fail(MJB_ERR_CUDA, "device allocation failed (state)");
  }
  double* d_sens = nullptr;
  const size_t nbytes = (size_t)nenv * nstep * nsens * sizeof(double);
  if (sensordata && nstep) {
    d_sens = reserve(2, nbytes);
    if (!d_sens) return fail(MJB_ERR_CUDA, "device allocation failed (sensordata)");
  }
  std::vector<EnvGroup> gs = env_groups(B, nstep);
  int rc = groups_fork(B, gs);
  // the states of a finished chunk of steps travel to the host while the next chunks are stepped: every launch is
  // enqueued first, an event marks the end of each chunk, and the (strided: [env][step][state]) copies follow on a
  // second stream.  Single group only; with several groups the copy follows the join.
  const int nchunk = (gs.size() == 1 && d_state && nstep >= 8) ? 4 : 1;
  std::vector<void*> chunk_ev;
  std::vector<int> chunk_end;
  // persistent kernel (mjb_krollout.cu): one launch per chunk of steps, no device-wide barrier inside a chunk
  bool persistent = !rc && gs.size() == 1 && !d_sens && (!d_control || control_spec == ST_CTRL) &&
                    backend::rollout_persistent_available(B->dm, B->b, nstep);
  if (persistent) {
    const int per = (nstep + nchunk - 1) / nchunk;
    for (int t0 = 0; t0 < nstep && !rc; t0 += per) {
      const int t1 = t0 + per < nstep ? t0 + per : nstep;
      rc = backend::launch_rollout_persistent(B->dm, B->b, t0, t1, nstep, 1 | 2, 4, 1, d_control, d_state, nstate, B->stream);
      if (rc == -1) { persistent = false; rc = 0; break; }   // the batch does not fit the mapping (decided before any launch)
      if (nchunk > 1 && !rc) {
        void* ev = backend::event_record(B->stream);
        if (ev) { chunk_ev.push_back(ev); chunk_end.push_back(t1); }
      }
    }
  }
  for (int t = 0; t < nstep && !rc && !persistent; t++) {
    for (size_t gi = 0; gi < gs.size(); gi++) {
      auto& g = gs[gi];
      if (d_control && !rc) rc = backend::launch_set_control(B->dm, g.b, d_control + (size_t)g.e0 * nstep * ncontrol, nstep, t, control_spec, ncontrol, g.stream);
      if (!rc) rc = run_step_on(B, g.b, g.stream, true, (t == 0 && gi + 1 < gs.size()) ? gs[gi + 1].stream : nullptr);
      if (d_state && !rc) rc = backend::launch_get_state(B->dm, g.b, d_state + (size_t)g.e0 * nstep * nstate, nstep, t, nstate, g.stream);
      if (d_sens && !rc) rc = backend::launch_get_sensor(B->dm, g.b, d_sens + (size_t)g.e0 * nstep * nsens, nstep, t, nsens, g.stream);
    }
    if (nchunk > 1 && !rc && ((t + 1) % ((nstep + nchunk - 1) / nchunk) == 0 || t + 1 == nstep)) {
      void* ev = backend::event_record(B->stream);
      if (ev) { chunk_ev.push_back(ev); chunk_end.push_back(t + 1); }
    }
  }
  if (!rc) rc = groups_join(B, gs);
  if (!rc && d_state) {
    if (nchunk > 1 && !chunk_end.empty() && chunk_end.back() == nstep) {
      if (!B->copy_stream) B->copy_stream = backend::stream_create();
      const size_t pitch = (size_t)nstep * nstate * sizeof(double);
      int t0 = 0;
      for (size_t c = 0; c < chunk_ev.size() && !rc; c++) {
        rc = backend::stream_wait_event(B->copy_stream, chunk_ev[c]);
        if (!rc) rc = backend::d2h_2d(state + (size_t)t0 * nstate, pitch, d_state + (size_t)t0 * nstate, pitch,
                                      (size_t)(chunk_end[c] - t0) * nstate * sizeof(double), (size_t)nenv, B->copy_stream);
        t0 = chunk_end[c];
      }
      if (!rc) rc = backend::sync(B->copy_stream);
    } else {
      for (void* ev : chunk_ev) backend::stream_wait_event(B->stream, ev);   // (releases the events)
      rc = backend::d2h(state, d_state, sbytes, B->stream);
    }
  }
  if (!rc && d_sens) rc = backend::d2h(sensordata, d_sens, nbytes, B->stream);
  if (!rc) rc = backend::sync(B->stream);
  return rc;
}

int mjb_step_host(mjbBatch* B, const double* ctrl, double* state_out) {
  if (!B || !ctrl || !state_out) return fail(MJB_ERR_ARG, "mjb_step_host: bad arguments");
  const int nenv = B->b.nenv, nu = B->hm.dm.sz.nu;
  const int nstate = 1 + B->hm.dm.sz.nq + B->hm.dm.sz.nv + B->hm.dm.sz.na + B->hm.dm.sz.nhistory;
  if (!B->io_ctrl) {
    B->io_ctrl = (double*)backend::dev_alloc((size_t)nenv * nu * sizeof(double));
    B->io_state = (double*)backend::dev_alloc((size_t)nenv * nstate * sizeof(double));
    if (!B->io_ctrl || !B->io_state) return fail(MJB_ERR_CUDA, "device allocation failed (io staging)");
  }
  int rc = backend::h2d(B->io_ctrl, ctrl, (size_t)nenv * nu * sizeof(double), B->stream);
  if (!rc) rc = backend::launch_set_control(B->dm, B->b, B->io_ctrl, 1, 0, ST_CTRL, nu, B->stream, /*skip_warned=*/false);
  if (!rc) rc = run_step(B, false);
  if (!rc) rc = backend::launch_get_state(B->dm, B->b, B->io_state, 1, 0, nstate, B->stream);
  if (!rc) rc = backend::d2h(state_out, B->io_state, (size_t)nenv * nstate * sizeof(double), B->stream);
  if (!rc) rc = backend::sync(B->stream);
  return rc;
}

int mjb_rollout_device(mjbBatch* B, int nstep, const double* d_ctrl, double* d_state) {
  if (!B || nstep < 0) return fail(MJB_ERR_ARG, "mjb_rollout_device: bad arguments");
  const int nstate = 1 + B->hm.dm.sz.nq + B->hm.dm.sz.nv + B->hm.dm.sz.na + B->hm.dm.sz.nhistory;
  // per-step launches (fused step or split step) unless the persistent rollout kernel applies; a persistent kernel
  // whose WARPS drift apart is slower (the instruction working set no longer fits the
  // instruction caches) - mjb_krollout.cu keeps the warps of a CTA in step and lets only the CTAs drift
  std::vector<EnvGroup> gs = env_groups(B, nstep);
  if (gs.size() == 1 && backend::rollout_persistent_available(B->dm, B->b, nstep)) {
    // every step in one persistent launch (mjb_krollout.cu): each CTA carries its own environments through the steps
    const int rc = backend::launch_rollout_persistent(B->dm, B->b, 0, nstep, nstep, 1, 0, 0, d_ctrl, d_state, nstate, B->stream);
    if (rc != -1) return rc;
  }
  int rc = groups_fork(B, gs);
  for (int t = 0; t < nstep && !rc; t++) {
    for (size_t gi = 0; gi < gs.size(); gi++) {   // native layouts are [..][elem][env]: a group starts e0 elements further
      auto& g = gs[gi];
      if (d_ctrl && !rc) rc = backend::launch_set_control_native(B->dm, g.b, d_ctrl + g.e0, t, g.stream);
      if (!rc) rc = run_step_on(B, g.b, g.stream, false, (t == 0 && gi + 1 < gs.size()) ? gs[gi + 1].stream : nullptr);
      if (d_state && !rc) rc = backend::launch_get_state_native(B->dm, g.b, d_state + g.e0, t, nstate, g.stream);
    }
  }
  if (!rc) rc = groups_join(B, gs);
  return rc;   // asynchronous: caller synchronises on mjb_stream()
}

// ---- field access ----------------------------------------------------------------------------------
static bool find_field(const mjbBatch* B, const char* name, long* off, long* cnt, bool* is_int) {
  const Sizes& S = B->hm.dm.sz;
  const Layout& L = B->b.L;
  (void)S;
#define X(fname, count) if (!strcmp(name, #fname)) { *off = L.fname; *cnt = (long)(count); *is_int = false; return true; }
  MJB_DATA_DBL_FIELDS(X, S)
  MJB_DATA_COLD_FIELDS(X, S)
  MJB_DATA_WRAP_FIELDS(X, S)
  MJB_DATA_HIST_FIELDS(X, S)
#undef X
#define X(fname, count) if (!strcmp(name, #fname)) { *off = L.fname; *cnt = (long)(count); *is_int = true; return true; }
  MJB_DATA_INT_FIELDS(X, S)
  MJB_DATA_WRAP_INT_FIELDS(X, S)
#undef X
  return false;
}

long mjb_field_size(const mjbBatch* B, const char* name) {
  long off, cnt; bool is_int;
  if (!B || !find_field(B, name, &off, &cnt, &is_int)) return -1;
  return cnt;
}

int mjb_get_field(mjbBatch* B, const char* name, double* out) {
  long off, cnt; bool is_int;
  if (!B || !out || !find_field(B, name, &off, &cnt, &is_int) || is_int) return fail(MJB_ERR_ARG, std::string("mjb_get_field: unknown double field ") + (name ? name : ""));
  return field_to_host(B, false, off, cnt, out);
}

int mjb_get_field_int(mjbBatch* B, const char* name, int* out) {
  long off, cnt; bool is_int;
  if (!B || !out || !find_field(B, name, &off, &cnt, &is_int) || !is_int) return fail(MJB_ERR_ARG, std::string("mjb_get_field_int: unknown int field ") + (name ? name : ""));
  return field_to_host(B, true, off, cnt, out);
}

int mjb_set_field(mjbBatch* B, const char* name, const double* in) {
  long off, cnt; bool is_int;
  if (!B || !in || !find_field(B, name, &off, &cnt, &is_int) || is_int) return fail(MJB_ERR_ARG, std::string("mjb_set_field: unknown double field ") + (name ? name : ""));
  if (!strcmp(name, "xfrc_applied")) B->b.xfrc = 1;
  return field_from_host(B, false, off, cnt, in);
}

// ---- mjData bridge: mj_step for a set of the reference's own mjData objects ---------------------------
// The reference steps one mjData per environment (`for k: mj_step(m, d[k])`, sample/testspeed.cc:123,
// rollout.cc:85-177).  mjb_step_mjdata is that loop as one call: inputs are read from every d[e]
// (time, qpos, qvel, ctrl, qfrc_applied, qacc_warmstart), the batch takes one mj_step, and the state plus
// every fixed-size mjData array the path computes is written back under the same member name, so code
// that reads mjData after mj_step keeps working.  Arena-allocated members (contact, efc_*) are not
// materialised on the host and ncon / nefc are published as ZERO (see bridge_mjdata); warning counters are added.
#define MJB_MJDATA_IN(X) X(qpos, nq) X(qvel, nv) X(act, na) X(mocap_pos, 3 * nmocap) X(mocap_quat, 4 * nmocap) X(xfrc_applied, 6 * nbody) X(ctrl, nu) X(qfrc_applied, nv) X(qacc_warmstart, nv)
// every fixed-size mjData array the path computes (position, velocity, acceleration stage; sensors and the
// rnePostConstraint / subtreeVel outputs where the model's sensors make the batch compute them)
#define MJB_MJDATA_OUT(X)                                                                                   \
  X(qpos, nq) X(qvel, nv) X(act, na) X(act_dot, na) X(qacc_warmstart, nv) X(qacc, nv)                       \
  X(xpos, 3 * nbody) X(xquat, 4 * nbody) X(xmat, 9 * nbody) X(xipos, 3 * nbody) X(ximat, 9 * nbody)         \
  X(xanchor, 3 * njnt) X(xaxis, 3 * njnt) X(geom_xpos, 3 * ngeom) X(geom_xmat, 9 * ngeom)                   \
  X(site_xpos, 3 * nsite) X(site_xmat, 9 * nsite)                                                           \
  X(subtree_com, 3 * nbody) X(cinert, 10 * nbody) X(cdof, 6 * nv) X(crb, 10 * nbody) X(M, nC) X(qLD, nC)    \
  X(qLDiagInv, nv) X(ten_length, ntendon) X(actuator_length, nu) X(ten_velocity, ntendon)                   \
  X(actuator_velocity, nu) X(cvel, 6 * nbody) X(cdof_dot, 6 * nv) X(qfrc_spring, nv) X(qfrc_damper, nv)     \
  X(qfrc_passive, nv) X(qfrc_bias, nv) X(actuator_force, nu) X(qfrc_actuator, nv) X(qfrc_smooth, nv)        \
  X(qacc_smooth, nv) X(qfrc_constraint, nv) X(sensordata, nsensordata) X(energy, 2)                                    \
  X(subtree_linvel, 3 * nbody * subtreevel) X(subtree_angmom, 3 * nbody * subtreevel)                       \
  X(cacc, 6 * nbody * rnepost) X(cfrc_int, 6 * nbody * rnepost) X(cfrc_ext, 6 * nbody * rnepost)

// what the bridge runs between copying the inputs in and the results out
enum BridgeOp { BR_STEP, BR_FORWARD, BR_FORWARD_NOSENSOR, BR_STEP1, BR_STEP2 };

static int bridge_mjdata(mjbBatch* B, mjData* const* d, int nd, BridgeOp op) {
  if (!B || !d || nd != B->b.nenv) return fail(MJB_ERR_ARG, "mjData bridge: need one mjData per environment");
  const Sizes& S = B->hm.dm.sz;
  const int nenv = B->b.nenv;
  const int nq = S.nq, nv = S.nv, nu = S.nu, na = S.na, nmocap = S.nmocap, nbody = S.nbody, njnt = S.njnt, ngeom = S.ngeom,
            ntendon = S.ntendon, nC = S.nC, nsite = S.nsite, nsensordata = S.nsensordata, subtreevel = S.subtreevel, rnepost = S.rnepost;
  (void)na; (void)nmocap; (void)nbody; (void)njnt; (void)ngeom; (void)ntendon; (void)nC; (void)nsite; (void)nsensordata; (void)subtreevel; (void)rnepost;
  std::vector<double> tmp;
  for (int e = 0; e < nenv && !B->b.xfrc; e++)
    for (int k = 0; k < 6 * nbody; k++) if (d[e]->xfrc_applied[k] != 0) { B->b.xfrc = 1; break; }
  {
    tmp.resize(nenv);
    for (int e = 0; e < nenv; e++) tmp[e] = d[e]->time;
    if (int rc = field_from_host(B, false, B->b.L.time, 1, tmp.data())) return rc;
  }
#define X(name, cnt)                                                                             \
  if ((cnt) > 0) {                                                                               \
    tmp.resize((size_t)nenv * (cnt));                                                            \
    for (int e = 0; e < nenv; e++) memcpy(tmp.data() + (size_t)e * (cnt), d[e]->name, sizeof(double) * (cnt)); \
    if (int rc = field_from_host(B, false, B->b.L.name, (cnt), tmp.data())) return rc;            \
  }
  MJB_MJDATA_IN(X)
  MJB_DATA_HIST_FIELDS(X, S)   // history buffers (allocated only for models with them)
#undef X
  if (S.neq) {   // mjData.eq_active is a byte array
    tmp.resize((size_t)nenv * S.neq);
    for (int e = 0; e < nenv; e++) for (int i = 0; i < S.neq; i++) tmp[(size_t)e * S.neq + i] = d[e]->eq_active[i];
    if (int rc = field_from_host(B, false, B->b.L.eq_active, S.neq, tmp.data())) return rc;
  }
  int rc = 0;
  switch (op) {
    case BR_STEP: rc = run_step(B, false); break;
    case BR_FORWARD: rc = backend::launch_stages(B->dm, B->b, 0x17, 0, B->stream); break;
    case BR_FORWARD_NOSENSOR: rc = backend::launch_stages(B->dm, B->b, 0x17, 8, B->stream); break;
    // mj_step1 (engine_forward.c:1884-1905): checks, position and velocity stages.  The velocity launch of this
    // path also evaluates actuation / acceleration; mj_step2 recomputes those from the controls it is given.
    case BR_STEP1: rc = backend::launch_stages(B->dm, B->b, 1 | 2, 1, B->stream); break;
    // mj_step2 (:1909-1940): actuation, acceleration, constraint, acceleration check, integration (Euler family)
    case BR_STEP2: rc = backend::launch_stages(B->dm, B->b, 2 | 4 | 8, 0, B->stream); break;
  }
  if (rc) return rc;
  {
    tmp.resize(nenv);
    if (int rc2 = field_to_host(B, false, B->b.L.time, 1, tmp.data())) return rc2;
    for (int e = 0; e < nenv; e++) d[e]->time = tmp[e];
  }
#define X(name, cnt)                                                                             \
  if ((cnt) > 0) {                                                                               \
    tmp.resize((size_t)nenv * (cnt));                                                            \
    if (int rc2 = field_to_host(B, false, B->b.L.name, (cnt), tmp.data())) return rc2;            \
    for (int e = 0; e < nenv; e++) memcpy(d[e]->name, tmp.data() + (size_t)e * (cnt), sizeof(double) * (cnt)); \
  }
  MJB_MJDATA_OUT(X)
  MJB_DATA_WRAP_FIELDS(X, S)   // spatial tendon paths (allocated only for models with spatial tendons)
  MJB_DATA_HIST_FIELDS(X, S)   // history buffers
#undef X
#define X(name, cnt)                                                                             \
  if ((cnt) > 0) {                                                                               \
    std::vector<int> it((size_t)nenv * (cnt));                                                   \
    if (int rc2 = field_to_host(B, true, B->b.L.name, (cnt), it.data())) return rc2;              \
    for (int e = 0; e < nenv; e++) memcpy(d[e]->name, it.data() + (size_t)e * (cnt), sizeof(int) * (cnt)); \
  }
  MJB_DATA_WRAP_INT_FIELDS(X, S)
#undef X
  // Arena members (contact, efc_*) are NOT materialised in the reference's mjData: the arena allocator is private
  // to the reference library.  The counts are therefore published as zero - an mjData that claims ncon contacts
  // without holding them would make mj_contactForce / the visualiser / `d.contact` read stale memory.  The batch's
  // own counts and lists are available by name (mjb_get_field_int(b, "ncon") ..., "con_*", "efc_*").
  for (int e = 0; e < nenv; e++) { d[e]->ncon = 0; d[e]->nefc = 0; d[e]->ne = 0; d[e]->nf = 0; d[e]->nl = 0; }
  std::vector<int> it((size_t)nenv * NWARNING);
  if (int rc2 = field_to_host(B, true, B->b.L.warning, NWARNING, it.data())) return rc2;
  for (int e = 0; e < nenv; e++)
    for (int w = 0; w < NWARNING && w < (int)mjNWARNING; w++) {
      // the batch counts warnings since its last reset; mjData accumulates: add what this step raised
      const int n = it[(size_t)e * NWARNING + w];
      if (n && !d[e]->warning[w].number) route_warning(w, d[e]->time);   // first occurrence: mju_warning, like mj_warning
      d[e]->warning[w].number += n;
    }
  return field_zero(B, true, B->b.L.warning, NWARNING) || backend::sync(B->stream);
}

int mjb_step_mjdata(mjbBatch* B, struct mjData_* const* dd, int nd) { return bridge_mjdata(B, (mjData* const*)dd, nd, BR_STEP); }
int mjb_forward_mjdata(mjbBatch* B, struct mjData_* const* dd, int nd) { return bridge_mjdata(B, (mjData* const*)dd, nd, BR_FORWARD); }

// _unsafe_rollout's own argument list (rollout.cc:67-78): one mjModel pointer per environment.  This path shares
// one flattened model among the environments of a batch, so the pointers must all name the same model; the
// batch is created for the call and released after it.
int mjb_rollout_models(const struct mjModel_* const* m, int nbatch, int nstep, unsigned int control_spec, const double* state0,
                       const double* warmstart0, const double* control, double* state, double* sensordata, int device) {
  if (!m || nbatch <= 0) return fail(MJB_ERR_ARG, "mjb_rollout_models: bad arguments");
  for (int e = 1; e < nbatch; e++)
    if (m[e] != m[0]) return fail(MJB_ERR_UNSUPPORTED, "unsupported: a different mjModel per environment (share one model, or make one batch per model)");
  mjbBatch* B = mjb_make_batch(m[0], nbatch, 0, 0, device);
  if (!B) return MJB_ERR_UNSUPPORTED;
  const int rc = mjb_rollout(B, nstep, control_spec, state0, warmstart0, control, state, sensordata);
  const std::string msg = rc ? get_error() : "";
  mjb_free_batch(B);
  if (rc) set_error(msg);
  return rc;
}

// ---- the reference's single-environment entry points (include/mujoco/mujoco.h:189-204) ------------------------
// Exported under their own names so that a host written against the reference (sample/testspeed.cc's loop, the
// Python bindings' functions.cc) can resolve them in libmjb200.so: each call is a batch of ONE environment on the
// mjData bridge above.  One batch is cached per mjModel pointer; call mjb_forget_model(m) after editing the model
// (options, parameters) or before freeing it.  Fatal conditions go to mju_error when the reference library is
// loaded in the process (the Python bindings intercept it, python/mujoco/errors.h:140-226), else to stderr + abort,
// which is what mju_error does by default.
namespace {
std::mutex g_shim_mutex;
std::map<const mjModel*, mjbBatch*> g_shim_batches;

void shim_call(const mjModel* m, mjData* d, BridgeOp op, const char* what) {
  std::lock_guard<std::mutex> lock(g_shim_mutex);
  mjbBatch*& B = g_shim_batches[m];
  if (!B) B = mjb_make_batch((const struct mjModel_*)m, 1, 0, 0, -1);
  if (!B) { g_shim_batches.erase(m); route_error(std::string(what) + ": " + get_error()); return; }
  mjData* one[1] = {d};
  if (bridge_mjdata(B, one, 1, op)) route_error(std::string(what) + ": " + get_error());
}
}  // namespace

void mjb_forget_model(const struct mjModel_* m) {
  std::lock_guard<std::mutex> lock(g_shim_mutex);
  auto it = g_shim_batches.find((const mjModel*)m);
  if (it == g_shim_batches.end()) return;
  mjb_free_batch(it->second);
  g_shim_batches.erase(it);
}

MJB_API void mj_step(const mjModel* m, mjData* d) { shim_call(m, d, BR_STEP, "mj_step"); }
MJB_API void mj_forward(const mjModel* m, mjData* d) { shim_call(m, d, BR_FORWARD, "mj_forward"); }
// skipstage only skips recomputation of stages whose inputs did not change (engine_forward.c:1783-1842): running
// them again gives the same values, so the shim honours skipsensor and recomputes the stages
MJB_API void mj_forwardSkip(const mjModel* m, mjData* d, int skipstage, int skipsensor) {
  (void)skipstage;
  shim_call(m, d, skipsensor ? BR_FORWARD_NOSENSOR : BR_FORWARD, "mj_forwardSkip");
}
MJB_API void mj_step1(const mjModel* m, mjData* d) { shim_call(m, d, BR_STEP1, "mj_step1"); }
MJB_API void mj_step2(const mjModel* m, mjData* d) {
  if (m->opt.integrator == mjINT_RK4) { route_error("mj_step2: the Runge-Kutta integrator cannot be split (engine_forward.c:1909), call mj_step"); return; }
  shim_call(m, d, BR_STEP2, "mj_step2");
}

int mjb_set_thread_mapping(int warp_per_env) {
  g_warp_per_env = warp_per_env ? 1 : 0;
  return 0;
}

int mjb_warning_counts(mjbBatch* B, int* out) { return mjb_get_field_int(B, "warning", out); }

}  // extern "C"
