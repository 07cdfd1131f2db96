/* mjb.h — C ABI of libmjb200: an H100-native (sm_90a) batched implementation of MuJoCo's mj_step hot path.
 *
 * Drop-in boundary.  The library consumes the reference's own `mjModel` (const, as produced by
 * mj_loadXML / mj_loadModel / the Python bindings' MjModel._address) and keeps the reference's
 * array contracts for state and control, so it slots in under python/mujoco/rollout.py:
 *
 *   reference interface replaced                         (file:line, /root/reference)
 *   --------------------------------------------------------------------------------------------
 *   mj_step(const mjModel*, mjData*)                     include/mujoco/mujoco.h:189   -> mjb_step
 *   mj_forward(const mjModel*, mjData*)                  include/mujoco/mujoco.h:198   -> mjb_forward
 *   mj_stateSize / mj_getState / mj_setState             include/mujoco/mujoco.h:505-515
 *                                                                     -> mjb_state_size/get/set_state
 *   _unsafe_rollout(m, d, start, end, nstep, control_spec, state0, warmstart0, control, state,
 *                   sensordata)                          python/mujoco/rollout.cc:67-178 -> mjb_rollout
 *   mj_resetData                                         include/mujoco/mujoco.h:249   -> mjb_reset
 *   mj_loadModel (MJB binary)                            include/mujoco/mujoco.h:117   -> mjb_load_model
 *
 * All arrays are C-contiguous fp64 (mjtNum == double) HOST buffers unless a function name says
 * "device"; layouts are the reference's: state vectors are the concatenation selected by the
 * mjtState bit signature (include/mujoco/mjtype.h:503-527) per environment.
 *
 * Errors: every int-returning entry point returns 0 on success and a negative code on failure;
 * mjb_last_error() returns a thread-local message.  The library FAILS LOUDLY (error return, no
 * CPU fallback) when no CUDA device is usable or when the model uses a feature outside the
 * supported hot path (mjb_check_model lists the reason).
 */
#ifndef MJB_H_
#define MJB_H_

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define MJB_API __attribute__((visibility("default")))
#else
#define MJB_API
#endif

struct mjModel_;                       /* the reference's mjModel (include/mujoco/mjmodel.h:242) */
typedef struct mjbBatch_ mjbBatch;     /* opaque: replicated device model + SoA batch of environments */

/* error codes */
enum {
  MJB_OK = 0,
  MJB_ERR_ARG = -1,          /* bad argument / size mismatch (rollout.cc raises value_error) */
  MJB_ERR_UNSUPPORTED = -2,  /* model feature outside the accelerated path */
  MJB_ERR_CUDA = -3,         /* CUDA runtime failure or no device */
  MJB_ERR_IO = -4            /* file / format error */
};

MJB_API const char* mjb_last_error(void);
MJB_API int mjb_version(void);

/* ---- model ------------------------------------------------------------------------------------ */
/* Load an MJB binary (written by the reference's mj_saveModel) into a heap mjModel with the
 * reference's struct layout.  Free with mjb_free_model.  Returns NULL on error. */
MJB_API struct mjModel_* mjb_load_model(const char* mjb_path);
MJB_API void mjb_free_model(struct mjModel_* m);
/* 0 if the model is fully supported by the accelerated path, else MJB_ERR_UNSUPPORTED and
 * mjb_last_error() names the first unsupported feature. */
MJB_API int mjb_check_model(const struct mjModel_* m);
/* integer model sizes by name ("nq","nv","nu","nbody","ngeom",...); -1 if unknown */
MJB_API long mjb_model_size(const struct mjModel_* m, const char* name);
/* read / write mjOption scalars by name ("timestep","solver","integrator","iterations",
 * "tolerance","disableflags",...) on a model; returns 0 or MJB_ERR_ARG */
MJB_API int mjb_get_option(const struct mjModel_* m, const char* name, double* value);
MJB_API int mjb_set_option(struct mjModel_* m, const char* name, double value);

/* ---- batch ------------------------------------------------------------------------------------ */
/* Create nenv environments of model m on CUDA device `device` (ordinal; -1 = current device).
 * nconmax / njmax are per-environment caps replacing the reference's per-mjData arena
 * (0 = library default for the model).  m->opt is captured at creation. */
MJB_API mjbBatch* mjb_make_batch(const struct mjModel_* m, int nenv, int nconmax, int njmax, int device);
MJB_API void mjb_free_batch(mjbBatch* b);
/* thread mapping used by batches created afterwards: 1 (default) = one warp per environment with
 * env-major storage, 0 = one lane per environment with field-major (SoA across envs) storage */
MJB_API int mjb_set_thread_mapping(int warp_per_env);
MJB_API int mjb_nenv(const mjbBatch* b);

/* mj_resetData on every environment: qpos = qpos0, everything else zero */
MJB_API int mjb_reset(mjbBatch* b);

/* state I/O with the reference's signature semantics; supported bits: mjSTATE_TIME, QPOS, QVEL,
 * ACT, HISTORY (the nhistory doubles of the actuator and sensor history buffers, mjData.history), WARMSTART, CTRL,
 * QFRC_APPLIED, XFRC_APPLIED, MOCAP_POS, MOCAP_QUAT,  (mjSTATE_FULLPHYSICS = TIME|QPOS|QVEL|ACT|HISTORY|...),
 * EQ_ACTIVE (0 / 1 as doubles, like mj_setState).  Once xfrc_applied has been written the
 * batch steps with the full kernels instead of the lean ones (a model without optional features otherwise). */
MJB_API int mjb_state_size(const mjbBatch* b, unsigned int sig);
MJB_API int mjb_set_state(mjbBatch* b, const double* state /* [nenv][size(sig)] */, unsigned int sig);
MJB_API int mjb_get_state(mjbBatch* b, double* state /* [nenv][size(sig)] */, unsigned int sig);

/* mj_forward / mj_step on all environments (nstep consecutive steps with the current ctrl) */
MJB_API int mjb_forward(mjbBatch* b);
MJB_API int mjb_step(mjbBatch* b, int nstep);

/* Batched rollout with the array contract of python/mujoco/rollout.cc:67-178:
 *   state0     [nenv][nstate]          mjSTATE_FULLPHYSICS initial states
 *   warmstart0 [nenv][nv] or NULL      initial qacc_warmstart (NULL -> zeros)
 *   control    [nenv][nstep][ncontrol] or NULL, ncontrol = mjb_state_size(control_spec)
 *   state      [nenv][nstep][nstate] or NULL  (output)
 *   sensordata [nenv][nstep][nsensordata] or NULL  (output; supported sensor types: mjb_check_model)
 * Environments that raise a warning stop stepping and pad their outputs with the current state,
 * as the reference does (rollout.cc:127-155). */
MJB_API int mjb_rollout(mjbBatch* b, int nstep, unsigned int control_spec,
                        const double* state0, const double* warmstart0, const double* control,
                        double* state, double* sensordata);

/* One mj_step for every environment with per-step host I/O (the end-to-end call an RL loop makes):
 * ctrl [nenv][nu] host (pinned for best speed) is copied in, the step runs, and the new
 * mjSTATE_FULLPHYSICS state [nenv][nstate] is copied back; returns after the copy completed. */
MJB_API int mjb_step_host(mjbBatch* b, const double* ctrl, double* state_out);

/* mj_step for the reference's own mjData objects, one per environment (replaces the per-thread loop
 * `for k: mj_step(m, d[k])`, sample/testspeed.cc:123 / python/mujoco/rollout.cc:85-177): reads time, qpos,
 * qvel, ctrl, qfrc_applied, qacc_warmstart and history from every d[e], steps the batch once, and writes the new state
 * and every fixed-size mjData array the path computes back under the same member names (plus ncon, nefc and
 * the warning counters; arena members - contact, efc_* - stay on the device: use mjb_get_field). */
struct mjData_;
MJB_API int mjb_step_mjdata(mjbBatch* b, struct mjData_* const* d, int nd);

/* Same, with DEVICE-resident control / state buffers in the library's native layout
 * ([nstep][ncontrol][nenv_stride] and [nstep][nstate][nenv_stride]); used by bench.py's
 * HBM-resident throughput measurement.  Either pointer may be NULL. */
MJB_API int mjb_rollout_device(mjbBatch* b, int nstep, const double* d_ctrl, double* d_state);
MJB_API long mjb_env_stride(const mjbBatch* b);

/* per-environment field access by mjData field name ("qpos","xpos","cinert","qM"/"M","qLD",
 * "efc_J","efc_AR","contact_dist",...).  Output is [nenv][count] in the reference's per-env
 * (row-major) layout.  count is returned by mjb_field_size (-1 if unknown). */
MJB_API long mjb_field_size(const mjbBatch* b, const char* name);
MJB_API int mjb_get_field(mjbBatch* b, const char* name, double* out);
MJB_API int mjb_get_field_int(mjbBatch* b, const char* name, int* out);
MJB_API int mjb_set_field(mjbBatch* b, const char* name, const double* in);

/* mj_forward on the reference's own mjData objects (as mjb_step_mjdata, without integration) */
MJB_API int mjb_forward_mjdata(mjbBatch* b, struct mjData_* const* d, int nd);

/* _unsafe_rollout's own argument list (python/mujoco/rollout.cc:67-78): one mjModel pointer per environment.  All
 * pointers must name the same model (this path shares one flattened model per batch; MJB_ERR_UNSUPPORTED
 * otherwise).  The batch lives for the call.  Arrays as in mjb_rollout. */
MJB_API int mjb_rollout_models(const struct mjModel_* const* m, int nbatch, int nstep, unsigned int control_spec,
                               const double* state0, const double* warmstart0, const double* control, double* state,
                               double* sensordata, int device);

/* The reference's single-environment entry points, include/mujoco/mujoco.h:189-204, with the reference's
 * signatures and semantics: a host linked (or dlopen-ed) against libmjb200.so instead of libmujoco for these five
 * symbols steps its mjData on the GPU, one environment per call (a batch of 1 on the mjData bridge; one cached
 * batch per mjModel pointer - mjb_forget_model() after editing or before freeing a model).  mjData.ncon / nefc
 * read 0 afterwards (arena members are not materialised, see INTEGRATION.md).  Fatal conditions are reported
 * through the process's mju_error when the reference library is loaded, else stderr + abort (mju_error's default);
 * first occurrences of a warning through mju_warning. */
MJB_API void mj_step(const struct mjModel_* m, struct mjData_* d);
MJB_API void mj_forward(const struct mjModel_* m, struct mjData_* d);
MJB_API void mj_forwardSkip(const struct mjModel_* m, struct mjData_* d, int skipstage, int skipsensor);
MJB_API void mj_step1(const struct mjModel_* m, struct mjData_* d);
MJB_API void mj_step2(const struct mjModel_* m, struct mjData_* d);
MJB_API void mjb_forget_model(const struct mjModel_* m);

/* statistics of the last mjb_step/mjb_rollout call */
MJB_API long mjb_kernel_launches(const mjbBatch* b);   /* cumulative number of kernels launched */
MJB_API int mjb_warning_counts(mjbBatch* b, int* out /* [nenv][8] */);

/* staged execution for tests/profiling: run only pipeline stages [first,last] of one step
 * (0 position, 1 velocity+actuation+acceleration, 2 constraint solve, 3 integrate) */
MJB_API int mjb_run_stages(mjbBatch* b, int first, int last);

/* one mj_step of every environment (as mjb_step(b, 1)) that also reports the duration in ms of the launches the
 * step is made of, timed with CUDA events on the batch's stream: ms4 = {position + velocity half, constraint
 * solve, finish + integrate half, redo launch}.  MJB_ERR_UNSUPPORTED when the batch steps with one fused launch. */
MJB_API int mjb_step_profile(mjbBatch* b, float* ms4);

/* test switches (process-wide).  "pgs4_slots" = 1: the PGS kernel takes its fallback shared-memory layout;
 * "persistent" = 0: multi-step rollouts of eligible batches step launch by launch instead of in the persistent
 * rollout kernel (1, the default). */
MJB_API int mjb_set_debug(const char* key, int value);

/* CUDA stream used by the batch (cudaStream_t as void*), e.g. for event timing by the caller */
MJB_API void* mjb_stream(mjbBatch* b);

/* Run the batch on the CALLER's stream from now on (cudaStream_t as void*; NULL: back to the batch's own stream).
 * Every launch and copy of the batch is then ordered with the caller's other work on that stream, as a caller of the
 * reference orders mj_step with its own code by program order.  The batch's own stream is drained first; the
 * caller keeps ownership of its stream and must keep it alive while it is set.  Multi-step rollouts of eligible
 * batches also run as ONE persistent launch on it (mjb_krollout.cu; mjb_set_debug("persistent", 0) turns that off). */
MJB_API int mjb_set_stream(mjbBatch* b, void* stream);

#ifdef __cplusplus
}
#endif
#endif  /* MJB_H_ */
