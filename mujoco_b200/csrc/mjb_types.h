// Device-side model (flattened, read-only, replicated per GPU) and the batch data layout for the
// batched mj_step path.
//
// Storage is env-major: every environment owns one contiguous block of doubles (hot fields first,
// the cold constraint matrices efc_J / efc_Y / efc_AR and the Newton factor last) and one of ints, so
// the cooperative lanes of an environment read/write consecutive elements (one 256-byte line per 32
// doubles) and the block stays hot in L1/L2.  Thread mappings over that storage (Env::lane/nlane):
//   cooperative (default): 32 lanes (one warp) per environment, or 16 lanes (two small environments
//       per warp) - MJB_PFOR / MJB_PSYNC / MJB_LANE0 below;
//   lane-per-env (validation): one lane runs the whole pipeline of one environment.
// Every mjData field the hot path touches (reference include/mujoco/mjxmacro.h:842-1030) exists
// per environment.  The per-env arena of the reference (contacts, efc_*) is replaced by fixed caps
// nconmax / njmax; overflow raises the same warning ids (mjWARN_CONTACTFULL / mjWARN_CNSTRFULL).
//
// This header is shared by the CUDA build (nvcc, sm_90a) and the test-only host emulation.
#pragma once
#include <stddef.h>
#include "mjb_math.h"

namespace mjb {

// ---- enum values mirrored from reference include/mujoco/mjtype.h (line numbers cited) ----------
enum { JNT_FREE = 0, JNT_BALL = 1, JNT_SLIDE = 2, JNT_HINGE = 3 };                       // :92-95
enum { GEOM_PLANE = 0, GEOM_HFIELD = 1, GEOM_SPHERE = 2, GEOM_CAPSULE = 3, GEOM_ELLIPSOID = 4,
       GEOM_CYLINDER = 5, GEOM_BOX = 6, GEOM_MESH = 7, GEOM_SDF = 8 };                   // :101-109
enum { CNSTR_EQUALITY = 0, CNSTR_FRICTION_DOF = 1, CNSTR_FRICTION_TENDON = 2, CNSTR_LIMIT_JOINT = 3,
       CNSTR_LIMIT_TENDON = 4, CNSTR_CONTACT_FRICTIONLESS = 5, CNSTR_CONTACT_PYRAMIDAL = 6,
       CNSTR_CONTACT_ELLIPTIC = 7 };                                                    // :532-539
enum { STATE_SATISFIED = 0, STATE_QUADRATIC = 1, STATE_LINEARNEG = 2, STATE_LINEARPOS = 3,
       STATE_CONE = 4 };                                                                // :544-548
enum { WARN_INERTIA = 0, WARN_CONTACTFULL = 1, WARN_CNSTRFULL = 2, WARN_BADQPOS = 3,
       WARN_BADQVEL = 4, WARN_BADQACC = 5, WARN_BADCTRL = 6, WARN_VGEOMFULL = 7, NWARNING = 8 };
enum { NISLAND = 20 };
enum { FEAT_SENSOR = 1, FEAT_EQUALITY = 2, FEAT_ISLAND = 4, FEAT_IMPLICITFAST = 8, FEAT_ACT = 16, FEAT_COLBOX = 32, FEAT_ALL = 63,
       FEAT_CONVEX = 64, FEAT_SPATIAL = 128, FEAT_HISTORY = 256 };   // FEAT_COLBOX: cylinder / box colliders (up to 8 contacts per pair)   // FEAT_ACT: stateful actuators (act), tendon transmissions, muscles
// FEAT_CONVEX: GJK / EPA narrow phase (mjb_convex.h).  Outside FEAT_ALL on purpose: only the convex instantiations
// carry its code and its polytope scratch, every other kernel compiles exactly as without it.
// FEAT_SPATIAL: spatial tendons (site paths, sphere / cylinder wrapping, pulleys) and their tendon-armature bias.
// Outside FEAT_ALL for the same reason: only the spatial instantiations (mjb_kstep_spatial32.cu) carry it.
// FEAT_HISTORY: actuator and sensor history buffers (delayed controls, delayed / sampled sensors, mjb_history.h).
// Outside FEAT_ALL as well: only the history instantiations (mjb_kstep_history32.cu) carry it.
enum { WRAP_NONE = 0, WRAP_JOINT = 1, WRAP_PULLEY = 2, WRAP_SITE = 3, WRAP_SPHERE = 4, WRAP_CYLINDER = 5 };   // mjtWrap (mjtype.h:220-227)
enum { EQ_JOINT = 0, EQ_TENDON = 1, EQ_CONNECT = 2, EQ_WELD = 3 };   // supported equality kinds (body semantics)
constexpr int kNEqData = 11;            // eq_data values per equality (mjNEQDATA): polycoef / anchors, relpose, torquescale
// sensors of the path (engine_sensor.c); internal codes, translated from mjtSensor by the host
enum { SENS_JOINTPOS, SENS_TENDONPOS, SENS_ACTUATORPOS, SENS_BALLQUAT, SENS_JOINTLIMITPOS, SENS_TENDONLIMITPOS,
       SENS_FRAMEPOS, SENS_FRAMEXAXIS, SENS_FRAMEYAXIS, SENS_FRAMEZAXIS, SENS_FRAMEQUAT, SENS_SUBTREECOM, SENS_CLOCK,
       SENS_JOINTVEL, SENS_TENDONVEL, SENS_ACTUATORVEL, SENS_BALLANGVEL, SENS_JOINTLIMITVEL, SENS_TENDONLIMITVEL,
       SENS_FRAMELINVEL, SENS_FRAMEANGVEL, SENS_ACTUATORFRC, SENS_JOINTACTFRC, SENS_JOINTLIMITFRC,
       SENS_TENDONLIMITFRC, SENS_VELOCIMETER, SENS_GYRO, SENS_ACCELEROMETER, SENS_FORCE, SENS_TORQUE,
       SENS_FRAMELINACC, SENS_FRAMEANGACC, SENS_SUBTREELINVEL, SENS_SUBTREEANGMOM, SENS_TOUCH, SENS_E_POTENTIAL, SENS_E_KINETIC, SENS_RANGEFINDER, SENS_CONTACT };
enum { SOBJ_XBODY = 0, SOBJ_BODY = 1, SOBJ_GEOM = 2, SOBJ_SITE = 3 };   // frame sensor object kinds (mjOBJ_*)   // mjNISLAND: islands with solver statistics (mjdata.h)  // :553-561
enum { SOL_PGS = 0, SOL_CG = 1, SOL_NEWTON = 2 };                                        // :202-204
enum { INT_EULER = 0, INT_RK4 = 1, INT_IMPLICIT = 2, INT_IMPLICITFAST = 3 };             // :181-184
enum { SAMEFRAME_NONE = 0, SAMEFRAME_BODY = 1, SAMEFRAME_INERTIA = 2, SAMEFRAME_BODYROT = 3,
       SAMEFRAME_INERTIAROT = 4 };                                                      // :457-461
enum { GAIN_FIXED = 0, GAIN_AFFINE = 1, GAIN_MUSCLE = 2 };                               // :256-258
enum { BIAS_NONE = 0, BIAS_AFFINE = 1, BIAS_MUSCLE = 2 };                                // :267-269
enum { DYN_NONE = 0, DYN_INTEGRATOR = 1, DYN_FILTER = 2, DYN_FILTEREXACT = 3, DYN_MUSCLE = 4 };   // :244-248
enum { TRN_JOINT = 0, TRN_TENDON = 1, TRN_BALL = 2, TRN_FREE = 3, TRN_SITE = 4, TRN_SITEREF = 5, TRN_SLIDERCRANK = 6 };   // >= TRN_SITE: dense moment row built by site_moment (site, site + reference site, slider-crank);   // TRN_SITE: 6D gear at a site (no refsite);   // TRN_BALL / TRN_FREE: 3D / 6D gear on a ball / free joint;   // transmissions built (mjTRN_JOINT / JOINTINPARENT on scalar joints, mjTRN_TENDON)
enum { DSBL_CONSTRAINT = 1 << 0, DSBL_EQUALITY = 1 << 1, DSBL_FRICTIONLOSS = 1 << 2, DSBL_LIMIT = 1 << 3,
       DSBL_CONTACT = 1 << 4, DSBL_SPRING = 1 << 5, DSBL_DAMPER = 1 << 6, DSBL_GRAVITY = 1 << 7,
       DSBL_CLAMPCTRL = 1 << 8, DSBL_WARMSTART = 1 << 9, DSBL_FILTERPARENT = 1 << 10,
       DSBL_ACTUATION = 1 << 11, DSBL_REFSAFE = 1 << 12, DSBL_EULERDAMP = 1 << 15,
       DSBL_AUTORESET = 1 << 16, DSBL_NATIVECCD = 1 << 17, DSBL_ISLAND = 1 << 18, DSBL_SENSOR = 1 << 13,
       DSBL_MULTICCD = 1 << 19 };
enum { ENBL_ENERGY = 1 << 1 };   // mjENBL_ENERGY (mjmodel.h mjtEnableBit)                                // :54-73
enum { LIM_HINGE = 0, LIM_BALL = 1, LIM_TENDON = 2 };   // kinds of limit candidates (host-built table)
constexpr int kNPoly = 2;   // mjNPOLY (include/mujoco/mjmodel.h:44)
constexpr int kNGain = 9;   // leading gain/bias parameters kept (affine: 3, muscle: 9)
constexpr int kNDyn = 3;    // leading dynprm values kept (filter tau; muscle tau_act, tau_deact, smoothing width)

// ---- model sizes and options --------------------------------------------------------------------
struct Sizes {
  int nq, nv, nu, na, nbody, njnt, ngeom, ntendon, nwrap, nJten, nC, ntree;
  int nsensor, nsensordata, nsite, neq, nmocap;
  int actfeat;   // 1 when an actuator is stateful, drives a tendon or is a muscle, or a body has gravcomp (FEAT_ACT code paths)
  int sitetrn;   // 1 when an actuator acts at a site (dense moment rows are allocated then)
  int fluid;     // 1 when the medium has density or viscosity (qfrc_fluid is allocated then)
  int gravcomp;  // 1 when a body has gravity compensation (qfrc_gravcomp is allocated then)
  int epot, ekin;   // 1 when the potential / kinetic energy is computed (mjENBL_ENERGY or an energy sensor)
  int subtreevel;   // 1 when a sensor needs mj_subtreeVel (subtree_linvel / subtree_angmom are allocated then)
  int rnepost;   // 1 when a sensor needs mj_rnePostConstraint (cacc / cfrc_int / cfrc_ext are allocated then)
  int freebody;  // 1 when implicitfast meets a standalone free body (local unsymmetric 6x6 solve, mjb_forward.h free_body_implicit)
  int colbox;    // 1 when a candidate pair needs a cylinder / box collider (FEAT_COLBOX code paths)
  int npair;     // static candidate geom pairs (host-built, reference order)
  int nconmax;   // per-env contact cap
  int njmax;     // per-env constraint-row cap
  int nlevel;    // depth levels of the body tree (level 0 = world)
  int ndlevel;   // depth levels of the dof tree
  int nlim;      // limit candidates (joint sides, ball joints, tendon sides) in row order
  int nfl;       // dofs, then tendons, with frictionloss, in row order (fl_dof: dof index, or -(tendon+1))
  int convex;    // 1 when a candidate pair needs the convex narrow phase (FEAT_CONVEX code paths, mjb_convex.h)
  int nconvex;   // candidate pairs that go through GJK / EPA (entries of the pre-contact store ccd_con)
  int ccdslots;  // polytope slots per environment (ccd_poly), 0 without GJK candidates
  int ccdslot;   // doubles per polytope slot (ccd_slot_doubles(ccd_iterations))
  int spatial;   // 1 when a tendon is spatial (FEAT_SPATIAL code paths; the wrap fields of the batch are allocated then)
  int nhistory;  // doubles of the actuator and sensor history buffers (FEAT_HISTORY code paths when > 0)
  int histflg;   // 1 when nhistory > 0 (the lazy-evaluation flags of the batch are allocated then)
};

struct Options {
  double timestep, impratio, tolerance, ls_tolerance, noslip_tolerance;
  double gravity[3];
  double density, viscosity, wind[3];   // medium (inertia-box fluid model)
  double meaninertia;   // m->stat.meaninertia
  int integrator, cone, solver, iterations, ls_iterations, noslip_iterations, disableflags, enableflags;
  int dense;            // mj_isSparse(m) == 0
  int eulerdamp;        // any dof takes the implicit-damping branch of mj_EulerSkip
  int has_limits;       // any limited joint or tendon
  int has_frictionloss; // any dof/tendon frictionloss
  int ccd_iterations;   // convex narrow phase: GJK / EPA iteration cap, also sizes the EPA polytope
  double ccd_tolerance; // convex narrow phase: GJK / EPA tolerance
};

// model arrays: one int blob and one double blob in device memory; members are pointers into them.
// The last group are host-built schedules that let a warp run the tree recursions level by level
// while reproducing the reference's serial accumulation order (see mjb_model.cc).
#define MJB_MODEL_INT_FIELDS(X)                                                             \
  X(body_parentid) X(body_rootid) X(body_weldid) X(body_jntnum) X(body_jntadr) X(body_dofnum) \
  X(body_dofadr) X(body_geomnum) X(body_geomadr) X(body_sameframe)                          \
  X(jnt_type) X(jnt_qposadr) X(jnt_dofadr) X(jnt_bodyid) X(jnt_limited) X(jnt_actfrclimited) \
  X(dof_bodyid) X(dof_jntid) X(dof_parentid) X(dof_simplenum) X(dof_treeid)                  \
  X(M_rownnz) X(M_rowadr) X(M_colind)                                                       \
  X(geom_type) X(geom_bodyid) X(geom_sameframe) X(body_treeid)                                              \
  X(tendon_adr) X(tendon_num) X(tendon_limited) X(wrap_type) X(wrap_objid)                   \
  X(ten_J_rownnz) X(ten_J_rowadr) X(ten_J_colind)                                            \
  X(actuator_trnjnt) X(actuator_gaintype) X(actuator_biastype) X(actuator_ctrllimited)       \
  X(actuator_forcelimited) X(actuator_trntype) X(actuator_dyntype) X(actuator_actadr)        \
  X(actuator_trnid2) X(actuator_refclear) X(actuator_actlimited) X(actuator_actearly) X(tendon_actfrclimited) X(body_mocapid) X(site_type) X(jnt_actgravcomp) X(actuator_inparent)        \
  X(pair_geom1) X(pair_geom2) X(pair_dim)                                                     \
  X(lvl_adr) X(lvl_body) X(child_adr) X(child_id)                                             \
  X(dlvl_adr) X(dlvl_dof) X(mt_adr) X(mt_dof) X(mt_qadr)                                      \
  X(fac_adr) X(fac_dst) X(fac_src) X(fac_cf)                                                  \
  X(lim_kind) X(lim_id) X(lim_side) X(fl_dof) X(body_dofanc)                                 \
  X(sensor_type) X(sensor_cutmode) X(sensor_objtype) X(sensor_objid) X(sensor_reftype) X(sensor_refid)   \
  X(sensor_dim) X(sensor_adr) X(sensor_intprm0) X(sensor_intprm1) X(sensor_objraw) X(sensor_refraw) X(geom_rayskip) X(site_bodyid) X(site_sameframe)                               \
  X(eq_kind) X(eq_obj1id) X(eq_obj2id) X(eq_active0)                                          \
  X(body_simple) X(tendon_slotadr)                                                            \
  X(actuator_history) X(actuator_historyadr) X(sensor_history) X(sensor_historyadr)

#define MJB_MODEL_DBL_FIELDS(X)                                                             \
  X(qpos0) X(qpos_spring) X(body_pos) X(body_quat) X(body_ipos) X(body_iquat) X(body_mass)   \
  X(body_subtreemass) X(body_inertia) X(body_invweight0)                                    \
  X(jnt_pos) X(jnt_axis) X(jnt_stiffness) X(jnt_stiffnesspoly) X(jnt_range) X(jnt_margin)    \
  X(jnt_solref) X(jnt_solimp) X(jnt_actfrcrange)                                            \
  X(dof_armature_eff) X(dof_damping_eff) X(dof_dampingpoly_eff) X(dof_invweight0) X(dof_M0)  \
  X(dof_frictionloss) X(dof_solref) X(dof_solimp)                                           \
  X(geom_pos) X(geom_quat) X(geom_size) X(geom_rbound)                                       \
  X(wrap_prm) X(tendon_range) X(tendon_margin) X(tendon_solref_lim) X(tendon_solimp_lim)     \
  X(tendon_invweight0) X(tendon_stiffness) X(tendon_stiffnesspoly) X(tendon_damping_eff)     \
  X(tendon_dampingpoly_eff) X(tendon_lengthspring) X(tendon_armature_eff)                    \
  X(actuator_gear0) X(actuator_gainprm) X(actuator_biasprm) X(actuator_ctrlrange)            \
  X(actuator_forcerange) X(actuator_dynprm) X(actuator_actrange) X(actuator_lengthrange) X(actuator_acc0) \
  X(site_size) X(body_gravcomp) X(actuator_gear6) X(actuator_cranklength) X(actuator_wrapperiod) X(tendon_frictionloss) X(tendon_solref_fri) X(tendon_solimp_fri) X(tendon_actfrcrange)      \
  X(pair_margin) X(pair_includemargin) X(pair_solref) X(pair_solimp) X(pair_friction) X(sensor_cutoff) X(site_pos) X(site_quat)            \
  X(eq_data) X(eq_solref) X(eq_solimp) X(tendon_length0)                                      \
  X(actuator_delay) X(sensor_delay) X(sensor_interval)

struct DModel {
  Sizes sz;
  Options opt;
#define X(name) const int* name;
  MJB_MODEL_INT_FIELDS(X)
#undef X
#define X(name) const double* name;
  MJB_MODEL_DBL_FIELDS(X)
#undef X
};

// ---- batch data fields (per environment), sizes in elements -------------------------------------
// HOT doubles: staged in shared memory by the fused warp-per-env kernel
#define MJB_DATA_DBL_FIELDS(X, S)                                                            \
  X(time, 1) X(energy, 2) X(qpos, S.nq) X(qvel, S.nv) X(act, S.na) X(act_dot, S.na) X(mocap_pos, 3 * S.nmocap) X(mocap_quat, 4 * S.nmocap) X(ctrl, S.nu) X(qacc_warmstart, S.nv)  \
  X(qfrc_applied, S.nv) X(xfrc_applied, 6 * S.nbody) X(eq_active, S.neq)                                         \
  X(xpos, 3 * S.nbody) X(xquat, 4 * S.nbody) X(xmat, 9 * S.nbody) X(xipos, 3 * S.nbody)      \
  X(ximat, 9 * S.nbody) X(xanchor, 3 * S.njnt) X(xaxis, 3 * S.njnt)                          \
  X(geom_xpos, 3 * S.ngeom) X(geom_xmat, 9 * S.ngeom) X(subtree_com, 3 * S.nbody)            \
  X(cinert, 10 * S.nbody) X(cdof, 6 * S.nv) X(crb, 10 * S.nbody) X(M, S.nC) X(qLD, S.nC)      \
  X(qLDiagInv, S.nv) X(ten_length, S.ntendon) X(ten_J, S.nJten)                              \
  X(actuator_length, S.nu) X(actuator_moment, S.nu) X(actuator_mom6, 6 * S.nu * S.actfeat) X(actuator_momrow, S.nu * S.nv * S.sitetrn)    \
  X(ten_velocity, S.ntendon) X(actuator_velocity, S.nu) X(cvel, 6 * S.nbody)                 \
  X(cdof_dot, 6 * S.nv) X(qfrc_gravcomp, S.nv * S.gravcomp) X(qfrc_fluid, S.nv * S.fluid) X(qfrc_spring, S.nv) X(qfrc_damper, S.nv) X(qfrc_passive, S.nv)      \
  X(qfrc_bias, S.nv) X(actuator_force, S.nu) X(qfrc_actuator, S.nv) X(qfrc_smooth, S.nv)     \
  X(qacc_smooth, S.nv) X(qfrc_constraint, S.nv) X(qacc, S.nv) X(qH, S.nC)                    \
  X(qHDiagInv, S.nv)                                                                         \
  X(con_dist, S.nconmax) X(con_pos, 3 * S.nconmax) X(con_frame, 9 * S.nconmax)               \
  X(con_includemargin, S.nconmax) X(con_friction, 5 * S.nconmax) X(con_solref, 2 * S.nconmax) \
  X(con_solimp, 5 * S.nconmax) X(con_mu, S.nconmax)                                          \
  X(efc_pos, S.njmax) X(efc_margin, S.njmax)                                                 \
  X(efc_frictionloss, S.njmax) X(efc_diagA, S.njmax) X(efc_KBIP, 4 * S.njmax)                \
  X(efc_D, S.njmax) X(efc_R, S.njmax) X(efc_vel, S.njmax) X(efc_aref, S.njmax)               \
  X(efc_b, S.njmax) X(efc_force, S.njmax)                                                    \
  X(scr_body, 12 * S.nbody) X(scr_nv, 8 * S.nv) X(scr_efc, 6 * S.njmax)                         \
  X(nwt_nv, 6 * S.nv) X(nwt_efc, 6 * S.njmax) X(rk_scr, S.nq + 8 * S.nv + 8 * S.na + 4) X(sensordata, S.nsensordata)  \
  X(site_xpos, 3 * S.nsite) X(site_xmat, 9 * S.nsite)                                        \
  X(subtree_linvel, 3 * S.nbody * S.subtreevel) X(subtree_angmom, 3 * S.nbody * S.subtreevel) X(subtree_bvel, 6 * S.nbody * S.subtreevel) \
  X(cacc, 6 * S.nbody * S.rnepost) X(cfrc_int, 6 * S.nbody * S.rnepost) X(cfrc_ext, 6 * S.nbody * S.rnepost)

// COLD doubles: stay in global memory / L2 in every mapping
#define MJB_DATA_COLD_FIELDS(X, S)                                                           \
  X(efc_J, S.njmax * S.nv) X(efc_Y, S.njmax * S.nv) X(efc_AR, S.njmax * S.njmax)                 \
  X(nwt_L, S.nv * S.nv)

// COLD doubles of the convex narrow phase (empty for models without GJK candidates): polytope slots and the stored
// pre-contacts of the GJK candidates.  Laid out after the other cold fields but declared last in Layout, so that the
// offsets of every other field stay where they are.
#define MJB_DATA_CCD_FIELDS(X, S)                                                            \
  X(ccd_poly, S.ccdslots * S.ccdslot) X(ccd_con, 36 * S.nconvex)

// spatial tendon paths (empty for models without spatial tendons): the path points of mj_tendon, as in mjData.
// Declared last in Layout and laid out after every other field, so that no other offset moves.
#define MJB_DATA_WRAP_FIELDS(X, S) X(wrap_xpos, 6 * S.nwrap * S.spatial)
#define MJB_DATA_WRAP_INT_FIELDS(X, S)                                                        \
  X(ten_wrapadr, S.ntendon * S.spatial) X(ten_wrapnum, S.ntendon * S.spatial) X(wrap_obj, 2 * S.nwrap * S.spatial)

// history buffers (empty for models without them): mjData.history, and the lazy-evaluation flags of
// mj_rnePostConstraint / mj_subtreeVel (mjData.flg_rnepost, flg_subtreevel).  Laid out after every other field.
#define MJB_DATA_HIST_FIELDS(X, S) X(history, S.nhistory)
#define MJB_DATA_HIST_INT_FIELDS(X, S) X(hist_flg, 2 * S.histflg)

// ints (all hot)
#define MJB_DATA_INT_FIELDS(X, S)                                                            \
  X(ncon, 1) X(nefc, 1) X(ne, 1) X(nf, 1) X(nl, 1) X(solver_niter, NISLAND) X(step_skip, 1) X(warning, NWARNING)  \
  X(nisland, 1) X(efc_island, S.njmax) X(map_iefc2efc, S.njmax) X(island_iefcadr, S.ntree + 2) X(tree_island, 2 * S.ntree + 2)            \
  X(island_idofadr, S.ntree + 2) X(map_idof2dof, S.nv) X(map_dof2idof, S.nv)     \
  X(con_geom1, S.nconmax) X(con_geom2, S.nconmax) X(con_dim, S.nconmax)                       \
  X(con_exclude, S.nconmax) X(con_efcadr, S.nconmax) X(con_pair, S.nconmax)                    \
  X(efc_type, S.njmax) X(efc_id, S.njmax) X(efc_state, S.njmax) X(nwt_state, S.njmax) X(scr_int, 4 * S.njmax)        \
  X(scr_ipair, S.npair + 4) X(scr_ilim, 2 * S.nlim + 4) X(scr_ieq, S.neq + 1)

struct Layout {
#define X(name, cnt) long name;
  MJB_DATA_DBL_FIELDS(X, _)
  MJB_DATA_COLD_FIELDS(X, _)
  MJB_DATA_INT_FIELDS(X, _)
#undef X
  long nhot;         // hot doubles per environment (offsets [0, nhot))
  long ndbl, nint;   // total doubles / ints per environment
#define X(name, cnt) long name;
  MJB_DATA_CCD_FIELDS(X, _)
  MJB_DATA_WRAP_FIELDS(X, _)
  MJB_DATA_WRAP_INT_FIELDS(X, _)
  MJB_DATA_HIST_FIELDS(X, _)
  MJB_DATA_HIST_INT_FIELDS(X, _)
#undef X
};

inline Layout make_layout(const Sizes& S) {
  Layout L;
  long o = 0;
#define X(name, cnt) L.name = o; o += (long)(cnt);
  MJB_DATA_DBL_FIELDS(X, S)
  o = (o + 15) / 16 * 16;
  L.nhot = o;
  MJB_DATA_COLD_FIELDS(X, S)
  MJB_DATA_CCD_FIELDS(X, S)
  MJB_DATA_WRAP_FIELDS(X, S)
  MJB_DATA_HIST_FIELDS(X, S)
  L.ndbl = o;
  o = 0;
  MJB_DATA_INT_FIELDS(X, S)
  MJB_DATA_WRAP_INT_FIELDS(X, S)
  MJB_DATA_HIST_INT_FIELDS(X, S)
  L.nint = o;
#undef X
  return L;
}

// view of one field of one environment (unit stride: storage is env-major in every mapping)
template <class T>
struct Fld {
  T* p;
  MJB_HD T& operator[](long i) const { return p[i]; }
  MJB_HD Fld operator+(long k) const { return Fld{p + k}; }
};
using FD = Fld<double>;
using FI = Fld<int>;

// batch storage handle (device or host pointers): env e owns dbl[e*dpitch ...] and itg[e*ipitch ...]
struct Batch {
  double* dbl;
  int* itg;
  size_t stride;   // padded number of environments (native ctrl/state buffers of the rollout)
  size_t dpitch, ipitch;
  int nenv;
  int warp_per_env;   // 0: one environment per lane (validation mapping), 1: cooperative lanes
  int nlane;          // cooperative lanes per environment: 32 (one warp) or 16 (two small environments per warp)
  int xfrc;           // 1 once the caller has written xfrc_applied: the step then runs the full (non-lean) kernels
  Layout L;
};

// per-environment accessor.  hd/hi may point at a shared-memory copy of the hot block.
struct Env {
  const DModel& m;
  const Batch& b;
  int e;
  int lane, nlane;   // cooperative lanes working on this environment (1 lane in lane-per-env mode)
  double* hd;        // hot doubles
  double* cd;        // cold doubles (same offsets, global memory)
  int* hi;           // ints
  double* sm = nullptr;   // per-warp shared-memory scratch (fused kernel only) and its capacity in doubles
  int smcap = 0;
  int solver = -1;   // constraint solver; a compile-time constant in the specialised fused kernels
  unsigned mask = 0xffffffffu;   // lanes of the warp that share this environment (sub-warp mapping)
  // optional parts of the pipeline this environment's model needs (FEAT_*); a compile-time constant in the
  // specialised fused kernels, so a model without sensors / equalities / several trees / implicitfast runs a
  // kernel that does not carry (or pay registers for) that code
  int feat = FEAT_ALL;
  MJB_HD Env(const DModel& m_, const Batch& b_, int e_, int lane_ = 0, int nlane_ = 1)
      : m(m_), b(b_), e(e_), lane(lane_), nlane(nlane_) {
    hd = b.dbl + (size_t)e * b.dpitch;
    cd = hd;
    hi = b.itg + (size_t)e * b.ipitch;
  }
  // hot block (doubles and ints) in a staged copy (shared memory in the fused kernel)
  MJB_HD Env(const DModel& m_, const Batch& b_, int e_, int lane_, int nlane_, double* hot, int* ints)
      : m(m_), b(b_), e(e_), lane(lane_), nlane(nlane_) {
    hd = hot;
    cd = b.dbl + (size_t)e * b.dpitch;
    hi = ints;
  }
#define X(name, cnt) MJB_HD FD name() const { return FD{hd + b.L.name}; }
  MJB_DATA_DBL_FIELDS(X, _)
#undef X
#define X(name, cnt) MJB_HD FD name() const { return FD{cd + b.L.name}; }
  MJB_DATA_COLD_FIELDS(X, _)
  MJB_DATA_CCD_FIELDS(X, _)
  MJB_DATA_WRAP_FIELDS(X, _)
  MJB_DATA_HIST_FIELDS(X, _)
#undef X
#define X(name, cnt) MJB_HD FI name() const { return FI{hi + b.L.name}; }
  MJB_DATA_INT_FIELDS(X, _)
  MJB_DATA_WRAP_INT_FIELDS(X, _)
  MJB_DATA_HIST_INT_FIELDS(X, _)
#undef X
  // barrier + memory ordering between the lanes that share this environment
  MJB_HD void sync() const {
#if defined(__CUDA_ARCH__)
    if (nlane > 1) __syncwarp(mask);
#endif
  }
};

// cooperative loop over n independent items, and the barrier that separates dependent regions
#define MJB_PFOR(i, n) for (int i = d.lane; i < (n); i += d.nlane)
#define MJB_PSYNC() d.sync()
#define MJB_LANE0 if (d.lane == 0)

// small load/store helpers between strided fields and value types
MJB_HD V3 ld3(FD f, long i) { return V3{f[i], f[i + 1], f[i + 2]}; }
MJB_HD void st3(FD f, long i, V3 v) { f[i] = v.x; f[i + 1] = v.y; f[i + 2] = v.z; }
MJB_HD Q4 ld4(FD f, long i) { return Q4{f[i], f[i + 1], f[i + 2], f[i + 3]}; }
MJB_HD void st4(FD f, long i, Q4 q) { f[i] = q.w; f[i + 1] = q.x; f[i + 2] = q.y; f[i + 3] = q.z; }
MJB_HD M3 ld9(FD f, long i) { M3 r; for (int k = 0; k < 9; k++) r.m[k] = f[i + k]; return r; }
MJB_HD void st9(FD f, long i, const M3& a) { for (int k = 0; k < 9; k++) f[i + k] = a.m[k]; }
MJB_HD S6 ld6(FD f, long i) { S6 r; for (int k = 0; k < 6; k++) r.v[k] = f[i + k]; return r; }
MJB_HD void st6(FD f, long i, const S6& a) { for (int k = 0; k < 6; k++) f[i + k] = a.v[k]; }
MJB_HD I10 ld10(FD f, long i) { I10 r; for (int k = 0; k < 10; k++) r.v[k] = f[i + k]; return r; }
MJB_HD void st10(FD f, long i, const I10& a) { for (int k = 0; k < 10; k++) f[i + k] = a.v[k]; }

// dot products in the reference's accumulation order (the summation order is part of parity):
// dense  : engine_util_blas.c:493-523 (mju_dot)   -> (r0+r2)+(r1+r3), tail added as one grouped sum
// sparse : engine_util_sparse.h:197-222 (mju_dotSparse) -> same 4 lanes, tail added one by one
template <class A, class B>
MJB_HD double dot_ref(int n, A a, B b) {
  double r0 = 0, r1 = 0, r2 = 0, r3 = 0;
  int i = 0;
  for (; i <= n - 4; i += 4) {
    r0 += a(i) * b(i);
    r1 += a(i + 1) * b(i + 1);
    r2 += a(i + 2) * b(i + 2);
    r3 += a(i + 3) * b(i + 3);
  }
  double res = (r0 + r2) + (r1 + r3);
  const int t = n - i;
  if (t == 3) res += a(i) * b(i) + a(i + 1) * b(i + 1) + a(i + 2) * b(i + 2);
  else if (t == 2) res += a(i) * b(i) + a(i + 1) * b(i + 1);
  else if (t == 1) res += a(i) * b(i);
  return res;
}
template <class A, class B>
MJB_HD double dot_sparse_ref(int n, A a, B b) {
  double r0 = 0, r1 = 0, r2 = 0, r3 = 0;
  int i = 0;
  for (; i <= n - 4; i += 4) {
    r0 += a(i) * b(i);
    r1 += a(i + 1) * b(i + 1);
    r2 += a(i + 2) * b(i + 2);
    r3 += a(i + 3) * b(i + 3);
  }
  double res = (r0 + r2) + (r1 + r3);
  for (; i < n; i++) res += a(i) * b(i);
  return res;
}

MJB_HD V3 ldc3(const double* p, long i) { return V3{p[i], p[i + 1], p[i + 2]}; }
MJB_HD Q4 ldc4(const double* p, long i) { return Q4{p[i], p[i + 1], p[i + 2], p[i + 3]}; }

}  // namespace mjb
