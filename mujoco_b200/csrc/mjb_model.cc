// Host side of libmjb200: read a reference mjModel (same struct layout, public headers only),
// check that it stays inside the accelerated hot path, and flatten it into the device model
// (mjb_types.h: DModel) — including the static candidate geom-pair table that replaces the
// reference's per-step broadphase/midphase bookkeeping with an order-preserving precomputation.
//
// Reference behaviour restated here (file:line under /root/reference):
//   src/engine/engine_io.c:514-690          MJB binary layout (mj_saveModel / mj_loadModelBuffer)
//   src/engine/engine_collision_driver.c:595-886  body-pair order, filters, per-pair geom order
//   src/engine/engine_collision_driver.c:288-343  filterBodyPair / canCollide2
//   src/engine/engine_collision_driver.c:410-443  contactcompare (midphase sort key)
//   src/engine/engine_collision_driver.c:1740-1835 mj_contactParam (static per geom pair)
//   src/engine/engine_core_util.c:1119-1215  mj_actuatorDamping / mj_actuatorArmature
//   src/engine/engine_forward.c:1409-1421    which dofs trigger implicit Euler damping
#include "mjb_model.h"
#include "mjb_collision.h"   // pair_gjk, kCcdSlots, ccd_slot_doubles (convex candidates and their scratch)

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include <mujoco/mjmodel.h>
#include <mujoco/mujoco.h>   // mjVERSION_HEADER (declarations only: the reference library is never linked)
#include <mujoco/mjxmacro.h>

namespace mjb {

static thread_local std::string g_err;
void set_error(const std::string& s) { g_err = s; }
const char* get_error() { return g_err.c_str(); }

// ------------------------------------------------------------------------------------------------
// MJB loader (header + sizes + option structs + arrays in MJMODEL_POINTERS order)
static const int kMjbId = 54321;

mjModel* load_mjb(const char* path) {
  FILE* f = fopen(path, "rb");
  if (!f) { set_error(std::string("cannot open ") + path); return nullptr; }
  fseek(f, 0, SEEK_END);
  long sz = ftell(f);
  fseek(f, 0, SEEK_SET);
  if (sz < 0 || sz > (1L << 34)) { fclose(f); set_error("cannot size the MJB file (or it is larger than 16 GB)"); return nullptr; }
  std::vector<unsigned char> buf;
  try { buf.resize((size_t)sz); } catch (...) { fclose(f); set_error("out of memory reading the MJB file"); return nullptr; }
  if (fread(buf.data(), 1, sz, f) != (size_t)sz) { fclose(f); set_error("short read"); return nullptr; }
  fclose(f);
  size_t p = 0;
  auto rd = [&](void* dst, size_t n) -> bool {
    if (p + n > (size_t)sz) return false;
    memcpy(dst, buf.data() + p, n);
    p += n;
    return true;
  };
  int header[5];
  if (!rd(header, sizeof(header)) || header[0] != kMjbId || header[1] != (int)sizeof(mjtNum)) {
    set_error("not an MJB file (bad header) or precision mismatch");
    return nullptr;
  }
  int nsize_expected = 0;
#define X(name) nsize_expected++;
  MJMODEL_SIZES
#undef X
  int nptr_expected = 0;
  {
#define X(type, name, nr, nc) nptr_expected++;
    MJMODEL_POINTERS
#undef X
  }
  // the reference compares all five header words (engine_io.c:568-580): id, precision, number of size fields,
  // library version, number of pointers
  if (header[2] != nsize_expected || header[3] != mjVERSION_HEADER || header[4] != nptr_expected) {
    set_error("MJB was written by a different mjModel revision (version / size-field / pointer count differs)");
    return nullptr;
  }
  std::vector<mjtSize> sizes(nsize_expected);
  if (!rd(sizes.data(), sizeof(mjtSize) * nsize_expected)) { set_error("truncated MJB (sizes)"); return nullptr; }
  for (mjtSize v : sizes) if (v < -1 || v > (mjtSize)1 << 40) { set_error("corrupt MJB (negative or absurd size field)"); return nullptr; }   // (nconmax / njmax are -1 by default)
  mjModel* m = (mjModel*)calloc(1, sizeof(mjModel));
  if (!m) { set_error("out of memory (mjModel)"); return nullptr; }
  {
    int k = 0;
#define X(name) m->name = sizes[k++];
    MJMODEL_SIZES
#undef X
  }
  bool ok = rd(&m->opt, sizeof(mjOption)) && rd(&m->vis, sizeof(mjVisual)) && rd(&m->stat, sizeof(mjStatistic)) &&
            rd(&m->flg_gravcomp, sizeof(mjtBool)) && rd(&m->flg_surfacevel, sizeof(mjtBool));
  if (!ok) { free(m); set_error("truncated MJB (structs)"); return nullptr; }
  // one allocation for all arrays, 64-byte aligned each
  size_t total = 0;
  {
    MJMODEL_POINTERS_PREAMBLE(m)
#define X(type, name, nr, nc) total += ((sizeof(type) * (size_t)(m->nr) * (size_t)(nc)) + 63) / 64 * 64;
    MJMODEL_POINTERS
#undef X
  }
  // the arrays of a well-formed file fit in the file: a larger total means corrupt size fields
  if (total > (size_t)sz + 64 * (size_t)nptr_expected) { free(m); set_error("corrupt MJB (array sizes exceed the file)"); return nullptr; }
  unsigned char* store = (unsigned char*)aligned_alloc(64, (total + 64 + 63) / 64 * 64);
  if (!store) { free(m); set_error("out of memory (mjModel arrays)"); return nullptr; }
  memset(store, 0, total + 64);
  m->buffer = store;
  size_t off = 0;
  {
    MJMODEL_POINTERS_PREAMBLE(m)
#define X(type, name, nr, nc)                                                  \
    {                                                                          \
      size_t nb = sizeof(type) * (size_t)(m->nr) * (size_t)(nc);               \
      m->name = (type*)(store + off);                                          \
      if (!rd(m->name, nb)) ok = false;                                        \
      off += (nb + 63) / 64 * 64;                                              \
    }
    MJMODEL_POINTERS
#undef X
  }
  if (!ok || p != (size_t)sz) {
    free(store); free(m);
    set_error("MJB array section does not match this mjModel revision");
    return nullptr;
  }
  return m;
}

void free_mjb(mjModel* m) {
  if (!m) return;
  free(m->buffer);
  free(m);
}

long model_size(const mjModel* m, const char* name) {
#define X(n) if (!strcmp(name, #n)) return (long)m->n;
  MJMODEL_SIZES
#undef X
  return -1;
}

int get_option(const mjModel* m, const char* name, double* v) {
#define X(T, n, sz) if (!strcmp(name, #n)) { *v = (double)m->opt.n; return 0; }
#define XVEC(T, n, sz)
  MJOPTION_FIELDS
#undef X
#undef XVEC
  if (!strcmp(name, "gravity_z")) { *v = m->opt.gravity[2]; return 0; }
  return -1;
}
int set_option(mjModel* m, const char* name, double v) {
#define X(T, n, sz) if (!strcmp(name, #n)) { m->opt.n = (T)v; return 0; }
#define XVEC(T, n, sz)
  MJOPTION_FIELDS
#undef X
#undef XVEC
  if (!strcmp(name, "gravity_z")) { m->opt.gravity[2] = v; return 0; }
  return -1;
}

// ------------------------------------------------------------------------------------------------
static bool is_sparse(const mjModel* m) {
  return m->opt.jacobian == mjJAC_SPARSE || (m->opt.jacobian == mjJAC_AUTO && m->nv >= 60);
}

// actuator-inherited joint/tendon damping (+poly) and armature
static double act_damping(const mjModel* m, bool tendon, int id, double poly[mjNPOLY]) {
  int aid = tendon ? m->tendon_actuatorid[id] : m->jnt_actuatorid[id];
  if (aid == -1) return 0;
  double damping = 0;
  auto add = [&](int k) {
    double g = m->actuator_gear[6 * m->actuator_outadr[k]];
    double g2 = g * g;
    damping += m->actuator_damping[k] * g2;
    for (int j = 0; j < mjNPOLY; j++) poly[j] += m->actuator_dampingpoly[mjNPOLY * k + j] * g2;
  };
  if (aid >= 0) {
    double g = m->actuator_gear[6 * m->actuator_outadr[aid]];
    double g2 = g * g;
    damping = m->actuator_damping[aid] * g2;
    for (int j = 0; j < mjNPOLY; j++) poly[j] += m->actuator_dampingpoly[mjNPOLY * aid + j] * g2;
  } else {
    for (int k = 0; k < m->nactuator; k++) {
      if (m->actuator_trnid[2 * k] != id) continue;
      int tt = m->actuator_trntype[k];
      if (!tendon && tt != mjTRN_JOINT && tt != mjTRN_JOINTINPARENT) continue;
      if (tendon && tt != mjTRN_TENDON) continue;
      add(k);
    }
  }
  return damping;
}
static double act_armature(const mjModel* m, bool tendon, int id) {
  int aid = tendon ? m->tendon_actuatorid[id] : m->jnt_actuatorid[id];
  if (aid == -1) return 0;
  double arm = 0;
  if (aid >= 0) {
    double g = m->actuator_gear[6 * m->actuator_outadr[aid]];
    arm = m->actuator_armature[aid] * (g * g);
  } else {
    for (int k = 0; k < m->nactuator; k++) {
      if (m->actuator_trnid[2 * k] != id) continue;
      int tt = m->actuator_trntype[k];
      if (!tendon && tt != mjTRN_JOINT && tt != mjTRN_JOINTINPARENT) continue;
      if (tendon && tt != mjTRN_TENDON) continue;
      double g = m->actuator_gear[6 * m->actuator_outadr[k]];
      arm += m->actuator_armature[k] * (g * g);
    }
  }
  return arm;
}

// cylinder / box colliders (mjb_collision.h, compiled into the FEAT_COLBOX kernels): up to 8 contacts per pair
static bool collider_boxfamily(int t1, int t2) {  // t1 <= t2
  auto is = [&](int a, int b) { return t1 == a && t2 == b; };
  return is(mjGEOM_PLANE, mjGEOM_CYLINDER) || is(mjGEOM_PLANE, mjGEOM_BOX) || is(mjGEOM_SPHERE, mjGEOM_CYLINDER) ||
         is(mjGEOM_SPHERE, mjGEOM_BOX) || is(mjGEOM_CAPSULE, mjGEOM_BOX) || is(mjGEOM_BOX, mjGEOM_BOX);
}
// convex narrow phase (mjb_convex.h, compiled into the FEAT_CONVEX kernels): plane-ellipsoid (mjc_PlaneConvex) and the
// primitive pairs the reference sends to mjc_Convex (GJK / EPA, up to five contacts per pair with multiCCD)
static bool collider_convex(int t1, int t2) {  // t1 <= t2
  return (t1 == mjGEOM_PLANE && t2 == mjGEOM_ELLIPSOID) || pair_gjk(t1, t2);
}
static bool collider_supported(int t1, int t2) {  // t1 <= t2
  auto is = [&](int a, int b) { return t1 == a && t2 == b; };
  return is(mjGEOM_PLANE, mjGEOM_SPHERE) || is(mjGEOM_PLANE, mjGEOM_CAPSULE) ||
         is(mjGEOM_SPHERE, mjGEOM_SPHERE) || is(mjGEOM_SPHERE, mjGEOM_CAPSULE) ||
         is(mjGEOM_CAPSULE, mjGEOM_CAPSULE) || collider_boxfamily(t1, t2) || collider_convex(t1, t2);
}
static bool collider_defined(int t1, int t2) {  // mjCOLLISIONFUNC != NULL, t1 <= t2
  if (t1 == mjGEOM_PLANE) return t2 != mjGEOM_PLANE && t2 != mjGEOM_HFIELD;
  return true;
}

struct Cand { int g1, g2; };

// static per-pair contact parameters (mj_contactParam with no <pair> overrides)
static void contact_param(const mjModel* m, int g1, int g2, int* condim, double* solref, double* solimp,
                          double* friction) {
  double fri[3];
  int p1 = m->geom_priority[g1], p2 = m->geom_priority[g2];
  if (p1 != p2) {
    int g = p1 > p2 ? g1 : g2;
    *condim = m->geom_condim[g];
    memcpy(solref, m->geom_solref + g * mjNREF, mjNREF * sizeof(double));
    memcpy(solimp, m->geom_solimp + g * mjNIMP, mjNIMP * sizeof(double));
    memcpy(fri, m->geom_friction + 3 * g, 3 * sizeof(double));
  } else {
    *condim = std::max(m->geom_condim[g1], m->geom_condim[g2]);
    double s1 = m->geom_solmix[g1], s2 = m->geom_solmix[g2], mix;
    if (s1 >= mjMINVAL && s2 >= mjMINVAL) mix = s1 / (s1 + s2);
    else if (s1 < mjMINVAL && s2 < mjMINVAL) mix = 0.5;
    else if (s1 < mjMINVAL) mix = 0.0;
    else mix = 1.0;
    const double* r1 = m->geom_solref + g1 * mjNREF;
    const double* r2 = m->geom_solref + g2 * mjNREF;
    if (r1[0] > 0 && r2[0] > 0) {
      for (int i = 0; i < mjNREF; i++) solref[i] = mix * r1[i] + (1 - mix) * r2[i];
    } else {
      for (int i = 0; i < mjNREF; i++) solref[i] = std::min(r1[i], r2[i]);
    }
    for (int i = 0; i < mjNIMP; i++)
      solimp[i] = mix * m->geom_solimp[g1 * mjNIMP + i] + (1 - mix) * m->geom_solimp[g2 * mjNIMP + i];
    for (int i = 0; i < 3; i++) fri[i] = std::max(m->geom_friction[3 * g1 + i], m->geom_friction[3 * g2 + i]);
  }
  friction[0] = fri[0]; friction[1] = fri[0]; friction[2] = fri[1]; friction[3] = fri[2]; friction[4] = fri[2];
  for (int i = 0; i < 5; i++) friction[i] = std::max((double)mjMINMU, friction[i]);  // mj_assignFriction
}

// sensors of the path: mjtSensor -> internal code, object kinds for the frame sensors; false = unsupported
static bool sensor_code(const mjModel* m, int i, int* code, int* okind, int* rkind) {
  auto kind = [](int objtype, int* k) {
    if (objtype == mjOBJ_XBODY) { *k = SOBJ_XBODY; return true; }
    if (objtype == mjOBJ_BODY) { *k = SOBJ_BODY; return true; }
    if (objtype == mjOBJ_GEOM) { *k = SOBJ_GEOM; return true; }
    if (objtype == mjOBJ_SITE) { *k = SOBJ_SITE; return true; }
    return false;
  };
  *okind = 0; *rkind = 0;
  bool frame = false;
  switch (m->sensor_type[i]) {
    case mjSENS_JOINTPOS: *code = SENS_JOINTPOS; break;
    case mjSENS_TENDONPOS: *code = SENS_TENDONPOS; break;
    case mjSENS_ACTUATORPOS: *code = SENS_ACTUATORPOS; break;
    case mjSENS_BALLQUAT: *code = SENS_BALLQUAT; break;
    case mjSENS_JOINTLIMITPOS: *code = SENS_JOINTLIMITPOS; break;
    case mjSENS_TENDONLIMITPOS: *code = SENS_TENDONLIMITPOS; break;
    case mjSENS_FRAMEPOS: *code = SENS_FRAMEPOS; frame = true; break;
    case mjSENS_FRAMEXAXIS: *code = SENS_FRAMEXAXIS; frame = true; break;
    case mjSENS_FRAMEYAXIS: *code = SENS_FRAMEYAXIS; frame = true; break;
    case mjSENS_FRAMEZAXIS: *code = SENS_FRAMEZAXIS; frame = true; break;
    case mjSENS_FRAMEQUAT: *code = SENS_FRAMEQUAT; frame = true; break;
    case mjSENS_SUBTREECOM: *code = SENS_SUBTREECOM; break;
    case mjSENS_CLOCK: *code = SENS_CLOCK; break;
    case mjSENS_E_POTENTIAL: *code = SENS_E_POTENTIAL; break;
    case mjSENS_E_KINETIC: *code = SENS_E_KINETIC; break;
    case mjSENS_JOINTVEL: *code = SENS_JOINTVEL; break;
    case mjSENS_TENDONVEL: *code = SENS_TENDONVEL; break;
    case mjSENS_ACTUATORVEL: *code = SENS_ACTUATORVEL; break;
    case mjSENS_BALLANGVEL: *code = SENS_BALLANGVEL; break;
    case mjSENS_JOINTLIMITVEL: *code = SENS_JOINTLIMITVEL; break;
    case mjSENS_TENDONLIMITVEL: *code = SENS_TENDONLIMITVEL; break;
    case mjSENS_FRAMELINVEL: *code = SENS_FRAMELINVEL; frame = true; break;
    case mjSENS_FRAMEANGVEL: *code = SENS_FRAMEANGVEL; frame = true; break;
    case mjSENS_ACTUATORFRC: *code = SENS_ACTUATORFRC; break;
    case mjSENS_JOINTACTFRC: *code = SENS_JOINTACTFRC; break;
    case mjSENS_JOINTLIMITFRC: *code = SENS_JOINTLIMITFRC; break;
    case mjSENS_TENDONLIMITFRC: *code = SENS_TENDONLIMITFRC; break;
    case mjSENS_VELOCIMETER: *code = SENS_VELOCIMETER; *okind = SOBJ_SITE; return m->sensor_objtype[i] == mjOBJ_SITE;
    case mjSENS_GYRO: *code = SENS_GYRO; *okind = SOBJ_SITE; return m->sensor_objtype[i] == mjOBJ_SITE;
    case mjSENS_ACCELEROMETER: *code = SENS_ACCELEROMETER; *okind = SOBJ_SITE; return m->sensor_objtype[i] == mjOBJ_SITE;
    case mjSENS_FORCE: *code = SENS_FORCE; *okind = SOBJ_SITE; return m->sensor_objtype[i] == mjOBJ_SITE;
    case mjSENS_TORQUE: *code = SENS_TORQUE; *okind = SOBJ_SITE; return m->sensor_objtype[i] == mjOBJ_SITE;
    case mjSENS_FRAMELINACC: *code = SENS_FRAMELINACC; frame = true; break;
    case mjSENS_FRAMEANGACC: *code = SENS_FRAMEANGACC; frame = true; break;
    case mjSENS_SUBTREELINVEL: *code = SENS_SUBTREELINVEL; break;
    case mjSENS_TOUCH: {   // contact normal forces inside a site volume (sphere, capsule, ellipsoid, cylinder, box zones)
      *code = SENS_TOUCH; *okind = SOBJ_SITE;
      if (m->sensor_objtype[i] != mjOBJ_SITE) return false;
      const int st = m->site_type[m->sensor_objid[i]];
      return st == mjGEOM_SPHERE || st == mjGEOM_CAPSULE || st == mjGEOM_ELLIPSOID || st == mjGEOM_CYLINDER || st == mjGEOM_BOX;
    }
    case mjSENS_SUBTREEANGMOM: *code = SENS_SUBTREEANGMOM; break;
    case mjSENS_CONTACT: {   // contacts selected by object / reference criteria (site volume, geom, body, subtree), reduced
      *code = SENS_CONTACT;
      auto okc = [&](int t, int id) {
        if (t == mjOBJ_UNKNOWN || t == mjOBJ_GEOM || t == mjOBJ_BODY || t == mjOBJ_XBODY) return true;
        if (t == mjOBJ_SITE) { const int st = m->site_type[id]; return st == mjGEOM_SPHERE || st == mjGEOM_CAPSULE || st == mjGEOM_ELLIPSOID || st == mjGEOM_CYLINDER || st == mjGEOM_BOX; }
        return false;
      };
      return okc(m->sensor_objtype[i], m->sensor_objid[i]) && okc(m->sensor_reftype[i], m->sensor_refid[i]) && m->sensor_reftype[i] != mjOBJ_SITE;
    }
    case mjSENS_RANGEFINDER: {   // site-attached ray along the site's z axis; every field of the data spec but the normal
      *code = SENS_RANGEFINDER; *okind = SOBJ_SITE;
      if (m->sensor_objtype[i] != mjOBJ_SITE) return false;            // (camera depth images are not built)
      if (m->sensor_intprm[i * mjNSENS] & (1 << mjRAYDATA_NORMAL)) return false;
      for (int g = 0; g < m->ngeom; g++) {   // every geom a ray can meet needs a closed-form ray test
        const bool invisible = (m->geom_matid[g] < 0 && m->geom_rgba[4 * g + 3] == 0) ||
                               (m->geom_matid[g] >= 0 && m->mat_rgba[4 * m->geom_matid[g] + 3] == 0);
        const int t = m->geom_type[g];
        if (!invisible && (t == mjGEOM_MESH || t == mjGEOM_HFIELD || t == mjGEOM_SDF)) return false;
      }
      return true;
    }
    default: return false;
  }
  if (frame) {
    if (!kind(m->sensor_objtype[i], okind)) return false;
    if (m->sensor_refid[i] >= 0 && !kind(m->sensor_reftype[i], rkind)) return false;
  }
  return true;
}

// ------------------------------------------------------------------------------------------------
int check_model(const mjModel* m) {
  char msg[256];
#define FAIL(...) do { snprintf(msg, sizeof(msg), __VA_ARGS__); set_error(std::string("unsupported: ") + msg); return -2; } while (0)
  if (m->nv <= 0 || m->nbody < 2) FAIL("model without degrees of freedom");
  if (m->nflex || m->nhfield || m->nplugin) FAIL("flex / hfield / plugin present");
  for (int i = 0; i < m->neq; i++) {
    if (m->eq_type[i] != mjEQ_JOINT && m->eq_type[i] != mjEQ_TENDON && m->eq_type[i] != mjEQ_CONNECT && m->eq_type[i] != mjEQ_WELD)
      FAIL("equality %d: joint, tendon, connect and weld equalities are built; flex equalities are not", i);
    if ((m->eq_type[i] == mjEQ_CONNECT || m->eq_type[i] == mjEQ_WELD) && m->eq_objtype[i] != mjOBJ_BODY) FAIL("equality %d: connect / weld with site semantics", i);
    if (m->eq_type[i] == mjEQ_JOINT) {
      for (int k = 0; k < 2; k++) {
        const int j = k ? m->eq_obj2id[i] : m->eq_obj1id[i];
        if (j >= 0 && m->jnt_type[j] != mjJNT_HINGE && m->jnt_type[j] != mjJNT_SLIDE) FAIL("equality %d couples a non-scalar joint", i);
      }
    }
  }
  if (m->opt.disableflags & mjDSBL_SENSOR) { /* sensordata simply stays untouched */ }
  for (int i = 0; i < m->nsensor; i++) {
    int code, okind, rkind;
    if (!sensor_code(m, i, &code, &okind, &rkind))
      FAIL("sensor %d: type %d / object type %d is outside the supported set", i, (int)m->sensor_type[i], (int)m->sensor_objtype[i]);
  }
  for (int i = 0; i < m->npair; i++) {
    // solreffriction only shapes the friction rows of ELLIPTIC cones (mj_makeImpedance); pyramidal rows take solref
    if ((m->pair_solreffriction[mjNREF * i] || m->pair_solreffriction[mjNREF * i + 1]) && m->opt.cone != mjCONE_PYRAMIDAL) FAIL("contact pair %d: solreffriction", i);
    if (m->pair_adhesion[i] != 0) FAIL("contact pair %d: adhesion", i);
  }
  // mj_resetData places the history samples on the timestep grid and refuses a non-positive timestep (engine_io.c)
  if (m->nhistory && !(m->opt.timestep > 0)) FAIL("history buffers with a timestep <= 0");
  if (m->flg_surfacevel) FAIL("geom surface velocity");
  if (m->opt.cone != mjCONE_PYRAMIDAL) FAIL("elliptic friction cones");
  if (m->opt.integrator == mjINT_IMPLICIT) FAIL("the fully implicit integrator (RNE velocity derivatives, sparse LU)");
  if (m->opt.integrator == mjINT_IMPLICITFAST) {
    if (m->ntendon > m->nv) FAIL("implicitfast with more tendons than dofs");
    // standalone free bodies take a separate unsymmetric 6x6 solve (mjd_freeMhat -> free_body_implicit); its matrix is
    // assembled from the lower triangle of qH, which is the whole story only while the body's qDeriv block is
    // diagonal (damping): actuators acting on such a body are refused
    for (int j = 0; j < m->njnt; j++) {
      const int b = m->jnt_bodyid[j];
      if (!(m->jnt_type[j] == mjJNT_FREE && m->body_jntnum[b] == 1 && m->tree_dofnum[m->dof_treeid[m->jnt_dofadr[j]]] == 6 &&
            m->body_subtreemass[b] == m->body_mass[b])) continue;
      for (int u = 0; u < m->nu; u++) {
        const int tt = m->actuator_trntype[u], id0 = m->actuator_trnid[2 * u], id1 = m->actuator_trnid[2 * u + 1];
        bool hit = false;
        if ((tt == mjTRN_JOINT || tt == mjTRN_JOINTINPARENT) && id0 == j) hit = true;
        if ((tt == mjTRN_SITE || tt == mjTRN_SLIDERCRANK) && (m->site_bodyid[id0] == b || (id1 >= 0 && m->site_bodyid[id1] == b))) hit = true;
        if (hit) FAIL("implicitfast: actuator %d acts on the standalone free body %d", u, b);
      }
    }
  }
  if (m->opt.noslip_iterations > 0 && m->opt.cone != mjCONE_PYRAMIDAL) FAIL("noslip solver with elliptic cones");
  if (m->opt.enableflags & (mjENBL_SLEEP | mjENBL_DIAGEXACT))
    FAIL("enable flags sleep/diagexact");
  if (m->opt.density != 0 || m->opt.viscosity != 0) {   // inertia-box fluid model only
    for (int i = 0; i < m->ngeom; i++) if (m->geom_fluid[mjNFLUID * i] > 0) FAIL("geom %d: ellipsoid fluid model", i);
    if (m->opt.integrator == mjINT_IMPLICITFAST) FAIL("fluid forces with implicitfast (velocity derivatives of the fluid forces)");
  }
  if (m->opt.disableflags & mjDSBL_ISLAND) { /* monolithic solve: fine for single-tree models */ }
  for (int i = 0; i < m->ngeom; i++) {
    if (m->geom_adhesion[i] != 0) FAIL("geom adhesion");
  }
  if (m->nout != m->nu || m->nactuator != m->nu) FAIL("multi-input/multi-output actuators");
  for (int i = 0; i < m->nactuator; i++) {
    int tt = m->actuator_trntype[i];
    if (tt != mjTRN_JOINT && tt != mjTRN_JOINTINPARENT && tt != mjTRN_TENDON && tt != mjTRN_SITE && tt != mjTRN_SLIDERCRANK) FAIL("actuator %d: body (adhesion) transmission", i);
    if ((tt == mjTRN_SITE || tt == mjTRN_SLIDERCRANK) && (m->actuator_damping[i] != 0 || m->actuator_armature[i] != 0)) FAIL("actuator %d: actuator damping / armature on a site / slider-crank transmission", i);
    // fwd_velocity gathers the nonzero moments of such an actuator into a list of 64 (mjb_forward.h)
    if ((tt == mjTRN_SITE || tt == mjTRN_SLIDERCRANK) && m->nv > 64) FAIL("actuator %d: site / slider-crank transmission on a model with nv > 64", i);
    if (tt != mjTRN_TENDON && tt != mjTRN_SITE && tt != mjTRN_SLIDERCRANK) {
      int jt = m->jnt_type[m->actuator_trnid[2 * i]];
      if ((jt == mjJNT_BALL || jt == mjJNT_FREE) && (m->actuator_damping[i] != 0 || m->actuator_armature[i] != 0))
        FAIL("actuator %d: actuator damping / armature on a ball or free joint", i);
    }
    int dt = m->actuator_dyntype[i], gt = m->actuator_gaintype[i], bt = m->actuator_biastype[i];
    if (dt != mjDYN_NONE && dt != mjDYN_INTEGRATOR && dt != mjDYN_FILTER && dt != mjDYN_FILTEREXACT && dt != mjDYN_MUSCLE)
      FAIL("actuator %d: dynamics type (none, integrator, filter, filterexact and muscle are built)", i);
    if (m->actuator_actnum[i] != (dt == mjDYN_NONE ? 0 : 1)) FAIL("actuator %d: activation block of %d states", i, (int)m->actuator_actnum[i]);
    if (gt != mjGAIN_FIXED && gt != mjGAIN_AFFINE && gt != mjGAIN_MUSCLE) FAIL("actuator %d: gain type", i);
    if (bt != mjBIAS_NONE && bt != mjBIAS_AFFINE && bt != mjBIAS_MUSCLE) FAIL("actuator %d: bias type", i);
    if (gt == mjGAIN_MUSCLE && m->opt.integrator == mjINT_IMPLICITFAST) FAIL("actuator %d: muscle gain with implicitfast (velocity derivative of the FLV curve)", i);
    if (m->actuator_ctrlnum[i] != 1 || m->actuator_outnum[i] != 1 || m->actuator_ctrladr[i] != i || m->actuator_outadr[i] != i)
      FAIL("actuator %d: non-scalar control block", i);
    if (m->actuator_plugin[i] >= 0) FAIL("actuator %d: plugin", i);
    if (m->opt.disableactuator & (1 << m->actuator_group[i])) FAIL("disabled actuator groups");
  }
  for (int i = 0; i < m->ngeom; i++) {
    int t = m->geom_type[i];
    if (t == mjGEOM_HFIELD || t == mjGEOM_SDF) FAIL("geom %d: hfield/sdf", i);
    if (m->geom_contype[i] == 0 && m->geom_conaffinity[i] == 0) continue;
    if (t == mjGEOM_MESH) FAIL("geom %d: mesh colliders are a 'next' row", i);
  }
#undef FAIL
  return 0;
}

// ------------------------------------------------------------------------------------------------
struct Builder {
  std::vector<int>& ib;
  std::vector<double>& db;
  std::vector<std::pair<const int**, size_t>> ifix;
  std::vector<std::pair<const double**, size_t>> dfix;
  template <class T>
  void addI(const int** slot, const T* src, size_t n) {
    size_t o = ib.size();
    for (size_t i = 0; i < n; i++) ib.push_back((int)src[i]);
    if (n == 0) ib.push_back(0);
    ifix.push_back({slot, o});
  }
  void addD(const double** slot, const double* src, size_t n) {
    size_t o = db.size();
    for (size_t i = 0; i < n; i++) db.push_back(src[i]);
    if (n == 0) db.push_back(0);
    dfix.push_back({slot, o});
  }
  void fix() {
    for (auto& f : ifix) *f.first = ib.data() + f.second;
    for (auto& f : dfix) *f.first = db.data() + f.second;
  }
};

int build_host_model(const mjModel* m, int nconmax, int njmax, HostModel* out) {
  if (int rc = check_model(m)) return rc;
  DModel& D = out->dm;
  memset(&D, 0, sizeof(D));
  Sizes& S = D.sz;
  S.actfeat = 0;
  for (int i = 0; i < m->nu; i++)
    if (m->actuator_dyntype[i] != mjDYN_NONE || m->actuator_trntype[i] == mjTRN_TENDON || m->actuator_trntype[i] == mjTRN_SITE || m->actuator_trntype[i] == mjTRN_SLIDERCRANK ||
        ((m->actuator_trntype[i] == mjTRN_JOINT || m->actuator_trntype[i] == mjTRN_JOINTINPARENT) &&
         (m->jnt_type[m->actuator_trnid[2 * i]] == mjJNT_BALL || m->jnt_type[m->actuator_trnid[2 * i]] == mjJNT_FREE)) || m->actuator_gaintype[i] == mjGAIN_MUSCLE ||
        m->actuator_biastype[i] == mjBIAS_MUSCLE) S.actfeat = 1;
  S.nmocap = m->nmocap;
  S.fluid = (m->opt.density != 0 || m->opt.viscosity != 0) ? 1 : 0;
  if (S.fluid) S.actfeat = 1;
  S.sitetrn = 0;
  for (int i = 0; i < m->nu; i++) if (m->actuator_trntype[i] == mjTRN_SITE || m->actuator_trntype[i] == mjTRN_SLIDERCRANK) S.sitetrn = 1;
  S.gravcomp = m->flg_gravcomp ? 1 : 0;
  S.colbox = 0;   // set while the candidate pairs are built
  S.convex = 0;
  S.nconvex = 0;
  S.freebody = 0;
  if (m->opt.integrator == mjINT_IMPLICITFAST)
    for (int j = 0; j < m->njnt; j++) {
      const int b = m->jnt_bodyid[j];
      if (m->jnt_type[j] == mjJNT_FREE && m->body_jntnum[b] == 1 && m->body_subtreemass[b] == m->body_mass[b]) S.freebody = 1;
    }
  if (S.gravcomp) S.actfeat = 1;
  S.nq = m->nq; S.nv = m->nv; S.nu = m->nu; S.na = m->na; S.nbody = m->nbody; S.njnt = m->njnt;
  S.ngeom = m->ngeom; S.ntendon = m->ntendon; S.nwrap = m->nwrap; S.nJten = m->nJten; S.nC = m->nC;
  S.ntree = m->ntree;
  S.nsensor = m->nsensor; S.nsensordata = m->nsensordata; S.nsite = m->nsite; S.neq = m->neq;
  S.rnepost = 0;
  S.subtreevel = 0;
  S.epot = S.ekin = (m->opt.enableflags & mjENBL_ENERGY) ? 1 : 0;
  for (int i = 0; i < m->nsensor; i++) {
    if (m->sensor_type[i] == mjSENS_E_POTENTIAL) S.epot = 1;
    if (m->sensor_type[i] == mjSENS_E_KINETIC) S.ekin = 1;
  }
  for (int i = 0; i < m->nsensor; i++)
    if (m->sensor_type[i] == mjSENS_SUBTREELINVEL || m->sensor_type[i] == mjSENS_SUBTREEANGMOM) S.subtreevel = 1;
  for (int i = 0; i < m->nsensor; i++) {
    const int t = m->sensor_type[i];
    if (t == mjSENS_ACCELEROMETER || t == mjSENS_FORCE || t == mjSENS_TORQUE || t == mjSENS_FRAMELINACC || t == mjSENS_FRAMEANGACC) S.rnepost = 1;
  }

  Options& O = D.opt;
  O.timestep = m->opt.timestep; O.impratio = m->opt.impratio; O.tolerance = m->opt.tolerance;
  O.ls_tolerance = m->opt.ls_tolerance;
  for (int i = 0; i < 3; i++) O.gravity[i] = m->opt.gravity[i];
  O.density = m->opt.density; O.viscosity = m->opt.viscosity;
  for (int i = 0; i < 3; i++) O.wind[i] = m->opt.wind[i];
  O.meaninertia = m->stat.meaninertia;
  O.ccd_iterations = m->opt.ccd_iterations; O.ccd_tolerance = m->opt.ccd_tolerance;
  O.integrator = m->opt.integrator; O.cone = m->opt.cone; O.solver = m->opt.solver;
  O.iterations = m->opt.iterations; O.ls_iterations = m->opt.ls_iterations;
  O.noslip_iterations = m->opt.noslip_iterations; O.noslip_tolerance = m->opt.noslip_tolerance;
  O.disableflags = m->opt.disableflags; O.enableflags = m->opt.enableflags;
  O.dense = is_sparse(m) ? 0 : 1;

  Builder B{out->ib, out->db, {}, {}};
  out->ib.clear(); out->db.clear();
  out->ib.reserve(1 << 16); out->db.reserve(1 << 16);

  B.addI(&D.body_parentid, m->body_parentid, m->nbody);
  B.addI(&D.body_rootid, m->body_rootid, m->nbody);
  B.addI(&D.body_weldid, m->body_weldid, m->nbody);
  B.addI(&D.body_jntnum, m->body_jntnum, m->nbody);
  B.addI(&D.body_jntadr, m->body_jntadr, m->nbody);
  B.addI(&D.body_dofnum, m->body_dofnum, m->nbody);
  B.addI(&D.body_dofadr, m->body_dofadr, m->nbody);
  B.addI(&D.body_geomnum, m->body_geomnum, m->nbody);
  B.addI(&D.body_geomadr, m->body_geomadr, m->nbody);
  B.addI(&D.body_sameframe, m->body_sameframe, m->nbody);
  B.addI(&D.jnt_type, m->jnt_type, m->njnt);
  B.addI(&D.jnt_qposadr, m->jnt_qposadr, m->njnt);
  B.addI(&D.jnt_dofadr, m->jnt_dofadr, m->njnt);
  B.addI(&D.jnt_bodyid, m->jnt_bodyid, m->njnt);
  B.addI(&D.jnt_limited, m->jnt_limited, m->njnt);
  B.addI(&D.jnt_actfrclimited, m->jnt_actfrclimited, m->njnt);
  B.addI(&D.dof_bodyid, m->dof_bodyid, m->nv);
  B.addI(&D.dof_jntid, m->dof_jntid, m->nv);
  B.addI(&D.dof_parentid, m->dof_parentid, m->nv);
  B.addI(&D.dof_simplenum, m->dof_simplenum, m->nv);
  B.addI(&D.dof_treeid, m->dof_treeid, m->nv);
  B.addI(&D.body_treeid, m->body_treeid, m->nbody);
  {   // sensors: internal type codes, cutoff mode (0 none, 1 real: both sides, 2 positive: upper side)
    std::vector<int> st(m->nsensor), cm(m->nsensor), ok(m->nsensor), rk(m->nsensor), rid(m->nsensor);
    for (int i = 0; i < m->nsensor; i++) {
      sensor_code(m, i, &st[i], &ok[i], &rk[i]);
      rid[i] = m->sensor_refid[i];
      cm[i] = 0;
      if (m->sensor_cutoff[i] > 0) {
        if (m->sensor_datatype[i] == mjDATATYPE_REAL) cm[i] = 1;
        else if (m->sensor_datatype[i] == mjDATATYPE_POSITIVE) cm[i] = 2;
      }
    }
    B.addI(&D.sensor_type, st.data(), m->nsensor);
    B.addI(&D.sensor_cutmode, cm.data(), m->nsensor);
    B.addI(&D.sensor_objtype, ok.data(), m->nsensor);
    B.addI(&D.sensor_objid, m->sensor_objid, m->nsensor);
    B.addI(&D.sensor_reftype, rk.data(), m->nsensor);
    B.addI(&D.sensor_refid, rid.data(), m->nsensor);
    B.addI(&D.sensor_dim, m->sensor_dim, m->nsensor);
    {
      std::vector<int> ip(m->nsensor), ip1(m->nsensor), skip(m->ngeom), oraw(m->nsensor), rraw(m->nsensor);
      for (int i = 0; i < m->nsensor; i++) {
        ip[i] = m->sensor_intprm[i * mjNSENS]; ip1[i] = m->sensor_intprm[i * mjNSENS + 1];
        // contact sensors match on the reference's own object kinds: 0 none, 1 site, 2 geom, 3 body, 4 xbody (subtree)
        auto raw = [](int t) { return t == mjOBJ_SITE ? 1 : t == mjOBJ_GEOM ? 2 : t == mjOBJ_BODY ? 3 : t == mjOBJ_XBODY ? 4 : 0; };
        oraw[i] = raw(m->sensor_objtype[i]); rraw[i] = raw(m->sensor_reftype[i]);
      }
      B.addI(&D.sensor_intprm1, ip1.data(), m->nsensor);
      B.addI(&D.sensor_objraw, oraw.data(), m->nsensor);
      B.addI(&D.sensor_refraw, rraw.data(), m->nsensor);
      for (int g = 0; g < m->ngeom; g++)   // ray_eliminate (engine_ray.c:68-99) with flg_static = 1 and no geom groups
        skip[g] = ((m->geom_matid[g] < 0 && m->geom_rgba[4 * g + 3] == 0) || (m->geom_matid[g] >= 0 && m->mat_rgba[4 * m->geom_matid[g] + 3] == 0)) ? 1 : 0;
      B.addI(&D.sensor_intprm0, ip.data(), m->nsensor);
      B.addI(&D.geom_rayskip, skip.data(), m->ngeom);
    }
    B.addI(&D.sensor_adr, m->sensor_adr, m->nsensor);
    {
      std::vector<int> kind(m->neq), act(m->neq);
      for (int i = 0; i < m->neq; i++) { kind[i] = (m->eq_type[i] == mjEQ_JOINT) ? EQ_JOINT : (m->eq_type[i] == mjEQ_TENDON) ? EQ_TENDON : (m->eq_type[i] == mjEQ_CONNECT) ? EQ_CONNECT : EQ_WELD; act[i] = m->eq_active0[i] ? 1 : 0; }
      B.addI(&D.eq_kind, kind.data(), m->neq);
      B.addI(&D.eq_obj1id, m->eq_obj1id, m->neq);
      B.addI(&D.eq_obj2id, m->eq_obj2id, m->neq);
      B.addI(&D.eq_active0, act.data(), m->neq);
    }
    B.addI(&D.site_bodyid, m->site_bodyid, m->nsite);
    B.addI(&D.site_sameframe, m->site_sameframe, m->nsite);
  }
  B.addI(&D.M_rownnz, m->M_rownnz, m->nv);
  B.addI(&D.M_rowadr, m->M_rowadr, m->nv);
  B.addI(&D.M_colind, m->M_colind, m->nC);
  B.addI(&D.geom_type, m->geom_type, m->ngeom);
  B.addI(&D.geom_bodyid, m->geom_bodyid, m->ngeom);
  B.addI(&D.geom_sameframe, m->geom_sameframe, m->ngeom);
  B.addI(&D.tendon_adr, m->tendon_adr, m->ntendon);
  B.addI(&D.tendon_num, m->tendon_num, m->ntendon);
  B.addI(&D.tendon_limited, m->tendon_limited, m->ntendon);
  B.addI(&D.wrap_type, m->wrap_type, m->nwrap);
  B.addI(&D.wrap_objid, m->wrap_objid, m->nwrap);
  B.addI(&D.ten_J_rownnz, m->ten_J_rownnz, m->ntendon);
  B.addI(&D.ten_J_rowadr, m->ten_J_rowadr, m->ntendon);
  B.addI(&D.ten_J_colind, m->ten_J_colind, m->nJten);
  {   // spatial tendons (mj_tendon, engine_core_smooth.c:985-1109): each tendon's path points are first written to a
      // slot of its own in wrap_xpos / wrap_obj, then packed to the running count ten_wrapadr.  A site or a pulley
      // gives at most one point and a wrapping geom at most two, so the slots fit the 2*nwrap points of mjData.
    S.spatial = 0;
    std::vector<int> slot(m->ntendon);
    int adr = 0;
    for (int i = 0; i < m->ntendon; i++) {
      slot[i] = adr;
      const int a = m->tendon_adr[i], n = m->tendon_num[i];
      if (m->wrap_type[a] == mjWRAP_JOINT) continue;
      S.spatial = 1;
      for (int j = 0; j < n; j++) adr += (m->wrap_type[a + j] == mjWRAP_SPHERE || m->wrap_type[a + j] == mjWRAP_CYLINDER) ? 2 : 1;
    }
    B.addI(&D.tendon_slotadr, slot.data(), m->ntendon);
    B.addI(&D.body_simple, m->body_simple, m->nbody);
  }
  {   // history buffers (mjData.history): [nsample, interp] and the buffer address of each actuator and sensor, the
      // delays, and the sensors' [period, phase]
    S.nhistory = (int)m->nhistory;
    S.histflg = m->nhistory > 0 ? 1 : 0;
    B.addI(&D.actuator_history, m->actuator_history, 2 * m->nu);
    B.addI(&D.actuator_historyadr, m->actuator_historyadr, m->nu);
    B.addI(&D.sensor_history, m->sensor_history, 2 * m->nsensor);
    B.addI(&D.sensor_historyadr, m->sensor_historyadr, m->nsensor);
    B.addD(&D.actuator_delay, m->actuator_delay, m->nu);
    B.addD(&D.sensor_delay, m->sensor_delay, m->nsensor);
    B.addD(&D.sensor_interval, m->sensor_interval, 2 * m->nsensor);
  }
  {
    std::vector<int> trn(m->nu);
    for (int i = 0; i < m->nu; i++) trn[i] = m->actuator_trnid[2 * i];
    B.addI(&D.actuator_trnjnt, trn.data(), m->nu);
  }
  B.addI(&D.actuator_gaintype, m->actuator_gaintype, m->nu);
  B.addI(&D.actuator_biastype, m->actuator_biastype, m->nu);
  B.addI(&D.actuator_ctrllimited, m->actuator_ctrllimited, m->nu);
  B.addI(&D.actuator_forcelimited, m->actuator_forcelimited, m->nu);
  {
    std::vector<int> tt(m->nu), al(m->nu), ae(m->nu);
    for (int i = 0; i < m->nu; i++) {
      tt[i] = (m->actuator_trntype[i] == mjTRN_TENDON) ? TRN_TENDON : (m->actuator_trntype[i] == mjTRN_SITE) ? (m->actuator_trnid[2 * i + 1] >= 0 ? TRN_SITEREF : TRN_SITE)
              : (m->actuator_trntype[i] == mjTRN_SLIDERCRANK) ? TRN_SLIDERCRANK : TRN_JOINT;
      if (tt[i] == TRN_JOINT && m->jnt_type[m->actuator_trnid[2 * i]] == mjJNT_BALL) tt[i] = TRN_BALL;
      if (tt[i] == TRN_JOINT && m->jnt_type[m->actuator_trnid[2 * i]] == mjJNT_FREE) tt[i] = TRN_FREE;
      al[i] = m->actuator_actlimited[i];
      ae[i] = m->actuator_actearly[i];
    }
    B.addI(&D.actuator_trntype, tt.data(), m->nu);
    {
      // second transmission target (reference site / slider site) and, for reference-site transmissions, the dofs of
      // the common ancestral chain of the two sites' bodies, whose Jacobian columns are cleared (:1606-1630)
      std::vector<int> t2(m->nu), clr((size_t)m->nu * m->nv * (S.sitetrn ? 1 : 0) + 1, 0);
      for (int i = 0; i < m->nu; i++) {
        t2[i] = m->actuator_trnid[2 * i + 1];
        if (tt[i] != TRN_SITEREF) continue;
        const int b0 = m->body_weldid[m->site_bodyid[m->actuator_trnid[2 * i]]], b1 = m->body_weldid[m->site_bodyid[t2[i]]];
        int d0 = m->body_dofadr[b0] + m->body_dofnum[b0] - 1, d1 = m->body_dofadr[b1] + m->body_dofnum[b1] - 1;
        int common = -1;
        if (d0 >= 0 && d1 >= 0) {
          while (d0 != d1) {
            if (d0 < d1) d1 = m->dof_parentid[d1]; else d0 = m->dof_parentid[d0];
            if (d0 == -1 || d1 == -1) break;
          }
          if (d0 == d1) common = d0;
        }
        for (int da = common; da >= 0; da = m->dof_parentid[da]) clr[(size_t)i * m->nv + da] = 1;
      }
      B.addI(&D.actuator_trnid2, t2.data(), m->nu);
      B.addI(&D.actuator_refclear, clr.data(), clr.size());
    }
    B.addI(&D.actuator_dyntype, m->actuator_dyntype, m->nu);
    B.addI(&D.actuator_actadr, m->actuator_actadr, m->nu);
    B.addI(&D.actuator_actlimited, al.data(), m->nu);
    B.addI(&D.actuator_actearly, ae.data(), m->nu);
    std::vector<int> ip(m->nu);
    for (int i = 0; i < m->nu; i++) ip[i] = (m->actuator_trntype[i] == mjTRN_JOINTINPARENT);
    B.addI(&D.actuator_inparent, ip.data(), m->nu);
    std::vector<int> tl(m->ntendon);
    for (int i = 0; i < m->ntendon; i++) tl[i] = m->tendon_actfrclimited[i];
    B.addI(&D.tendon_actfrclimited, tl.data(), m->ntendon);
    B.addI(&D.body_mocapid, m->body_mocapid, m->nbody);
    std::vector<int> ag(m->njnt);
    for (int i = 0; i < m->njnt; i++) ag[i] = m->jnt_actgravcomp[i];
    B.addI(&D.jnt_actgravcomp, ag.data(), m->njnt);
  }

  B.addD(&D.qpos0, m->qpos0, m->nq);
  B.addD(&D.qpos_spring, m->qpos_spring, m->nq);
  B.addD(&D.body_pos, m->body_pos, 3 * m->nbody);
  B.addD(&D.body_quat, m->body_quat, 4 * m->nbody);
  B.addD(&D.body_ipos, m->body_ipos, 3 * m->nbody);
  B.addD(&D.body_iquat, m->body_iquat, 4 * m->nbody);
  B.addD(&D.body_mass, m->body_mass, m->nbody);
  B.addD(&D.body_subtreemass, m->body_subtreemass, m->nbody);
  B.addD(&D.body_inertia, m->body_inertia, 3 * m->nbody);
  B.addD(&D.body_invweight0, m->body_invweight0, 2 * m->nbody);
  B.addD(&D.jnt_pos, m->jnt_pos, 3 * m->njnt);
  B.addD(&D.jnt_axis, m->jnt_axis, 3 * m->njnt);
  B.addD(&D.jnt_stiffness, m->jnt_stiffness, m->njnt);
  B.addD(&D.jnt_stiffnesspoly, m->jnt_stiffnesspoly, mjNPOLY * m->njnt);
  B.addD(&D.jnt_range, m->jnt_range, 2 * m->njnt);
  B.addD(&D.jnt_margin, m->jnt_margin, m->njnt);
  B.addD(&D.jnt_solref, m->jnt_solref, mjNREF * m->njnt);
  B.addD(&D.jnt_solimp, m->jnt_solimp, mjNIMP * m->njnt);
  B.addD(&D.jnt_actfrcrange, m->jnt_actfrcrange, 2 * m->njnt);
  {
    std::vector<double> arm(m->nv), dmp(m->nv), dpoly(mjNPOLY * m->nv);
    int eulerdamp = 0;
    for (int i = 0; i < m->nv; i++) {
      int j = m->dof_jntid[i];
      arm[i] = m->dof_armature[i] + act_armature(m, false, j);
      double poly[mjNPOLY];
      for (int k = 0; k < mjNPOLY; k++) poly[k] = m->dof_dampingpoly[mjNPOLY * i + k];
      dmp[i] = m->dof_damping[i] + act_damping(m, false, j, poly);
      for (int k = 0; k < mjNPOLY; k++) dpoly[mjNPOLY * i + k] = poly[k];
      bool polynz = false;
      for (int k = 0; k < mjNPOLY; k++) polynz |= (m->dof_dampingpoly[mjNPOLY * i + k] != 0);
      if (m->dof_damping[i] > 0 || polynz || m->jnt_actuatorid[j] != -1) eulerdamp = 1;
    }
    if ((m->opt.disableflags & mjDSBL_EULERDAMP) || (m->opt.disableflags & mjDSBL_DAMPER)) eulerdamp = 0;
    O.eulerdamp = eulerdamp;
    B.addD(&D.dof_armature_eff, arm.data(), m->nv);
    B.addD(&D.dof_damping_eff, dmp.data(), m->nv);
    B.addD(&D.dof_dampingpoly_eff, dpoly.data(), mjNPOLY * m->nv);
  }
  B.addD(&D.dof_invweight0, m->dof_invweight0, m->nv);
  B.addD(&D.dof_M0, m->dof_M0, m->nv);
  B.addD(&D.dof_frictionloss, m->dof_frictionloss, m->nv);
  B.addD(&D.dof_solref, m->dof_solref, mjNREF * m->nv);
  B.addD(&D.dof_solimp, m->dof_solimp, mjNIMP * m->nv);
  B.addD(&D.geom_pos, m->geom_pos, 3 * m->ngeom);
  B.addD(&D.geom_quat, m->geom_quat, 4 * m->ngeom);
  B.addD(&D.geom_size, m->geom_size, 3 * m->ngeom);
  B.addD(&D.geom_rbound, m->geom_rbound, m->ngeom);
  B.addD(&D.wrap_prm, m->wrap_prm, m->nwrap);
  B.addD(&D.tendon_range, m->tendon_range, 2 * m->ntendon);
  B.addD(&D.tendon_margin, m->tendon_margin, m->ntendon);
  B.addD(&D.tendon_solref_lim, m->tendon_solref_lim, mjNREF * m->ntendon);
  B.addD(&D.tendon_solimp_lim, m->tendon_solimp_lim, mjNIMP * m->ntendon);
  B.addD(&D.tendon_invweight0, m->tendon_invweight0, m->ntendon);
  B.addD(&D.tendon_stiffness, m->tendon_stiffness, m->ntendon);
  B.addD(&D.tendon_stiffnesspoly, m->tendon_stiffnesspoly, mjNPOLY * m->ntendon);
  {
    std::vector<double> tdmp(m->ntendon), tpoly(mjNPOLY * m->ntendon), tarm(m->ntendon);
    for (int i = 0; i < m->ntendon; i++) {
      double poly[mjNPOLY];
      for (int k = 0; k < mjNPOLY; k++) poly[k] = m->tendon_dampingpoly[mjNPOLY * i + k];
      tdmp[i] = m->tendon_damping[i] + act_damping(m, true, i, poly);
      for (int k = 0; k < mjNPOLY; k++) tpoly[mjNPOLY * i + k] = poly[k];
      tarm[i] = m->tendon_armature[i] + act_armature(m, true, i);
      // mj_tendonDot (the bias of tendon armature) has no geom-wrapping branch in the reference either
      if (tarm[i] != 0 && m->wrap_type[m->tendon_adr[i]] != mjWRAP_JOINT)
        for (int j = 0; j < m->tendon_num[i]; j++)
          if (m->wrap_type[m->tendon_adr[i] + j] == mjWRAP_SPHERE || m->wrap_type[m->tendon_adr[i] + j] == mjWRAP_CYLINDER) {
            set_error("unsupported: tendon armature (incl. actuator armature) on a spatial tendon with geom wrapping");
            return -2;
          }
    }
    B.addD(&D.tendon_damping_eff, tdmp.data(), m->ntendon);
    B.addD(&D.tendon_dampingpoly_eff, tpoly.data(), mjNPOLY * m->ntendon);
    B.addD(&D.tendon_armature_eff, tarm.data(), m->ntendon);
  }
  B.addD(&D.tendon_lengthspring, m->tendon_lengthspring, 2 * m->ntendon);
  {
    std::vector<double> g0(m->nu), gp(kNGain * m->nu), bp(kNGain * m->nu);
    for (int i = 0; i < m->nu; i++) {
      g0[i] = m->actuator_gear[6 * i];
      for (int k = 0; k < kNGain; k++) {
        gp[kNGain * i + k] = m->actuator_gainprm[mjNGAIN * i + k];
        bp[kNGain * i + k] = m->actuator_biasprm[mjNBIAS * i + k];
      }
    }
    B.addD(&D.actuator_gear0, g0.data(), m->nu);
    B.addD(&D.actuator_gainprm, gp.data(), kNGain * m->nu);
    B.addD(&D.actuator_biasprm, bp.data(), kNGain * m->nu);
  }
  B.addD(&D.actuator_ctrlrange, m->actuator_ctrlrange, 2 * m->nu);
  B.addD(&D.actuator_forcerange, m->actuator_forcerange, 2 * m->nu);
  {
    std::vector<double> dp(kNDyn * (size_t)m->nu);
    for (int i = 0; i < m->nu; i++) for (int k = 0; k < kNDyn; k++) dp[kNDyn * i + k] = m->actuator_dynprm[mjNDYN * i + k];
    B.addD(&D.actuator_dynprm, dp.data(), dp.size());
  }
  B.addD(&D.actuator_actrange, m->actuator_actrange, 2 * m->nu);
  B.addD(&D.actuator_lengthrange, m->actuator_lengthrange, 2 * m->nu);
  B.addD(&D.actuator_acc0, m->actuator_acc0, m->nu);
  B.addD(&D.actuator_gear6, m->actuator_gear, 6 * m->nu);
  B.addD(&D.actuator_cranklength, m->actuator_cranklength, m->nu);
  {   // wrapPeriod (engine_forward.c:296-328): servo-shaped actuators on a ball joint take the setpoint nearest the length
    std::vector<double> wp(m->nu, 0.0);
    for (int i = 0; i < m->nu; i++) {
      const int dt = m->actuator_dyntype[i], tt = m->actuator_trntype[i];
      const bool servo = m->actuator_gaintype[i] == mjGAIN_FIXED && m->actuator_biastype[i] == mjBIAS_AFFINE &&
                         m->actuator_gainprm[mjNGAIN * i] == -m->actuator_biasprm[mjNBIAS * i + 1] &&
                         (dt == mjDYN_NONE || dt == mjDYN_INTEGRATOR);
      if (servo && (tt == mjTRN_JOINT || tt == mjTRN_JOINTINPARENT) && m->jnt_type[m->actuator_trnid[2 * i]] == mjJNT_BALL)
      {
        const mjtNum* g = m->actuator_gear + 6 * i;
        wp[i] = 2 * mjPI * std::sqrt(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]);   // 2*mjPI * mju_norm3(gear)
      }
    }
    B.addD(&D.actuator_wrapperiod, wp.data(), m->nu);
  }
  B.addD(&D.tendon_frictionloss, m->tendon_frictionloss, m->ntendon);
  B.addD(&D.tendon_solref_fri, m->tendon_solref_fri, mjNREF * m->ntendon);
  B.addD(&D.tendon_solimp_fri, m->tendon_solimp_fri, mjNIMP * m->ntendon);
  B.addD(&D.tendon_actfrcrange, m->tendon_actfrcrange, 2 * m->ntendon);
  B.addD(&D.sensor_cutoff, m->sensor_cutoff, m->nsensor);
  {
    std::vector<double> ed(kNEqData * (size_t)m->neq);
    for (int i = 0; i < m->neq; i++) for (int k = 0; k < kNEqData; k++) ed[kNEqData * i + k] = m->eq_data[mjNEQDATA * i + k];
    B.addD(&D.eq_data, ed.data(), ed.size());
    B.addD(&D.eq_solref, m->eq_solref, 2 * (size_t)m->neq);
    B.addD(&D.eq_solimp, m->eq_solimp, 5 * (size_t)m->neq);
    B.addD(&D.tendon_length0, m->tendon_length0, m->ntendon);
  }
  B.addD(&D.site_pos, m->site_pos, 3 * m->nsite);
  B.addD(&D.site_size, m->site_size, 3 * m->nsite);
  B.addD(&D.body_gravcomp, m->body_gravcomp, m->nbody);
  B.addI(&D.site_type, m->site_type, m->nsite);
  B.addD(&D.site_quat, m->site_quat, 4 * m->nsite);

  int has_lim = 0, has_fl = 0;
  for (int i = 0; i < m->njnt; i++) has_lim |= m->jnt_limited[i];
  for (int i = 0; i < m->ntendon; i++) has_lim |= m->tendon_limited[i];
  for (int i = 0; i < m->nv; i++) has_fl |= (m->dof_frictionloss[i] != 0);
  for (int i = 0; i < m->ntendon; i++) has_fl |= (m->tendon_frictionloss[i] > 0);
  O.has_limits = has_lim; O.has_frictionloss = has_fl;

  // ---- static candidate geom pairs, in the order the reference emits their contacts -----------
  std::vector<int> pg1, pg2, pdim;
  std::vector<double> pmargin, pinc, psolref, psolimp, pfric;
  const bool filterparent = !(m->opt.disableflags & mjDSBL_FILTERPARENT);
  const bool midphase = !(m->opt.disableflags & mjDSBL_MIDPHASE);
  const bool contacts_on = !(m->opt.disableflags & (mjDSBL_CONSTRAINT | mjDSBL_CONTACT));
  auto can_collide = [&](int b) { return m->body_contype[b] || m->body_conaffinity[b]; };
  auto has_plane = [&](int b) {
    for (int g = m->body_geomadr[b]; g < m->body_geomadr[b] + m->body_geomnum[b]; g++)
      if (m->geom_type[g] == mjGEOM_PLANE) return true;
    return false;
  };
  auto always = [&](int b) {
    return (b == 0 && m->body_geomnum[b] > 0) || (m->body_dofnum[m->body_weldid[b]] == 0 && has_plane(b));
  };
  // predefined <pair>s (engine_collision_driver.c:651-662,820-826): merged into the body-pair walk by signature -
  // a pair is tested before the first body pair whose signature is not smaller, the rest after the walk - with the
  // pair's own parameters and none of the body / bitmask filters
  int pairadr = 0;
  // convex candidates: the libccd path that mjDSBL_NATIVECCD selects for the GJK pairs is not built (plane-ellipsoid
  // never uses it), and ccd_iterations sizes the EPA polytope, whose faces name their vertices in 10 bits
  auto note_convex = [&](int t1, int t2) -> int {
    if (!collider_convex(t1, t2)) return 0;
    if (pair_gjk(t1, t2)) {
      if (m->opt.disableflags & mjDSBL_NATIVECCD) {
        set_error("unsupported: mjDSBL_NATIVECCD (the libccd convex collision path) is not built; only native GJK / EPA is");
        return -2;
      }
      if (m->opt.ccd_iterations < 1 || m->opt.ccd_iterations > 1000) {
        set_error("unsupported: ccd_iterations outside [1, 1000] with convex collision pairs");
        return -2;
      }
      S.nconvex++;
    }
    S.convex = 1;
    return 0;
  };
  auto push_predefined = [&](int k) -> int {
    int x = m->pair_geom1[k], y = m->pair_geom2[k];
    if (m->geom_type[x] > m->geom_type[y]) std::swap(x, y);
    if (!collider_defined(m->geom_type[x], m->geom_type[y])) return 0;
    if (!collider_supported(m->geom_type[x], m->geom_type[y])) {
      char msg[160];
      snprintf(msg, sizeof(msg), "unsupported: collider for geom types (%d,%d) (contact pair %d) is a 'next' row", m->geom_type[x], m->geom_type[y], k);
      set_error(msg);
      return -2;
    }
    if (collider_boxfamily(m->geom_type[x], m->geom_type[y])) S.colbox = 1;
    if (int rc = note_convex(m->geom_type[x], m->geom_type[y])) return rc;
    pg1.push_back(x); pg2.push_back(y); pdim.push_back(m->pair_dim[k]);
    pmargin.push_back(m->pair_margin[k] + m->pair_gap[k]); pinc.push_back(m->pair_margin[k]);
    for (int c = 0; c < mjNREF; c++) psolref.push_back(m->pair_solref[mjNREF * k + c]);
    for (int c = 0; c < mjNIMP; c++) psolimp.push_back(m->pair_solimp[mjNIMP * k + c]);
    for (int c = 0; c < 5; c++) pfric.push_back(m->pair_friction[5 * k + c]);
    return 0;
  };
  for (int b1 = 0; contacts_on && b1 < m->nbody; b1++) {
    for (int b2 = b1 + 1; b2 < m->nbody; b2++) {
      const unsigned sig0 = ((unsigned)b1 << 16) + (unsigned)b2;
      const int startadr = pairadr;
      bool merged = false;
      for (; pairadr < m->npair && (unsigned)m->pair_signature[pairadr] <= sig0; pairadr++) {
        merged = ((unsigned)m->pair_signature[pairadr] == sig0);
        if (int rc = push_predefined(pairadr)) return rc;
      }
      if (!can_collide(b1) || !can_collide(b2)) continue;
      // broadphase membership: SAP covers bodies >= 1; the world body only through always-collide
      if (b1 == 0 && !always(0)) continue;
      int w1 = m->body_weldid[b1], w2 = m->body_weldid[b2];
      int pw1 = m->body_weldid[m->body_parentid[w1]], pw2 = m->body_weldid[m->body_parentid[w2]];
      if (w1 == w2) continue;
      if (m->body_dofnum[w1] == 0 && m->body_dofnum[w2] == 0) continue;
      if (filterparent && w1 != 0 && w2 != 0 && (w1 == pw2 || w2 == pw1)) continue;
      // add_pair: OR of geom bitmasks
      int ct1 = 0, ca1 = 0, ct2 = 0, ca2 = 0;
      for (int g = m->body_geomadr[b1]; g < m->body_geomadr[b1] + m->body_geomnum[b1]; g++) { ct1 |= m->geom_contype[g]; ca1 |= m->geom_conaffinity[g]; }
      for (int g = m->body_geomadr[b2]; g < m->body_geomadr[b2] + m->body_geomnum[b2]; g++) { ct2 |= m->geom_contype[g]; ca2 |= m->geom_conaffinity[g]; }
      if (!(ct1 & ca2) && !(ct2 & ca1)) continue;
      if (!(m->body_contype[b1] & m->body_conaffinity[b2]) && !(m->body_contype[b2] & m->body_conaffinity[b1])) continue;
      unsigned sig = ((unsigned)b1 << 16) + (unsigned)b2;
      bool excluded = false;
      for (int e = 0; e < m->nexclude; e++) if ((unsigned)m->exclude_signature[e] == sig) excluded = true;
      if (excluded) continue;

      std::vector<Cand> cand;
      int n1 = m->body_geomnum[b1], n2 = m->body_geomnum[b2];
      int a1 = m->body_geomadr[b1], a2 = m->body_geomadr[b2];
      for (int g1 = a1; g1 < a1 + n1; g1++)
        for (int g2 = a2; g2 < a2 + n2; g2++) {
          if (!(m->geom_contype[g1] & m->geom_conaffinity[g2]) && !(m->geom_contype[g2] & m->geom_conaffinity[g1])) continue;
          bool predefined = false;   // the geom pair of a merged <pair> is not collided a second time
          for (int k = startadr; merged && k < pairadr; k++)
            if ((m->pair_geom1[k] == g1 && m->pair_geom2[k] == g2) || (m->pair_geom1[k] == g2 && m->pair_geom2[k] == g1)) predefined = true;
          if (predefined) continue;
          int x = g1, y = g2;
          if (m->geom_type[x] > m->geom_type[y]) std::swap(x, y);
          if (!collider_defined(m->geom_type[x], m->geom_type[y])) continue;
          cand.push_back({x, y});
        }
      bool single = (n1 == 1 && n2 == 1);
      if (!single && midphase && m->body_bvhadr[b1] >= 0 && m->body_bvhadr[b2] >= 0) {
        // midphase emits leaves in traversal order, then stable-sorts the pair's contacts by
        // (geom[0], geom[1]) with geom[0] the lower-type geom: a static order
        std::stable_sort(cand.begin(), cand.end(), [](const Cand& a, const Cand& b) {
          if (a.g1 != b.g1) return a.g1 < b.g1;
          return a.g2 < b.g2;
        });
      }
      for (auto& c : cand) {
        if (!collider_supported(m->geom_type[c.g1], m->geom_type[c.g2])) {
          char msg[160];
          snprintf(msg, sizeof(msg), "unsupported: collider for geom types (%d,%d) (geoms %d,%d) is a 'next' row",
                   m->geom_type[c.g1], m->geom_type[c.g2], c.g1, c.g2);
          set_error(msg);
          return -2;
        }
        if (collider_boxfamily(m->geom_type[c.g1], m->geom_type[c.g2])) S.colbox = 1;
        if (int rc = note_convex(m->geom_type[c.g1], m->geom_type[c.g2])) return rc;
        int condim; double solref[mjNREF], solimp[mjNIMP], fr[5];
        contact_param(m, c.g1, c.g2, &condim, solref, solimp, fr);
        double margin = m->geom_margin[c.g1] + m->geom_margin[c.g2];
        double gap = m->geom_gap[c.g1] + m->geom_gap[c.g2];
        pg1.push_back(c.g1); pg2.push_back(c.g2); pdim.push_back(condim);
        pmargin.push_back(margin + gap); pinc.push_back(margin);
        for (int k = 0; k < mjNREF; k++) psolref.push_back(solref[k]);
        for (int k = 0; k < mjNIMP; k++) psolimp.push_back(solimp[k]);
        for (int k = 0; k < 5; k++) pfric.push_back(fr[k]);
      }
    }
  }
  for (; contacts_on && pairadr < m->npair; pairadr++)   // predefined pairs past the last body pair
    if (int rc = push_predefined(pairadr)) return rc;
  // mjENBL_OVERRIDE (mj_assignMargin / Ref / Imp / Friction, engine_core_constraint.c:176-217): every contact takes the
  // margin, solver parameters and friction of mjOption; the gap stays the pair's own
  if (m->opt.enableflags & mjENBL_OVERRIDE) {
    for (size_t p = 0; p < pg1.size(); p++) {
      const double gap = pmargin[p] - pinc[p];
      pinc[p] = m->opt.o_margin;
      pmargin[p] = m->opt.o_margin + gap;
      for (int c = 0; c < mjNREF; c++) psolref[mjNREF * p + c] = m->opt.o_solref[c];
      for (int c = 0; c < mjNIMP; c++) psolimp[mjNIMP * p + c] = m->opt.o_solimp[c];
      for (int c = 0; c < 5; c++) pfric[5 * p + c] = std::max((double)mjMINMU, m->opt.o_friction[c]);
    }
  }
  S.npair = (int)pg1.size();
  if (S.nhistory && S.spatial) {
    set_error("unsupported: history buffers (delays) together with spatial tendons: no kernel carries both");
    return -2;
  }
  if (S.nhistory && S.convex) {
    set_error("unsupported: history buffers (delays) together with convex (GJK / EPA) collision pairs: no kernel carries both");
    return -2;
  }
  if (S.spatial && S.convex) {
    set_error("unsupported: spatial tendons together with convex (GJK / EPA) collision pairs: no kernel carries both");
    return -2;
  }
  // polytope scratch of the GJK candidates (mjb_convex.h): kCcdSlots slots per environment, fewer when the model has
  // fewer GJK candidates; nothing at all for models without them, whose layout is unchanged
  S.ccdslots = std::min(kCcdSlots, S.nconvex);
  S.ccdslot = S.nconvex ? (int)ccd_slot_doubles(m->opt.ccd_iterations) : 0;
  B.addI(&D.pair_geom1, pg1.data(), pg1.size());
  B.addI(&D.pair_geom2, pg2.data(), pg2.size());
  B.addI(&D.pair_dim, pdim.data(), pdim.size());
  B.addD(&D.pair_margin, pmargin.data(), pmargin.size());
  B.addD(&D.pair_includemargin, pinc.data(), pinc.size());
  B.addD(&D.pair_solref, psolref.data(), psolref.size());
  B.addD(&D.pair_solimp, psolimp.data(), psolimp.size());
  B.addD(&D.pair_friction, pfric.data(), pfric.size());

  // ---- schedules for the cooperative (warp-per-env) tree recursions --------------------------------
  // Every schedule reproduces the reference's SERIAL accumulation order per output element, so the
  // level-parallel recursions stay bit-compatible with engine_core_smooth.c.
  {
    // body depth levels (level 0 = world) and per-body child lists in DESCENDING id order:
    // the reference's backward passes run i = nbody-1..1 and add body i into its parent, so each
    // parent receives its children in descending id order (mj_comPos :262-275, mj_crb :1911-1917)
    std::vector<int> depth(m->nbody, 0);
    int nlevel = 1;
    for (int i = 1; i < m->nbody; i++) { depth[i] = depth[m->body_parentid[i]] + 1; nlevel = std::max(nlevel, depth[i] + 1); }
    std::vector<int> ladr(nlevel + 1, 0), lbody;
    for (int l = 0; l < nlevel; l++) {
      ladr[l] = (int)lbody.size();
      for (int i = 0; i < m->nbody; i++) if (depth[i] == l) lbody.push_back(i);
    }
    ladr[nlevel] = (int)lbody.size();
    std::vector<int> cadr(m->nbody + 1, 0), cid;
    for (int p = 0; p < m->nbody; p++) {
      cadr[p] = (int)cid.size();
      for (int i = m->nbody - 1; i >= 1; i--) if (m->body_parentid[i] == p) cid.push_back(i);
    }
    cadr[m->nbody] = (int)cid.size();
    S.nlevel = nlevel;
    B.addI(&D.lvl_adr, ladr.data(), ladr.size());
    B.addI(&D.lvl_body, lbody.data(), lbody.size());
    B.addI(&D.child_adr, cadr.data(), cadr.size());
    B.addI(&D.child_id, cid.data(), cid.size());

    // dof depth levels (depth = number of dof ancestors) and, per dof j, its strict descendants i in
    // DESCENDING order with the CSR address of M(i,j): gather form of the L^-T pass of mj_solveLD
    int nv = m->nv, ndl = 1;
    std::vector<int> dd(nv, 0);
    for (int i = 0; i < nv; i++) { dd[i] = m->M_rownnz[i] - 1; ndl = std::max(ndl, dd[i] + 1); }
    std::vector<int> dadr(ndl + 1, 0), ddof;
    for (int l = 0; l < ndl; l++) {
      dadr[l] = (int)ddof.size();
      for (int i = 0; i < nv; i++) if (dd[i] == l) ddof.push_back(i);
    }
    dadr[ndl] = (int)ddof.size();
    std::vector<int> madr(nv + 1, 0), mdof, mq;
    for (int j = 0; j < nv; j++) {
      madr[j] = (int)mdof.size();
      for (int i = nv - 1; i > j; i--) {
        int start = m->M_rowadr[i], nnz = m->M_rownnz[i];
        for (int a = start; a < start + nnz - 1; a++)
          if (m->M_colind[a] == j) { mdof.push_back(i); mq.push_back(a); }
      }
    }
    madr[nv] = (int)mdof.size();
    S.ndlevel = ndl;
    B.addI(&D.dlvl_adr, dadr.data(), dadr.size());
    B.addI(&D.dlvl_dof, ddof.data(), ddof.size());
    B.addI(&D.mt_adr, madr.data(), madr.size());
    B.addI(&D.mt_dof, mdof.data(), mdof.size());
    B.addI(&D.mt_qadr, mq.data(), mq.size());

    // L'DL "program": for pivot row k the independent element updates
    //   mat[dst] += mat[src] * (-mat[cf] * invD)      (mj_factorI :1997-2029)
    std::vector<int> fadr(nv + 1, 0), fdst, fsrc, fcf;
    for (int k = 0; k < nv; k++) {
      fadr[k] = (int)fdst.size();
      int start = m->M_rowadr[k], diag = m->M_rownnz[k] - 1, end = start + diag;
      for (int adr = end - 1; adr >= start; adr--) {
        int i = m->M_colind[adr];
        for (int c = 0; c < m->M_rownnz[i]; c++) { fdst.push_back(m->M_rowadr[i] + c); fsrc.push_back(start + c); fcf.push_back(adr); }
      }
    }
    fadr[nv] = (int)fdst.size();
    B.addI(&D.fac_adr, fadr.data(), fadr.size());
    B.addI(&D.fac_dst, fdst.data(), fdst.size());
    B.addI(&D.fac_src, fsrc.data(), fsrc.size());
    B.addI(&D.fac_cf, fcf.data(), fcf.size());

    // limit candidates in the reference's row order (mj_instantiateLimit :1388-1517) and
    // friction-loss dofs (mj_instantiateFriction :1291-1320)
    std::vector<int> lk, lid, ls, fl;
    for (int i = 0; i < m->njnt; i++) {
      if (!m->jnt_limited[i]) continue;
      if (m->jnt_type[i] == mjJNT_SLIDE || m->jnt_type[i] == mjJNT_HINGE) {
        for (int side = -1; side <= 1; side += 2) { lk.push_back(LIM_HINGE); lid.push_back(i); ls.push_back(side); }
      } else if (m->jnt_type[i] == mjJNT_BALL) {
        lk.push_back(LIM_BALL); lid.push_back(i); ls.push_back(0);
      }
    }
    for (int i = 0; i < m->ntendon; i++) {
      if (!m->tendon_limited[i]) continue;
      for (int side = -1; side <= 1; side += 2) { lk.push_back(LIM_TENDON); lid.push_back(i); ls.push_back(side); }
    }
    for (int i = 0; i < nv; i++) if (m->dof_frictionloss[i] != 0) fl.push_back(i);
    for (int i = 0; i < m->ntendon; i++) if (m->tendon_frictionloss[i] > 0) fl.push_back(-(i + 1));   // engine_core_constraint.c:1323
    S.nlim = (int)lk.size();
    S.nfl = (int)fl.size();
    B.addI(&D.lim_kind, lk.data(), lk.size());
    B.addI(&D.lim_id, lid.data(), lid.size());
    B.addI(&D.lim_side, ls.data(), ls.size());
    B.addI(&D.fl_dof, fl.data(), fl.size());

    // body x dof ancestry: 1 if dof c is on the kinematic chain of body b's weld root (mj_jac :197-225)
    std::vector<int> anc((size_t)m->nbody * nv, 0);
    for (int b = 0; b < m->nbody; b++) {
      int wb = m->body_weldid[b];
      if (m->body_dofnum[wb] == 0) continue;
      int i = m->body_dofadr[wb] + m->body_dofnum[wb] - 1;
      while (i >= 0) { anc[(size_t)b * nv + i] = 1; i = m->dof_parentid[i]; }
    }
    B.addI(&D.body_dofanc, anc.data(), anc.size());
  }

  // caps replacing the reference arena (larger caps cost memory, not time, so the defaults lean generous)
  if (nconmax <= 0) nconmax = std::min(std::max(S.npair / 2, 16), 48);
  if (njmax <= 0) njmax = S.nfl + 6 * S.neq + 128;
  S.nconmax = nconmax;
  S.njmax = njmax;
  if (O.solver == mjSOL_PGS && !O.dense) { set_error("unsupported: PGS with sparse Jacobian (nv >= 60)"); return -2; }
  if (!O.dense) { set_error("unsupported: sparse-Jacobian models (nv >= 60) are a 'next' row"); return -2; }
  if (O.solver != mjSOL_PGS && O.solver != mjSOL_NEWTON && O.solver != mjSOL_CG) { set_error("unsupported: unknown solver"); return -2; }

  B.fix();
  return 0;
}

}  // namespace mjb
