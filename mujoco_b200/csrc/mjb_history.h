// History buffers of delayed actuators and delayed / sampled sensors (FEAT_HISTORY), restated operation for operation
// from the reference: historyFindIndex, mju_historyInsert and mju_historyRead (src/engine/engine_util_misc.c:1355-1561).
// A buffer of n samples of dim values is laid out as [user, cursor, times[n], values[n*dim]]; the cursor is the
// physical index of the newest sample, logical index 0 is the oldest.
#pragma once
#include "mjb_types.h"

// On the device the call sites of this code in the shared pipeline headers are compiled only in the translation unit
// that defines MJB_HISTORY_UNIT (the FEAT_HISTORY instantiations, mjb_kstep_history32.cu): every other kernel is the
// same code as without history buffers.  Host compilations (the emulation of the device path) always carry them.
#if defined(MJB_HISTORY_UNIT) || !defined(__CUDA_ARCH__)
#define MJB_HISTORY_CODE
#endif

namespace mjb {

MJB_HD int hist_phys(int cursor, int n, int logical) { return (cursor + 1 + logical) % n; }

// logical i with times[i-1] < t <= times[i]: 0 at or before the oldest sample, n after the newest (circular bisection)
MJB_HD int hist_find(FD times, int n, int cursor, double t) {
  if (t <= times[hist_phys(cursor, n, 0)]) return 0;
  if (t > times[hist_phys(cursor, n, n - 1)]) return n;
  int lo = 0, hi = n - 1;
  while (hi - lo > 1) {
    const int mid = (lo + hi) / 2;
    if (times[hist_phys(cursor, n, mid)] < t) lo = mid;
    else hi = mid;
  }
  return hi;
}

// slot for a sample at time t (the caller writes its dim values there): an existing sample at the same time is
// reused; a time before the oldest replaces the oldest; a time after the newest advances the cursor; a time in between
// shifts the older samples down, dropping the oldest
MJB_HD FD hist_insert(FD buf, int n, int dim, double t) {
  int cursor = (int)buf[1];
  FD times = buf + 2, values = buf + 2 + n;
  const int i = hist_find(times, n, cursor, t);
  if (i < n) {
    const int p = hist_phys(cursor, n, i);
    if (fabs(t - times[p]) < kMinVal) return values + (long)p * dim;
  }
  if (i == 0) {
    const int p = hist_phys(cursor, n, 0);
    times[p] = t;
    return values + (long)p * dim;
  }
  if (i == n) {
    cursor = (cursor + 1) % n;
    buf[1] = (double)cursor;
    times[cursor] = t;
    return values + (long)cursor * dim;
  }
  for (int j = 0; j < i - 1; j++) {
    const int src = hist_phys(cursor, n, j + 1), dst = hist_phys(cursor, n, j);
    times[dst] = times[src];
    for (int k = 0; k < dim; k++) values[(long)dst * dim + k] = values[(long)src * dim + k];
  }
  const int p = hist_phys(cursor, n, i - 1);
  times[p] = t;
  return values + (long)p * dim;
}

// value at time t into res[dim]: clamped to the oldest / newest sample, an exact match as stored, else zero-order hold
// (interp 0), linear (1) or cubic Hermite with Catmull-Rom slopes that are zero at the ends (2)
template <class R>
MJB_HD void hist_read(FD buf, int n, int dim, R res, double t, int interp) {
  const int cursor = (int)buf[1];
  FD times = buf + 2, values = buf + 2 + n;
  const int po = hist_phys(cursor, n, 0), pn = hist_phys(cursor, n, n - 1);
  int src = -1;
  int i = 0;
  if (t <= times[po] + kMinVal) src = po;
  else if (t >= times[pn] - kMinVal) src = pn;
  else {
    i = hist_find(times, n, cursor, t);
    const int pi = hist_phys(cursor, n, i);
    if (fabs(t - times[pi]) < kMinVal) src = pi;
    else if (interp == 0) src = hist_phys(cursor, n, i - 1);
  }
  if (src >= 0) {
    for (int k = 0; k < dim; k++) res[k] = values[(long)src * dim + k];
    return;
  }
  const int plo = hist_phys(cursor, n, i - 1), phi = hist_phys(cursor, n, i);
  const double dt = times[phi] - times[plo];
  const double alpha = (t - times[plo]) / dt;
  if (interp == 1) {
    for (int k = 0; k < dim; k++) res[k] = values[(long)plo * dim + k] + alpha * (values[(long)phi * dim + k] - values[(long)plo * dim + k]);
    return;
  }
  const double a2 = alpha * alpha, a3 = a2 * alpha;
  const double h00 = 2 * a3 - 3 * a2 + 1, h10 = a3 - 2 * a2 + alpha, h01 = -2 * a3 + 3 * a2, h11 = a3 - a2;
  for (int k = 0; k < dim; k++) {
    double mlo = 0, mhi = 0;
    if (i > 1) {
      const int pp = hist_phys(cursor, n, i - 2);
      mlo = (values[(long)phi * dim + k] - values[(long)pp * dim + k]) / (times[phi] - times[pp]);
    }
    if (i < n - 1) {
      const int pq = hist_phys(cursor, n, i + 1);
      mhi = (values[(long)pq * dim + k] - values[(long)plo * dim + k]) / (times[pq] - times[plo]);
    }
    res[k] = h00 * values[(long)plo * dim + k] + h10 * dt * mlo + h01 * values[(long)phi * dim + k] + h11 * dt * mhi;
  }
}

}  // namespace mjb
