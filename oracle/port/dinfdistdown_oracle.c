/* TEST INFRASTRUCTURE ONLY — CPU restatement of dinfdistdown (src/DinfDistDown.cpp:95-1398), line by line: the receiver counts of
 * prop() > 0, the stream cells reset to 0, the FIFO queue that starts with the cells at 0, the flow algebra of a dequeued cell in
 * each of the four methods (h, v, p, s) and three statistics (ave, max, min), and the decrements of its donors, exactly as the
 * reference's one-rank run does.  The GPU's levels are checked against this (tests/test_dinfdistdown.py); this in turn replays the
 * reference's recorded outputs (tests/golden/dinfdistdown_reference.json).  Conventions as oracle/port/taudem_oracle.c: row 0 =
 * north, cell (i = column, j = row) at [j * nx + i]; nodata test fabsf(v - nodata) < 1e-5f.  Build: make -C oracle -f
 * dinfdistdown.mk port.
 *
 * One deliberate difference: the reference takes the shares inside the algebra of v, p and s from fel's per-row cell sizes and
 * everything else from ang's; here (and on the GPU) ang's cell sizes serve throughout (dxc / dyc).
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

static const int d1[9] = {0, 1, 1, 0, -1, -1, -1, 0, 1};   /* column offset */
static const int d2[9] = {0, 0, -1, -1, -1, 0, 1, 1, 1};   /* row offset    */
#define PI 3.14159265359
#define MISSINGFLOAT (-FLT_MAX)
#define IDX(i, j) ((size_t)(j) * nx + (i))
#define INSIDE(i, j) ((i) >= 0 && (i) < nx && (j) >= 0 && (j) < ny)

static int ndf(float v, float nd) { return fabsf(v - nd) < 1e-5f; }

/* src/commonLib.cpp:76-91 */
static double prop(float a, int k, double dx1, double dy1) {
  double aref[10] = {-atan2(dy1, dx1), 0., 0., (double)(0.5 * PI), 0., (double)PI, 0., (double)(1.5 * PI), 0., (double)(2. * PI)};
  aref[2] = -aref[0];
  aref[4] = PI - aref[2];
  aref[6] = PI + aref[2];
  aref[8] = 2. * PI - aref[2];
  double p = 0.;
  if (k <= 0) k = k + 8;
  if (k == 1 && a > PI) a = (float)(a - 2.0 * PI);
  if (a > aref[k - 1] && a < aref[k + 1]) {
    if (a > aref[k]) p = (aref[k + 1] - a) / (aref[k + 1] - aref[k]);
    else p = (a - aref[k - 1]) / (aref[k] - aref[k - 1]);
  }
  if (p < 1e-5) return -1.;
  return p;
}

/* typemethod 0 h, 1 v, 2 p, 3 s; statmethod 0 ave, 1 max, 2 min; fel NULL for h; w NULL: no weights; dxc / dyc per-row cell sizes.
 * dd out (float32, nodata MISSINGFLOAT).  Returns the number of cells dequeued. */
long long orc_dinfdistdown(const float* ang, const float* fel, const float* w, const int16_t* src, float* dd, int nx, int ny, float andv,
                           float fnd, float wnd, const double* dxc, const double* dyc, int statmethod, int typemethod, int concheck) {
  const size_t n = (size_t)nx * ny;
  const int usew = w != NULL && typemethod != 1;
  short* nb = (short*)malloc(n * sizeof(short));
  int32_t* q = (int32_t*)malloc(n * 4 + 4);
  float* dist = (float*)malloc((size_t)ny * 9 * 4);
  float* dv = typemethod == 2 ? (float*)malloc(n * 4) : NULL;   /* p: the vertical values */
  size_t qh = 0, qt = 0;
  for (int m = 0; m < ny; m++)
    for (int kk = 1; kk <= 8; kk++) dist[(size_t)m * 9 + kk] = (float)sqrt(dxc[m] * dxc[m] * d1[kk] * d1[kk] + dyc[m] * dyc[m] * d2[kk] * d2[kk]);
  for (size_t c = 0; c < n; c++) {
    nb[c] = -32768;
    dd[c] = MISSINGFLOAT;
    if (dv) dv[c] = MISSINGFLOAT;
  }
  /* src/DinfDistDown.cpp:207-233 */
  for (int j = 0; j < ny; j++)
    for (int i = 0; i < nx; i++) {
      const size_t c = IDX(i, j);
      if (ndf(ang[c], andv)) continue;
      nb[c] = 0;
      for (int k = 1; k <= 8; k++) {
        const int in = i + d1[k], jn = j + d2[k];
        const double p = prop(ang[c], k, dxc[j], dyc[j]);
        if (p > 0. && INSIDE(in, jn) && !ndf(ang[IDX(in, jn)], andv)) nb[c]++;
      }
      if (src[c] >= 1) nb[c] = 0;
      if (nb[c] == 0) q[qt++] = (int32_t)c;
    }
  long long dequeued = 0;
  while (qh < qt) {
    const size_t c = (size_t)q[qh++];
    const int i = (int)(c % nx), j = (int)(c / nx);
    dequeued++;
    if (src[c] >= 1) {
      dd[c] = 0.0f;
      if (dv) dv[c] = 0.0f;
    } else if (typemethod != 0 && ndf(fel[c], fnd)) {
      dd[c] = MISSINGFLOAT;
      if (dv) dv[c] = MISSINGFLOAT;
    } else {
      int con = 0, first = 1;
      float distr = 0.0f, distrv = 0.0f, sump = 0.0f;
      const float angle = ang[c];
      const float elv = typemethod != 0 ? fel[c] : 0.0f;
      for (int k = 1; k <= 8; k++) {
        const int in = i + d1[k], jn = j + d2[k];
        const double p = prop(angle, k, dxc[j], dyc[j]);
        if (!(p > 0.)) continue;
        if (!INSIDE(in, jn) || ndf(dd[IDX(in, jn)], MISSINGFLOAT)) { con = 1; continue; }
        const size_t r = IDX(in, jn);
        if (typemethod != 0 && ndf(fel[r], fnd)) { con = 1; continue; }
        sump = sump + p;
        const float dtss = dd[r];
        float wt = 1.f;
        if (usew) {
          if (ndf(w[r], wnd)) con = 1;
          else wt = w[r];
        }
        float x, xv = 0.0f;
        if (typemethod == 0) x = dist[(size_t)j * 9 + k] * wt + dtss;
        else if (typemethod == 1) {
          const float distk = elv - fel[r];
          x = distk * 1.0f + dtss;
        } else if (typemethod == 2) {
          const float distk = elv - fel[r];
          x = dist[(size_t)j * 9 + k] * wt + dtss;
          xv = distk + dv[r];
        } else {
          const float elvn = fel[r];
          const float distk = sqrtf((elv - elvn) * (elv - elvn) + (dist[(size_t)j * 9 + k] * wt) * (dist[(size_t)j * 9 + k] * wt));
          x = distk + dtss;
        }
        if (statmethod == 0) {
          distr = distr + p * x;
          distrv = distrv + p * xv;
        } else if (statmethod == 1 && typemethod == 0) {
          if (x > distr) distr = x;
        } else if (first) {
          distr = x;
          distrv = xv;
          first = 0;
        } else if (statmethod == 1) {
          if (x > distr) distr = x;
          if (xv > distrv) distrv = xv;
        } else {
          if (x < distr) distr = x;
          if (xv < distrv) distrv = xv;
        }
      }
      if ((con && concheck == 1) || sump <= 0.) {
        dd[c] = MISSINGFLOAT;
        if (dv) dv[c] = MISSINGFLOAT;
      } else {
        dd[c] = statmethod == 0 ? (float)(distr / sump) : distr;
        if (dv) dv[c] = statmethod == 0 ? (float)(distrv / sump) : distrv;
      }
    }
    /* src/DinfDistDown.cpp:311-329 */
    for (int k = 1; k <= 8; k++) {
      const int in = i + d1[k], jn = j + d2[k];
      if (!INSIDE(in, jn) || ndf(ang[IDX(in, jn)], andv)) continue;
      const size_t r = IDX(in, jn);
      if (prop(ang[r], (k + 4) % 8, dxc[jn], dyc[jn]) > 0.) {
        nb[r]--;
        if (nb[r] == 0) q[qt++] = (int32_t)r;
      }
    }
  }
  /* src/DinfDistDown.cpp:1014-1025 */
  if (dv)
    for (size_t c = 0; c < n; c++) {
      if (ndf(dv[c], MISSINGFLOAT)) dd[c] = MISSINGFLOAT;
      else if (!ndf(dd[c], MISSINGFLOAT)) {
        const float h = dd[c], v = dv[c];
        dd[c] = sqrtf(h * h + v * v);
      }
    }
  free(nb); free(q); free(dist); free(dv);
  return dequeued;
}
