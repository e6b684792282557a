/* TEST INFRASTRUCTURE ONLY — CPU restatement of slopeavedown (src/SlopeAveDown.cpp:59-330), line by line: every pass re-runs
 * the aread8 queue of initNeighborD8up (src/commonLib.cpp:240-283) and evaluates the cells in queue order, reading and writing
 * ed, dd and sd in place, exactly as the reference's one-rank run does.  The GPU's Jacobi passes over the D8 sweep's cells are
 * checked against this (tests/test_slopeavedown.py); this in turn replays the reference's recorded outputs
 * (tests/golden/slopeavedown_reference.json).  Conventions as oracle/port/taudem_oracle.c: row 0 = north, cell (i = column,
 * j = row) at [j * nx + i]; nodata test fabsf(v - nodata) < 1e-5f.  Build: make -C oracle -f downslope.mk port.
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

static const int d1[9] = {0, 1, 1, 0, -1, -1, -1, 0, 1};   /* column offset */
static const int d2[9] = {0, 0, -1, -1, -1, 0, 1, 1, 1};   /* row offset    */
#define MISSINGSHORT ((int16_t)-32768)
#define MISSINGFLOAT (-FLT_MAX)
#define IDX(i, j) ((size_t)(j) * nx + (i))
#define INSIDE(i, j) ((i) >= 0 && (i) < nx && (j) >= 0 && (j) < ny)

static int ndf(float v, float nd) { return fabsf(v - nd) < 1e-5f; }
static int nds(int16_t v, int16_t nd) { return fabsf((float)((int)v - (int)nd)) < 1e-5f; }

/* niter = dn / min(dxA, dyA) + 1 (src/SlopeAveDown.cpp:172); returns 1 where that conversion is undefined */
int orc_slopeavedown_niter(double dn, double dxA, double dyA, int* niter) {
  const double v = dn / (dyA < dxA ? dyA : dxA) + 1;     /* std::min(dxA, dyA) */
  if (!isfinite(dn) || !(v > -2147483649.0 && v < 2147483648.0)) return 1;
  *niter = (int)v;
  return 0;
}

/* z = fel (nodata znd), p (nodata pnd); dxc / dyc per-row cell sizes; dxA / dyA the header's.  sd out.  Returns 0, or 1 when niter
 * is undefined.  *passes (may be NULL): the number of the last pass that changed any of ed, dd, sd (0: none did). */
int orc_slopeavedown(const float* z, const int16_t* p, float* sd, int nx, int ny, float znd, int16_t pnd, const double* dxc, const double* dyc,
                     double dxA, double dyA, double dn, int* passes) {
  int niter = 0;
  if (orc_slopeavedown_niter(dn, dxA, dyA, &niter)) return 1;
  const size_t n = (size_t)nx * ny;
  float* ed = (float*)malloc(n * 4);
  float* dd = (float*)malloc(n * 4);
  int16_t* nb = (int16_t*)malloc(n * 2);
  int32_t* q = (int32_t*)malloc(n * 4);
  float* dist = (float*)malloc((size_t)ny * 9 * 4);
  /* src/SlopeAveDown.cpp:119-128 */
  for (int m = 0; m < ny; m++)
    for (int kk = 1; kk <= 8; kk++) dist[(size_t)m * 9 + kk] = (float)sqrt(d1[kk] * d1[kk] * dxc[m] * dxc[m] + d2[kk] * d2[kk] * dyc[m] * dyc[m]);
  /* src/SlopeAveDown.cpp:133-163 */
  for (size_t c = 0; c < n; c++) { ed[c] = MISSINGFLOAT; dd[c] = MISSINGFLOAT; sd[c] = MISSINGFLOAT; }
  for (size_t c = 0; c < n; c++)
    if (!ndf(z[c], znd) && !nds(p[c], pnd)) { ed[c] = z[c]; dd[c] = 0.0f; }
  if (passes) *passes = 0;
  for (int iter = 0; iter < niter; iter++) {
    int moved = 0;
    /* initNeighborD8up (src/commonLib.cpp:250-281) */
    size_t qh = 0, qt = 0;
    for (int j = 0; j < ny; j++)
      for (int i = 0; i < nx; i++) {
        const size_t c = IDX(i, j);
        nb[c] = MISSINGSHORT;
        if (nds(p[c], pnd) || p[c] < 0 || p[c] > 8) continue;
        nb[c] = 0;
        for (int k = 1; k <= 8; k++) {
          const int in = i + d1[k], jn = j + d2[k];
          if (!INSIDE(in, jn) || nds(p[IDX(in, jn)], pnd)) continue;
          const int16_t t = p[IDX(in, jn)];
          if (t >= 0 && t <= 8 && (t - k == 4 || t - k == -4)) nb[c]++;
        }
        if (nb[c] == 0) q[qt++] = (int32_t)c;
      }
    /* src/SlopeAveDown.cpp:222-264 */
    while (qh < qt) {
      const size_t c = q[qh++];
      const int i = (int)(c % nx), j = (int)(c / nx);
      const int k = p[c];
      if (k < 1 || k > 8) continue;               /* (the reference prints a warning here) */
      const int in = i + d1[k], jn = j + d2[k];
      if (INSIDE(in, jn) && !ndf(ed[IDX(in, jn)], MISSINGFLOAT)) {
        const float ddi = dist[(size_t)j * 9 + k] + dd[IDX(in, jn)];
        const float zi = ed[IDX(in, jn)];
        if (ndf(sd[c], MISSINGFLOAT)) {
          if (ddi > dn) {
            const float slp = (z[c] - zi) / ddi;
            union { float f; uint32_t u; } a = {slp}, b = {sd[c]};
            moved |= a.u != b.u;
            sd[c] = slp;
          }
        }
        union { float f; uint32_t u; } e0 = {ed[c]}, e1 = {zi}, d0 = {dd[c]}, d1v = {ddi};
        moved |= e0.u != e1.u || d0.u != d1v.u;
        ed[c] = zi;
        dd[c] = ddi;
      }
      if (INSIDE(in, jn) && !nds(p[IDX(in, jn)], pnd)) {
        const size_t r = IDX(in, jn);
        nb[r] = (int16_t)(nb[r] - 1);
        if (nb[r] == 0) q[qt++] = (int32_t)r;
      }
    }
    if (moved && passes) *passes = iter + 1;
  }
  free(ed); free(dd); free(nb); free(q); free(dist);
  return 0;
}
