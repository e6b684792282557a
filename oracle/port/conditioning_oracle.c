/* TEST INFRASTRUCTURE ONLY — CPU restatements of flowdircond and retlimflow.
 *
 * flowdircond (src/flowdircond.cpp:56-236), line by line: the aread8 queue of
 * initNeighborD8up (src/commonLib.cpp:240-283), then the cells in queue order, lowering z in place (float compares, the
 * reference's strict test in increasing k) and draining into the receiver, exactly as the reference's one-rank run does.  The
 * GPU's algebra 11 of the contributing-area sweep is checked against this (tests/test_conditioning.py); this in turn replays the
 * reference's recorded outputs (tests/golden/conditioning_reference.json).  Conventions as oracle/port/taudem_oracle.c: row 0 =
 * north, cell (i = column, j = row) at [j * nx + i]; nodata test fabsf(v - nodata) < 1e-5f.
 * Build: make -C oracle -f conditioning.mk port.
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static const int d1[9] = {0, 1, 1, 0, -1, -1, -1, 0, 1};   /* column offset */
static const int d2[9] = {0, 0, -1, -1, -1, 0, 1, 1, 1};   /* row offset    */
#define MISSINGSHORT ((int16_t)-32768)
#define MISSINGFLOAT (-FLT_MAX)
#define PI 3.14159265359
#define IDX(i, j) ((size_t)(j) * nx + (i))
#define INSIDE(i, j) ((i) >= 0 && (i) < nx && (j) >= 0 && (j) < ny)

static int ndf(float v, float nd) { return fabsf(v - nd) < 1e-5f; }
static int nds(int16_t v, int16_t nd) { return fabsf((float)((int)v - (int)nd)) < 1e-5f; }

/* p (nodata pnd), z (nodata znd) in; zfdc out (starts as z, lowered in place).  *processed (may be NULL): cells dequeued. */
void orc_flowdircond(const int16_t* p, const float* z, float* zfdc, int nx, int ny, int16_t pnd, float znd, long long* processed) {
  const size_t n = (size_t)nx * ny;
  int16_t* nb = (int16_t*)malloc(n * 2);
  int32_t* q = (int32_t*)malloc(n * 4 + 4);
  memcpy(zfdc, z, n * 4);
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
  long long done = 0;
  /* src/flowdircond.cpp:147-194 */
  while (qh < qt) {
    const size_t c = (size_t)q[qh++];
    const int i = (int)(c % (size_t)nx), j = (int)(c / (size_t)nx);
    ++done;
    if (!ndf(zfdc[c], znd)) {
      float zval = zfdc[c];
      for (int k = 1; k <= 8; k++) {
        const int in = i + d1[k], jn = j + d2[k];
        if (!INSIDE(in, jn)) continue;           /* the partition's getData off the grid: nodata, never in 1..8 */
        const int16_t sdir = p[IDX(in, jn)];
        if (sdir >= 1 && sdir <= 8) {
          if (!ndf(zfdc[IDX(in, jn)], znd)) {
            if (zfdc[IDX(in, jn)] < zval && (sdir - k == 4 || sdir - k == -4)) {
              zval = zfdc[IDX(in, jn)];
              zfdc[c] = zval;
            }
          }
        }
      }
    }
    /* drain into the receiver (code 0: the cell itself) */
    const int k = p[c];
    const int in = i + d1[k], jn = j + d2[k];
    if (INSIDE(in, jn) && !nds(p[IDX(in, jn)], pnd)) {
      const int16_t t = p[IDX(in, jn)];
      if (t >= 0 && t <= 8) {
        nb[IDX(in, jn)]--;
        if (nb[IDX(in, jn)] == 0) q[qt++] = (int32_t)IDX(in, jn);
      }
    }
  }
  if (processed) *processed = done;
  free(nb);
  free(q);
}

/* retlimflow (src/RetlimFlow.cpp:53-240), line by line: the queue of initNeighborDinfup (src/commonLib.cpp:92-136: a contributor is a
 * neighbour whose angle is not nodata and sends a share (float)prop(angle, direction to me) > 0, with its row's cell sizes), then
 * the cells in queue order: a cell whose wg or rc is nodata keeps MISSINGFLOAT and decrements nothing; the others sum the float
 * share times qrl of every neighbour with p > 0 in increasing k (the angle is not tested for nodata there), add wg, subtract rc,
 * clip at 0 by `< 0.`, and decrement every neighbour they send a share to.
 * edge_quirk = 1 follows the reference's one-rank run also where a share leaves the grid through the top or bottom edge: the drain
 * does not test hasAccess, so the decrement lands in the partition's border row (src/linearpart.h:554-564), and addBorders adds that
 * border back into the grid's own first / last row of the same column (src/linearpart.h:313-326; passBorders does nothing on one
 * rank), after which a count that reached 0 there is queued (src/RetlimFlow.cpp:204-215).  Such an edge cell can be evaluated
 * before, or without, its contributors.  edge_quirk = 0: flow that leaves the grid decrements nothing (the GPU's contract). */
static double prop(float a, int k, double dx1, double dy1) {
  double aref[10] = {-atan2(dy1, dx1), 0., 0., (double)(0.5 * PI), 0., (double)PI, 0., (double)(1.5 * PI), 0., (double)(2. * PI)};
  aref[2] = -aref[0]; aref[4] = PI - aref[2]; aref[6] = PI + aref[2]; aref[8] = 2. * PI - aref[2];
  double pp = 0.;
  if (k <= 0) k = k + 8;
  if (k == 1 && a > PI) a = (float)(a - 2.0 * PI);
  if (a > aref[k - 1] && a < aref[k + 1]) {
    if (a > aref[k]) pp = (aref[k + 1] - a) / (aref[k + 1] - aref[k]);
    else pp = (a - aref[k - 1]) / (aref[k] - aref[k - 1]);
  }
  return pp < 1e-5 ? -1. : pp;
}

void orc_retlimflow(const float* ang, const float* wg, const float* rc, float* qrl, int nx, int ny, float andv, float wnd, float rcnd, const double* dxc,
                    const double* dyc, int edge_quirk, long long* processed) {
  const size_t n = (size_t)nx * ny;
  int16_t* nb = (int16_t*)malloc(n * 2);
  int32_t* q = (int32_t*)malloc(n * 4 * 4 + 4);                /* (edge cells can be queued more than once) */
  int* topb = (int*)calloc((size_t)nx, sizeof(int));
  int* botb = (int*)calloc((size_t)nx, sizeof(int));
  size_t qh = 0, qt = 0;
  for (size_t c = 0; c < n; c++) qrl[c] = MISSINGFLOAT;
  for (int j = 0; j < ny; j++)
    for (int i = 0; i < nx; i++) {
      const size_t c = IDX(i, j);
      nb[c] = MISSINGSHORT;
      if (ndf(ang[c], andv)) continue;
      nb[c] = 0;
      for (int k = 1; k <= 8; k++) {
        const int in = i + d1[k], jn = j + d2[k];
        if (!INSIDE(in, jn) || ndf(ang[IDX(in, jn)], andv)) continue;
        const float pf = (float)prop(ang[IDX(in, jn)], (k + 4) % 8, dxc[jn], dyc[jn]);
        if (pf > 0.0) nb[c]++;
      }
      if (nb[c] == 0) q[qt++] = (int32_t)c;
    }
  long long done = 0;
  for (;;) {
  while (qh < qt) {
    const size_t c = (size_t)q[qh++];
    const int i = (int)(c % (size_t)nx), j = (int)(c / (size_t)nx);
    ++done;
    float qrlval = 0.;
    if (!ndf(wg[c], wnd) && !ndf(rc[c], rcnd)) {
      for (int k = 1; k <= 8; k++) {
        const int in = i + d1[k], jn = j + d2[k];
        if (INSIDE(in, jn)) {
          const float p = (float)prop(ang[IDX(in, jn)], (k + 4) % 8, dxc[jn], dyc[jn]);
          if (p > 0.) qrlval = qrlval + p * qrl[IDX(in, jn)];
        }
      }
      qrlval = qrlval + wg[c] - rc[c];
      if (qrlval < 0.) qrlval = 0.;
      qrl[c] = qrlval;
      for (int k = 1; k <= 8; k++) {
        const float p = (float)prop(ang[c], k, dxc[j], dyc[j]);
        if (p > 0.0) {
          const int in = i + d1[k], jn = j + d2[k];
          if (INSIDE(in, jn) && nb[IDX(in, jn)] != MISSINGSHORT) { nb[IDX(in, jn)]--; if (nb[IDX(in, jn)] == 0) q[qt++] = (int32_t)IDX(in, jn); }
          else if (edge_quirk && in >= 0 && in < nx) { if (jn == -1) topb[in]--; else if (jn == ny) botb[in]--; }
        }
      }
    }
  }
  if (!edge_quirk) break;
  /* addBorders, the border queue, clearBorders (src/RetlimFlow.cpp:201-218) */
  for (int i = 0; i < nx; i++) {
    if (nb[IDX(i, 0)] != MISSINGSHORT) nb[IDX(i, 0)] += topb[i];
    if (nb[IDX(i, ny - 1)] != MISSINGSHORT) nb[IDX(i, ny - 1)] += botb[i];
  }
  for (int i = 0; i < nx; i++) {
    if (topb[i] != 0 && nb[IDX(i, 0)] == 0) q[qt++] = (int32_t)IDX(i, 0);
    if (botb[i] != 0 && nb[IDX(i, ny - 1)] == 0) q[qt++] = (int32_t)IDX(i, ny - 1);
    topb[i] = botb[i] = 0;
  }
  if (qh == qt) break;
  }
  if (processed) *processed = done;
  free(nb);
  free(q);
  free(topb);
  free(botb);
}
