/* TEST INFRASTRUCTURE ONLY — CPU restatement of d8hdisttostrm and d8vdisttostrm (src/D8HDistToStrm.cpp:57-226,
 * src/D8VDistToStrm.cpp:58-240), line by line: the neighbour counts, the FIFO queue that starts with the stream cells, the flow
 * algebra of a dequeued cell and the decrements of its upslope neighbours, exactly as the reference's one-rank run does.  The GPU's
 * BFS levels are checked against this (tests/test_disttostrm.py); this in turn replays the reference's recorded outputs
 * (tests/golden/disttostrm_reference.json).  Conventions as oracle/port/taudem_oracle.c: row 0 = north, cell (i = column, j = row)
 * at [j * nx + i]; nodata test fabsf(v - nodata) < 1e-5f.  Build: make -C oracle -f disttostrm.mk port.
 *
 * One deliberate difference: a dequeued cell whose code is -3..-1 or 9..12 (the reference matches them with its +-4 test, then
 * indexes d1 / d2 out of bounds) gets MISSINGFLOAT, as on the GPU.
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
static int stream(const int32_t* src, size_t c, int32_t snd, int thresh) { return src[c] != snd && src[c] >= thresh; }

/* vertical = 0: d8hdisttostrm (fel unused; dxc / dyc per-row cell sizes), 1: d8vdisttostrm (dxc / dyc unused).  dist out. */
int orc_disttostrm(int vertical, const int16_t* p, const float* fel, const int32_t* src, float* dist, int nx, int ny, int16_t pnd, int32_t snd,
                   int thresh, const double* dxc, const double* dyc) {
  const size_t n = (size_t)nx * ny;
  int16_t* nb = (int16_t*)malloc(n * 2);
  int32_t* q = (int32_t*)malloc(n * 4 + 4);
  float* dd = (float*)malloc((size_t)ny * 9 * 4);
  size_t qh = 0, qt = 0;
  /* src/D8HDistToStrm.cpp:121-130 */
  if (!vertical)
    for (int m = 0; m < ny; m++)
      for (int kk = 1; kk <= 8; kk++) dd[(size_t)m * 9 + kk] = (float)sqrt(d1[kk] * d1[kk] * dxc[m] * dxc[m] + d2[kk] * d2[kk] * dyc[m] * dyc[m]);
  /* src/D8HDistToStrm.cpp:133-150 */
  for (size_t c = 0; c < n; c++) { nb[c] = MISSINGSHORT; dist[c] = MISSINGFLOAT; }
  for (int j = 0; j < ny; j++)
    for (int i = 0; i < nx; i++) {
      const size_t c = IDX(i, j);
      if (!nds(p[c], pnd)) nb[c] = 1;
      if (stream(src, c, snd, thresh)) { nb[c] = 0; q[qt++] = (int32_t)c; }
    }
  /* src/D8HDistToStrm.cpp:161-201 */
  while (qh < qt) {
    const size_t c = (size_t)q[qh++];
    const int i = (int)(c % nx), j = (int)(c / nx);
    if (stream(src, c, snd, thresh)) dist[c] = 0.0f;
    else {
      const int k = p[c];
      if (k < 0 || k > 8) dist[c] = MISSINGFLOAT;           /* the reference reads d1[k] / d2[k] out of bounds here */
      else {
        const int in = i + d1[k], jn = j + d2[k];
        if (!INSIDE(in, jn) || ndf(dist[IDX(in, jn)], MISSINGFLOAT)) dist[c] = MISSINGFLOAT;
        else if (vertical) dist[c] = (fel[c] - fel[IDX(in, jn)]) + dist[IDX(in, jn)];
        else dist[c] = dd[(size_t)j * 9 + k] + dist[IDX(in, jn)];
      }
    }
    for (int k = 1; k <= 8; k++) {
      const int in = i + d1[k], jn = j + d2[k];
      if (!INSIDE(in, jn) || nds(p[IDX(in, jn)], pnd)) continue;
      const int t = p[IDX(in, jn)];
      if (t - k == 4 || t - k == -4) {
        const size_t r = IDX(in, jn);
        nb[r] = (int16_t)(nb[r] - 1);
        if (nb[r] == 0) q[qt++] = (int32_t)r;
      }
    }
  }
  free(nb); free(q); free(dd);
  return 0;
}
