/* TEST INFRASTRUCTURE ONLY — CPU restatement ("port") of the TauDEM hot path on plain arrays.
 *
 * Parity status: PINNED.  tests/test_cpu.py checks every function below against the committed
 * golden vectors (tests/golden/*.npz) and the recorded output digests (tests/golden/reference.json),
 * which are outputs of the reference's own tools compiled unchanged (oracle/_ref, see
 * oracle/Makefile and tests/golden/make_golden.py).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may load this library.
 * It is a checker: single-threaded, written for clarity, and never on a product path.
 *
 * Conventions (reference src/commonLib.h:76-84, src/linearpart.h:471-483): row 0 = north, cell
 * (i = column, j = row) at [j*nx + i]; neighbour k = 1..8 = E,NE,N,NW,W,SW,S,SE; nodata test
 * fabsf(v - nodata) < 1e-5f; PI is the reference's truncated literal.
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define PI 3.14159265359
static const int d1[9] = {0, 1, 1, 0, -1, -1, -1, 0, 1};   /* column offset */
static const int d2[9] = {0, 0, -1, -1, -1, 0, 1, 1, 1};   /* row offset    */
#define MISSINGSHORT ((int16_t)-32768)
#define MISSINGFLOAT (-FLT_MAX)
#define IDX(i, j) ((size_t)(j) * nx + (i))
#define INSIDE(i, j) ((i) >= 0 && (i) < nx && (j) >= 0 && (j) < ny)

static int ndf(float v, float nd) { return fabsf(v - nd) < 1e-5f; }
static int nds(int16_t v, int16_t nd) { return fabsf((float)((int)v - (int)nd)) < 1e-5f; }
static int on_edge(int i, int j, int nx, int ny) { return i == 0 || j == 0 || i == nx - 1 || j == ny - 1; }

/* ------------------------------------------------------------------------------------------------
 * pitremove: reference src/flood.cpp:243-479.  Seeds (src/flood.cpp:243-271): nodata -> -3.0e38f,
 * mask == 1, grid-edge cells and cells with a nodata neighbour keep z; every other cell ends at
 * max(z, min over neighbours of W), the unique fixed point of the reference's stack sweeps
 * (:292-479) = the minimax path elevation to a seed.  Restated as a priority flood (binary heap).
 * ---------------------------------------------------------------------------------------------- */
typedef struct { float w; int32_t c; } hnode;
static void hpush(hnode* h, size_t* n, hnode v) {
  size_t i = (*n)++;
  while (i > 0) { size_t p = (i - 1) / 2; if (h[p].w <= v.w) break; h[i] = h[p]; i = p; }
  h[i] = v;
}
static hnode hpop(hnode* h, size_t* n) {
  hnode top = h[0], last = h[--(*n)];
  size_t i = 0;
  for (;;) {
    size_t l = 2 * i + 1, r = l + 1, m;
    if (l >= *n) break;
    m = (r < *n && h[r].w < h[l].w) ? r : l;
    if (h[m].w >= last.w) break;
    h[i] = h[m]; i = m;
  }
  h[i] = last;
  return top;
}

int orc_flood(const float* z, float* W, const int16_t* mask, int nx, int ny, float nodata, int four_way) {
  const int step = four_way ? 2 : 1;
  const size_t n = (size_t)nx * ny;
  hnode* heap = (hnode*)malloc(sizeof(hnode) * (n + 1));
  uint8_t* done = (uint8_t*)calloc(n, 1);
  size_t hn = 0;
  if (!heap || !done) return 1;
  for (int j = 0; j < ny; j++)
    for (int i = 0; i < nx; i++) {
      const size_t c = IDX(i, j);
      int seed = 0;
      if (ndf(z[c], nodata)) { W[c] = -3.0e38f; done[c] = 1; continue; }
      if (mask && mask[c] == 1) seed = 1;
      else if (on_edge(i, j, nx, ny)) seed = 1;
      else for (int k = 1; k <= 8 && !seed; k += step) if (ndf(z[IDX(i + d1[k], j + d2[k])], nodata)) seed = 1;
      if (seed) { W[c] = z[c]; done[c] = 1; hnode v = {z[c], (int32_t)c}; hpush(heap, &hn, v); }
      else W[c] = FLT_MAX;
    }
  while (hn) {
    const hnode t = hpop(heap, &hn);
    const int i = t.c % nx, j = t.c / nx;
    for (int k = 1; k <= 8; k += step) {
      const int in = i + d1[k], jn = j + d2[k];
      if (!INSIDE(in, jn)) continue;
      const size_t c = IDX(in, jn);
      if (done[c]) continue;
      W[c] = z[c] > t.w ? z[c] : t.w;
      done[c] = 1;
      hnode v = {W[c], (int32_t)c};
      hpush(heap, &hn, v);
    }
  }
  free(heap); free(done);
  return 0;
}

/* ------------------------------------------------------------------------------------------------
 * Garbrecht-Martz flat resolution shared by D8 and D-infinity (reference src/d8.cpp:459-680 and
 * src/dinf.cpp:598-833), written as the reference's own repeated passes over the flat list.
 * `drains(c)`: neighbour has a direction (D8: 1..8; Dinf: angle >= 0).
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int nx, ny, dinf;
  float* elev;        /* mutable copy of the DEM (overwritten by elev2 between outer iterations) */
  int16_t* dir8;      /* D8 directions   */
  float* ang;         /* Dinf angles     */
  const double *dxc, *dyc;
} flatctx;

static int fc_drains(const flatctx* f, size_t c) { return f->dinf ? f->ang[c] >= 0.0f : (f->dir8[c] > 0 && f->dir8[c] < 9); }
static int fc_eq(const flatctx* f, size_t c, int v) { return f->dinf ? f->ang[c] == (float)v : f->dir8[c] == v; }
/* dontCross: src/d8.cpp:54-100 / src/dinf.cpp:58-105 */
static int dont_cross(const flatctx* f, int k, int i, int j) {
  const int nx = f->nx;
  switch (k) {
    case 2: return fc_eq(f, IDX(i + 1, j), 4) || fc_eq(f, IDX(i, j - 1), 8);
    case 4: return fc_eq(f, IDX(i, j - 1), 6) || fc_eq(f, IDX(i - 1, j), 2);
    case 6: return fc_eq(f, IDX(i, j + 1), 4) || fc_eq(f, IDX(i - 1, j), 8);
    case 8: return fc_eq(f, IDX(i + 1, j), 6) || fc_eq(f, IDX(i, j + 1), 2);
    default: return 0;
  }
}
/* does flat cell (i,j) still increment in pass `st`?  src/d8.cpp:516-541 */
static int still_rising(const flatctx* f, const int16_t* elev2, int i, int j, int st) {
  const int nx = f->nx;
  for (int k = 1; k <= 8; k++) {
    if (dont_cross(f, k, i, j)) continue;
    const size_t n = IDX(i + d1[k], j + d2[k]);
    const float ed = f->elev[IDX(i, j)] - f->elev[n];
    if (ed >= 0 && fc_drains(f, n)) return 0;
    else if (ed == 0 && elev2[n] >= 0 && elev2[n] < st) return 0;
  }
  return 1;
}

/* VSLOPE: src/dinf.cpp:286-313 */
static void vslope(double E0, double E1, double E2, double D1, double D2, double DD, double* S, double* A) {
  const double S1 = (E0 - E1) / D1, S2 = (E1 - E2) / D2;
  const double AD = atan2(D2, D1);
  *A = (S2 == 0 && S1 == 0) ? 0 : atan2(S2, S1);
  if (*A < 0.) { *A = 0.; *S = S1; }
  else if (*A > AD) { *A = AD; *S = (E0 - E2) / DD; }
  else *S = sqrt(S1 * S1 + S2 * S2);
}
static const int FI1[9] = {0, 0, -1, -1, 0, 0, 1, 1, 0}, FI2[9] = {0, -1, -1, -1, -1, 1, 1, 1, 1};
static const int FJ1[9] = {0, 1, 0, 0, -1, -1, 0, 0, 1}, FJ2[9] = {0, 1, 1, -1, -1, -1, -1, 1, 1};
static const int FD1[9] = {0, 1, 2, 2, 1, 1, 2, 2, 1}, FD2[9] = {0, 2, 1, 1, 2, 2, 1, 1, 2};
static const float ANGC[9] = {0, 0., 1., 1., 2., 2., 3., 3., 4.}, ANGF[9] = {0, 1., -1., 1., -1., 1., -1., 1., -1.};

/* setFlow2: src/d8.cpp:412-454 */
static void set_flow2(flatctx* f, const int16_t* elev2, const int16_t* dn, int i, int j) {
  static const int order[8] = {1, 3, 5, 7, 2, 4, 6, 8};
  const int nx = f->nx;
  const double dx = f->dxc[j], dy = f->dyc[j];
  float smax = 0.f;
  for (int ii = 0; ii < 8; ii++) {
    const int k = order[ii];
    const size_t n = IDX(i + d1[k], j + d2[k]);
    if (dn[n] > 0) {
      const double fact = 1. / sqrt(d1[k] * d1[k] * dx * dx + d2[k] * d2[k] * dy * dy);
      const float slope = (float)(fact * (elev2[IDX(i, j)] - elev2[n]));
      if (slope > smax) { f->dir8[IDX(i, j)] = (int16_t)k; smax = slope; }
    } else {
      const float ed = f->elev[IDX(i, j)] - f->elev[n];
      if (ed >= 0) { f->dir8[IDX(i, j)] = (int16_t)k; break; }
    }
  }
}
/* flat SET2: src/dinf.cpp:375-528 */
static void set2_flat(flatctx* f, const int16_t* elev2, const int16_t* dn, int J /*col*/, int I /*row*/) {
  const int nx = f->nx;
  const double DXX[3] = {0, f->dxc[I], f->dyc[I]};
  const double DD = sqrt(DXX[1] * DXX[1] + DXX[2] * DXX[2]);
  double SK[9], ANGLE[9], SMAX = 0.0;
  int KD = 0, diag = 0;
  const size_t c0 = IDX(J, I);
  for (int K = 1; K <= 8; K++) {
    const size_t c1 = IDX(J + FJ1[K], I + FI1[K]), c2 = IDX(J + FJ2[K], I + FI2[K]);
    const int t1 = dn[c1], t2 = dn[c2];
    const double D1 = DXX[FD1[K]], D2 = DXX[FD2[K]];
    if (t1 <= 0 && t2 <= 0) {
      const double a = f->elev[c0], b = f->elev[c1], c = f->elev[c2];
      vslope(a, b, c, D1, D2, DD, &SK[K], &ANGLE[K]);
      if (SK[K] >= 0.0) {
        if (b > a) { if (!diag) { diag = 1; KD = K; } }
        else { KD = K; break; }
      }
    } else if (t1 <= 0 && t2 > 0) {
      const double a = f->elev[c0], b = f->elev[c1];
      if (a >= b) { ANGLE[K] = 0.0; SK[K] = 0.0; KD = K; break; }
      const int16_t a1 = elev2[c0], cc = elev2[c2], b1 = a1 > cc ? a1 : cc;
      vslope(a1, b1, cc, D1, D2, DD, &SK[K], &ANGLE[K]);
      if (SK[K] > SMAX) { SMAX = SK[K]; KD = K; }
    } else if (t1 > 0 && t2 <= 0) {
      const double a = f->elev[c0], c = f->elev[c2];
      if (a >= c) { if (!diag) { ANGLE[K] = atan2(D2, D1); SK[K] = 0.0; KD = K; diag = 1; } }
      else {
        const int16_t a1 = elev2[c0], b1 = elev2[c1], cc = a1 > b1 ? a1 : b1;
        vslope(a1, b1, cc, D1, D2, DD, &SK[K], &ANGLE[K]);
        if (SK[K] > SMAX) { SMAX = SK[K]; KD = K; }
      }
    } else {
      vslope(elev2[c0], elev2[c1], elev2[c2], D1, D2, DD, &SK[K], &ANGLE[K]);
      if (SK[K] > SMAX) { SMAX = SK[K]; KD = K; }
    }
  }
  if (!ndf(f->ang[c0], MISSINGFLOAT)) f->ang[c0] = -1.0f;
  if (KD > 0) {
    const float t = (float)(ANGC[KD] * (PI / 2) + ANGF[KD] * ANGLE[KD]);
    if (t >= 0.0f) f->ang[c0] = t;
  }
}

static long resolve_once(flatctx* f, int32_t* q, long nflat) {
  const int nx = f->nx, ny = f->ny;
  const size_t n = (size_t)nx * ny;
  int16_t* elev2 = (int16_t*)malloc(n * 2); int16_t* dn = (int16_t*)calloc(n, 2); int16_t* s = (int16_t*)calloc(n, 2);
  for (size_t c = 0; c < n; c++) elev2[c] = 1;
  /* incfall: src/d8.cpp:509-558 */
  long inc_old = -1, inc = 0; int st = 1;
  while (inc != inc_old) {
    inc_old = inc; inc = 0;
    for (long q0 = 0; q0 < nflat; q0++) {
      const int i = q[q0] % nx, j = q[q0] / nx;
      if (still_rising(f, elev2, i, j, st)) { elev2[q[q0]]++; inc++; }
    }
    st++;
  }
  if (inc > 0)   /* pits: src/d8.cpp:559-593 */
    for (long q0 = 0; q0 < nflat; q0++) {
      const int i = q[q0] % nx, j = q[q0] / nx;
      if (still_rising(f, elev2, i, j, st)) { if (f->dinf) f->ang[q[q0]] = MISSINGFLOAT; else f->dir8[q[q0]] = MISSINGSHORT; }
    }
  /* incrise: src/d8.cpp:595-638 */
  long marked_old = 0;
  for (;;) {
    for (long q0 = 0; q0 < nflat; q0++) {
      const int i = q[q0] % nx, j = q[q0] / nx;
      for (int k = 1; k <= 8; k++) {
        const size_t nb = IDX(i + d1[k], j + d2[k]);
        if (f->elev[q[q0]] - f->elev[nb] < 0) dn[q[q0]] = 1;
        if (dn[nb] > 0 && s[nb] > 0) dn[q[q0]] = 1;
      }
    }
    long marked = 0;
    for (size_t c = 0; c < n; c++) if (dn[c] > 0) { s[c]++; marked++; }
    if (marked == marked_old) break;
    marked_old = marked;
  }
  for (long q0 = 0; q0 < nflat; q0++) elev2[q[q0]] = (int16_t)(elev2[q[q0]] + s[q[q0]]);
  /* directions from the artificial surface; what is still flat stays in the queue */
  long left = 0;
  for (long q0 = 0; q0 < nflat; q0++) {
    const int i = q[q0] % nx, j = q[q0] / nx;
    if (f->dinf) { set2_flat(f, elev2, dn, i, j); if (!ndf(f->ang[q[q0]], MISSINGFLOAT) && f->ang[q[q0]] < 0.) q[left++] = q[q0]; }
    else { set_flow2(f, elev2, dn, i, j); if (f->dir8[q[q0]] == 0) q[left++] = q[q0]; }
  }
  if (left > 0) for (size_t c = 0; c < n; c++) f->elev[c] = (float)elev2[c];   /* src/d8.cpp:669-675 */
  free(elev2); free(dn); free(s);
  return left;
}

/* test hook: stop after the positive-slope stencil (the input state of the flat resolution) */
static int g_skip_flats = 0;
void orc_set_skip_flats(int v) { g_skip_flats = v; }

static void resolve_flats(flatctx* f) {
  const int nx = f->nx, ny = f->ny;
  if (g_skip_flats) return;
  int32_t* q = (int32_t*)malloc(sizeof(int32_t) * (size_t)nx * ny);
  long nflat = 0;
  for (int j = 0; j < ny; j++)
    for (int i = 0; i < nx; i++) {
      const size_t c = IDX(i, j);
      if (f->dinf ? (!ndf(f->ang[c], MISSINGFLOAT) && f->ang[c] < 0.0f) : f->dir8[c] == 0) q[nflat++] = (int32_t)c;
    }
  if (nflat > 0) {   /* outer loop: src/d8.cpp:302-317 */
    long last = nflat, left = resolve_once(f, q, nflat);
    while (left > 0 && left < last) { last = left; left = resolve_once(f, q, left); }
  }
  free(q);
}

/* ------------------------------------------------------------------------------------------------
 * d8flowdir: setPosDir + setFlow + calcSlope (src/d8.cpp:359-409, 103-150, 153-177), then flats.
 * ---------------------------------------------------------------------------------------------- */
int orc_d8(const float* fel, int16_t* p, float* sd8, int nx, int ny, float nodata, const double* dxc, const double* dyc) {
  static const int order[8] = {1, 3, 5, 7, 2, 4, 6, 8};
  for (int j = 0; j < ny; j++)
    for (int i = 0; i < nx; i++) {
      const size_t c = IDX(i, j);
      int bad = ndf(fel[c], nodata) || on_edge(i, j, nx, ny);
      for (int k = 1; k <= 8 && !bad; k++) bad = ndf(fel[IDX(i + d1[k], j + d2[k])], nodata);
      if (bad) { p[c] = MISSINGSHORT; sd8[c] = -1.0f; continue; }
      int dir = 0; float smax = 0.f;
      for (int ii = 0; ii < 8; ii++) {
        const int k = order[ii];
        const double fact = 1. / sqrt(d1[k] * d1[k] * dxc[j] * dxc[j] + d2[k] * d2[k] * dyc[j] * dyc[j]);
        const float slope = (float)(fact * (fel[c] - fel[IDX(i + d1[k], j + d2[k])]));
        if (slope > smax) { smax = slope; dir = k; }
      }
      p[c] = (int16_t)dir; sd8[c] = smax;
    }
  float* elev = (float*)malloc(sizeof(float) * (size_t)nx * ny);
  memcpy(elev, fel, sizeof(float) * (size_t)nx * ny);
  flatctx f = {nx, ny, 0, elev, p, NULL, dxc, dyc};
  resolve_flats(&f);
  free(elev);
  return 0;
}

/* dinfflowdir: setPosDirDinf + SET2 (src/dinf.cpp:530-595, 317-373), then flats. */
int orc_dinf(const float* fel, float* ang, float* slp, int nx, int ny, float nodata, const double* dxc, const double* dyc) {
  for (int j = 0; j < ny; j++)
    for (int i = 0; i < nx; i++) {
      const size_t c = IDX(i, j);
      int bad = ndf(fel[c], nodata) || on_edge(i, j, nx, ny);
      for (int k = 1; k <= 8 && !bad; k++) bad = ndf(fel[IDX(i + d1[k], j + d2[k])], nodata);
      if (bad) { ang[c] = MISSINGFLOAT; slp[c] = -1.0f; continue; }
      const double DXX[3] = {0, dxc[j], dyc[j]};
      const double DD = sqrt(DXX[1] * DXX[1] + DXX[2] * DXX[2]);
      double SK[9], ANGLE[9], SMAX = 0.; int KD = 0;
      for (int K = 1; K <= 8; K++)
        vslope(fel[c], fel[IDX(i + FJ1[K], j + FI1[K])], fel[IDX(i + FJ2[K], j + FI2[K])], DXX[FD1[K]], DXX[FD2[K]], DD, &SK[K], &ANGLE[K]);
      for (int K = 1; K <= 8; K++) if (SK[K] > SMAX) { SMAX = SK[K]; KD = K; }
      ang[c] = KD > 0 ? (float)(ANGC[KD] * (PI / 2) + ANGF[KD] * ANGLE[KD]) : -1.0f;
      slp[c] = (float)SMAX;
    }
  float* elev = (float*)malloc(sizeof(float) * (size_t)nx * ny);
  memcpy(elev, fel, sizeof(float) * (size_t)nx * ny);
  flatctx f = {nx, ny, 1, elev, NULL, ang, dxc, dyc};
  resolve_flats(&f);
  free(elev);
  return 0;
}

/* ------------------------------------------------------------------------------------------------
 * The D8 and D-infinity sweeps: dependency counts, then a FIFO queue of cells whose count is zero;
 * evaluate, decrement the receivers, push those that reach zero.  One count / drain pair per flow
 * model, shared by the tools of that model.
 * ---------------------------------------------------------------------------------------------- */
/* -o outlets (grid cells; n < 0 = none).  Set before any of the sweep tools below. */
static int g_nout = -1;
static const int32_t *g_ocol = NULL, *g_orow = NULL;
void orc_set_outlets(const int32_t* cols, const int32_t* rows, int n) { g_ocol = cols; g_orow = rows; g_nout = n; }

static int d8_drains_to(int16_t d, int k) { return d >= 0 && d <= 8 && (d - k == 4 || d - k == -4); }

/* initNeighborD8up (src/commonLib.cpp:240-385): nb = number of neighbours that drain into the cell, MISSINGSHORT where the
 * cell is not a node (direction nodata or outside 0..8; with outlets: not upstream of one).  Cells with no contributor go
 * to q; returns their number. */
static size_t d8_counts(const int16_t* p, int16_t* nb, int32_t* q, int nx, int ny, int16_t pnd) {
  const size_t n = (size_t)nx * ny;
  size_t qt = 0;
  if (g_nout >= 0) {
    /* outlets: src/commonLib.cpp:285-385 — a breadth-first walk up from the outlets */
    int32_t* tb = (int32_t*)malloc(n * 4 * 9);
    size_t th = 0, tt = 0;
    for (size_t c = 0; c < n; c++) nb[c] = MISSINGSHORT;
    for (int o = 0; o < g_nout; o++) if (INSIDE(g_ocol[o], g_orow[o])) tb[tt++] = (int32_t)IDX(g_ocol[o], g_orow[o]);
    while (th < tt) {
      const size_t c = tb[th++];
      const int i = c % nx, j = c / nx;
      if (nb[c] != MISSINGSHORT) continue;
      nb[c] = 0;
      for (int k = 1; k <= 8; k++) {
        const int in = i + d1[k], jn = j + d2[k];
        if (!INSIDE(in, jn) || nds(p[IDX(in, jn)], pnd)) continue;
        if (d8_drains_to(p[IDX(in, jn)], k)) { tb[tt++] = (int32_t)IDX(in, jn); nb[c]++; }
      }
      if (nb[c] == 0) q[qt++] = (int32_t)c;
    }
    free(tb);
    return qt;
  }
  for (int j = 0; j < ny; j++)
    for (int i = 0; i < nx; i++) {
      const size_t c = IDX(i, j);
      nb[c] = MISSINGSHORT;
      if (nds(p[c], pnd) || p[c] < 0 || p[c] > 8) continue;
      nb[c] = 0;
      for (int k = 1; k <= 8; k++) {
        const int in = i + d1[k], jn = j + d2[k];
        if (!INSIDE(in, jn) || nds(p[IDX(in, jn)], pnd)) continue;
        if (d8_drains_to(p[IDX(in, jn)], k)) nb[c]++;
      }
      if (nb[c] == 0) q[qt++] = (int32_t)c;
    }
  return qt;
}
/* the receiver of an evaluated D8 cell loses a dependency (src/aread8.cpp:261-272) */
static void d8_drain(const int16_t* p, int16_t* nb, int32_t* q, size_t* qt, int nx, int ny, size_t c) {
  const int i = c % nx, j = c / nx, k = p[c];
  if (k < 1 || k > 8) return;
  const int in = i + d1[k], jn = j + d2[k];
  if (INSIDE(in, jn) && nb[IDX(in, jn)] != MISSINGSHORT) { nb[IDX(in, jn)]--; if (nb[IDX(in, jn)] == 0) q[(*qt)++] = (int32_t)IDX(in, jn); }
}

/* aread8: the evaluation loop of src/aread8.cpp:216-304. */
int orc_aread8(const int16_t* p, const float* w, float* ad8, int nx, int ny, int16_t pnd, float wnd, int usew, int contcheck) {
  const size_t n = (size_t)nx * ny;
  int16_t* nb = (int16_t*)malloc(n * 2);
  int32_t* q = (int32_t*)malloc(n * 4);
  size_t qh = 0, qt;
  for (size_t c = 0; c < n; c++) ad8[c] = -1.0f;
  qt = d8_counts(p, nb, q, nx, ny, pnd);
  while (qh < qt) {
    const size_t c = q[qh++];
    const int i = c % nx, j = c / nx;
    int con = 0;
    if (usew) { if (!ndf(w[c], wnd)) ad8[c] = w[c]; } else ad8[c] = 1.0f;
    for (int k = 1; k <= 8; k++) {
      const int in = i + d1[k], jn = j + d2[k];
      if (!INSIDE(in, jn) || nds(p[IDX(in, jn)], pnd)) { con = 1; continue; }
      const int16_t d = p[IDX(in, jn)];
      if (d - k == 4 || d - k == -4) { if (ndf(ad8[IDX(in, jn)], -1.0f)) con = 1; else ad8[c] = ad8[c] + ad8[IDX(in, jn)]; }
    }
    if (con && contcheck) ad8[c] = -1.0f;
    d8_drain(p, nb, q, &qt, nx, ny, c);
  }
  free(nb); free(q);
  return 0;
}

/* d8flowpathextremeup: the evaluation loop of src/D8flowpathextremeup.cpp:172-228.  The cell starts from its own sa value
 * (nodata or not) and takes the largest (usemax) / smallest ssa of the neighbours that drain into it; a neighbour outside the
 * grid or with a nodata direction, or a contributor whose ssa is nodata, contaminates.  nodata = MISSINGFLOAT. */
int orc_flowpathextremeup(const int16_t* p, const float* sa, float* ssa, int nx, int ny, int16_t pnd, int usemax, int contcheck) {
  const size_t n = (size_t)nx * ny;
  int16_t* nb = (int16_t*)malloc(n * 2);
  int32_t* q = (int32_t*)malloc(n * 4);
  size_t qh = 0, qt;
  for (size_t c = 0; c < n; c++) ssa[c] = MISSINGFLOAT;
  qt = d8_counts(p, nb, q, nx, ny, pnd);
  while (qh < qt) {
    const size_t c = q[qh++];
    const int i = c % nx, j = c / nx;
    int con = 0;
    ssa[c] = sa[c];
    for (int k = 1; k <= 8; k++) {
      const int in = i + d1[k], jn = j + d2[k];
      if (!INSIDE(in, jn) || nds(p[IDX(in, jn)], pnd)) { con = 1; continue; }
      const int16_t d = p[IDX(in, jn)];
      if (d - k == 4 || d - k == -4) {
        const float v = ssa[IDX(in, jn)];
        if (ndf(v, MISSINGFLOAT)) con = 1;
        else if (usemax ? v > ssa[c] : v < ssa[c]) ssa[c] = v;
      }
    }
    if (con && contcheck) ssa[c] = MISSINGFLOAT;
    d8_drain(p, nb, q, &qt, nx, ny, c);
  }
  free(nb); free(q);
  return 0;
}

/* gridnet: src/gridnet.cpp:193-209 (float distances per row), 226-374 (start values, counts), 378-445 (evaluation).
 * mask == NULL: every cell is inside (the reference's mask of ones with threshold 0).  gord starts at 1 on data cells inside
 * the mask (with outlets: 1 on the cells upstream of an outlet, 0 on the other data cells).  A cell inside the mask
 * (mask >= thresh) is evaluated from the neighbours inside the mask whose direction 1..8 points at it, with dist[] of the
 * RECEIVING row: plen = max(plen + dist), tlen = sum(tlen + dist) in float, gord = Strahler order (a tie of the two largest
 * orders raises it).  nodata: plen / tlen -1, gord -1.
 * Where gridnet.cpp reads past its arrays the restatement keeps to the D8 tools' graph: counts as initNeighborD8up (codes
 * outside 0..8 are not nodes; the reference would index d1[] / d2[] with them), neighbours outside the grid never contribute
 * (the reference would compare a stale direction there). */
int orc_gridnet(const int16_t* p, const int32_t* mask, int thresh, float* plen, float* tlen, int16_t* gord, int nx, int ny, int16_t pnd,
                const double* dxc, const double* dyc) {
  const size_t n = (size_t)nx * ny;
  int16_t* nb = (int16_t*)malloc(n * 2);
  int32_t* q = (int32_t*)malloc(n * 4);
  float* dist = (float*)malloc(sizeof(float) * 9 * (size_t)ny);
  size_t qh = 0, qt;
  const int thr = mask ? thresh : 0;
#define MSK(c) (mask ? mask[c] : 1)
  for (int m = 0; m < ny; m++)
    for (int k = 1; k <= 8; k++) dist[m * 9 + k] = (float)sqrt(dxc[m] * dxc[m] * d1[k] * d1[k] + dyc[m] * dyc[m] * d2[k] * d2[k]);
  qt = d8_counts(p, nb, q, nx, ny, pnd);
  for (size_t c = 0; c < n; c++) {
    plen[c] = -1.0f; tlen[c] = -1.0f; gord[c] = -1;
    if (g_nout >= 0) { if (nb[c] != MISSINGSHORT) gord[c] = 1; else if (!nds(p[c], pnd)) gord[c] = 0; }
    else if (!nds(p[c], pnd) && MSK(c) >= thr) gord[c] = 1;
    if (nds(p[c], pnd)) nb[c] = MISSINGSHORT;   /* nothing drains into a nodata cell (src/gridnet.cpp:434): an outlet there is evaluated only
                                                   if nothing drains towards it */
  }
  while (qh < qt) {
    const size_t c = q[qh++];
    const int i = c % nx, j = c / nx;
    if (MSK(c) >= thr) {
      int16_t a1 = 0, a2 = 0;
      plen[c] = 0.0f; tlen[c] = 0.0f;
      for (int k = 1; k <= 8; k++) {
        const int in = i + d1[k], jn = j + d2[k];
        if (!INSIDE(in, jn)) continue;
        const size_t cn = IDX(in, jn);
        const int16_t sdir = p[cn];
        if (sdir < 1 || sdir > 8 || nds(sdir, pnd) || MSK(cn) < thr || !(sdir - k == 4 || sdir - k == -4)) continue;
        if (gord[cn] >= a1) { a2 = a1; a1 = gord[cn]; }
        else if (gord[cn] > a2) a2 = gord[cn];
        const float ld = plen[cn] + dist[j * 9 + sdir];
        tlen[c] = tlen[c] + (float)(tlen[cn] + dist[j * 9 + sdir]);
        if (ld > plen[c]) plen[c] = ld;
      }
      gord[c] = (int16_t)(a2 + 1 > a1 ? a2 + 1 : a1);
    }
    d8_drain(p, nb, q, &qt, nx, ny, c);
  }
#undef MSK
  free(nb); free(q); free(dist);
  return 0;
}

/* prop: src/commonLib.cpp:76-91 */
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

/* initNeighborDinfup (src/commonLib.cpp:92-237): as d8_counts, a contributor being a neighbour whose angle sends a share
 * prop(angle, direction to me) > 0, with the contributor's row cell sizes. */
static size_t dinf_counts(const float* ang, int16_t* nb, int32_t* q, int nx, int ny, float and_, const double* dxc, const double* dyc) {
  const size_t n = (size_t)nx * ny;
  size_t qt = 0;
  if (g_nout >= 0) {
    /* outlets: src/commonLib.cpp:137-237 */
    int32_t* tb = (int32_t*)malloc(n * 4 * 9);
    size_t th = 0, tt = 0;
    for (size_t c = 0; c < n; c++) nb[c] = MISSINGSHORT;
    for (int o = 0; o < g_nout; o++) if (INSIDE(g_ocol[o], g_orow[o])) tb[tt++] = (int32_t)IDX(g_ocol[o], g_orow[o]);
    while (th < tt) {
      const size_t c = tb[th++];
      const int i = c % nx, j = c / nx;
      if (nb[c] != MISSINGSHORT) continue;
      nb[c] = 0;
      for (int k = 1; k <= 8; k++) {
        const int in = i + d1[k], jn = j + d2[k];
        if (!INSIDE(in, jn) || ndf(ang[IDX(in, jn)], and_)) continue;
        const float pf = (float)prop(ang[IDX(in, jn)], (k + 4) % 8, dxc[jn], dyc[jn]);
        if (pf > 0.0) { tb[tt++] = (int32_t)IDX(in, jn); nb[c]++; }
      }
      if (nb[c] == 0) q[qt++] = (int32_t)c;
    }
    free(tb);
    return qt;
  }
  for (int j = 0; j < ny; j++)
    for (int i = 0; i < nx; i++) {
      const size_t c = IDX(i, j);
      nb[c] = MISSINGSHORT;
      if (ndf(ang[c], and_)) continue;
      nb[c] = 0;
      for (int k = 1; k <= 8; k++) {
        const int in = i + d1[k], jn = j + d2[k];
        if (!INSIDE(in, jn) || ndf(ang[IDX(in, jn)], and_)) continue;
        const float pf = (float)prop(ang[IDX(in, jn)], (k + 4) % 8, dxc[jn], dyc[jn]);
        if (pf > 0.0) nb[c]++;
      }
      if (nb[c] == 0) q[qt++] = (int32_t)c;
    }
  return qt;
}
/* the receivers of an evaluated D-infinity cell lose a dependency (src/areadinf.cpp:221-239): its own row's cell sizes */
static void dinf_drain(const float* ang, int16_t* nb, int32_t* q, size_t* qt, int nx, int ny, size_t c, const double* dxc, const double* dyc) {
  const int i = c % nx, j = c / nx;
  for (int k = 1; k <= 8; k++)
    if (prop(ang[c], k, dxc[j], dyc[j]) > 0.0) {
      const int in = i + d1[k], jn = j + d2[k];
      if (INSIDE(in, jn) && nb[IDX(in, jn)] != MISSINGSHORT) { nb[IDX(in, jn)]--; if (nb[IDX(in, jn)] == 0) q[(*qt)++] = (int32_t)IDX(in, jn); }
    }
}
/* share that the contributor in direction k of cell (i, j) sends to the cell: > 0 if it contributes, -1 if it does not, -2 if it
 * is outside the grid or its angle is nodata (contamination) */
static double dinf_share(const float* ang, int nx, int ny, int i, int j, int k, float and_, const double* dxc, const double* dyc) {
  const int in = i + d1[k], jn = j + d2[k];
  if (!INSIDE(in, jn) || ndf(ang[IDX(in, jn)], and_)) return -2.0;
  return prop(ang[IDX(in, jn)], (k + 4) % 8, dxc[jn], dyc[jn]);
}

/* areadinf: the area() loop of src/areadinf.cpp:173-265. */
int orc_areadinf(const float* ang, const float* w, float* sca, int nx, int ny, float and_, int usew, int contcheck, const double* dxc,
                 const double* dyc) {
  const size_t n = (size_t)nx * ny;
  int16_t* nb = (int16_t*)malloc(n * 2);
  int32_t* q = (int32_t*)malloc(n * 4);
  size_t qh = 0, qt;
  for (size_t c = 0; c < n; c++) sca[c] = -1.0f;
  qt = dinf_counts(ang, nb, q, nx, ny, and_, dxc, dyc);
  while (qh < qt) {
    const size_t c = q[qh++];
    const int i = c % nx, j = c / nx;
    float areares = 0.f; int con = 0;
    for (int k = 1; k <= 8; k++) {
      const double pr = dinf_share(ang, nx, ny, i, j, k, and_, dxc, dyc);
      const size_t cn = IDX(i + d1[k], j + d2[k]);
      if (pr == -2.0) con = 1;
      else if (pr > 0.0) { if (ndf(sca[cn], -1.0f)) con = 1; else areares = (float)(areares + pr * sca[cn]); }
    }
    if (usew) areares = areares + w[c]; else areares = (float)(areares + dxc[j]);
    sca[c] = (con && contcheck) ? -1.0f : areares;
    dinf_drain(ang, nb, q, &qt, nx, ny, c, dxc, dyc);
  }
  free(nb); free(q);
  return 0;
}

/* dinfdecayaccum: the evaluation loop of src/dinfdecayaccum.cpp:203-258.  The cell starts from its weight (nodata or not) or its
 * row's dx, then adds (float)(dm * area * p) per contributor in increasing k — dm * area in float, times the double share.
 * A contributor whose result or decay multiplier is nodata contaminates.  nodata = MISSINGFLOAT. */
int orc_dinfdecayaccum(const float* ang, const float* dm, const float* w, float* dsca, int nx, int ny, float and_, float dmnd, int usew, int contcheck,
                       const double* dxc, const double* dyc) {
  const size_t n = (size_t)nx * ny;
  int16_t* nb = (int16_t*)malloc(n * 2);
  int32_t* q = (int32_t*)malloc(n * 4);
  size_t qh = 0, qt;
  for (size_t c = 0; c < n; c++) dsca[c] = MISSINGFLOAT;
  qt = dinf_counts(ang, nb, q, nx, ny, and_, dxc, dyc);
  while (qh < qt) {
    const size_t c = q[qh++];
    const int i = c % nx, j = c / nx;
    int con = 0;
    dsca[c] = usew ? w[c] : (float)dxc[j];
    for (int k = 1; k <= 8; k++) {
      const double pr = dinf_share(ang, nx, ny, i, j, k, and_, dxc, dyc);
      const size_t cn = IDX(i + d1[k], j + d2[k]);
      if (pr == -2.0) con = 1;
      else if (pr > 0.0) {
        if (ndf(dsca[cn], MISSINGFLOAT) || ndf(dm[cn], dmnd)) con = 1;
        else { const float da = dm[cn] * dsca[cn]; dsca[c] = dsca[c] + (float)(da * pr); }
      }
    }
    if (con && contcheck) dsca[c] = MISSINGFLOAT;
    dinf_drain(ang, nb, q, &qt, nx, ny, c, dxc, dyc);
  }
  free(nb); free(q);
  return 0;
}

/* DinfConcLimAccum: the evaluation loop of src/DinfConcLimAccum.cpp:226-287.  Only cells with q > 0 are evaluated (the others
 * are nodata); an indicator cell (dg > 0) has the concentration csol and is never contaminated; any other cell the float sum,
 * in increasing k, of p * ctpt * q * dm (double products) over its contributors, divided by its own q.  A contributor whose
 * ctpt, dm or q is nodata contaminates.  nodata = MISSINGFLOAT. */
int orc_dinfconclimaccum(const float* ang, const float* dm, const float* qv, const int16_t* dg, float* ctpt, int nx, int ny, float and_, float dmnd,
                         float qnd, float csol, int contcheck, const double* dxc, const double* dyc) {
  const size_t n = (size_t)nx * ny;
  int16_t* nb = (int16_t*)malloc(n * 2);
  int32_t* q = (int32_t*)malloc(n * 4);
  size_t qh = 0, qt;
  for (size_t c = 0; c < n; c++) ctpt[c] = MISSINGFLOAT;
  qt = dinf_counts(ang, nb, q, nx, ny, and_, dxc, dyc);
  while (qh < qt) {
    const size_t c = q[qh++];
    const int i = c % nx, j = c / nx;
    if (qv[c] > 0.) {
      int con = 0;
      if (dg[c] > 0) ctpt[c] = csol;
      else {
        float conc = 0.0f;
        for (int k = 1; k <= 8; k++) {
          const double pr = dinf_share(ang, nx, ny, i, j, k, and_, dxc, dyc);
          const size_t cn = IDX(i + d1[k], j + d2[k]);
          if (pr == -2.0) con = 1;
          else if (pr > 0.0) {
            if (ndf(ctpt[cn], MISSINGFLOAT) || ndf(dm[cn], dmnd) || ndf(qv[cn], qnd)) con = 1;
            else conc = (float)(conc + pr * ctpt[cn] * qv[cn] * dm[cn]);
          }
        }
        ctpt[c] = conc / qv[c];
      }
      if (con && contcheck) ctpt[c] = MISSINGFLOAT;
    }
    dinf_drain(ang, nb, q, &qt, nx, ny, c, dxc, dyc);
  }
  free(nb); free(q);
  return 0;
}

/* DinfTransLimAccum: the evaluation loop of src/DinfTransLimAccum.cpp:226-311.  Cells whose supply or capacity (or, with cs,
 * supply concentration) is nodata are not evaluated.  transin = float sum of p * tla over the contributors in increasing k;
 * the transport out is min(transin + supply, capacity), the rest is deposited.  With cs: loadin = float sum of p * tla * ctpt
 * (a contributor whose tla is nodata carries no load), and ctpt = loadout / transout (0 without transport).  A contributor
 * whose tla (or ctpt) is nodata contaminates: all outputs of the cell are nodata then.  nodata = MISSINGFLOAT. */
int orc_dinftranslimaccum(const float* ang, const float* tsup, const float* tc, const float* cs, float* tla, float* tdep, float* ctpt, int nx, int ny,
                          float and_, float tsnd, float tcnd, float csnd, int contcheck, const double* dxc, const double* dyc) {
  const size_t n = (size_t)nx * ny;
  int16_t* nb = (int16_t*)malloc(n * 2);
  int32_t* q = (int32_t*)malloc(n * 4);
  size_t qh = 0, qt;
  for (size_t c = 0; c < n; c++) { tla[c] = MISSINGFLOAT; tdep[c] = MISSINGFLOAT; if (cs) ctpt[c] = MISSINGFLOAT; }
  qt = dinf_counts(ang, nb, q, nx, ny, and_, dxc, dyc);
  while (qh < qt) {
    const size_t c = q[qh++];
    const int i = c % nx, j = c / nx;
    if (!ndf(tsup[c], tsnd) && !ndf(tc[c], tcnd) && (!cs || !ndf(cs[c], csnd))) {
      float transin = 0.f, loadin = 0.f, transout, depp;
      int con = 0;
      for (int k = 1; k <= 8; k++) {
        const double pr = dinf_share(ang, nx, ny, i, j, k, and_, dxc, dyc);
        const size_t cn = IDX(i + d1[k], j + d2[k]);
        if (pr == -2.0) con = 1;
        else if (pr > 0.0) {
          float nt = 0.0f;
          if (ndf(tla[cn], MISSINGFLOAT)) con = 1; else { nt = tla[cn]; transin = (float)(transin + pr * nt); }
          if (cs) { if (ndf(ctpt[cn], MISSINGFLOAT)) con = 1; else loadin = (float)(loadin + pr * nt * ctpt[cn]); }
        }
      }
      if ((transin + tsup[c]) > tc[c]) { transout = tc[c]; depp = transin + tsup[c] - transout; }
      else { transout = transin + tsup[c]; depp = 0.f; }
      tla[c] = transout; tdep[c] = depp;
      if (cs) {
        float loadout;
        if (transout < transin) loadout = transin > 0 ? loadin * transout / transin : 0.f;
        else loadout = loadin + cs[c] * (transout - transin);
        ctpt[c] = transout > 0. ? (float)(loadout / transout) : 0.0f;
      }
      if (con && contcheck) { tdep[c] = MISSINGFLOAT; tla[c] = MISSINGFLOAT; if (cs) ctpt[c] = MISSINGFLOAT; }
    }
    dinf_drain(ang, nb, q, &qt, nx, ny, c, dxc, dyc);
  }
  free(nb); free(q);
  return 0;
}
