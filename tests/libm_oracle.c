// TEST INFRASTRUCTURE ONLY — the host libm's logf / powf, a correctly rounded float log / power, and the reference's slopearea
// product and lengtharea decision, over whole arrays and over ranges of float bit patterns, on all cores (pthreads).  Built by
// tests/libm_oracle.py with the system C compiler (-O2 -ffp-contract=off) and loaded with ctypes; the point-wise tests compare the
// kernels with it cell by cell, and the whole-float sweeps need its speed (2^31 inputs in seconds).
//
// The correctly rounded value: the double log / pow rounded to float, except where the double lies within a few double ulps of a
// float midpoint (or beyond the float range): there logl / powl (64-bit significand) rounded once to float decides.
#include <float.h>
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <string.h>
#include <unistd.h>

static float asf(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static uint32_t asu(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

// d rounds to a float unambiguously: it is finite, inside the float range, and more than 8 double ulps away from both midpoints
// around (float)d; beyond the float range it must be clear of the overflow threshold FLT_MAX + half an ulp (= 2^128 - 2^103)
static int clear_of_midpoints(double d) {
  if (!isfinite(d)) return 0;
  if (fabs(d) > (double)FLT_MAX) return fabs(d) > 0x1p128;
  const float f = (float)d;
  const double lo = 0.5 * ((double)f + (double)nextafterf(f, -INFINITY)), hi = 0.5 * ((double)f + (double)nextafterf(f, INFINITY));
  const double tol = 8.0 * fmax(fabs(d) * 0x1p-52, 0x1p-1074);
  return fabs(d - lo) > tol && fabs(d - hi) > tol;
}
static float cr_log(float x) {
  const double d = log((double)x);
  return clear_of_midpoints(d) || !isfinite(d) ? (float)d : (float)logl((long double)x);
}
static float cr_pow(float x, float e) {
  const double d = pow((double)x, (double)e);
  if (clear_of_midpoints(d)) return (float)d;
  return (float)powl((long double)x, (long double)e);
}

// ---- a parallel loop over [0, n)
typedef void (*body_fn)(void* arg, long i0, long i1, int t);
struct job { body_fn f; void* arg; long n; int t, nt; };
static void* run_job(void* p) {
  struct job* j = (struct job*)p;
  const long a = j->n * j->t / j->nt, b = j->n * (j->t + 1) / j->nt;
  j->f(j->arg, a, b, j->t);
  return NULL;
}
enum { MAXT = 64 };
static int nthreads(void) {
  const long c = sysconf(_SC_NPROCESSORS_ONLN);
  return c < 1 ? 1 : c > MAXT ? MAXT : (int)c;
}
static void parallel(body_fn f, void* arg, long n) {
  const int nt = n < 65536 ? 1 : nthreads();
  pthread_t th[MAXT];
  struct job jobs[MAXT];
  for (int t = 0; t < nt; ++t) {
    jobs[t] = (struct job){f, arg, n, t, nt};
    if (t > 0) pthread_create(&th[t], NULL, run_job, &jobs[t]);
  }
  run_job(&jobs[0]);
  for (int t = 1; t < nt; ++t) pthread_join(th[t], NULL);
}

// ---- element-wise
struct ew { const float *x, *y; const int* a; float e, m; float* out; short* s; int which; };
static void ew_body(void* p, long i0, long i1, int t) {
  (void)t;
  const struct ew* w = (const struct ew*)p;
  for (long i = i0; i < i1; ++i) switch (w->which) {
      case 0: w->out[i] = logf(w->x[i]); break;
      case 1: w->out[i] = powf(w->x[i], w->e); break;
      case 2: w->out[i] = cr_log(w->x[i]); break;
      case 3: w->out[i] = cr_pow(w->x[i], w->e); break;
      case 4: w->out[i] = powf(w->x[i], w->m) * powf(w->y[i], w->e); break;             // slp^m * sca^n, two floats
      case 5: w->s[i] = w->x[i] >= 0.0f ? (short)((float)w->a[i] >= w->m * powf(w->x[i], w->e) ? 1 : 0) : (short)-32768; break;
    }
}
void lo_logf(const float* x, float* out, long n) { struct ew w = {x, 0, 0, 0, 0, out, 0, 0}; parallel(ew_body, &w, n); }
void lo_powf(const float* x, float e, float* out, long n) { struct ew w = {x, 0, 0, e, 0, out, 0, 1}; parallel(ew_body, &w, n); }
void lo_log_cr(const float* x, float* out, long n) { struct ew w = {x, 0, 0, 0, 0, out, 0, 2}; parallel(ew_body, &w, n); }
void lo_pow_cr(const float* x, float e, float* out, long n) { struct ew w = {x, 0, 0, e, 0, out, 0, 3}; parallel(ew_body, &w, n); }
// the reference's slopearea product powf(slp, m) * powf(sca, n) (no nodata test: the caller masks)
void lo_slopearea(const float* slp, const float* sca, float m, float n, float* out, long cnt) {
  struct ew w = {slp, sca, 0, n, m, out, 0, 4};
  parallel(ew_body, &w, cnt);
}
// the reference's lengtharea cell: (float)ad8 >= M * powf(plen, y) ? 1 : 0 where plen >= 0, else -32768
void lo_lengtharea(const float* plen, const int* ad8, float m, float y, short* out, long n) {
  struct ew w = {plen, 0, ad8, y, m, 0, out, 5};
  parallel(ew_body, &w, n);
}

// ---- sweeps over float bit patterns [u0, u0 + n)
// Compares a kernel's results gpu[i] for x = asf(u0 + i) (which 0: log x, 1: x^e) with libm and the correctly rounded value.
// cnt[0] = cells where gpu differs from libm, cnt[1] = inputs where libm is not correctly rounded, cnt[2] = cells where gpu is
// not correctly rounded, cnt[3] = cells where exactly one of the first two holds.  The first `cap` cells of the last two kinds go
// to bad[] (as bit patterns).
struct sweep { int which; float e; uint32_t u0; const float* gpu; long long cnt[MAXT][4]; uint32_t* bad; long cap; long nbad; pthread_mutex_t mu; };
static void sweep_body(void* p, long i0, long i1, int t) {
  struct sweep* s = (struct sweep*)p;
  long long c[4] = {0, 0, 0, 0};
  for (long i = i0; i < i1; ++i) {
    const float x = asf(s->u0 + (uint32_t)i);
    const float lib = s->which == 0 ? logf(x) : powf(x, s->e), cr = s->which == 0 ? cr_log(x) : cr_pow(x, s->e);
    const uint32_t g = asu(s->gpu ? s->gpu[i] : cr);
    const int d = g != asu(lib), b = asu(lib) != asu(cr), w = g != asu(cr);
    c[0] += d; c[1] += b; c[2] += w; c[3] += d != b;
    if (w || d != b) {
      pthread_mutex_lock(&s->mu);
      if (s->nbad < s->cap) s->bad[s->nbad] = s->u0 + (uint32_t)i;
      ++s->nbad;
      pthread_mutex_unlock(&s->mu);
    }
  }
  memcpy(s->cnt[t], c, sizeof c);
}
// returns the number of cells of the last two kinds; gpu = NULL compares libm with the correctly rounded value only
long lo_sweep(int which, float e, uint32_t u0, const float* gpu, long n, long long* cnt, uint32_t* bad, long cap) {
  static struct sweep s;
  memset(&s, 0, sizeof s);
  s.which = which; s.e = e; s.u0 = u0; s.gpu = gpu; s.bad = bad; s.cap = cap;
  pthread_mutex_init(&s.mu, NULL);
  parallel(sweep_body, &s, n);
  for (int k = 0; k < 4; ++k) {
    cnt[k] = 0;
    for (int t = 0; t < MAXT; ++t) cnt[k] += s.cnt[t][k];
  }
  pthread_mutex_destroy(&s.mu);
  return s.nbad;
}

// libm's powf is faithful at exponent e on [u0, u0 + n): it is the correctly rounded value or the float on the other side of the
// exact power.  Returns the number of inputs where it is neither; the first `cap` go to bad[].
struct faith { float e; uint32_t u0; long long cnt[MAXT]; uint32_t* bad; long cap; long nbad; pthread_mutex_t mu; };
static void faith_body(void* p, long i0, long i1, int t) {
  struct faith* s = (struct faith*)p;
  long long c = 0;
  for (long i = i0; i < i1; ++i) {
    const float x = asf(s->u0 + (uint32_t)i), lib = powf(x, s->e), cr = cr_pow(x, s->e);
    if (asu(lib) == asu(cr)) continue;
    const long double exact = powl((long double)x, (long double)s->e);
    const int ok = ((long double)cr < exact && lib == nextafterf(cr, INFINITY)) || ((long double)cr > exact && lib == nextafterf(cr, -INFINITY));
    if (ok) continue;
    ++c;
    pthread_mutex_lock(&s->mu);
    if (s->nbad < s->cap) s->bad[s->nbad] = s->u0 + (uint32_t)i;
    ++s->nbad;
    pthread_mutex_unlock(&s->mu);
  }
  s->cnt[t] = c;
}
long lo_powf_unfaithful(float e, uint32_t u0, long n, uint32_t* bad, long cap) {
  static struct faith s;
  memset(&s, 0, sizeof s);
  s.e = e; s.u0 = u0; s.bad = bad; s.cap = cap;
  pthread_mutex_init(&s.mu, NULL);
  parallel(faith_body, &s, n);
  pthread_mutex_destroy(&s.mu);
  return s.nbad;
}

// lengtharea cells whose decision depends on the last bit of the power: plen = asf(u0 + i) and an integer ad8 < 2^31 that
// (float)ad8 >= M * p decides differently for p = libm's powf and p = the correctly rounded power.  Writes up to cap pairs,
// returns how many exist in the range.
struct flips { float m, y; uint32_t u0; float* plen; int* ad8; long cap; long n; pthread_mutex_t mu; };
static void flips_body(void* p, long i0, long i1, int t) {
  (void)t;
  struct flips* s = (struct flips*)p;
  for (long i = i0; i < i1; ++i) {
    const float x = asf(s->u0 + (uint32_t)i), r = powf(x, s->y);
    const float g = cr_pow(x, s->y);
    if (asu(r) == asu(g)) continue;
    const float tr = s->m * r, tg = s->m * g;
    if (!(tr != tg) || !isfinite(tr) || !isfinite(tg)) continue;
    const float k = ceilf(fminf(tr, tg));
    if (!(k <= fmaxf(tr, tg)) || !(k < 2147483648.0f) || !(k > -2147483648.0f) || (k >= tr) == (k >= tg)) continue;
    pthread_mutex_lock(&s->mu);
    if (s->n < s->cap) { s->plen[s->n] = x; s->ad8[s->n] = (int)k; }
    ++s->n;
    pthread_mutex_unlock(&s->mu);
  }
}
long lo_lengtharea_flips(float m, float y, uint32_t u0, long n, float* plen, int* ad8, long cap) {
  static struct flips s;
  memset(&s, 0, sizeof s);
  s.m = m; s.y = y; s.u0 = u0; s.plen = plen; s.ad8 = ad8; s.cap = cap;
  pthread_mutex_init(&s.mu, NULL);
  parallel(flips_body, &s, n);
  pthread_mutex_destroy(&s.mu);
  return s.n;
}
