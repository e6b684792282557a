// Garbrecht-Martz flat resolution for D8 and D-infinity, as breadth-first searches.
//
// reference: D8   resolveflats src/d8.cpp:459-680,  setFlow2 :412-454, dontCross :54-100,
//                 outer loop src/d8.cpp:302-317
//            Dinf resolveflats src/dinf.cpp:598-833, flat SET2 :375-528, dontCross :58-105
//
// The reference sweeps a queue of flat cells repeatedly (one pass per unit of
// artificial elevation).  Its passes are order independent (SURVEY.md A.4), so each
// of the two gradients is a multi-source BFS over the flat cells F:
//   fall: level(c) = 1 if c has a lower-or-equal draining neighbour (not crossing),
//         2 if it has an equal neighbour outside F, else 1 + min level over equal
//         neighbours in F; elev2 = level, or 1+T for cells never reached (pits),
//         T = number of reference passes = first t >= 2 with no cell at level t
//         (T = 1 when every flat cell is at level 1);
//   rise: m(c) = 1 if a neighbour is strictly higher, else 1 + min m over marked
//         neighbours in F; s = U - m + 1 with U = first pass that marks nothing.
// elev2 += s; then directions are set per flat cell from elev2/dn (setFlow2 / SET2),
// the still-flat cells form the next F, and the whole DEM is overwritten by
// (float)elev2 before the next outer iteration — all exactly as the reference does.
// Frontiers are int64 cell-index lists appended with warp-aggregated atomics; one
// kernel launch per BFS level, total work O(|F|).
//
// Row strips (one per process, src/linearpart.h): every strip runs the same loop on its own flat cells; the
// caller supplies three callbacks (td_strip_comm: share edge rows, collect halo rows, all-reduce) that stand
// where the reference calls share()/MPI_Allreduce in resolveflats.  A BFS level may claim a cell of the
// neighbour strip: the claim is made on the local halo copy of lev / mk, sent to the owner and merged there
// (k_merge appends the cell to the owner's frontier; a claim on a cell the owner has already assigned is ignored), so that the
// levels — and with them T, U and every elev2 — are those of the undivided grid.
#include <stdlib.h>

#include <algorithm>
#include <vector>

#include "ctx.h"
#include "dinf_common.cuh"

namespace td {
namespace {

constexpr int UNASSIGNED = 0x7fffffff;
constexpr int MAXPASS = 32767;          // fall / rise passes at which the reference's short pass counter wraps

struct D8Pol {
  using DirT = short;
  __device__ static bool drains(short d) { return d > 0 && d < 9; }
  __device__ static bool is_flat(short d) { return d == 0; }
  __device__ static bool eqc(short d, int c) { return (int)d == c; }
  __device__ static short pit() { return TD_MISSINGSHORT; }
};
struct DinfPol {
  using DirT = float;
  __device__ static bool drains(float a) { return a >= 0.0f; }
  __device__ static bool is_flat(float a) { return !nd_f(a, TD_MISSINGFLOAT) && a < 0.0f; }
  __device__ static bool eqc(float a, int c) { return a == (float)c; }
  __device__ static float pit() { return TD_MISSINGFLOAT; }
};

__device__ __forceinline__ void append(long long* list, unsigned long long* ctr, bool pred, long long v) {
  const unsigned m = __ballot_sync(__activemask(), pred);
  if (!pred) return;
  const int lane = threadIdx.x & 31;
  const int leader = __ffs(m) - 1;
  unsigned long long base = 0;
  if (lane == leader) base = atomicAdd(ctr, (unsigned long long)__popc(m));
  base = __shfl_sync(m, base, leader);
  if (list) list[base + __popc(m & ((1u << lane) - 1u))] = v;     // list == NULL: counting pass
}

template <class P>
__global__ void k_collect(const typename P::DirT* __restrict__ dir, Strip s, long long* __restrict__ list,
                          unsigned long long* __restrict__ ctr) {
  const int c = blockIdx.y * blockDim.x + threadIdx.x, r = 1 + blockIdx.x;   // rows on grid.x (no 65535 limit)
  const bool in = c < s.nx;
  const long long ci = s.idx(r, in ? c : 0);
  append(list, ctr, in && P::is_flat(dir[ci]), ci);
}

__global__ void k_mark(const long long* __restrict__ list, unsigned long long n, int* __restrict__ lev) {
  const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n) lev[list[t]] = UNASSIGNED;
}

// dontCross for direction k at cell ci (needs the directions of the four cardinal neighbours)
template <class P>
__device__ __forceinline__ bool dont_cross(const typename P::DirT* __restrict__ dir, long long ci, int pitch, int k) {
  switch (k) {
    case 2: return P::eqc(dir[ci + 1], 4) || P::eqc(dir[ci - pitch], 8);
    case 4: return P::eqc(dir[ci - pitch], 6) || P::eqc(dir[ci - 1], 2);
    case 6: return P::eqc(dir[ci + pitch], 4) || P::eqc(dir[ci - 1], 8);
    case 8: return P::eqc(dir[ci + 1], 6) || P::eqc(dir[ci + pitch], 2);
    default: return false;
  }
}

// Pass-1 classification of every flat cell (src/d8.cpp:516-541 with st = 1,2 and :604-610)
template <class P>
__global__ void k_classify(const long long* __restrict__ list, unsigned long long n, const float* __restrict__ elev,
                           const typename P::DirT* __restrict__ dir, int* __restrict__ lev, int* __restrict__ mk, int pitch) {
  const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const long long ci = list[t];
  const float z = elev[ci];
  bool low = false, seed2 = false, higher = false;
#pragma unroll
  for (int k = 1; k <= 8; ++k) {
    const long long ni = ci + (long long)drow(k) * pitch + dcol(k);
    const float ed = z - elev[ni];
    if (ed < 0) higher = true;
    if (!dont_cross<P>(dir, ci, pitch, k)) {
      if (ed >= 0 && P::drains(dir[ni])) low = true;
      else if (ed == 0 && lev[ni] == 0) seed2 = true;    // equal neighbour outside the flat set: elev2 = 1 < st from pass 2 on
    }
  }
  if (low) lev[ci] = 1;
  else if (seed2) lev[ci] = 2;
  if (higher) mk[ci] = 1;
}

// append the cells of `list` whose arr[] value equals v
__global__ void k_gather(const long long* __restrict__ list, unsigned long long n, const int* __restrict__ arr, int v,
                         long long* __restrict__ out, unsigned long long* __restrict__ ctr) {
  const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = t < n;
  const long long ci = in ? list[t] : 0;
  append(out, ctr, in && arr[ci] == v, ci);
}

// fall BFS: frontier cells stopped at level t-1; an unassigned neighbour c with an
// equal-elevation, non-crossing link to the frontier cell stops at level t.
template <class P>
__global__ void k_expand_fall(const long long* __restrict__ fr, unsigned long long n, int t, const float* __restrict__ elev,
                              const typename P::DirT* __restrict__ dir, int* __restrict__ lev, int pitch, int ny,
                              long long* __restrict__ out, unsigned long long* __restrict__ ctr) {
  const unsigned long long tid = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = tid < n;
  const long long ni = in ? fr[tid] : 0;
  const float zn = in ? elev[ni] : 0.f;
#pragma unroll
  for (int kk = 1; kk <= 8; ++kk) {            // direction from the frontier cell to the candidate c
    bool push = false;
    const long long ci = ni + (long long)drow(kk) * pitch + dcol(kk);
    if (in && lev[ci] == UNASSIGNED) {
      const int k = kk > 4 ? kk - 4 : kk + 4;  // direction from c back to the frontier cell
      if (elev[ci] - zn == 0 && !dont_cross<P>(dir, ci, pitch, k)) push = atomicCAS(lev + ci, UNASSIGNED, t) == UNASSIGNED;
      if (ci < pitch || ci >= (long long)(ny + 1) * pitch) push = false;   // a cell of the neighbour strip: its owner appends it (k_merge)
    }
    append(out, ctr, push, ci);
  }
}

// rise BFS: any flat neighbour of a cell marked in pass u-1 is marked in pass u (src/d8.cpp:611-618)
__global__ void k_expand_rise(const long long* __restrict__ fr, unsigned long long n, int u, const int* __restrict__ lev,
                              int* __restrict__ mk, int pitch, int ny, long long* __restrict__ out, unsigned long long* __restrict__ ctr) {
  const unsigned long long tid = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = tid < n;
  const long long ni = in ? fr[tid] : 0;
#pragma unroll
  for (int kk = 1; kk <= 8; ++kk) {
    bool push = false;
    const long long ci = ni + (long long)drow(kk) * pitch + dcol(kk);
    if (in && lev[ci] != 0 && mk[ci] == 0) push = atomicCAS(mk + ci, 0, u) == 0;
    if (ci < pitch || ci >= (long long)(ny + 1) * pitch) push = false;     // neighbour strip's cell: see k_merge
    append(out, ctr, push, ci);
  }
}

// One BFS level without a host round trip (single strip, TAUDEM_B200_FLATS_BATCH): a fixed grid strides over the
// frontier of level t-1 = fr[bounds[t-2], bounds[t-1]) — the bounds live in device memory — and the last block to
// finish records where level t ends, bounds[t] = *ctr.  The host enqueues a batch of levels and reads the bounds
// back once; levels past the last non-empty one find an empty frontier and do nothing.
template <class P, bool FALL>
__global__ void __launch_bounds__(256) k_bfs_level(const long long* __restrict__ fr, unsigned long long* __restrict__ bounds, int t,
                                                   const float* __restrict__ elev, const typename P::DirT* __restrict__ dir,
                                                   int* __restrict__ lev, int* __restrict__ mk, int pitch, int ny, long long* __restrict__ out,
                                                   unsigned long long* __restrict__ ctr, unsigned* __restrict__ blkdone) {
  const unsigned long long lo = bounds[t - 2], hi = bounds[t - 1];
  const unsigned long long n = hi - lo;
  for (unsigned long long base = (unsigned long long)blockIdx.x * 256; base < n; base += (unsigned long long)gridDim.x * 256) {
    const unsigned long long i = base + threadIdx.x;
    const bool in = i < n;
    const long long ni = in ? fr[lo + i] : 0;
    const float zn = (FALL && in) ? elev[ni] : 0.f;
#pragma unroll
    for (int kk = 1; kk <= 8; ++kk) {
      bool push = false;
      const long long ci = ni + (long long)drow(kk) * pitch + dcol(kk);
      if (FALL) {
        if (in && lev[ci] == UNASSIGNED) {
          const int k = kk > 4 ? kk - 4 : kk + 4;
          if (elev[ci] - zn == 0 && !dont_cross<P>(dir, ci, pitch, k)) push = atomicCAS(lev + ci, UNASSIGNED, t) == UNASSIGNED;
        }
      } else if (in && lev[ci] != 0 && mk[ci] == 0) push = atomicCAS(mk + ci, 0, t) == 0;
      if (ci < pitch || ci >= (long long)(ny + 1) * pitch) push = false;
      append(out, ctr, push, ci);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(blkdone, 1u) == gridDim.x - 1) {          // the last block: every append of this level is done
      __threadfence();
      bounds[t] = *reinterpret_cast<volatile unsigned long long*>(ctr);
      *blkdone = 0;
    }
  }
}

// finalise elev2 = level (+T+1 for unreachable cells, which are marked as pits) + s, stored as the reference's 16-bit elev2:
// level + s wraps to a negative value past 32767 (T, U < 32767 keep level and s themselves in range)
template <class P>
__global__ void k_combine(const long long* __restrict__ list, unsigned long long n, int* __restrict__ lev,
                          const int* __restrict__ mk, typename P::DirT* __restrict__ dir, int T, int U) {
  const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const long long ci = list[t];
  int l = lev[ci];
  if (l == UNASSIGNED) { l = 1 + T; dir[ci] = P::pit(); }    // src/d8.cpp:559-593
  const int m = mk[ci];
  if (m > 0) l += U - m + 1;                                   // src/d8.cpp:640-646
  lev[ci] = (short)l;
}

// setFlow2 (src/d8.cpp:412-454)
__global__ void k_setflow2(const long long* __restrict__ list, unsigned long long n, const float* __restrict__ elev,
                           const int* __restrict__ lev, const int* __restrict__ mk, short* __restrict__ dir, Strip s,
                           const double* __restrict__ dxc, const double* __restrict__ dyc, long long* __restrict__ out,
                           unsigned long long* __restrict__ ctr) {
  const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = t < n;
  const long long ci = in ? list[t] : 0;
  bool still = false;
  if (in) {
    const int r = (int)(ci / s.pitch);
    const double dx = dxc[r - 1], dy = dyc[r - 1];
    const double fE = 1. / sqrt(dx * dx), fN = 1. / sqrt(dy * dy), fD = 1. / sqrt(dx * dx + dy * dy);
    const float z = elev[ci];
    const int e2 = lev[ci];
    short d = dir[ci];
    float smax = 0.f;
    const int order[8] = {1, 3, 5, 7, 2, 4, 6, 8};
#pragma unroll
    for (int ii = 0; ii < 8; ++ii) {
      const int k = order[ii];
      const long long ni = ci + (long long)drow(k) * s.pitch + dcol(k);
      if (mk[ni] > 0) {
        const double f = (k & 1) ? ((k == 1 || k == 5) ? fE : fN) : fD;
        const float sl = (float)(f * (double)(e2 - lev[ni]));
        if (sl > smax) { d = (short)k; smax = sl; }
      } else {
        const float ed = z - elev[ni];
        if (ed >= 0) { d = (short)k; break; }
      }
    }
    dir[ci] = d;
    still = d == 0;
  }
  append(out, ctr, still, ci);
}

// flat SET2 (src/dinf.cpp:375-528)
__global__ void k_set2_flat(const long long* __restrict__ list, unsigned long long n, const float* __restrict__ elev,
                            const int* __restrict__ lev, const int* __restrict__ mk, float* __restrict__ ang, Strip s,
                            const double* __restrict__ dxc, const double* __restrict__ dyc, const double* __restrict__ thA,
                            const double* __restrict__ thB, long long* __restrict__ out, unsigned long long* __restrict__ ctr) {
  const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = t < n;
  const long long ci = in ? list[t] : 0;
  bool still = false;
  if (in) {
    const int r = (int)(ci / s.pitch);
    const double dx = dxc[r - 1], dy = dyc[r - 1];
    const double DD = sqrt(dx * dx + dy * dy);
    const double adA = thA[r - 1], adB = thB[r - 1];
    double SMAX = 0.0, AKD = 0.0;
    int KD = 0;
    bool diagOutFound = false;
    const double a = (double)elev[ci];
    const int a1 = lev[ci];
#pragma unroll 1
    for (int K = 1; K <= 8; ++K) {
      const long long i1 = ci + (long long)fI1(K) * s.pitch + fJ1(K), i2 = ci + (long long)fI2(K) * s.pitch + fJ2(K);
      const bool d1x = fD1isDx(K);
      const double D1 = d1x ? dx : dy, D2 = d1x ? dy : dx, AD = d1x ? adA : adB;
      const bool t1 = mk[i1] > 0, t2 = mk[i2] > 0;
      if (!t1 && !t2) {
        const double b = (double)elev[i1], c = (double)elev[i2];
        const Facet f = vslope_dev(a, b, c, D1, D2, DD);
        if (f.S >= 0.0) {
          if (b > a) { if (!diagOutFound) { diagOutFound = true; KD = K; AKD = facet_angle(f, AD); } }
          else { KD = K; AKD = facet_angle(f, AD); break; }
        }
      } else if (!t1 && t2) {
        const double b = (double)elev[i1];
        if (a >= b) { AKD = 0.0; KD = K; break; }
        const int c1 = lev[i2], b1 = max(a1, c1);
        const Facet f = vslope_dev((double)a1, (double)b1, (double)c1, D1, D2, DD);
        if (f.S > SMAX) { SMAX = f.S; KD = K; AKD = facet_angle(f, AD); }
      } else if (t1 && !t2) {
        const double c = (double)elev[i2];
        if (a >= c) { if (!diagOutFound) { AKD = AD; KD = K; diagOutFound = true; } }
        else {
          const int b1 = lev[i1], c1 = max(a1, b1);
          const Facet f = vslope_dev((double)a1, (double)b1, (double)c1, D1, D2, DD);
          if (f.S > SMAX) { SMAX = f.S; KD = K; AKD = facet_angle(f, AD); }
        }
      } else {
        const Facet f = vslope_dev((double)a1, (double)lev[i1], (double)lev[i2], D1, D2, DD);
        if (f.S > SMAX) { SMAX = f.S; KD = K; AKD = facet_angle(f, AD); }
      }
    }
    float v = ang[ci];
    if (!nd_f(v, TD_MISSINGFLOAT)) v = -1.0f;
    if (KD > 0) {
      const float tf = dinf_angle(KD, AKD);
      if (tf >= 0.0f) v = tf;
    }
    ang[ci] = v;
    still = !nd_f(v, TD_MISSINGFLOAT) && v < 0.0f;
  }
  append(out, ctr, still, ci);
}

// src/d8.cpp:669-675: elevDEM := (float)elev2 on every cell (elev2 = 1 outside the flat set)
__global__ void k_overwrite(float* __restrict__ elev, const int* __restrict__ lev, Strip s) {
  const int c = blockIdx.y * blockDim.x + threadIdx.x, r = 1 + blockIdx.x;   // rows on grid.x (no 65535 limit)
  if (c >= s.nx) return;
  const long long ci = s.idx(r, c);
  const int l = lev[ci];
  elev[ci] = (float)(l != 0 ? l : 1);
}

__global__ void k_reset(const long long* __restrict__ list, unsigned long long n, int* __restrict__ lev, int* __restrict__ mk) {
  const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n) { lev[list[t]] = 0; mk[list[t]] = 0; }
}

// Claims the neighbour strips made on their halo copies of my first / last row during BFS level t:
// recv_top[c] / recv_bot[c] = the neighbour's lev (FALL) or mk (rise) value for (row 1, c) / (row ny, c).
template <bool FALL>
__global__ void k_merge(const int* __restrict__ recv_top, const int* __restrict__ recv_bot, Strip s, int t, int* __restrict__ lev,
                        int* __restrict__ mk, long long* __restrict__ out, unsigned long long* __restrict__ ctr) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = c < s.nx;
#pragma unroll
  for (int side = 0; side < 2; ++side) {
    const int* recv = side == 0 ? recv_top : recv_bot;
    const long long ci = s.idx(side == 0 ? 1 : s.ny, in ? c : 0);
    bool push = false;
    if (in && recv != nullptr && recv[c] == t) {
      if (FALL) { if (lev[ci] == UNASSIGNED) { lev[ci] = t; push = true; } }
      else if (lev[ci] != 0 && mk[ci] == 0) { mk[ci] = t; push = true; }
    }
    append(out, ctr, push, ci);
  }
}

inline unsigned nblk(unsigned long long n) { return (unsigned)((n + 255) / 256); }

struct Geo { const double *dxc, *dyc, *thA, *thB; };

template <class P>
int resolve_flats(td_ctx* ctx, float* elev, typename P::DirT* dir, const Strip& s, const Geo& g, long long* nleft,
                  const td_strip_comm* comm, cudaStream_t st) {
  const bool multi = s.has_top || s.has_bot;
  if (multi && (!comm || !comm->share || !comm->collect || !comm->allreduce_sum)) {
    set_error("flat resolution over row strips needs the td_strip_comm callbacks"); return TD_ERR_ARG;
  }
  if (!multi) comm = nullptr;
  const size_t ncell = (size_t)s.cells();
  unsigned long long* dc = ctx->d_ctr;   // [0] list append, [1] frontier append
  auto read_ctr = [&](int i, unsigned long long* v) -> cudaError_t {
    cudaError_t e = cudaMemcpyAsync(ctx->h_ctr + i, dc + i, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st);
    if (e != cudaSuccess) return e;
    e = cudaStreamSynchronize(st);
    *v = ctx->h_ctr[i];
    return e;
  };
  // the three places where the reference's resolveflats talks to the other ranks
  auto gsum = [&](unsigned long long v, unsigned long long* out) -> int {
    *out = v;
    if (comm && comm->allreduce_sum(comm->user, out, 1) != 0) { set_error("td_strip_comm.allreduce_sum failed"); return TD_ERR_ARG; }
    return TD_OK;
  };
  auto share = [&](void* arr, int elem) -> int {
    if (!comm) return TD_OK;
    TD_CUDA(cudaStreamSynchronize(st));
    if (comm->share(comm->user, arr, elem) != 0) { set_error("td_strip_comm.share failed"); return TD_ERR_ARG; }
    return TD_OK;
  };
  int* recv_top = nullptr; int* recv_bot = nullptr;
  if (multi) {
    TD_CUDA(ctx->halo.ensure(sizeof(int) * 2 * (size_t)s.pitch));
    if (s.has_top) recv_top = ctx->halo.as<int>();
    if (s.has_bot) recv_bot = ctx->halo.as<int>() + s.pitch;
  }
  auto collect = [&](const void* arr) -> int {      // halo rows -> owners (recv_top / recv_bot)
    TD_CUDA(cudaStreamSynchronize(st));
    if (comm->collect(comm->user, arr, 4, recv_top, recv_bot) != 0) { set_error("td_strip_comm.collect failed"); return TD_ERR_ARG; }
    return TD_OK;
  };
  // --- collect the flat cells (first call of the reference: src/d8.cpp:492-503)
  // a counting pass sizes the lists (8 bytes per FLAT cell, not per cell of the strip)
  unsigned long long n = 0, ntot = 0;      // flat cells of this strip / of the whole grid
  {
    dim3 grid(s.ny, (s.nx + 255) / 256);
    TD_CUDA(cudaMemsetAsync(dc, 0, 4 * sizeof(unsigned long long), st));
    k_collect<P><<<grid, 256, 0, st>>>(dir, s, nullptr, dc);
    TD_LAUNCHED();
    TD_CUDA(read_ctr(0, &n));
    TD_CUDA(ctx->listA.ensure(sizeof(long long) * (n + 1)));
    TD_CUDA(cudaMemsetAsync(dc, 0, 4 * sizeof(unsigned long long), st));
    k_collect<P><<<grid, 256, 0, st>>>(dir, s, ctx->listA.as<long long>(), dc);
    TD_LAUNCHED();
  }
  TD_CUDA(read_ctr(0, &n));
  if (int rc = gsum(n, &ntot)) return rc;
  *nleft = (long long)ntot;
  if (ntot == 0) return TD_OK;
  TD_CUDA(ctx->lev.ensure(ncell * 4));
  TD_CUDA(ctx->mk.ensure(ncell * 4));
  TD_CUDA(ctx->listB.ensure(sizeof(long long) * (n + 1)));
  TD_CUDA(ctx->listC.ensure(sizeof(long long) * (n + 1)));
  TD_CUDA(cudaMemsetAsync(ctx->lev.p, 0, ncell * 4, st));
  TD_CUDA(cudaMemsetAsync(ctx->mk.p, 0, ncell * 4, st));
  int* lev = ctx->lev.as<int>();
  int* mk = ctx->mk.as<int>();
  long long* cur = ctx->listA.as<long long>();
  long long* nxt = ctx->listB.as<long long>();
  long long* fr = ctx->listC.as<long long>();
  const unsigned colblk = (unsigned)((s.nx + 255) / 256);

  // single strip: 64 BFS levels per host round trip (k_bfs_level; TAUDEM_B200_FLATS_BATCH = K overrides, 0 = one launch + read-back per level)
  int batch = 0;
  if (!multi) { const char* e = getenv("TAUDEM_B200_FLATS_BATCH"); batch = e ? std::max(0, std::min(atoi(e), 4096)) : 64; }
  constexpr unsigned long long MAXLEV = 1ull << 22;
  unsigned long long* bounds = nullptr; unsigned* blkdone = nullptr;
  int bgrid = 1;
  if (batch > 0) {
    TD_CUDA(ctx->tileflags.ensure(sizeof(unsigned long long) * (MAXLEV + 2)));
    bounds = ctx->tileflags.as<unsigned long long>();
    blkdone = reinterpret_cast<unsigned*>(bounds + MAXLEV + 1);
    TD_CUDA(cudaMemsetAsync(blkdone, 0, sizeof(unsigned long long), st));
    int dev = 0, sms = 1;
    cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    bgrid = std::max(1, sms * 4);
  }
  std::vector<unsigned long long> hb;
  // runs BFS levels 2, 3, ... in batches from the frontier fr[0, hi1) of level 1; *passes = first level that assigns nothing
  auto bfs_batched = [&](bool fall, unsigned long long hi1, int* passes) -> int {
    const unsigned long long b01[2] = {0ull, hi1};
    TD_CUDA(cudaMemcpyAsync(bounds, b01, sizeof b01, cudaMemcpyHostToDevice, st));
    unsigned long long prev = hi1;
    for (int t0 = 2;; t0 += batch) {
      if ((unsigned long long)(t0 + batch) >= MAXLEV) { set_error("flat resolution: too many BFS levels for the batched mode"); return TD_ERR_ALLOC; }
      for (int t = t0; t < t0 + batch; ++t) {
        if (fall) k_bfs_level<P, true><<<bgrid, 256, 0, st>>>(fr, bounds, t, elev, dir, lev, mk, s.pitch, s.ny, fr, dc + 1, blkdone);
        else k_bfs_level<P, false><<<bgrid, 256, 0, st>>>(fr, bounds, t, elev, dir, lev, mk, s.pitch, s.ny, fr, dc + 1, blkdone);
        TD_LAUNCHED();
      }
      hb.resize(batch);
      TD_CUDA(cudaMemcpyAsync(hb.data(), bounds + t0, sizeof(unsigned long long) * batch, cudaMemcpyDeviceToHost, st));
      TD_CUDA(cudaStreamSynchronize(st));
      for (int j = 0; j < batch; ++j) {
        if (hb[j] == prev) { *passes = t0 + j; return TD_OK; }
        prev = hb[j];
      }
    }
  };

  unsigned long long last = ntot + 1;
  // outer loop: src/d8.cpp:302-317
  while (ntot > 0 && ntot < last) {
    last = ntot;
    if (n) { k_mark<<<nblk(n), 256, 0, st>>>(cur, n, lev); TD_LAUNCHED(); }
    if (int rc = share(lev, 4)) return rc;                       // who is in the flat set on the other side of the boundary
    if (n) { k_classify<P><<<nblk(n), 256, 0, st>>>(cur, n, elev, dir, lev, mk, s.pitch); TD_LAUNCHED(); }
    if (int rc = share(lev, 4)) return rc;
    if (int rc = share(mk, 4)) return rc;
    // ---- fall BFS
    TD_CUDA(cudaMemsetAsync(dc + 1, 0, sizeof(unsigned long long), st));
    if (n) { k_gather<<<nblk(n), 256, 0, st>>>(cur, n, lev, 1, fr, dc + 1); TD_LAUNCHED(); }
    unsigned long long lo = 0, hi = 0, hitot = 0;
    TD_CUDA(read_ctr(1, &hi));
    if (int rc = gsum(hi, &hitot)) return rc;
    int T = 1;
    if (hitot != ntot) {
      // pass 2: seeds (equal neighbour outside F) + expansion of level 1
      if (n) { k_gather<<<nblk(n), 256, 0, st>>>(cur, n, lev, 2, fr, dc + 1); TD_LAUNCHED(); }
      int t = 2;
      if (batch > 0) {
        if (int rc = bfs_batched(true, hi, &T)) return rc;
      } else
      for (;;) {
        if (hi > lo) { k_expand_fall<P><<<nblk(hi - lo), 256, 0, st>>>(fr + lo, hi - lo, t, elev, dir, lev, s.pitch, s.ny, fr, dc + 1); TD_LAUNCHED(); }
        if (multi) {
          // (the halo copies are not refreshed per level: a stale "unassigned" only produces a claim the owner ignores)
          if (int rc = collect(lev)) return rc;
          k_merge<true><<<colblk, 256, 0, st>>>(recv_top, recv_bot, s, t, lev, mk, fr, dc + 1); TD_LAUNCHED();
        }
        unsigned long long end = 0, nt = 0;
        TD_CUDA(read_ctr(1, &end));
        // level t occupies [hi', end): for t == 2 the seeds were appended before the expansion
        if (int rc = gsum(end - hi, &nt)) return rc;
        if (nt == 0) { T = t; break; }
        lo = hi; hi = end; ++t;
      }
    }
    // ---- rise BFS
    TD_CUDA(cudaMemsetAsync(dc + 1, 0, sizeof(unsigned long long), st));
    if (n) { k_gather<<<nblk(n), 256, 0, st>>>(cur, n, mk, 1, fr, dc + 1); TD_LAUNCHED(); }
    lo = 0; hi = 0;
    TD_CUDA(read_ctr(1, &hi));
    if (int rc = gsum(hi, &hitot)) return rc;
    int U = 1;
    if (hitot > 0) {
      int u = 2;
      if (batch > 0) {
        if (int rc = bfs_batched(false, hi, &U)) return rc;
      } else
      for (;;) {
        if (hi > lo) { k_expand_rise<<<nblk(hi - lo), 256, 0, st>>>(fr + lo, hi - lo, u, lev, mk, s.pitch, s.ny, fr, dc + 1); TD_LAUNCHED(); }
        if (multi) {
          if (int rc = collect(mk)) return rc;
          k_merge<false><<<colblk, 256, 0, st>>>(recv_top, recv_bot, s, u, lev, mk, fr, dc + 1); TD_LAUNCHED();
        }
        unsigned long long end = 0, nu = 0;
        TD_CUDA(read_ctr(1, &end));
        if (int rc = gsum(end - hi, &nu)) return rc;
        if (nu == 0) { U = u; break; }
        lo = hi; hi = end; ++u;
      }
    }
    // The reference counts passes in a short (src/d8.cpp:514, src/dinf.cpp:655): from pass 32767 on its counter wraps and its
    // elev2 no longer follows the gradients, so there is no result to reproduce.
    if (T >= MAXPASS || U >= MAXPASS) {
      set_error("flat resolution: a flat needs " + std::to_string(std::max(T, U)) + " " + (T >= MAXPASS ? "fall" : "rise") +
                " passes; the reference's 16-bit pass counter allows at most 32766");
      return TD_ERR_FLAT_PASSES;
    }
    // ---- combine, set directions, collect what is still flat
    if (n) { k_combine<P><<<nblk(n), 256, 0, st>>>(cur, n, lev, mk, dir, T, U); TD_LAUNCHED(); }
    if (int rc = share(lev, 4)) return rc;                        // elev2 of the neighbours' edge cells
    if (int rc = share(mk, 4)) return rc;                         // and whether they rise (k_setflow2 / k_set2_flat read both)
    if (int rc = share(dir, (int)sizeof(typename P::DirT))) return rc;   // pits marked by k_combine
    TD_CUDA(cudaMemsetAsync(dc, 0, sizeof(unsigned long long), st));
    if (n) {
      if constexpr (sizeof(typename P::DirT) == 2)
        k_setflow2<<<nblk(n), 256, 0, st>>>(cur, n, elev, lev, mk, (short*)dir, s, g.dxc, g.dyc, nxt, dc);
      else
        k_set2_flat<<<nblk(n), 256, 0, st>>>(cur, n, elev, lev, mk, (float*)dir, s, g.dxc, g.dyc, g.thA, g.thB, nxt, dc);
      TD_LAUNCHED();
    }
    unsigned long long nn = 0, nntot = 0;
    TD_CUDA(read_ctr(0, &nn));
    if (int rc = gsum(nn, &nntot)) return rc;
    if (int rc = share(dir, (int)sizeof(typename P::DirT))) return rc;   // the directions just set (dontCross of the next iteration)
    if (nntot > 0) {
      dim3 grid(s.ny, colblk);
      k_overwrite<<<grid, 256, 0, st>>>(elev, lev, s); TD_LAUNCHED();
      if (int rc = share(elev, 4)) return rc;
    }
    if (n) { k_reset<<<nblk(n), 256, 0, st>>>(cur, n, lev, mk); TD_LAUNCHED(); }
    if (multi) {        // the halo copies of lev / mk are reset with their owners' cells
      TD_CUDA(cudaMemsetAsync(lev, 0, sizeof(int) * (size_t)s.pitch, st));
      TD_CUDA(cudaMemsetAsync(mk, 0, sizeof(int) * (size_t)s.pitch, st));
      TD_CUDA(cudaMemsetAsync(lev + (size_t)(s.ny + 1) * s.pitch, 0, sizeof(int) * (size_t)s.pitch, st));
      TD_CUDA(cudaMemsetAsync(mk + (size_t)(s.ny + 1) * s.pitch, 0, sizeof(int) * (size_t)s.pitch, st));
    }
    std::swap(cur, nxt);
    n = nn; ntot = nntot;
  }
  TD_CUDA(cudaGetLastError());
  *nleft = (long long)ntot;
  return TD_OK;
}
}  // namespace

int resolve_flats_d8(td_ctx* ctx, float* elev, short* dir, const Strip& s, const double* dxc, const double* dyc, long long* nleft,
                     const td_strip_comm* comm, cudaStream_t st) {
  Geo g{dxc, dyc, nullptr, nullptr};
  return resolve_flats<D8Pol>(ctx, elev, dir, s, g, nleft, comm, st);
}
int resolve_flats_dinf(td_ctx* ctx, float* elev, float* ang, const Strip& s, const double* dxc, const double* dyc, const double* thA,
                       const double* thB, long long* nleft, const td_strip_comm* comm, cudaStream_t st) {
  Geo g{dxc, dyc, thA, thB};
  return resolve_flats<DinfPol>(ctx, elev, ang, s, g, nleft, comm, st);
}

}  // namespace td
