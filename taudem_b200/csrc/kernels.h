// Internal launcher prototypes (one per kernel family).
#pragma once
#include "ctx.h"

namespace td {
struct RowFact;
int launch_d8_stencil(const float* elev, short* dir, float* slope, const RowFact* rowf, const Strip& s, float nodata,
                      unsigned long long* nflat, cudaStream_t st);
int launch_dinf_stencil(const float* elev, float* ang, float* slp, const RowFact* rowf, const Strip& s, float nodata,
                        unsigned long long* nflat, cudaStream_t st);
int resolve_flats_d8(td_ctx* ctx, float* elev, short* dir, const Strip& s, const double* dxc, const double* dyc,
                     long long* nleft, const td_strip_comm* comm, cudaStream_t st);
int resolve_flats_dinf(td_ctx* ctx, float* elev, float* ang, const Strip& s, const double* dxc, const double* dyc,
                       const double* thA, const double* thB, long long* nleft, const td_strip_comm* comm, cudaStream_t st);
cudaError_t launch_deps_d8(const short* p, unsigned short* node, unsigned char* cnt, float* area, const Strip& s,
                           short nodata, cudaStream_t st, float area_init = -1.0f);
cudaError_t launch_halo_codes_d8(const short* p, unsigned short* node, const Strip& s, short nodata, cudaStream_t st);   // gridnet on row strips
cudaError_t launch_deps_dinf(const float* ang, unsigned short* node, unsigned char* cnt, float* area, const Strip& s,
                             float nodata, const double* theta, cudaStream_t st, float area_init = -1.0f);
cudaError_t zero_words(void* p, size_t bytes, cudaStream_t st);
// retlimflow: cells of the owned rows whose wg or rc is nodata lose their receivers in the node words (sweep_warp.cu)
cudaError_t launch_block_cells(unsigned short* node, const float* wg, float wg_nodata, const float* rc, float rc_nodata, const Strip& s, cudaStream_t st);     // a multiple of 4 bytes, zeroed by a kernel (never by a copy engine)
int wsweep_begin(td_ctx* ctx, const Strip& s, cudaStream_t st);
int wsweep_apply_halo(td_ctx* ctx, const Strip& s, const int* dec_top, const int* dec_bot, cudaStream_t st);
// the extra grids of the concentration- and transport-limited accumulations (algebras 7-9 of the D-infinity sweep, sweep_warp.cu)
struct SweepExtra {
  const short* dg = nullptr;       // ALG 7: indicator grid (> 0: the cell is a source at the solubility threshold)
  float csol = 0.f;                // ALG 7: the concentration of such a cell
  const float* cin = nullptr;      // ALG 9: concentration of the supply
  float cin_nodata = 0.f;
  float* out2 = nullptr;           // ALG 8 / 9: deposition (written, never read; must start as nodata)
  float* out3 = nullptr;           // ALG 9: concentration in the transported flux (written and read by receivers; must start as nodata)
};
int wsweep_run(td_ctx* ctx, bool dinf, float* area, const float* w, const float* ang, const Strip& s, float w_nodata, int usew,
               int contcheck, const double* theta, const double* dxc, int* halo, cudaStream_t st, int alg = 0, const float* dm = nullptr,
               float dm_nodata = 0.f, const float* dist = nullptr, const SweepExtra* extra = nullptr);
cudaError_t fill_floats(float* p, const Strip& s, float v, cudaStream_t st);   // every cell of the strip := v
int sweep_restrict_round(td_ctx* ctx, const Strip& s, const int* cols, const int* rows, int nout, const int* in_top, const int* in_bot,
                         int* req_out, int finish, cudaStream_t st);
int sweep_restrict_upstream(td_ctx* ctx, const Strip& s, const int* cols, const int* rows, int nout, cudaStream_t st);
int sweep_peer_export(td_ctx* ctx, const Strip& s, int dinf, unsigned char* handles, int* meta, cudaStream_t st);
int sweep_peer_connect(td_ctx* ctx, int which, const unsigned char* handles, const int* meta);
int sweep_peer_begin(td_ctx* ctx, const Strip& s, cudaStream_t st);
void sweep_peer_off(td_ctx* ctx);
int fill_init(const float* dem, const short* mask, float* W, const Strip& s, float nodata, int four, cudaStream_t st);
int fill_relax(td_ctx* ctx, const float* dem, float* W, const Strip& s, int four, int* changed, cudaStream_t st, bool edges_only = false);
int launch_threshold(const float* ssa, const float* mask, short* src, const Strip& s, float thresh, float ssa_nodata, cudaStream_t st);
// twi, slopearea and lengtharea synchronise st; pend holds the cells they decide on the host (a context's buffer; nullptr: one
// allocated for the call, pointwise.cu)
int launch_slopearea(const float* slp, const float* sca, float* sa, const Strip& s, float m, float n, cudaStream_t st,
                     td_ctx::Buf* pend = nullptr);
int launch_slopearearatio(const float* slp, const float* sca, float* sar, const Strip& s, float sca_nodata, cudaStream_t st);
int launch_twi(const float* slp, const float* sca, float* twi, const Strip& s, float slp_nodata, float sca_nodata, cudaStream_t st,
               td_ctx::Buf* pend = nullptr);
int launch_lengtharea(const float* plen, const int* ad8, short* ss, const Strip& s, float m, float y, cudaStream_t st,
                      td_ctx::Buf* pend = nullptr);
int launch_pd_smooth(const float* fel, float* sm, const Strip& s, float nodata, const float* p /* host: w_mid, w_side, w_diag */, cudaStream_t st);
int launch_pd_mark(const float* sm, short* ss, const Strip& s, float nodata, cudaStream_t st);
// slopeavedown.cu: s0 / s1 = the two (ed, dd) state buffers (float2 per strip cell)
int launch_sad_init(const short* p, const unsigned char* cnt, const float* fel, unsigned char* code, float* s0, float* s1, float* sd,
                    const Strip& s, short p_nodata, float fel_nodata, cudaStream_t st);
int launch_sad_pass(const unsigned char* code, const float* fel, const float* src, float* dst, float* sd, const float* dist, const Strip& s,
                    double dn, int* changed, cudaStream_t st);
// disttostrm.cu: the BFS from the stream cells of d8hdisttostrm / d8vdisttostrm.  list: one entry per strip cell at most;
// ctr[0] = entries appended, ctr[1] = entries consumed by the levels run so far; bounds: DTS_BATCH + 2 words; blkdone: one word.
constexpr int DTS_BATCH = 64;     // BFS levels per host read-back
struct DtsBufs { unsigned* list; unsigned long long* ctr; unsigned long long* bounds; unsigned* blkdone; };
int dts_seed(const short* p, const int* src, float* val, unsigned char* code, const Strip& s, int thresh, short p_nodata, int src_nodata,
             const DtsBufs& b, cudaStream_t st);
// the edge-row cells of a row strip whose receiver is in a halo row with a value, then levels until the frontier is empty (grid
// blocks per level); *cells = the list entries added since the last call (with the seeds), *levels = the non-empty levels run
int dts_levels(bool vertical, const unsigned char* code, const float* fel, const float* dist, float* val, const Strip& s, const DtsBufs& b, int grid,
               unsigned long long* cells, long long* levels, cudaStream_t st);
// dinfdistdown.cu: Kahn's algorithm over the D-infinity receivers, one level per launch on the same frontier machinery (flood.cuh).
// theta: the strip's per-row angle table (theta_of_row); dist: the cell-to-cell distances of the owned rows (8 per row); val2: the
// vertical values of the p mode (else NULL); state: one byte per strip cell, the strip's size a multiple of 4 bytes; halo_out: the
// decrements of the donors in the halo rows, [0, pitch) row 0 (sent up), [pitch, 2 pitch) row ny + 1 (sent down); NULL on one strip.
struct DddArgs {
  const float* ang; const float* fel; const float* w; const float* dist; const double* theta;
  float* val; float* val2; unsigned char* state; int* halo_out;
  float fel_nodata, w_nodata;
  int concheck;
};
int ddd_seed(const float* ang, const short* src, float ang_nodata, const DddArgs& A, const Strip& s, const DtsBufs& b, cudaStream_t st);
// mode 0..3 = h, v, p, s; stat 0..2 = ave, max, min
int ddd_levels(int mode, int stat, const DddArgs& A, const Strip& s, const DtsBufs& b, int grid, unsigned long long* cells, long long* levels,
               cudaStream_t st);
// the decrements received for the first / last owned row (NULL: no neighbour there); the released cells join the frontier
int ddd_edge(unsigned char* state, const int* dec_top, const int* dec_bot, const Strip& s, const DtsBufs& b, cudaStream_t st);
int ddd_pythagoras(float* h, const float* v, const Strip& s, cudaStream_t st);
int launch_mask_ok(const int* mask, float* ok, const Strip& s, int thresh, cudaStream_t st);
int launch_gord_finish(const float* g, const short* p, const float* ok, const unsigned short* node, short* gord, const Strip& s, short p_nodata,
                       int outlets, cudaStream_t st);
void gridnet_dist_table(const double* dxc, const double* dyc, int ny, float* dist);   // host: gridnet's per-row distances (capi.cu)
cudaError_t launch_gen_dem(float* dem, const Strip& s, int row0, int total_ny, unsigned seed, float hurst, float tilt, cudaStream_t st);
cudaError_t launch_gen_w(float* w, const Strip& s, int row0, unsigned seed, cudaStream_t st);
}  // namespace td
