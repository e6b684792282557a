/* taudem_b200 — C ABI of the H100-native TauDEM flow-direction / contributing-area path.
 *
 * Three layers, all `extern "C"`, plain pointers and sizes only:
 *
 *  1. FILE level  — drop-in replacements for the five reference library
 *     functions that the reference's mains call (same parameter lists, bool -> int):
 *       td_flood      <- int flood(...)     reference src/flood.h,  src/flood.cpp:50
 *       td_setdird8   <- int setdird8(...)  reference src/d8.h:7,   src/d8.cpp:181
 *       td_setdir     <- int setdir(...)    reference src/tardemlib.h:70, src/dinf.cpp:109
 *       td_aread8     <- int aread8(...)    reference src/aread8.h:3,   src/aread8.cpp:56
 *       td_area       <- int area(...)      reference src/areadinf.h:2, src/areadinf.cpp:53
 *     They read/write rasters with the tiffIO contract (src/tiffIO.cpp) and return 0 on
 *     success, non-zero on error, like the reference.
 *
 *  2. HOST-GRID level — the same computations on caller-owned host arrays
 *     (row-major, row 0 = north, `nx` columns, `ny` rows, dense).  Host<->device
 *     copies happen inside the call.  This is what a binding that already holds
 *     the rasters in memory (e.g. a GDAL- or numpy-based caller) uses.
 *
 *  3. DEVICE-STRIP level — kernels on device-resident row strips, the unit the
 *     reference distributes over MPI ranks (src/linearpart.h:125-166).  A strip
 *     buffer holds `ny + 2` rows of `pitch` elements: row 0 is the halo row
 *     above, rows 1..ny are owned, row ny+1 is the halo row below
 *     (topBorder/bottomBorder, src/linearpart.h:66-67).  `has_top/has_bot` say
 *     whether a neighbouring strip exists (hasAccess, src/linearpart.h:178-190).
 *     `stream` is a cudaStream_t passed as void*.
 *
 * No CPU fallback exists: every compute entry point fails (TD_ERR_CUDA) when no
 * CUDA device is usable.
 */
#ifndef TAUDEM_B200_H
#define TAUDEM_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TD_OK 0
#define TD_ERR_ARG 1      /* bad argument / size mismatch (reference: return 1)        */
#define TD_ERR_IO 21      /* cannot open raster (reference: MPI_Abort(MCW,21))          */
#define TD_ERR_DRIVER 22  /* output driver unavailable (reference: MPI_Abort(MCW,22))   */
#define TD_ERR_MISMATCH 5 /* companion raster mismatch (reference: MPI_Abort(MCW,5))    */
#define TD_ERR_CUDA 90    /* CUDA runtime failure / no device                           */
#define TD_ERR_ALLOC 91   /* device or host allocation failure (reference: -999)        */
#define TD_ERR_FLAT_PASSES 92 /* a flat needs >= 32767 fall or rise passes: the reference's
                                 16-bit pass counter wraps there (DESIGN.md §2)            */

/* ---- version / diagnostics -------------------------------------------------------- */
const char* td_version(void);            /* "5.4.0-b200" (TDVERSION, src/commonLib.h:63)  */
const char* td_last_error(void);         /* thread-local message for the last failure     */
int td_device_count(void);               /* number of CUDA devices, 0 if none             */
int td_warmup(void);                     /* creates the CUDA context now (callable from a helper thread while inputs are read) */
int td_set_device(int dev);
/* Kernels launched by this library since the last reset (bench `gpu_launches`). */
unsigned long long td_launch_count(void);
void td_reset_launch_count(void);
/* Seconds spent inside the device-resident compute part of the last host-grid or
 * file-level call (the reference's "Compute time", e.g. src/aread8.cpp:175,307). */
double td_last_compute_seconds(void);

/* ---- 1. file level ---------------------------------------------------------------- */
int td_flood(const char* demfile, const char* felfile, const char* sfdrfile, int usesfdr,
             int verbose, int is_4Point, int use_mask, const char* maskfile);
int td_setdird8(const char* demfile, const char* pointfile, const char* slopefile,
                const char* flowfile, int useflowfile);
int td_setdir(const char* demfile, const char* angfile, const char* slopefile,
              const char* flowfile, int useflowfile);
int td_aread8(const char* pfile, const char* afile, const char* datasrc, const char* lyrname,
              int uselyrname, int lyrno, const char* wfile, int useOutlets, int usew,
              int contcheck);
int td_area(const char* angfile, const char* scafile, const char* datasrc, const char* lyrname,
            int uselyrname, int lyrno, const char* wfile, int useOutlets, int usew,
            int contcheck);
/* reference src/commonLib.cpp:53-73 */
int td_nameadd(char* full, const char* arg, const char* suff);

/* raster file helpers (tiffIO contract) used by the CLI, tests and bindings */
int td_raster_info(const char* path, int* nx, int* ny, double* nodata, int* has_nodata,
                   double* dx, double* dy, int* is_geographic, int* bits, int* sample_format);
/* dtype: 0 = int16, 1 = int32, 2 = float32 (SHORT_TYPE/LONG_TYPE/FLOAT_TYPE) */
int td_raster_read(const char* path, int dtype, void* dest, int nx, int ny);
int td_raster_cell_sizes(const char* path, double* dxc, double* dyc, int ny);
/* like_path may be NULL (no georeferencing); compression: 1 none, 5 LZW, 8 Deflate */
int td_raster_write(const char* path, int dtype, const void* src, int nx, int ny, double nodata,
                    const char* like_path, double dx, double dy, int compression);

/* ---- 2. host-grid level ------------------------------------------------------------ */
/* dxc/dyc: per-row cell sizes (ny doubles each; tiffIO::getdxc/getdyc). */
int td_flood_host(const float* dem, float* fel, const int16_t* depmask /*may be NULL*/,
                  int nx, int ny, float dem_nodata, int is_4Point);
int td_setdird8_host(const float* fel, int16_t* p, float* sd8, int nx, int ny,
                     float fel_nodata, const double* dxc, const double* dyc);
int td_setdir_host(const float* fel, float* ang, float* slp, int nx, int ny, float fel_nodata,
                   const double* dxc, const double* dyc);
int td_aread8_host(const int16_t* p, const float* w /*NULL unless usew*/, float* ad8, int nx,
                   int ny, int16_t p_nodata, float w_nodata, int contcheck);
int td_area_host(const float* ang, const float* w /*NULL unless usew*/, float* sca, int nx, int ny,
                 float ang_nodata, float w_nodata, const double* dxc, const double* dyc,
                 int contcheck);
/* Point-wise consumers of the area rasters (SURVEY.md 8(f) rank 4).  File level = the reference prototypes
 * `int threshold(char* ssafile, char* srcfile, char* maskfile, float thresh, int usemask)` (src/Threshold.cpp:48) and
 * `int twigrid(char* slopefile, char* areafile, char* twifile)` (src/TWI.cpp:47); host-grid and device-strip level like
 * the other tools.  src: int16, nodata -32768; twi: float32, nodata -1 (the correctly rounded logarithm: one ulp from the
 * reference's logf exactly where glibc's logf is not correctly rounded; slopearea likewise with powf). */
/* Sibling of aread8 on the same sweep (SURVEY.md 8(f) rank 3): the largest / smallest value of a grid on the D8 flow paths above
 * each cell.  File level = `int d8flowpathextremeup(char* pfile, char* safile, char* ssafile, int usemax, char* datasrc, char* lyrname,
 * int uselyrname, int lyrno, int useOutlets, int contcheck)` (src/D8flowpathextremeup.cpp:58); ssa: float32, nodata -FLT_MAX. */
int td_d8flowpathextremeup(const char* pfile, const char* safile, const char* ssafile, int usemax, const char* datasrc, const char* lyrname,
                           int uselyrname, int lyrno, int useOutlets, int contcheck);
int td_d8flowpathextremeup_host(const int16_t* p, const float* sa, float* ssa, int nx, int ny, int16_t p_nodata, int usemax, int contcheck,
                                const int* outlet_cols, const int* outlet_rows, int nout /* < 0: no outlets */);
/* Sibling of areadinf on the same sweep: decaying accumulation.  File level = `int dmarea(char* angfile, char* adecfile, char* dmfile,
 * char* datasrc, char* lyrname, int uselyrname, int lyrno, char* wfile, int useOutlets, int usew, int contcheck)`
 * (src/dinfdecayaccum.cpp:61); dsca: float32, nodata -FLT_MAX.  A cell starts from its weight (or its cell size dx) and receives
 * (float)(dm * area * p) from every contributor, dm = the contributor's decay multiplier (src/dinfdecayaccum.cpp:205-235). */
int td_dmarea(const char* angfile, const char* adecfile, const char* dmfile, const char* datasrc, const char* lyrname, int uselyrname, int lyrno,
              const char* wfile, int useOutlets, int usew, int contcheck);
int td_dinfdecayaccum_host(const float* ang, const float* dm, const float* w /*NULL unless usew*/, float* dsca, int nx, int ny, float ang_nodata,
                           float dm_nodata, const double* dxc, const double* dyc, int contcheck, const int* outlet_cols, const int* outlet_rows,
                           int nout /* < 0: no outlets */);
/* Siblings of areadinf on the same sweep: the concentration- and the transport-limited accumulation.  File level =
 * `int dsllArea(char* angfile, char* ctptfile, char* dmfile, char* datasrc, char* lyrname, int uselyrname, int lyrno, char* qfile, char* dgfile,
 * int useOutlets, int contcheck, float cSol)` (src/DinfConcLimAccum.cpp:61) and `int tlaccum(char* angfile, char* tsupfile, char* tcfile,
 * char* tlafile, char* depfile, char* cinfile, char* coutfile, char* datasrc, char* lyrname, int uselyrname, int lyrno, int useOutlets, int usec,
 * int contcheck)` (src/DinfTransLimAccum.cpp:61).  All outputs float32 with nodata -FLT_MAX.
 * ctpt: cells with q > 0 only; an indicator cell (dg > 0) has the concentration cSol, any other the float sum of p * ctpt * q * dm over its
 * contributors divided by its own q (src/DinfConcLimAccum.cpp:242-270).  tla / tdep / ctpt: transport out = min(transport in + supply,
 * capacity), deposition = the rest, concentration = load out / transport out (src/DinfTransLimAccum.cpp:237-302); cs and ctpt are
 * both NULL or both given. */
int td_dsllarea(const char* angfile, const char* ctptfile, const char* dmfile, const char* datasrc, const char* lyrname, int uselyrname, int lyrno,
                const char* qfile, const char* dgfile, int useOutlets, int contcheck, float cSol);
int td_tlaccum(const char* angfile, const char* tsupfile, const char* tcfile, const char* tlafile, const char* depfile, const char* cinfile,
               const char* coutfile, const char* datasrc, const char* lyrname, int uselyrname, int lyrno, int useOutlets, int usec, int contcheck);
int td_dinfconclimaccum_host(const float* ang, const float* dm, const float* q, const int16_t* dg, float* ctpt, int nx, int ny, float ang_nodata,
                             float dm_nodata, float q_nodata, float csol, const double* dxc, const double* dyc, int contcheck, const int* outlet_cols,
                             const int* outlet_rows, int nout /* < 0: no outlets */);
int td_dinftranslimaccum_host(const float* ang, const float* tsup, const float* tc, const float* cs /*NULL unless usec*/, float* tla, float* tdep,
                              float* ctpt /*NULL unless usec*/, int nx, int ny, float ang_nodata, float tsup_nodata, float tc_nodata, float cs_nodata,
                              const double* dxc, const double* dyc, int contcheck, const int* outlet_cols, const int* outlet_rows,
                              int nout /* < 0: no outlets */);
/* Sibling of aread8 on the same sweep: gridnet.  File level = `int gridnet(char* pfile, char* plenfile, char* tlenfile, char* gordfile,
 * char* maskfile, char* datasrc, char* lyrname, int uselyrname, int lyrno, int useMask, int useOutlets, int thresh)`
 * (src/gridnet.cpp:55); plen / tlen: float32, nodata -1; gord: int16, nodata -1.  mask (int32, NULL = none): only cells with
 * mask >= thresh are evaluated and contribute (src/gridnet.cpp:383-399).  Inputs are D8 rasters as d8flowdir writes them (no
 * direction on the grid's edge cells: the reference reads stale temporaries for neighbours beyond the left / right edge). */
int td_gridnet(const char* pfile, const char* plenfile, const char* tlenfile, const char* gordfile, const char* maskfile, const char* datasrc,
               const char* lyrname, int uselyrname, int lyrno, int useMask, int useOutlets, int thresh);
int td_gridnet_host(const int16_t* p, const int32_t* mask /*NULL unless useMask*/, int thresh, float* plen, float* tlen, int16_t* gord, int nx, int ny,
                    int16_t p_nodata, const double* dxc, const double* dyc, const int* outlet_cols, const int* outlet_rows, int nout /* < 0: no outlets */);
int td_threshold(const char* ssafile, const char* srcfile, const char* maskfile, float thresh, int usemask);
int td_twigrid(const char* slopefile, const char* areafile, const char* twifile);
int td_threshold_host(const float* ssa, const float* mask /*NULL unless usemask*/, int16_t* src, int nx, int ny, float thresh, float ssa_nodata);
int td_twi_host(const float* slp, const float* sca, float* twi, int nx, int ny, float slp_nodata, float sca_nodata);
/* The other two point-wise consumers of SURVEY.md 8(f) rank 4.  File level = `int slopearea(char* slopefile, char* scafile, char* safile,
 * float* p)` (src/SlopeArea.cpp:52; p[0] = m, p[1] = n: sa = slp^m * sca^n where both are >= 0) and `int atanbgrid(char* slopefile,
 * char* areafile, char* atanbfile)` (src/SlopeAreaRatio.cpp:49: sar = slp / sca where sca is data).  sa, sar: float32, nodata -1.
 * sar is bit-exact; sa is within a few float ulps of the reference's powf * powf (nodata masks identical). */
int td_slopearea(const char* slopefile, const char* scafile, const char* safile, const float* p /* m, n */);
int td_atanbgrid(const char* slopefile, const char* areafile, const char* atanbfile);
int td_slopearea_host(const float* slp, const float* sca, float* sa, int nx, int ny, float m, float n);
int td_slopearearatio_host(const float* slp, const float* sca, float* sar, int nx, int ny, float sca_nodata);
/* The two stream definitions besides the area threshold.  File level = `int peukerdouglas(char* felfile, char* ssfile, float* p)`
 * (src/PeukerDouglas.cpp:54; p = the smoothing weights of the centre, side and diagonal cells, default 0.4 0.1 0.05) and
 * `int lengtharea(char* plenfile, char* ad8file, char* ssfile, float* p)` (src/LengthArea.cpp:51; p[0] = M, p[1] = y: ss = 1 where
 * ad8 >= M plen^y, ad8 read as 32-bit integers; TD_ERR_ARG when the two grids do not match; the output takes ad8's georeference).
 * peukerdouglas ss: int16, 0 / 1 on every cell, nodata tag -2; lengtharea ss: int16, nodata -32768 where plen < 0.
 * Both bit-exact (lengtharea decides the cells that depend on the last bit of the power with libm's powf: see pointwise.cu). */
int td_peukerdouglas(const char* felfile, const char* ssfile, const float* p /* w_mid, w_side, w_diag */);
int td_lengtharea(const char* plenfile, const char* ad8file, const char* ssfile, const float* p /* M, y */);
int td_peukerdouglas_host(const float* fel, int16_t* ss, int nx, int ny, float fel_nodata, const float* p);
int td_lengtharea_host(const float* plen, const int32_t* ad8, int16_t* ss, int nx, int ny, float m, float y);
/* slopeavedown: the D8 slope averaged over the downslope distance dn (the downslope gradient index).  File level = `int sloped(char*
 * pfile, char* felfile, char* slpdfile, double dn)` (src/SlopeAveDown.cpp:59; TD_ERR_MISMATCH when fel and p differ in size).
 * slpd: float32, nodata MISSINGFLOAT, the georeference of p.  Host-grid level: dxc / dyc = per-row cell sizes (the distances),
 * dx / dy = the header's cell sizes (niter = dn / min(dx, dy) + 1 passes).  TD_ERR_ARG when dn is not finite or niter does not fit
 * an int.  Bit-exact; stops early, with the same result, once a pass changes nothing. */
int td_sloped(const char* pfile, const char* felfile, const char* slpdfile, double dn);
int td_slopeavedown_host(const float* fel, const int16_t* p, float* slpd, int nx, int ny, float fel_nodata, int16_t p_nodata, const double* dxc,
                         const double* dyc, double dx, double dy, double dn);
/* d8hdisttostrm / d8vdisttostrm: the distance from every cell down its D8 path to the first stream cell (src >= thresh where src,
 * read as int32, is data), horizontal (the path length) or vertical (the drop: height above the nearest drainage).  File level =
 * `int distgrid(char* pfile, char* srcfile, char* distfile, int thresh)` (src/D8HDistToStrm.cpp:57) and `int d8vdistdown(char*
 * pfile, char* felfile, char* srcfile, char* distfile, int thresh)` (src/D8VDistToStrm.cpp:58); TD_ERR_MISMATCH, after "File sizes
 * do not match", when src or fel differs from p in size.  dist: float32, nodata MISSINGFLOAT, the georeference of p.  Stream cells
 * get 0; cells whose path leaves the grid, meets a non-stream cell whose p is nodata, 0 or outside 1..8, or ends in a cycle without
 * a stream cell keep MISSINGFLOAT.  Host-grid level: dxc / dyc = per-row cell sizes (horizontal only).  One GPU takes a grid whose
 * strip, (ny + 2) * td_pitch_for(nx) cells, holds fewer than 2^32 cells (TD_ERR_ARG otherwise) and whose rasters fit its memory: 15
 * bytes per strip cell (horizontal; 19 vertical).  Bit-exact.  td_disttostrm_last_levels: the
 * BFS levels of the last host-grid call. */
int td_distgrid(const char* pfile, const char* srcfile, const char* distfile, int thresh);
int td_d8vdistdown(const char* pfile, const char* felfile, const char* srcfile, const char* distfile, int thresh);
int td_d8hdisttostrm_host(const int16_t* p, const int32_t* src, float* dist, int nx, int ny, int16_t p_nodata, int32_t src_nodata, int thresh,
                          const double* dxc, const double* dyc);
int td_d8vdisttostrm_host(const int16_t* p, const float* fel, const int32_t* src, float* dist, int nx, int ny, int16_t p_nodata, int32_t src_nodata,
                          int thresh);
long long td_disttostrm_last_levels(void);
/* dinfdistdown: the D-infinity distance from every cell down to the stream (stream cells: src, read as int16, >= 1; no threshold,
 * src's nodata not tested).  File level = `int dinfdistdown(char* angfile, char* felfile, char* slpfile, char* wfile, char* srcfile,
 * char* dtsfile, int statmethod, int typemethod, int usew, int concheck)` (src/DinfDistDown.cpp:66; slp is never opened; TD_ERR_MISMATCH,
 * after "File sizes do not match", when fel, wg or src differs from ang in size; the output takes ang's georeference).  typemethod 0 h (horizontal), 1 v (vertical: the height above the nearest
 * drainage), 2 p (Pythagoras: sqrt(h^2 + v^2)), 3 s (surface); statmethod 0 ave, 1 max, 2 min over the cell's receivers.  Host-grid
 * level: fel = NULL for h, w = NULL for no weights (ignored by v), dxc / dyc = ang's per-row cell sizes, used for the shares and the
 * distances of every mode; concheck = 1: a receiver that is off the grid or nodata (or whose fel or weight is nodata) makes the cell
 * nodata.  dd: float32, nodata MISSINGFLOAT.  Cells on a cycle of angles and every cell upslope of one keep MISSINGFLOAT.  One GPU
 * takes a grid whose strip, (ny + 2) * td_pitch_for(nx) cells, holds fewer than 2^32 cells (TD_ERR_ARG otherwise) and whose rasters
 * fit its memory: 15 bytes per strip cell for h, 19 for v and s, 23 for p, and 4 more with weights (27 for p with weights).
 * Bit-exact.  td_dinfdistdown_last_levels: the levels of the last host-grid call. */
int td_dinfdistdown(const char* angfile, const char* felfile, const char* slpfile, const char* wfile, const char* srcfile, const char* dtsfile,
                    int statmethod, int typemethod, int usew, int concheck);
int td_dinfdistdown_host(const float* ang, const float* fel, const float* w, const int16_t* src, float* dd, int nx, int ny, float ang_nodata,
                         float fel_nodata, float w_nodata, const double* dxc, const double* dyc, int statmethod, int typemethod, int concheck);
long long td_dinfdistdown_last_levels(void);
/* flowdircond: D8-conditioned elevations.  Every cell the D8 queue of p reaches gets the smallest conditioned elevation among the
 * cells that drain into it, or its own z if that is smaller, so that elevations never rise downstream along p; the other cells keep
 * their z.  A cell whose z is nodata keeps it and still drains.  File level = `int flowdircond(char* pfile, char* zfile, char*
 * zfdcfile)` (src/flowdircond.cpp:56; TD_ERR_MISMATCH when z and p differ in size).  zfdc: float32, the nodata value and the
 * georeference of z.  Bit-exact. */
int td_flowdircond(const char* pfile, const char* zfile, const char* zfdcfile);
int td_flowdircond_host(const int16_t* p, const float* z, float* zfdc, int nx, int ny, int16_t p_nodata, float z_nodata);
/* retlimflow: D-infinity retention-limited runoff, qrl = max(0, sum of p * qrl of the contributors + wg - rc) in float.  A cell whose
 * wg or rc is nodata gets nodata and passes nothing on, so every cell downstream of it stays nodata.  File level = `int
 * retlimro(char* angfile, char* wgfile, char* rcfile, char* qrlfile)` (src/RetlimFlow.cpp:53; TD_ERR_MISMATCH when a grid differs
 * in size from ang).  qrl: float32, nodata MISSINGFLOAT, the georeference of rc.  dxc / dyc: per-row cell sizes.  TD_ERR_ARG when
 * the angle nodata value is one prop() reads as a flow direction (above about -pi/4): the reference would add its share times
 * MISSINGFLOAT.  Bit-exact. */
int td_retlimro(const char* angfile, const char* wgfile, const char* rcfile, const char* qrlfile);
int td_retlimflow_host(const float* ang, const float* wg, const float* rc, float* qrl, int nx, int ny, float ang_nodata, float wg_nodata, float rc_nodata,
                       const double* dxc, const double* dyc);

/* aread8 + areadinf of one DEM in one call (no weights, no outlets), the host<->device copies overlapped with the kernels
 * on three streams: p in -> aread8 || ang in -> areadinf || ad8 out -> sca out.  Same results as the two calls above.
 * Pinned host rasters make the copies asynchronous.  (No counterpart in the reference: its tools are one process each,
 * src/aread8.cpp:56, src/areadinf.cpp:53; this is what a caller that wants both rasters of a DEM would bind.) */
int td_contributing_areas_host(const int16_t* p, const float* ang, float* ad8, float* sca, int nx, int ny, int16_t p_nodata,
                               float ang_nodata, const double* dxc, const double* dyc, int contcheck);

/* The same with outlets (-o; the outlet branches of initNeighborD8up / initNeighborDinfup,
 * src/commonLib.cpp:285-385, 137-237): only the cells upstream of the outlet cells (column, row; points
 * off the grid are ignored) are evaluated, everything else keeps the nodata value -1.  nout < 0: no
 * outlets, the whole grid.                                                                            */
int td_aread8_outlets_host(const int16_t* p, const float* w, float* ad8, int nx, int ny,
                           int16_t p_nodata, float w_nodata, int contcheck,
                           const int* outlet_cols, const int* outlet_rows, int nout);
int td_area_outlets_host(const float* ang, const float* w, float* sca, int nx, int ny,
                         float ang_nodata, float w_nodata, const double* dxc, const double* dyc,
                         int contcheck, const int* outlet_cols, const int* outlet_rows, int nout);

/* Outlet points of a data source (src/ReadOutlets.cpp:49-189 reads them through OGR): ESRI shapefile
 * (.shp, Point / PointZ / PointM) or GeoJSON Point features; a directory is a data source whose layers are
 * its .shp files.  Writes up to cap points, *n = number of points in the layer.  No GPU needed.        */
int td_outlets_read(const char* datasrc, const char* lyrname, int uselyrname, int lyrno,
                    double* x, double* y, int cap, int* n);

/* ---- 3. device-strip level ----------------------------------------------------------- */
typedef struct td_strip {
  int nx;       /* columns of the grid                                                  */
  int ny;       /* rows owned by this strip                                             */
  int pitch;    /* elements per stored row, multiple of 32, >= nx                       */
  int has_top;  /* 1 if a strip exists above (row 0 holds its last row)                 */
  int has_bot;  /* 1 if a strip exists below (row ny+1 holds its first row)             */
} td_strip;

typedef struct td_ctx td_ctx;   /* per-device scratch (frontier queues, counters) */
td_ctx* td_ctx_create(void);
void td_ctx_destroy(td_ctx*);
int td_pitch_for(int nx);        /* smallest legal pitch */
/* diagnostics: device counter i of the context (27 = tile visits of the last sweep) */
unsigned long long td_ctx_counter(td_ctx*, int i);

/* synthetic fractal DEM written straight into a strip (bench/test input generator) */
int td_gen_dem_dev(float* dem, td_strip s, int row0_global, int total_ny, unsigned seed,
                   float hurst, float tilt, void* stream);
int td_gen_weights_dev(float* w, td_strip s, int row0_global, unsigned seed, void* stream);

/* pit filling: init (src/flood.cpp:243-271) + relaxation to the fixed point (:292-479).
 * td_flood_relax_dev runs tile-local relaxation rounds until no tile of this strip changes
 * given the current halo rows; *changed_out (host) tells whether anything moved.          */
int td_flood_init_dev(td_ctx*, const float* dem, const int16_t* depmask, float* planchon,
                      td_strip s, float dem_nodata, int is_4Point, void* stream);
int td_flood_relax_dev(td_ctx*, const float* dem, float* planchon, td_strip s, int is_4Point,
                       int* changed_out, void* stream);
/* the same after the neighbours' edge rows were copied into the halo rows again: starts from the tiles next to them only */
int td_flood_relax_edges_dev(td_ctx*, const float* dem, float* planchon, td_strip s, int is_4Point,
                             int* changed_out, void* stream);

/* D8: setPosDir+calcSlope stencil (src/d8.cpp:359-409,153-177); dxc/dyc are DEVICE arrays
 * of ny doubles.  *nflat_out (host) = number of dir==0 cells in the strip.                */
int td_d8_slopes_dev(td_ctx*, const float* fel, int16_t* p, float* sd8, td_strip s,
                     float fel_nodata, const double* dxc, const double* dyc,
                     long long* nflat_out, void* stream);
/* Garbrecht-Martz flat resolution, all iterations (src/d8.cpp:302-317,459-680).
 * fel is modified like the reference modifies elevDEM.  Single strip only.              */
int td_d8_flats_dev(td_ctx*, float* fel, int16_t* p, td_strip s, const double* dxc,
                    const double* dyc, long long* nflat_left, void* stream);

/* The same over row strips (one per process).  The callbacks stand where the reference's
 * resolveflats calls linearpart::share() and MPI_Allreduce (src/d8.cpp:459-680,
 * src/linearpart.h:195-219); they are invoked on the calling thread with the stream
 * synchronised, the pointers are DEVICE pointers.  Return 0 on success.
 *   share     : first / last owned row of a strip array (ny+2 rows of pitch cells,
 *               elem_bytes per cell) -> bottom / top halo row of the strips above / below
 *   collect   : the reverse: my halo row 0 -> the strip above, my halo row ny+1 -> the strip
 *               below; recv_top / recv_bot (pitch cells, NULL at the grid edge) receive what
 *               the strips above / below hold in their halo rows for my first / last row
 *   allreduce_sum : element-wise sum of v[0..n) over all strips (host memory)
 * fel, p / ang must have current halo rows on entry; nflat_left is the global count.     */
typedef struct td_strip_comm {
  void* user;
  int (*share)(void* user, void* strip_array, int elem_bytes);
  int (*collect)(void* user, const void* strip_array, int elem_bytes, void* recv_top, void* recv_bot);
  int (*allreduce_sum)(void* user, unsigned long long* v, int n);
} td_strip_comm;
int td_d8_flats_strip_dev(td_ctx*, float* fel, int16_t* p, td_strip s, const double* dxc, const double* dyc,
                          long long* nflat_left, const td_strip_comm* comm, void* stream);
int td_dinf_flats_strip_dev(td_ctx*, float* fel, float* ang, td_strip s, const double* dxc, const double* dyc,
                            long long* nflat_left, const td_strip_comm* comm, void* stream);

/* D-infinity: setPosDirDinf/SET2/VSLOPE stencil (src/dinf.cpp:530-595,317-373,286-313) */
int td_dinf_slopes_dev(td_ctx*, const float* fel, float* ang, float* slp, td_strip s,
                       float fel_nodata, const double* dxc, const double* dyc,
                       long long* nflat_out, void* stream);
int td_dinf_flats_dev(td_ctx*, float* fel, float* ang, td_strip s, const double* dxc,
                      const double* dyc, long long* nflat_left, void* stream);

/* Row strips of a raster whose rows have different cell sizes (geographic rasters): the cell sizes of the rows just above / below
 * the strip (the neighbour strips' edge rows; <= 0 = none).  The D-infinity dependency stencil and sweep evaluate a contributor in a
 * halo row with ITS row's cell sizes like the reference (getdxdyc(jn), src/areadinf.cpp:199-201).  Call before td_area_deps_dev;
 * stays in effect for the context until changed. */
void td_set_halo_cell_sizes_dev(td_ctx*, double dx_top, double dy_top, double dx_bot, double dy_bot);

/* -o: restricts the dependency state built by *_deps_dev to the cells upstream of the outlets (host
 * arrays of grid coordinates, row 0 = first owned row); call between *_deps_dev and *_sweep_dev.       */
int td_sweep_restrict_dev(td_ctx*, td_strip s, const int* cols, const int* rows, int nout, void* stream);
/* Row strips: one round (outlet seeds with nout >= 0 in the first round; in_top / in_bot = the neighbour strips'
 * requests for my first / last row, device arrays of pitch ints or NULL; req_out = my requests to them, device,
 * 2 x pitch ints: [0,pitch) to the strip above, [pitch,2 pitch) below).  Exchange req_out like the sweeps' halo
 * counts and repeat until no strip requests anything, then call once more with finish = 1.              */
int td_sweep_restrict_round_dev(td_ctx*, td_strip s, const int* cols, const int* rows, int nout,
                                const int* in_top, const int* in_bot, int* req_out, int finish, void* stream);

/* contributing area.  *_deps_dev = initNeighborD8up / initNeighborDinfup
 * (src/commonLib.cpp:240-283, 92-136): fills the strip's dependency state inside ctx.
 * *_sweep_dev = the evaluation wavefront (src/aread8.cpp:216-304, src/areadinf.cpp:173-265)
 * run until this strip has no ready cell left.  For one strip that is the whole job.
 * *_deps_dev also initialises the output raster to its nodata value (-1).                 */
int td_aread8_deps_dev(td_ctx*, const int16_t* p, float* ad8, td_strip s, int16_t p_nodata, void* stream);
int td_aread8_sweep_dev(td_ctx*, const float* w, float* ad8, td_strip s, float w_nodata, int usew,
                        int contcheck, void* stream);
int td_area_deps_dev(td_ctx*, const float* ang, float* sca, td_strip s, float ang_nodata,
                     const double* dxc, const double* dyc, void* stream);
int td_area_sweep_dev(td_ctx*, const float* ang, const float* w, float* sca, td_strip s, int usew,
                      int contcheck, const double* dxc, void* stream);

/* Row-strip partitioned sweeps (one strip per GPU, src/aread8.cpp:280-304 / src/areadinf.cpp:241-265):
 *   td_*_deps_dev (after the halo rows of p / ang were exchanged), td_sweep_begin_dev, then rounds of
 *     td_*_sweep_run_dev      - evaluates until no cell of the strip is ready; halo_out (2*pitch ints,
 *                               zeroed by the caller) counts the decrements that crossed into the strip
 *                               above ([0,pitch)) and below ([pitch,2*pitch));
 *     (caller) exchange the first/last area rows and the halo_out arrays with the neighbour ranks;
 *     td_sweep_apply_halo_dev - applies the received decrements to the first (dec_top) / last (dec_bot)
 *                               row and queues the tiles whose cells became ready;
 *   until no rank sent a decrement (ringTerm, src/linearpart.h:344-384).                               */
int td_sweep_begin_dev(td_ctx*, td_strip s, void* stream);
int td_sweep_apply_halo_dev(td_ctx*, td_strip s, const int* dec_top, const int* dec_bot, void* stream);
int td_aread8_sweep_run_dev(td_ctx*, const float* w, float* ad8, td_strip s, float w_nodata, int usew,
                            int contcheck, int* halo_out, void* stream);
int td_area_sweep_run_dev(td_ctx*, const float* ang, const float* w, float* sca, td_strip s, int usew,
                          int contcheck, const double* dxc, int* halo_out, void* stream);

/* The five sibling sweep tools on row strips, with the same protocol: the tool's *_deps_dev (it initialises the outputs to the
 * tool's nodata), td_sweep_begin_dev, then rounds of the tool's *_sweep_run_dev(..., halo_out, ...) and td_sweep_apply_halo_dev;
 * or peer mode (td_sweep_peer_export_dev with dinf = 0 for the D8 tools, 1 for the D-infinity ones, ..., td_sweep_peer_begin_dev,
 * a barrier, one *_sweep_run_dev per rank).  Every round the caller exchanges, with the halo_out arrays, the first / last owned
 * rows of the value the sweep carries (ssa, plen / tlen / the Strahler order, dsca, ctpt, tla) into the neighbours' halo rows.
 * Inputs read at a neighbour cell need valid halo rows before the deps call (like p / ang): listed per tool.  D-infinity tools on
 * rasters whose rows have different cell sizes call td_set_halo_cell_sizes_dev first.  dxc / dyc: DEVICE arrays of ny doubles.
 *
 * d8flowpathextremeup: halo rows of p.  ssa starts as MISSINGFLOAT; sa needs no halo rows.                                     */
int td_d8flowpathextremeup_deps_dev(td_ctx*, const int16_t* p, float* ssa, td_strip s, int16_t p_nodata, void* stream);
int td_d8flowpathextremeup_sweep_run_dev(td_ctx*, const float* sa, float* ssa, td_strip s, int usemax, int contcheck, int* halo_out,
                                         void* stream);
/* flowdircond: halo rows of p and of z (the deps call starts zfdc as a copy of the whole strip of z, halo rows included; the sweep
 * reads a halo row's value only after an exchange or a peer delivery) and overwrites the cells it evaluates.                    */
int td_flowdircond_deps_dev(td_ctx*, const int16_t* p, const float* z, float* zfdc, td_strip s, int16_t p_nodata, void* stream);
int td_flowdircond_sweep_run_dev(td_ctx*, const float* z, float* zfdc, td_strip s, float z_nodata, int* halo_out, void* stream);
/* retlimflow: halo rows of ang (wg, rc: owned rows only).  qrl starts as MISSINGFLOAT.  The deps call reads dxc / dyc back to the
 * host to check the angle nodata value (it synchronises the stream) and blocks the cells whose wg or rc is nodata.              */
int td_retlimflow_deps_dev(td_ctx*, const float* ang, const float* wg, const float* rc, float* qrl, td_strip s, float ang_nodata,
                           float wg_nodata, float rc_nodata, const double* dxc, const double* dyc, void* stream);
int td_retlimflow_sweep_run_dev(td_ctx*, const float* ang, const float* wg, const float* rc, float* qrl, td_strip s, float wg_nodata,
                                float rc_nodata, const double* dxc, int* halo_out, void* stream);
/* dinfdecayaccum: halo rows of ang and dm (w: owned rows only, NULL = no weights).  dsca starts as MISSINGFLOAT.                */
int td_dinfdecayaccum_deps_dev(td_ctx*, const float* ang, float* dsca, td_strip s, float ang_nodata, const double* dxc,
                               const double* dyc, void* stream);
int td_dinfdecayaccum_sweep_run_dev(td_ctx*, const float* ang, const float* dm, const float* w, float* dsca, td_strip s,
                                    float dm_nodata, int contcheck, const double* dxc, int* halo_out, void* stream);
/* dinfconclimaccum: halo rows of ang, dm and q (dg: owned rows only).  ctpt starts as MISSINGFLOAT.                              */
int td_dinfconclimaccum_deps_dev(td_ctx*, const float* ang, float* ctpt, td_strip s, float ang_nodata, const double* dxc,
                                 const double* dyc, void* stream);
int td_dinfconclimaccum_sweep_run_dev(td_ctx*, const float* ang, const float* dm, const float* q, const int16_t* dg, float* ctpt,
                                      td_strip s, float dm_nodata, float q_nodata, float csol, int contcheck, const double* dxc,
                                      int* halo_out, void* stream);
/* dinftranslimaccum: halo rows of ang (tsup, tc, cs: owned rows only).  tla, tdep and ctpt start as MISSINGFLOAT.  With -cs
 * (cs and ctpt given) the caller exchanges the first / last owned rows of ctpt every round too, together with those of tla.    */
int td_dinftranslimaccum_deps_dev(td_ctx*, const float* ang, float* tla, float* tdep, float* ctpt /*NULL unless cs*/, td_strip s,
                                  float ang_nodata, const double* dxc, const double* dyc, void* stream);
int td_dinftranslimaccum_sweep_run_dev(td_ctx*, const float* ang, const float* tsup, const float* tc, const float* cs /*NULL or*/,
                                       float* tla, float* tdep, float* ctpt /*with cs*/, td_strip s, float tsup_nodata, float tc_nodata,
                                       float cs_nodata, int contcheck, const double* dxc, int* halo_out, void* stream);
/* gridnet: three sweeps in turn (which = 0 longest path plen, 1 total path tlen, 2 Strahler order), each with its own
 * td_gridnet_deps_dev + begin + rounds (or peer begin + barrier + run), then td_gridnet_order_dev turns the third sweep's floats
 * into gord (int16, -1 = nodata).  Halo rows of p, and of the mask when there is one: td_gridnet_mask_dev turns it (int32, with
 * halo rows) into the 0 / 1 grid `ok` (NULL = no mask) of the owned rows and the halo rows.  dist: DEVICE array of ny x 8 floats,
 * dist[row][k - 1] = (float)sqrt(dxc^2 d1[k]^2 + dyc^2 d2[k]^2) of the strip's own rows (src/gridnet.cpp:190-200).  outlets = 1
 * after td_sweep_restrict_dev (single strip).  Every sweep starts its output as -1.                                            */
int td_gridnet_mask_dev(td_ctx*, const int32_t* mask, float* ok, td_strip s, int thresh, void* stream);
int td_gridnet_deps_dev(td_ctx*, const int16_t* p, float* out, td_strip s, int16_t p_nodata, void* stream);
int td_gridnet_sweep_run_dev(td_ctx*, int which, const float* ok /*NULL = no mask*/, const float* dist, float* out, td_strip s,
                             int outlets, int* halo_out, void* stream);
int td_gridnet_order_dev(td_ctx*, const float* order, const int16_t* p, const float* ok, int16_t* gord, td_strip s, int16_t p_nodata,
                         int outlets, void* stream);

/* point-wise consumers on device strips (pointwise.cu) */
int td_threshold_dev(td_ctx*, const float* ssa, const float* mask, int16_t* src, td_strip s, float thresh, float ssa_nodata, void* stream);
int td_twi_dev(td_ctx*, const float* slp, const float* sca, float* twi, td_strip s, float slp_nodata, float sca_nodata, void* stream);
int td_slopearea_dev(td_ctx*, const float* slp, const float* sca, float* sa, td_strip s, float m, float n, void* stream);
int td_slopearearatio_dev(td_ctx*, const float* slp, const float* sca, float* sar, td_strip s, float sca_nodata, void* stream);
/* peukerdouglas on row strips: td_peukerdouglas_smooth_dev (fel with valid halo rows -> the smoothed grid sm; p: host array of the
 * three weights), then the caller copies the first / last owned rows of sm into the neighbours' halo rows (the reference's second
 * share()), then td_peukerdouglas_mark_dev (sm -> ss).  fel_nodata: the elevations' nodata value, in both passes.               */
int td_peukerdouglas_smooth_dev(td_ctx*, const float* fel, float* sm, td_strip s, float fel_nodata, const float* p, void* stream);
int td_peukerdouglas_mark_dev(td_ctx*, const float* sm, int16_t* ss, td_strip s, float fel_nodata, void* stream);
/* td_twi_dev, td_slopearea_dev and td_lengtharea_dev synchronise the stream: they read back the number of cells they leave to
 * the host (a logarithm or power too close to a float midpoint; a length-area decision that depends on the last bit of powf) and
 * decide those there (pointwise.cu).                                                                                             */
int td_lengtharea_dev(td_ctx*, const float* plen, const int32_t* ad8, int16_t* ss, td_strip s, float m, float y, void* stream);
/* slopeavedown on a strip (slopeavedown.cu).  First the D8 dependency stencil and sweep of p on the same context (td_aread8_deps_dev,
 * then td_aread8_sweep_dev or the row-strip / peer protocol): the cells the sweep evaluates are the cells the reference's queue
 * processes.  Then td_slopeavedown_init_dev (p and fel with valid halo rows) writes code (one byte per strip cell), both state
 * buffers ed_dd0 and ed_dd1 (two floats per strip cell: the elevation and the distance carried up from downslope, the halo rows
 * included) and sd (MISSINGFLOAT).  Each td_slopeavedown_pass_dev is one of the reference's passes: state in -> state out (swap the
 * two between passes), sd updated in place; *changed (host) = whether any bit of the state or sd changed (it synchronises the
 * stream).  On row strips the caller copies the first / last owned rows of the pass's output state (8 bytes per cell) into the
 * neighbours' halo rows between passes (the reference's ed->share(); dd->share()).  dist: device table of the strip's own rows,
 * dist[8 * (row - 1) + k - 1] = (float)sqrt(d1[k]^2 dxc^2 + d2[k]^2 dyc^2).  td_slopeavedown_niter: the reference's pass count. */
int td_slopeavedown_init_dev(td_ctx*, const int16_t* p, const float* fel, uint8_t* code, float* ed_dd0, float* ed_dd1, float* sd, td_strip s,
                             int16_t p_nodata, float fel_nodata, void* stream);
int td_slopeavedown_pass_dev(td_ctx*, const uint8_t* code, const float* fel, const float* ed_dd_in, float* ed_dd_out, float* sd, td_strip s,
                             const float* dist, double dn, int* changed, void* stream);
int td_slopeavedown_niter(double dn, double dx, double dy, int* niter);
/* d8hdisttostrm / d8vdisttostrm on a strip (disttostrm.cu).  td_disttostrm_seed_dev writes dist (MISSINGFLOAT, 0 on the owned stream
 * cells) and code (one byte per strip cell) and starts the BFS frontier with the stream cells; td_disttostrm_levels_dev first gives
 * the owned edge-row cells whose receiver lies in a halo row of dist that holds a value their values, then runs BFS levels until the
 * frontier is empty (a batch of levels per host read-back).  vertical = 0: rowdist = the device table of the strip's own rows
 * (td_slopeavedown_pass_dev's dist); vertical = 1: fel with valid halo rows.  On row strips the caller copies the first / last owned
 * rows of dist into the neighbours' halo rows after each levels call and repeats until no strip added a cell: *cells (may be NULL) =
 * the cells that joined the frontier since the previous call, the seeds included; *levels (may be NULL) = the non-empty levels run.
 * The frontier lives on the context (its listA / listB): nothing else may run on it between the seed and the last levels call. */
int td_disttostrm_seed_dev(td_ctx*, const int16_t* p, const int32_t* src, float* dist, uint8_t* code, td_strip s, int thresh, int16_t p_nodata,
                           int32_t src_nodata, void* stream);
int td_disttostrm_levels_dev(td_ctx*, int vertical, const uint8_t* code, const float* fel, const float* rowdist, float* dist, td_strip s,
                             unsigned long long* cells, long long* levels, void* stream);
/* dinfdistdown on a strip (dinfdistdown.cu).  td_dinfdistdown_seed_dev loads the strip's row angles from dxc / dyc (device arrays, one
 * per owned row; td_set_halo_cell_sizes_dev gives the halo rows theirs), writes dd (and dd2, the vertical values, in the p mode; NULL
 * otherwise) as MISSINGFLOAT and state (one byte per strip cell: the receivers, the receivers not yet evaluated, the stream bit; the
 * strip's cells are a multiple of 4), and starts the frontier with the owned cells that wait for no receiver.  ang needs valid halo
 * rows.  td_dinfdistdown_levels_dev runs levels until the frontier is empty: rowdist = the device table of the strip's own rows
 * (td_slopeavedown_pass_dev's dist; unused by v), fel (v, p, s) and w (NULL: no weights) with valid halo rows; halo_out (2 pitch ints,
 * zeroed by the caller; NULL on a strip without neighbours) counts the decrements of the donors in row 0 ([0, pitch), for the strip
 * above) and row ny + 1 ([pitch, 2 pitch), for the strip below).  *cells / *levels as td_disttostrm_levels_dev.  On row strips the
 * caller then hands halo_out and the first / last owned rows of dd (and dd2) to the neighbours, puts the rows it receives into the
 * halo rows, gives the decrements it receives to td_dinfdistdown_edge_dev (dec_top for the first owned row, dec_bot for the last,
 * NULL where there is no neighbour), which starts the next levels from the cells they release, and repeats until no strip handed a
 * decrement over.  p mode: td_dinfdistdown_pythagoras_dev then turns dd into sqrt(dd^2 + dd2^2).  The frontier lives on the context
 * (its listA / listB, shared with disttostrm): nothing else may run on it between the seed and the last levels call. */
int td_dinfdistdown_seed_dev(td_ctx*, const float* ang, const int16_t* src, float* dd, float* dd2, uint8_t* state, td_strip s, float ang_nodata,
                             const double* dxc, const double* dyc, void* stream);
int td_dinfdistdown_levels_dev(td_ctx*, int typemethod, int statmethod, const float* ang, const float* fel, const float* w, const float* rowdist,
                               float* dd, float* dd2, uint8_t* state, td_strip s, float fel_nodata, float w_nodata, int concheck, int* halo_out,
                               unsigned long long* cells, long long* levels, void* stream);
int td_dinfdistdown_edge_dev(td_ctx*, uint8_t* state, const int* dec_top, const int* dec_bot, td_strip s, void* stream);
int td_dinfdistdown_pythagoras_dev(td_ctx*, float* dd, const float* dd2, td_strip s, void* stream);

/* Peer mode (one process per GPU on one NVSwitch box): every rank exports the IPC handles of the buffers
 * its neighbours write (counts, tile scheduler, halo areas, rank 0 also the global pending counter), opens
 * its neighbours' (which: 0 = strip above, 1 = strip below, 2 = counter owner; NULL handles = none / self),
 * then td_sweep_peer_begin_dev + a barrier + ONE td_*_sweep_run_dev per rank complete the whole sweep:
 * tiles deliver into the neighbour GPU over NVLink (remote store + system-scope atomics) and queue its
 * tiles directly.  td_sweep_peer_off_dev returns to the round-based mode.                                */
int td_sweep_peer_export_dev(td_ctx*, td_strip s, int dinf, unsigned char* handles_5x64, int* meta_8, void* stream);
int td_sweep_peer_connect_dev(td_ctx*, int which, const unsigned char* handles_5x64, const int* meta_8);
int td_sweep_peer_begin_dev(td_ctx*, td_strip s, void* stream);
void td_sweep_peer_off_dev(td_ctx*);

#ifdef __cplusplus
}
#endif
#endif /* TAUDEM_B200_H */
