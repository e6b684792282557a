// Command line front ends: pitremove, d8flowdir, dinfflowdir, aread8, areadinf (+ the point-wise consumers threshold, twi, slopearea, slopearearatio,
// the sibling sweep tools, the stream definitions peukerdouglas and lengtharea, slopeavedown, flowdircond, retlimflow, d8hdisttostrm,
// d8vdisttostrm and dinfdistdown).
// Same flags, same two invocation styles and the same "print usage and exit(0)" error
// behaviour as the reference mains (src/PitRemovemn.cpp:48-172, src/D8FlowDirmn.cpp:49-146,
// src/DinfFlowDirmn.cpp:54-147, src/aread8mn.cpp:49-193, src/areadinfmn.cpp:49-178);
// one table-driven parser instead of five strcmp chains.  Build with -DTOOL_<name>.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include "../../../include/taudem_b200.h"

// the outputs are on disk: leave without tearing the CUDA context down (hundreds of milliseconds with gigabytes allocated)
static int done() { fflush(stdout); fflush(stderr); _exit(0); return 0; }

#define MAXLN 4096

struct Opt {
  const char* flag;
  int kind;        // 0 = file name, 1 = switch, 2 = integer, 3 = float (ival points to a float), 4 = two floats, 5 = three floats,
                   // 6 = double (ival points to a double), 7 = two method tokens (ival points to {typemethod, statmethod}: method_token)
  char* sval;      // kind 0
  int* ival;       // kind 1 (set to `set`) / kind 2 (parsed) / kind 0 (set to `set` when given, may be NULL)
  int set;
};

static void usage(const char* prog);

// one token of dinfdistdown's -m (src/DinfDistDownmn.cpp:138-195): h / v / p / s set the method, ave / max / min the statistic, anything
// else leaves both as they are
static void method_token(const char* t, int* m) {
  if (strcmp(t, "h") == 0) m[0] = 0;
  else if (strcmp(t, "v") == 0) m[0] = 1;
  else if (strcmp(t, "p") == 0) m[0] = 2;
  else if (strcmp(t, "s") == 0) m[0] = 3;
  if (strcmp(t, "ave") == 0) m[1] = 0;
  else if (strcmp(t, "max") == 0) m[1] = 1;
  else if (strcmp(t, "min") == 0) m[1] = 2;
}

// argc == 2 -> "simple usage" (nothing parsed, names derived with nameadd);
// argc  > 2 -> flags; unknown flag or missing value -> usage, exit(0).
static void parse(int argc, char** argv, Opt* opts, int nopts) {
  if (argc < 2) {
    printf("Error: To run this program, use either the Simple Usage option or\n");
    printf("the Usage with Specific file names option\n");
    usage(argv[0]);
  }
  int i = argc > 2 ? 1 : 2;
  while (argc > i) {
    Opt* o = NULL;
    for (int k = 0; k < nopts; k++) if (strcmp(argv[i], opts[k].flag) == 0) o = &opts[k];
    if (!o) usage(argv[0]);
    i++;
    if (o->kind == 1) { *o->ival = o->set; continue; }
    if (argc <= i) usage(argv[0]);
    if (o->kind == 0) { strncpy(o->sval, argv[i], MAXLN - 1); o->sval[MAXLN - 1] = 0; if (o->ival) *o->ival = o->set; }
    else if (o->kind == 3) sscanf(argv[i], "%f", (float*)o->ival);
    else if (o->kind == 6) sscanf(argv[i], "%lf", (double*)o->ival);
    else if (o->kind == 4) { if (argc <= i + 1) usage(argv[0]); sscanf(argv[i], "%f", (float*)o->ival); i++; sscanf(argv[i], "%f", (float*)o->ival + 1); }
    else if (o->kind == 7) { if (argc <= i + 1) usage(argv[0]); method_token(argv[i], o->ival); i++; method_token(argv[i], o->ival); }
    else if (o->kind == 5) { if (argc <= i + 2) usage(argv[0]); for (int k = 0; k < 3; ++k, ++i) sscanf(argv[i], "%f", (float*)o->ival + k); i--; }
    else sscanf(argv[i], "%d", o->ival);
    i++;
  }
}

#if defined(TOOL_pitremove)
static void usage(const char* prog) {
  printf("Simple use:\n %s <demfile>\n", prog);
  printf("Simple use derives the output name by inserting 'fel' into the input file name;\n");
  printf("a depression mask or 4 way filling cannot be requested this way.\n\n");
  printf("General use with specific file names:\n %s -z <demfile> -fel <newfile> [-depmask <maskfile>] [ -4way] [-v] \n", prog);
  printf("<demfile> is the name of the input elevation grid file.\n");
  printf("<newfile> is the output elevation grid with pits filled.\n");
  printf("<depmaskfile> is depression mask indicator grid.\n");
  printf("-4way (optional) is flag to set 4 way depression filling.\n");
  printf("-v (optional) is flag to set verbose (more detailed) output messages.\n");
  exit(0);
}
int main(int argc, char** argv) {
  static char dem[MAXLN], fel[MAXLN], mask[MAXLN];
  int verbose = 0, four = 0, use_mask = 0;
  Opt opts[] = {{"-z", 0, dem, NULL, 0}, {"-fel", 0, fel, NULL, 0}, {"-v", 1, NULL, &verbose, 1},
                {"-4way", 1, NULL, &four, 1}, {"-depmask", 0, mask, &use_mask, 1}};
  parse(argc, argv, opts, 5);
  if (argc == 2) { strncpy(dem, argv[1], MAXLN - 1); td_nameadd(fel, argv[1], "fel"); }
  if (verbose) {
    printf("On input demfile: %s\n", dem);
    printf("On input newfile: %s\n", fel);
    printf("%ssing mask file: %s\n", use_mask ? "U" : "Not U", use_mask ? mask : "N/A");
    fflush(stdout);
  }
  int err = td_flood(dem, fel, "", 0, verbose, four, use_mask, mask);
  if (err != 0) printf("PitRemove error %d\n", err);
  return done();
}

#elif defined(TOOL_d8flowdir)
static void usage(const char* prog) {
  printf("Simple Usage:\n %s <basefilename>\n", prog);
  printf("Usage with specific file names:\n %s -fel <demfile>\n", prog);
  printf("-sd8 <slopefile> -p <angfile> [-sfdr <flowfile>]\n");
  printf("<basefilename> is the name of the raw digital elevation model\n");
  printf("<demfile> is the pit filled or carved DEM input file.\n");
  printf("<slopefile> is the slope output file.\n");
  printf("<pointfile> is the output d8 flow direction file.\n");
  printf("[-sfdr <flowfile>] is the optional user imposed stream flow direction file.\n");
  printf("Suffixes appended to the base name in simple usage: fel (input), sd8, p (outputs)\n");
  exit(0);
}
int main(int argc, char** argv) {
  static char dem[MAXLN], p[MAXLN], sd8[MAXLN], flow[MAXLN];
  int useflow = 0;
  Opt opts[] = {{"-fel", 0, dem, NULL, 0}, {"-sd8", 0, sd8, NULL, 0}, {"-p", 0, p, NULL, 0}, {"-sfdr", 0, flow, &useflow, 1}};
  parse(argc, argv, opts, 4);
  if (argc == 2) { td_nameadd(dem, argv[1], "fel"); td_nameadd(p, argv[1], "p"); td_nameadd(sd8, argv[1], "sd8"); }
  int err = td_setdird8(dem, p, sd8, flow, useflow);
  if (err != 0) printf("setdird8 error %d\n", err);
  return done();
}

#elif defined(TOOL_dinfflowdir)
static void usage(const char* prog) {
  printf("Simple Usage:\n %s <basefilename>\n", prog);
  printf("Usage with specific file names:\n %s -fel <demfile>\n", prog);
  printf("-slp <slopefile> -ang <angfile> [-sfdr <flowfile>]\n");
  printf("<basefilename> is the name of the raw digital elevation model\n");
  printf("<demfile> is the pit filled or carved DEM input file.\n");
  printf("<slopefile> is the slope output file.\n");
  printf("<angfile> is the output D-infinity flow direction file.\n");
  printf("[-sfdr <flowfile>] is the optional user imposed stream flow direction file.\n");
  printf("Suffixes appended to the base name in simple usage: fel (input), slp, ang (outputs)\n");
  exit(0);
}
int main(int argc, char** argv) {
  static char dem[MAXLN], ang[MAXLN], slp[MAXLN], flow[MAXLN];
  int useflow = 0;
  Opt opts[] = {{"-fel", 0, dem, NULL, 0}, {"-slp", 0, slp, NULL, 0}, {"-ang", 0, ang, NULL, 0}, {"-sfdr", 0, flow, &useflow, 1}};
  parse(argc, argv, opts, 4);
  if (argc == 2) { td_nameadd(dem, argv[1], "fel"); td_nameadd(ang, argv[1], "ang"); td_nameadd(slp, argv[1], "slp"); }
  int err = td_setdir(dem, ang, slp, flow, useflow);
  if (err != 0) printf("Setdir error %d\n", err);
  return done();
}

#elif defined(TOOL_aread8) || defined(TOOL_areadinf)
#if defined(TOOL_aread8)
#define IN_FLAG "-p"
#define OUT_FLAG "-ad8"
#define IN_SUFF "p"
#define OUT_SUFF "ad8"
#define IN_DESC "<pfile> is the D8 flow direction input file."
#define OUT_DESC "<afile> is the D8 area output file."
#define CALL td_aread8
#else
#define IN_FLAG "-ang"
#define OUT_FLAG "-sca"
#define IN_SUFF "ang"
#define OUT_SUFF "sca"
#define IN_DESC "<angfile> is the D-infinity flow direction input file."
#define OUT_DESC "<scafile> is the D-infinity specific catchment area output file."
#define CALL td_area
#endif
static void usage(const char* prog) {
  printf("Simple Usage:\n %s <basefilename>\n", prog);
  printf("Usage with specific file names:\n %s %s <infile>\n", prog, IN_FLAG);
  printf("%s <outfile> [-o <outletfile>] [-lyrno <n>] [-lyrname <name>] [-wg <wfile>] [-nc]\n", OUT_FLAG);
  printf("<basefilename> is the name of the raw digital elevation model\n");
  printf("%s\n%s\n", IN_DESC, OUT_DESC);
  printf("[-o <outletfile>] is the optional outlet point input file.\n");
  printf("[-wg <wfile>] is the optional weight grid input file.\n");
  printf("The flag -nc overrides edge contamination checking\n");
  printf("Suffixes appended to the base name in simple usage: %s (input), %s (output)\n", IN_SUFF, OUT_SUFF);
  exit(0);
}
int main(int argc, char** argv) {
  static char in[MAXLN], out[MAXLN], wfile[MAXLN], datasrc[MAXLN], lyrname[MAXLN];
  int useOutlets = 0, uselyrname = 0, usew = 0, contcheck = 1, lyrno = 0;
  Opt opts[] = {{IN_FLAG, 0, in, NULL, 0},        {OUT_FLAG, 0, out, NULL, 0},          {"-o", 0, datasrc, &useOutlets, 1},
                {"-lyrno", 2, NULL, &lyrno, 0},   {"-lyrname", 0, lyrname, &uselyrname, 1}, {"-wg", 0, wfile, &usew, 1},
                {"-nc", 1, NULL, &contcheck, 0}};
  parse(argc, argv, opts, 7);
  if (argc == 2) { td_nameadd(out, argv[1], OUT_SUFF); td_nameadd(in, argv[1], IN_SUFF); }
  int err = CALL(in, out, datasrc, lyrname, uselyrname, lyrno, wfile, useOutlets, usew, contcheck);
  if (err != 0) printf("area error %d\n", err);
  return done();
}
#elif defined(TOOL_d8flowpathextremeup)
// src/D8FlowPathExtremeUpmn.cpp:57-174
static void usage(const char* prog) {
  printf("Simple Use:\n %s <basefilename>\n", prog);
  printf("Use with specific file names:\n %s -p <pfile>\n", prog);
  printf("-sa <safile> -ssa <ssafile> [-min] [-nc] [-o <outletsfile>]\n");
  printf("<basefilename> is the name of the base digital elevation model without suffixes for simple input. Suffixes 'p', 'sa' and 'ssa' will be appended. \n");
  printf("<pfile> is the name of D8 flow directions file.\n");
  printf("<safile> is the name of input file with values from which extreme upslope is to be found.\n");
  printf("<ssa> is the name of the output file with extreme upslope values.\n");
  printf("-min indicates to search for a minimum (default is max)\n");
  printf("-nc indicates to override edge contamination checking (checking is on by default)\n");
  exit(0);
}
int main(int argc, char** argv) {
  static char pf[MAXLN], sa[MAXLN], ssa[MAXLN], datasrc[MAXLN], lyrname[MAXLN];
  int useOutlets = 0, uselyrname = 0, usemax = 1, contcheck = 1, lyrno = 0;
  if (argc < 2) usage(argv[0]);
  Opt opts[] = {{"-p", 0, pf, NULL, 0}, {"-sa", 0, sa, NULL, 0}, {"-ssa", 0, ssa, NULL, 0}, {"-o", 0, datasrc, &useOutlets, 1},
                {"-lyrno", 2, NULL, &lyrno, 0}, {"-lyrname", 0, lyrname, &uselyrname, 1}, {"-min", 1, NULL, &usemax, 0}, {"-nc", 1, NULL, &contcheck, 0}};
  parse(argc, argv, opts, 8);
  if (argc == 2) { td_nameadd(pf, argv[1], "p"); td_nameadd(sa, argv[1], "sa"); td_nameadd(ssa, argv[1], "ssa"); }
  int err = td_d8flowpathextremeup(pf, sa, ssa, usemax, datasrc, lyrname, uselyrname, lyrno, useOutlets, contcheck);
  if (err != 0) printf("Flow Path Extreme Up Error %d\n", err);
  return done();
}

#elif defined(TOOL_gridnet)
// src/gridnetmn.cpp:51-215
static void usage(const char* prog) {
  printf("Simple Usage:\n %s <basefilename>\n", prog);
  printf("<basefilename> is the name of the raw digital elevation model\n");
  printf("The following are appended to the file names\nbefore the files are opened:\n");
  printf("p   D8 flow direction output file\nplen   the longest flow length upstream of each point output file.\n");
  printf("tlen   the total path length upstream of each point output file.\ngord   the grid of strahler order output file.\n\n");
  printf("Usage with specific file names:\n %s -p <pfile>\n", prog);
  printf("-plen <plenfile> -tlen <tlenfile> -gord <gordfile> [-o <outletfine>] [-lyrname <layer name>] [-lyrno <layer number>] [-mask <maskfile> [-thresh <threshold>]]\n");
  printf("<pfile> is the D8 flow direction input file.\n");
  printf("[-mask <maskfile> [-thresh <threshold>]].  maskfile is an optional mask grid input file; the grid network is evaluated for\n");
  printf("grid cells where values of the maskfile grid read as 4 byte integers are >= threshold.\n");
  exit(0);
}
int main(int argc, char** argv) {
  static char pf[MAXLN], plen[MAXLN], tlen[MAXLN], gord[MAXLN], maskfile[MAXLN], datasrc[MAXLN], lyrname[MAXLN];
  int useOutlets = 0, uselyrname = 0, useMask = 0, lyrno = 0, thresh = 0, havethresh = 0;
  if (argc < 2) usage(argv[0]);
  Opt opts[] = {{"-p", 0, pf, NULL, 0}, {"-plen", 0, plen, NULL, 0}, {"-tlen", 0, tlen, NULL, 0}, {"-gord", 0, gord, NULL, 0}, {"-o", 0, datasrc, &useOutlets, 1},
                {"-lyrno", 2, NULL, &lyrno, 0}, {"-lyrname", 0, lyrname, &uselyrname, 1}, {"-mask", 0, maskfile, &useMask, 1}, {"-thresh", 2, NULL, &thresh, 0}};
  parse(argc, argv, opts, 9);
  for (int i = 1; i < argc; ++i) if (strcmp(argv[i], "-thresh") == 0) havethresh = 1;
  if (useMask && !havethresh) usage(argv[0]);          // src/gridnetmn.cpp:160-166: -mask must be followed by -thresh
  if (argc == 2) { td_nameadd(pf, argv[1], "p"); td_nameadd(plen, argv[1], "plen"); td_nameadd(tlen, argv[1], "tlen"); td_nameadd(gord, argv[1], "gord"); }
  int err = td_gridnet(pf, plen, tlen, gord, maskfile, datasrc, lyrname, uselyrname, lyrno, useMask, useOutlets, thresh);
  if (err != 0) printf("gridnet error %d\n", err);
  return done();
}

#elif defined(TOOL_dinfdecayaccum)
// src/DinfDecayAccummn.cpp:51-192
static void usage(const char* prog) {
  printf("Simple Usage:\n %s <basefilename>\n", prog);
  printf("Usage with specific file names:\n %s -ang <angfile>\n", prog);
  printf("-dm <dmfile> -dsca <adecfile> [-o <outletshapefile>] [-wg <wfile>] [-nc]\n");
  printf("<basefilename> is the name of the raw digital elevation model\n");
  printf("<angfile> is the D-infinity flow direction input file.\n");
  printf("<dmfile> is the decay multiplier input grid file.\n");
  printf("<adecfile> is the decayed specific catchment area output grid file.\n");
  printf("[-o <outletshapefile>] is the optional outlet shape input file.\n");
  printf("[-wg <wfile>] is the optional weight grid input file.\n");
  printf("The flag -nc overrides edge contamination checking\n");
  printf("The following are appended to the file names before the files are opened:\n");
  printf("ang    D-infinity flow direction input file\ndm    decay multiplier input file\ndsca   decayed specific catchment area output file\n");
  exit(0);
}
int main(int argc, char** argv) {
  static char ang[MAXLN], dm[MAXLN], dsca[MAXLN], wfile[MAXLN], datasrc[MAXLN], lyrname[MAXLN];
  int useOutlets = 0, uselyrname = 0, usew = 0, contcheck = 1, lyrno = 0;
  if (argc < 2) usage(argv[0]);
  Opt opts[] = {{"-ang", 0, ang, NULL, 0}, {"-dm", 0, dm, NULL, 0}, {"-dsca", 0, dsca, NULL, 0}, {"-wg", 0, wfile, &usew, 1}, {"-o", 0, datasrc, &useOutlets, 1},
                {"-lyrno", 2, NULL, &lyrno, 0}, {"-lyrname", 0, lyrname, &uselyrname, 1}, {"-nc", 1, NULL, &contcheck, 0}};
  parse(argc, argv, opts, 8);
  if (argc == 2) { td_nameadd(ang, argv[1], "ang"); td_nameadd(dm, argv[1], "dm"); td_nameadd(dsca, argv[1], "dsca"); }
  int err = td_dmarea(ang, dsca, dm, datasrc, lyrname, uselyrname, lyrno, wfile, useOutlets, usew, contcheck);
  if (err != 0) printf("area error %d\n", err);
  return done();
}

#elif defined(TOOL_dinfconclimaccum)
// src/DinfConcLimAccummn.cpp:50-221
static void usage(const char* prog) {
  printf("Simple Usage:\n %s <basefilename>\n", prog);
  printf("Usage with specific file names:\n %s -ang <angfile>\n", prog);
  printf("-dg <indicatorFile> -dm <dmfile> -ctpt <afile>\n");
  printf("-q <qfile> [-o <outletshapefile>] [-csol <cSol>] [<-nc>]\n");
  printf("<basefilename> is the name of the raw digital elevation model\n");
  printf("<angfile> is the D-infinity flow direction input file.\n");
  printf("<indicatorFile> is the disturbance indicator input grid file.\n");
  printf("<dmfile> is the decay multiplier input grid file.\n");
  printf("<ctptfile> is the concentration output grid file.\n");
  printf("<qfile> is the specific discharge input grid file.\n");
  printf("<outletshapefile> is the optional outlet shape input file.\n");
  printf("<cSol> is the optional concentration threshold.\n");
  printf("The flag -nc overrides edge contamination checking\n");
  printf("The following are appended to the file names\nbefore the files are opened:\n");
  printf("ang    D-infinity flow direction input file\ndg     Disturbance indicator input file\ndm     Decay multiplier grid (input)\n");
  printf("q      Specific discharge grid (input)\nctpt   Concentration grid (output)\n");
  exit(0);
}
int main(int argc, char** argv) {
  static char ang[MAXLN], ctpt[MAXLN], dm[MAXLN], q[MAXLN], dg[MAXLN], datasrc[MAXLN], lyrname[MAXLN];
  int useOutlets = 0, uselyrname = 0, lyrno = 0, contcheck = 1;
  float csol = 1.f;
  Opt opts[] = {{"-ang", 0, ang, NULL, 0}, {"-dg", 0, dg, NULL, 0}, {"-dm", 0, dm, NULL, 0}, {"-ctpt", 0, ctpt, NULL, 0}, {"-q", 0, q, NULL, 0},
                {"-csol", 3, NULL, (int*)&csol, 0}, {"-o", 0, datasrc, &useOutlets, 1}, {"-lyrno", 2, NULL, &lyrno, 0},
                {"-lyrname", 0, lyrname, &uselyrname, 1}, {"-nc", 1, NULL, &contcheck, 0}};
  parse(argc, argv, opts, 10);
  if (argc == 2) { td_nameadd(ang, argv[1], "ang"); td_nameadd(dg, argv[1], "dg"); td_nameadd(dm, argv[1], "dm"); td_nameadd(q, argv[1], "q"); td_nameadd(ctpt, argv[1], "ctpt"); }
  int err = td_dsllarea(ang, ctpt, dm, datasrc, lyrname, uselyrname, lyrno, q, dg, useOutlets, contcheck, csol);
  if (err != 0) printf("area error %d\n", err);
  return done();
}

#elif defined(TOOL_dinftranslimaccum)
// src/DinfTransLimAccummn.cpp:51-234
static void usage(const char* prog) {
  printf("Simple Usage:\n %s <basefilename>\n", prog);
  printf("Usage with specific file names:\n %s -ang <pfile>\n", prog);
  printf("-tsup <wfile> -tc <tcfile> [-cs <cfile> -ctpt <coutfile>]\n");
  printf("-tla <tlafile> -tdep <depfile> [-o <shfile>] [<-nc>]\n");
  printf("<basefilename> is the name of the raw digital elevation model\n");
  printf("<angfile> is the D-infinity flow direction input file.\n");
  printf("<wfile> is the input transport supply grid file.\n");
  printf("<tcfile> is the input transport capacity grid file.\n");
  printf("<cfile> is the optional input concentration grid file.\n");
  printf("<coutfile> is the optional output concentration grid file.\n");
  printf("<tlafile> is the output transport limitted accumulation grid file.\n");
  printf("<depfile> is the output deposition grid file.\n");
  printf("<shfile> is the optional outlet shapefile.\n");
  printf("The flag -nc overrides edge contamination checking\n");
  printf("The following are appended to the file names\nbefore the files are opened:\n");
  printf("ang    D-infinity flow direction input file\ntsup   Input transport supply grid\ntc     Input transport capacity grid\n");
  printf("tla    Output transport limitted accumulation grid\ntdep   output deposition grid\n");
  exit(0);
}
int main(int argc, char** argv) {
  static char ang[MAXLN], tsup[MAXLN], tc[MAXLN], tla[MAXLN], dep[MAXLN], cin[MAXLN], cout[MAXLN], datasrc[MAXLN], lyrname[MAXLN];
  int useOutlets = 0, usec = 0, compctpt = 0, uselyrname = 0, lyrno = 0, contcheck = 1;
  Opt opts[] = {{"-ang", 0, ang, NULL, 0}, {"-tsup", 0, tsup, NULL, 0}, {"-tc", 0, tc, NULL, 0}, {"-cs", 0, cin, &usec, 1}, {"-ctpt", 0, cout, &compctpt, 1},
                {"-tla", 0, tla, NULL, 0}, {"-tdep", 0, dep, NULL, 0}, {"-o", 0, datasrc, &useOutlets, 1}, {"-lyrno", 2, NULL, &lyrno, 0},
                {"-lyrname", 0, lyrname, &uselyrname, 1}, {"-nc", 1, NULL, &contcheck, 0}};
  parse(argc, argv, opts, 11);
  if (argc == 2) { td_nameadd(ang, argv[1], "ang"); td_nameadd(tsup, argv[1], "tsup"); td_nameadd(tc, argv[1], "tc"); td_nameadd(tla, argv[1], "tla"); td_nameadd(dep, argv[1], "tdep"); }
  usec = usec * compctpt;            // both -cs and -ctpt, or no concentration at all (src/DinfTransLimAccummn.cpp:202)
  int err = td_tlaccum(ang, tsup, tc, tla, dep, cin, cout, datasrc, lyrname, uselyrname, lyrno, useOutlets, usec, contcheck);
  if (err != 0) printf("tlaccum error %d\n", err);
  return done();
}

#elif defined(TOOL_threshold)
// src/Thresholdmn.cpp:50-130 (its usage text names the flags wrongly; the flags themselves are -ssa -src -thresh -mask)
static void usage(const char* prog) {
  printf("Simple Use:\n %s <basefilename>\n", prog);
  printf("Use with specific file names:\n %s -fel <ssafile>\n", prog);
  printf("-ss <srcfile> [-thresh <thresholdvalue>] [-mask <maskfile>]\n");
  printf("<basefilename> is the name of the base digital elevation model without suffixes for simple input. Suffixes 'ssa' and 'src' will be appended. \n");
  printf("<ssafile> is the name of file to be thresholded.\n");
  printf("<srcfile> is the name of file with the thresholded output.\n");
  printf("<maskfile> is the name of a file that masks the domain.\n");
  printf("<thresholdvalue> is the value of the threshold.\n");
  printf("The threshold logic is src = ((ssa >= thresh) & (mask >=0)) ? 1:0.\n");
  exit(0);
}
int main(int argc, char** argv) {
  static char ssa[MAXLN], src[MAXLN], mask[MAXLN];
  int usemask = 0;
  float thresh = 100.f;
  if (argc < 2) usage(argv[0]);                 // (no "Error:" preamble in this tool)
  Opt opts[] = {{"-ssa", 0, ssa, NULL, 0}, {"-src", 0, src, NULL, 0}, {"-mask", 0, mask, &usemask, 1}, {"-thresh", 3, NULL, (int*)&thresh, 0}};
  parse(argc, argv, opts, 4);
  if (argc == 2) { td_nameadd(ssa, argv[1], "ssa"); td_nameadd(src, argv[1], "src"); }
  int err = td_threshold(ssa, src, mask, thresh, usemask);
  if (err != 0) printf("Threshold Error %d\n", err);
  return done();
}

#elif defined(TOOL_twi)
// src/TWImn.cpp:48-129
static void usage(const char* prog) {
  printf("Simple Usage:\n %s <basefilename>\n", prog);
  printf("Usage with specific file names:\n %s -sca <areafile>\n", prog);
  printf("-slp <slopefile> -twi <twifile>\n");
  printf("<basefilename> is the name of the raw digital elevation model\n");
  printf("<areafile> is the D-infinity specific catchment area input file.\n");
  printf("<slopefile> is the D-infinity slope input file.\n");
  printf("<twifile> is the topographic wetness index (ln(a/S) output file.\n");
  printf("The following are appended to the file names\n");
  printf("before the files are opened:\n");
  printf("sca    D-infinity specific catchment area grid (input)\n");
  printf("slp     D-infinity slope grid (input)\n");
  printf("twi    output topographic wetness index grid grid\n");
  exit(0);
}
int main(int argc, char** argv) {
  static char slp[MAXLN], sca[MAXLN], twi[MAXLN];
  Opt opts[] = {{"-sca", 0, sca, NULL, 0}, {"-slp", 0, slp, NULL, 0}, {"-twi", 0, twi, NULL, 0}};
  parse(argc, argv, opts, 3);
  if (argc == 2) { td_nameadd(sca, argv[1], "sca"); td_nameadd(slp, argv[1], "slp"); td_nameadd(twi, argv[1], "twi"); }
  int err = td_twigrid(slp, sca, twi);
  if (err != 0) printf("TWI error %d\n", err);
  return done();
}
#elif defined(TOOL_slopearea)
// src/SlopeAreamn.cpp:50-138 (no "Error:" preamble; -par takes two floats; errors leave through `return 0`)
static void usage(const char* prog) {
  printf("Simple Use:\n %s <basefilename>\n", prog);
  printf("Use with specific file names:\n %s -slp <slopefile>\n", prog);
  printf("-sca <scafile> -sa <safile> [-par <m> <n>] \n");
  printf("<basefilename> is the name of the base digital elevation model without suffixes for simple input. Suffixes 'slp', 'sca' and 'sa' will be appended. \n");
  printf("<slopefile> is the name of the input slope file.\n");
  printf("<scafile> is the name of input contributing area file.\n");
  printf("<safile> is the name of the output file with the result slope^m x (contributing area)^n.\n");
  printf("<m> is the exponent on slope, default value 2 if not specified.\n");
  printf("<n> is the exponent on contributing area, default value 1 if not specified.\n");
  exit(0);
}
int main(int argc, char** argv) {
  static char slp[MAXLN], sca[MAXLN], sa[MAXLN];
  float par[2] = {2.f, 1.f};
  if (argc < 2) usage(argv[0]);
  Opt opts[] = {{"-slp", 0, slp, NULL, 0}, {"-sca", 0, sca, NULL, 0}, {"-sa", 0, sa, NULL, 0}, {"-par", 4, NULL, (int*)par, 0}};
  parse(argc, argv, opts, 4);
  if (argc == 2) { td_nameadd(slp, argv[1], "slp"); td_nameadd(sca, argv[1], "sca"); td_nameadd(sa, argv[1], "sa"); }
  int err = td_slopearea(slp, sca, sa, par);
  if (err != 0) printf("SlopeArea Error %d\n", err);
  return done();
}

#elif defined(TOOL_slopearearatio)
// src/SlopeAreaRatiomn.cpp:48-136
static void usage(const char* prog) {
  printf("Simple Usage:\n %s <basefilename>\n", prog);
  printf("Usage with specific file names:\n %s -sca <areafile>\n", prog);
  printf("-slp <slopefile> -sar <atanbfile>\n");
  printf("<basefilename> is the name of the raw digital elevation model\n");
  printf("<areafile> is the D-infinity specific catchment area input file.\n");
  printf("<slopefile> is the D-infinity slope input file.\n");
  printf("<atanbfile> is the slope area ratio output file.\n");
  printf("The following are appended to the file names\n");
  printf("before the files are opened:\n");
  printf("sca    D-infinity specific catchment area grid (input)\n");
  printf("slp     D-infinity slope grid (input)\n");
  printf("sar    output slope area ratio grid\n");
  exit(0);
}
int main(int argc, char** argv) {
  static char slp[MAXLN], sca[MAXLN], sar[MAXLN];
  Opt opts[] = {{"-sca", 0, sca, NULL, 0}, {"-slp", 0, slp, NULL, 0}, {"-sar", 0, sar, NULL, 0}};
  parse(argc, argv, opts, 3);
  if (argc == 2) { td_nameadd(sca, argv[1], "sca"); td_nameadd(slp, argv[1], "slp"); td_nameadd(sar, argv[1], "sar"); }
  int err = td_atanbgrid(slp, sca, sar);
  if (err != 0) printf("Slope area ratio error %d\n", err);
  return done();
}

#elif defined(TOOL_peukerdouglas)
// src/PeukerDouglasmn.cpp:53-128 (no "Error:" preamble; -par takes three floats)
static void usage(const char* prog) {
  printf("Simple Use:\n %s <basefilename>\n", prog);
  printf("Use with specific file names:\n %s -fel <elevationfile>\n", prog);
  printf("-ss <streamsource> [-par <weightMiddle> <weightSide> <weightDiagonal>]\n");
  printf("<basefilename> is the name of the base digital elevation model without suffixes for simple input. 'fel' will be appended. \n");
  printf("<elevationfile> is the name of the elevation input file.\n");
  printf("<streamsource> is the name of the stream source file output.\n");
  printf("The elevation input is smoothed by averaging using the center and eight surrounding grid cells.\n");
  printf("<weightMiddle> is the weight given to the center cell in the smoothing of the input elevations.\n");
  printf("<weightSide> is the weight given to the 4 side cells in the smoothing of the input elevations.\n");
  printf("<weightDiagonal> is the weight given to the 4 diagonal cells in the smoothing of the input elevations.\n");
  printf("Default weights are 0.4 0.1 0.05 if -par is not specified.\n");
  exit(0);
}
int main(int argc, char** argv) {
  static char fel[MAXLN], ss[MAXLN];
  float par[3] = {0.4f, 0.1f, 0.05f};
  if (argc < 2) usage(argv[0]);
  Opt opts[] = {{"-fel", 0, fel, NULL, 0}, {"-ss", 0, ss, NULL, 0}, {"-par", 5, NULL, (int*)par, 0}};
  parse(argc, argv, opts, 3);
  if (argc == 2) { td_nameadd(fel, argv[1], "fel"); td_nameadd(ss, argv[1], "ss"); }
  int err = td_peukerdouglas(fel, ss, par);
  if (err != 0) printf("Peuker Douglas Error %d\n", err);
  return done();
}

#elif defined(TOOL_lengtharea)
// src/LengthAreamn.cpp:50-133 (no "Error:" preamble; -par takes two floats)
static void usage(const char* prog) {
  printf("Simple Use:\n %s <basefilename>\n", prog);
  printf("Use with specific file names:\n %s -plen <plenfile>\n", prog);
  printf("-ad8 <ad8file> -ss <ssfile> [-par <M> <y>] \n");
  printf("<basefilename> is the name of the base digital elevation model without suffixes for simple input. Suffixes 'plen', 'ad8' and 'ss' will be appended. \n");
  printf("<plenfile> is the name of the input upslope longest path length file.\n");
  printf("<ad8file> is the name of input contributing area file.\n");
  printf("<ssfile> is the name of the output file with the result A >= M L^y ? 1:0.\n");
  printf("<M> is the coefficient, default value 0.03 if not specified.\n");
  printf("<y> is the exponent on upslope length, default value 1.3 if not specified.\n");
  exit(0);
}
int main(int argc, char** argv) {
  static char plen[MAXLN], ad8[MAXLN], ss[MAXLN];
  float par[2] = {0.03f, 1.3f};
  if (argc < 2) usage(argv[0]);
  Opt opts[] = {{"-plen", 0, plen, NULL, 0}, {"-ad8", 0, ad8, NULL, 0}, {"-ss", 0, ss, NULL, 0}, {"-par", 4, NULL, (int*)par, 0}};
  parse(argc, argv, opts, 4);
  if (argc == 2) { td_nameadd(plen, argv[1], "plen"); td_nameadd(ad8, argv[1], "ad8"); td_nameadd(ss, argv[1], "ss"); }
  int err = td_lengtharea(plen, ad8, ss, par);
  if (err != 0) printf("Length Area Error %d\n", err);
  return done();
}
#elif defined(TOOL_slopeavedown)
// src/SlopeAveDownmn.cpp:49-145 (the reference's usage text, typos included; -dn is read with %lf, default 50)
static void usage(const char* prog) {
  printf("Simple Usage:\n %s <basefilename>\n", prog);
  printf("Usage with specific file names:\n %s -p <pfile>\n", prog);
  printf("-fel <felfile> -slpd <slpdfile> -dn <dn>\n");
  printf("<basefilename> is the name of the base digital elevation model\n");
  printf("<pfile> is the D8 flow direction input file.\n");
  printf("<felfile> is the pit filled or carved elevation input file.\n");
  printf("<slpdfile> is the output D8 slope distance averaged grid file.\n");
  printf("<dn is the optional user selected downslope distance.\n");
  printf("The following are appended to the file names\n");
  printf("before the files are opened:\n");
  printf("fel   pit filled or carved elevation grid (input)\n");
  printf("p   D-infinity flow direction grid (Input)\n");
  printf("slpd   avalanche source site grod (input)\n");
  exit(0);
}
int main(int argc, char** argv) {
  static char p[MAXLN], fel[MAXLN], slpd[MAXLN];
  double dn = 50.0;
  Opt opts[] = {{"-fel", 0, fel, NULL, 0}, {"-p", 0, p, NULL, 0}, {"-slpd", 0, slpd, NULL, 0}, {"-dn", 6, NULL, (int*)&dn, 0}};
  parse(argc, argv, opts, 4);
  if (argc == 2) { td_nameadd(fel, argv[1], "fel"); td_nameadd(p, argv[1], "p"); td_nameadd(slpd, argv[1], "slpd"); }
  int err = td_sloped(p, fel, slpd, dn);
  if (err != 0) printf("sloped error %d\n", err);
  return done();
}
#elif defined(TOOL_flowdircond)
// src/flowdirconditionmn.cpp:55-128 (the reference's usage text, without a "Simple Usage" line, and its error line as printed)
static void usage(const char* prog) {
  printf("Use with specific file names:\n %s -p <pfile>\n", prog);
  printf("-z <zfile> -zfdc <zfdcfile> \n");
  printf("<pfile> is the name of the input D8 flow direction raster file.\n");
  printf("<zfile> is the name of the input elevation raster file.\n");
  printf("<zfdcfile> is the name of the output conditioned elevation raster file.\n");
  exit(0);
}
int main(int argc, char** argv) {
  static char p[MAXLN], z[MAXLN], zfdc[MAXLN];
  Opt opts[] = {{"-z", 0, z, NULL, 0}, {"-p", 0, p, NULL, 0}, {"-zfdc", 0, zfdc, NULL, 0}};
  parse(argc, argv, opts, 3);
  if (argc == 2) { td_nameadd(z, argv[1], "z"); td_nameadd(p, argv[1], "p"); td_nameadd(zfdc, argv[1], "zfdc"); }
  int err = td_flowdircond(p, z, zfdc);
  if (err != 0) printf("flowdiircond error %d\n", err);
  return done();
}
#elif defined(TOOL_retlimflow)
// src/RetLimFlowmn.cpp:51-146 (the reference's usage text; its error line always shows 1: `err=retlimro(...) != 0` assigns the
// comparison)
static void usage(const char* prog) {
  printf("Simple Usage:\n %s <basefilename>\n", prog);
  printf("Usage with specific file names:\n %s -ang <angfile>", prog);
  printf("-rc <rcfile> -wg <wgfile> -qrl <qrlfile>\n");
  printf("<basefilename> is the name of the raw digital elevation model\n");
  printf("<angfile> is the D-infinity flow direction input file.\n");
  printf("<rcfile> retention capacity file.\n");
  printf("<wgfile> is the input weight at each grid cell.\n");
  printf("<qrlfile> is retention limited runoff that is output.\n");
  printf("With simple use the following are appended to the file names\n");
  printf("before the files are opened:\n");
  printf("ang    D-infinity flow direction input file\n");
  printf("rc    retention capacity (input)\n");
  printf("wg     weight grid (input)\n");
  printf("qrl   retention limited runoff (output)\n");
  exit(0);
}
int main(int argc, char** argv) {
  static char ang[MAXLN], wg[MAXLN], rc[MAXLN], qrl[MAXLN];
  Opt opts[] = {{"-ang", 0, ang, NULL, 0}, {"-wg", 0, wg, NULL, 0}, {"-rc", 0, rc, NULL, 0}, {"-qrl", 0, qrl, NULL, 0}};
  parse(argc, argv, opts, 4);
  if (argc == 2) { td_nameadd(ang, argv[1], "ang"); td_nameadd(rc, argv[1], "rc"); td_nameadd(qrl, argv[1], "qrl"); td_nameadd(wg, argv[1], "wg"); }
  int err = td_retlimro(ang, wg, rc, qrl) != 0;
  if (err) printf("RetlimFlow error %d\n", err);
  return done();
}
#elif defined(TOOL_d8hdisttostrm) || defined(TOOL_d8vdisttostrm)
// src/D8HDistToStrmmn.cpp:51-149 and src/D8VDistToStrmmn.cpp:52-163 (the reference's usage texts; -thresh is read with %d, default 1).
// Their error line always shows 1 (`err=distgrid(...) != 0` assigns the comparison).  Rasters whose sizes differ end the program
// with exit status 5 after "File sizes do not match", as the reference's MPI_Abort(MCW, 5) does.
#if defined(TOOL_d8vdisttostrm)
#define DTS_V 1
#else
#define DTS_V 0
#endif
static void usage(const char* prog) {
  printf("Simple Usage:\n %s <basefilename>\n", prog);
  printf("Usage with specific file names:\n %s -p <pfile>\n", prog);
  printf(DTS_V ? "-fel <felfile> -src <srcfile> -dist <distfile> [-thresh <thresh>]\n" : "-src <srcfile> -dist <distfile> [-thresh <thresh>]\n");
  printf("<basefilename> is the name of the base digital elevation model\n");
  printf("<pfile> is the d8 flow direction input file.\n");
  if (DTS_V) printf("<felfile> is the pit filled or carved elevation input file.\n");
  printf("<srcfile> is the stream raster input file.\n");
  printf(DTS_V ? "<distfile> is the vertical distance to stream output file.\n" : "<distfile> is the distance to stream output file.\n");
  printf("The optional <thresh> is the user input threshold number.\n");
  printf("The following are appended to the file names\n");
  printf("before the files are opened:\n");
  printf("p      D8 flow directions (input)\n");
  if (DTS_V) printf("fel    pit filled or carved elevation file\n");
  printf("src    stream raster file (Input)\n");
  printf("dist   distance to stream file(output)\n");
  exit(0);
}
int main(int argc, char** argv) {
  static char p[MAXLN], fel[MAXLN], src[MAXLN], dist[MAXLN];
  int thresh = 1;
  Opt opts[] = {{"-p", 0, p, NULL, 0}, {"-src", 0, src, NULL, 0}, {"-dist", 0, dist, NULL, 0}, {"-thresh", 2, NULL, &thresh, 0}, {"-fel", 0, fel, NULL, 0}};
  parse(argc, argv, opts, DTS_V ? 5 : 4);
  if (argc == 2) {
    td_nameadd(p, argv[1], "p");
    if (DTS_V) td_nameadd(fel, argv[1], "fel");
    td_nameadd(src, argv[1], "src");
    td_nameadd(dist, argv[1], "dist");
  }
  const int rc = DTS_V ? td_d8vdistdown(p, fel, src, dist, thresh) : td_distgrid(p, src, dist, thresh);
  if (rc == TD_ERR_MISMATCH) { fflush(stdout); _exit(5); }
  const int err = rc != 0;
  if (err) printf(DTS_V ? "D8 distance down error %d\n" : "D8 distance error %d\n", err);
  return done();
}
#elif defined(TOOL_dinfdistdown)
// src/DinfDistDownmn.cpp:50-269.  -m reads the next two tokens, each either a method or a statistic, in either order; an unknown token
// leaves the default (ave h).  `-m x` as the last argument prints the usage here (the reference reads argv[argc] there).  -slp is
// read and never opened.  Simple usage derives every name, -wg's included, but never uses the weights.  Rasters whose sizes differ end
// the program with exit status 5 after "File sizes do not match", as the reference's MPI_Abort(MCW, 5) does.
static void usage(const char* prog) {
  printf("Simple Usage:\n %s <basefilename>\n", prog);
  printf("Usage with specific file names:\n %s -ang <angfile>\n", prog);
  printf("-fel <felfile> -slp <slpfile> -src <srcfile> [-wg <wfile>] -dd <dtsfile>\n");
  printf("[-m ave h] [-nc]\n");
  printf("<basefilename> is the name of the raw digital elevation model\n");
  printf("<angfile> is the D-infinity flow direction input file.\n");
  printf("<felfile> is the pit filled or carved elevation input file.\n");
  printf("<slpfile> is the D-infinity slope input file.\n");
  printf("<srcfile> is the stream raster input file.\n");
  printf("<wgfile> is the D-infinity flow direction input file.\n");
  printf("<dtsfile> is the D-infinity distance output file.\n");
  printf("[-m ave h] is the optional method flag.\n");
  printf("The flag -nc overrides edge contamination checking\n");
  printf("The following are appended to the file names\n");
  printf("before the files are opened:\n");
  printf("ang   D-infinity contributing area file (output)\n");
  printf("fel   pit filled or carved elevation file\n");
  printf("slp   D-infinity slope input file file\n");
  printf("src   Stream raster input file\n");
  printf("wg   weight input file\n");
  printf("dd   distance to stream output file\n");
  exit(0);
}
int main(int argc, char** argv) {
  static char ang[MAXLN], fel[MAXLN], slp[MAXLN], wfile[MAXLN], src[MAXLN], dd[MAXLN];
  int usew = 0, concheck = 1, m[2] = {0, 0};     // {typemethod, statmethod}
  Opt opts[] = {{"-ang", 0, ang, NULL, 0}, {"-fel", 0, fel, NULL, 0}, {"-slp", 0, slp, NULL, 0},   {"-src", 0, src, NULL, 0},
                {"-wg", 0, wfile, &usew, 1}, {"-dd", 0, dd, NULL, 0}, {"-m", 7, NULL, m, 0},        {"-nc", 1, NULL, &concheck, 0}};
  parse(argc, argv, opts, 8);
  if (argc == 2) {
    td_nameadd(ang, argv[1], "ang");
    td_nameadd(fel, argv[1], "fel");
    td_nameadd(slp, argv[1], "slp");
    td_nameadd(src, argv[1], "src");
    td_nameadd(wfile, argv[1], "wg");
    td_nameadd(dd, argv[1], "dd");
  }
  const int err = td_dinfdistdown(ang, fel, slp, wfile, src, dd, m[1], m[0], usew, concheck);
  if (err == TD_ERR_MISMATCH) { fflush(stdout); _exit(5); }
  if (err != 0) printf("area error %d\n", err);
  return done();
}
#else
#error "define TOOL_<name>"
#endif
