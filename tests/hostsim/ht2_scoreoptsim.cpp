// ht2_scoreoptsim.cpp -- TEST-ONLY host build of ht2_hostsim with the mate orientation and the N ceiling of
// ht2gpu_options_t, applied as applyOptions (ht2_gpu.cu) applies them:
//   HT2_SCORE_OPTS="pe_orient=<0 fr|1 rf|2 ff>,n_ceil=<C|L|S|G>:<const>:<coeff>,rna_strandness=<0..4>"
// The read filter and the --bowtie2-dp extension read Ht2Params::nCeilTab, the formatter the SAM setting.
//   --nceil-table <type> <const> <coeff>: prints nCeilTab, one "len value" line per read length.
//   --scpen <sp_max> <sp_min>: prints ht2_scpen for qualities 0 .. 80, one "q value" line each.
// usage and every other variable as ht2_hostsim.
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <string>
#include <vector>
#include <chrono>
#include "../../hisat2_b200/csrc/ht2_host.h"
#include "../../hisat2_b200/csrc/ht2_seed.h"
#include "../../hisat2_b200/csrc/ht2_ssdb.h"

static int g_peOrient = HT2GPU_PE_FR;
static char g_nCeilType = 0;
static double g_nCeilConst = 0, g_nCeilCoeff = 0;
static Ht2SamOutput g_samOut;

static void scoreoptDefaultParams(Ht2Params& P, const Ht2Image& img, bool noSplicedAlignment)
{
    ht2_default_params(P, img, noSplicedAlignment);
    if (g_nCeilType) ht2_set_n_ceil(P, g_nCeilType, g_nCeilConst, g_nCeilCoeff);
    P.gMate1fw = g_peOrient != HT2GPU_PE_RF; P.gMate2fw = g_peOrient != HT2GPU_PE_FR;
    P.pePolicy = g_peOrient == HT2GPU_PE_FF ? 0 : g_peOrient == HT2GPU_PE_RF ? 3 : 2;
}
static bool scoreoptFormat(const Ht2Image& img, const Ht2Params& P, const ht2gpu_read_batch_t* b, const char* nm,
                           const ht2gpu_result_batch_t* res, char** out, size_t* out_len, unsigned nth, const uint8_t* ssT = NULL,
                           uint32_t* colCount = NULL, Ht2SsRec* colRecs = NULL, uint32_t colCap = 0)
{
    return ht2_format_batch(img, P, b, nm, res, out, out_len, nth, ssT, colCount, colRecs, colCap, &g_samOut);
}

// ht2_hostsim.cpp's headers are already included (include guards), so only its own calls are renamed.  Its filter
// calls sit where its parameters are in scope as P.
#define ht2_default_params scoreoptDefaultParams
#define ht2_format_batch scoreoptFormat
#define ht2_filters(rd, minsc) ht2_filters(rd, minsc, P.nCeilTab)
#define main ht2_hostsim_main
#include "ht2_hostsim.cpp"
#undef main
#undef ht2_filters
#undef ht2_format_batch
#undef ht2_default_params

int main(int argc, char** argv)
{
    if (argc == 5 && !strcmp(argv[1], "--nceil-table")) {
        static Ht2Params P;
        if (!ht2_set_n_ceil(P, argv[2][0], atof(argv[3]), atof(argv[4]))) { fprintf(stderr, "bad type %s\n", argv[2]); return 2; }
        for (uint32_t len = 0; len <= HT2_PARAMS_MAX_RDLEN; len++) printf("%u %d\n", len, P.nCeilTab[len]);
        return 0;
    }
    if (argc == 4 && !strcmp(argv[1], "--scpen")) {
        Ht2ParamsCore P; memset(&P, 0, sizeof(P));
        P.scpMax = (int32_t)atoll(argv[2]); P.scpMin = (int32_t)atoll(argv[3]);
        for (int q = 0; q <= 80; q++) printf("%d %d\n", q, ht2_scpen(P, q));
        return 0;
    }
    if (const char* so = getenv("HT2_SCORE_OPTS")) {
        std::string s(so); size_t p0 = 0;
        while (p0 < s.size()) {
            size_t c = s.find(',', p0); if (c == std::string::npos) c = s.size();
            const std::string kv = s.substr(p0, c - p0); p0 = c + 1;
            const size_t e = kv.find('=');
            if (e == std::string::npos) { fprintf(stderr, "bad HT2_SCORE_OPTS entry %s\n", kv.c_str()); return 2; }
            const std::string k = kv.substr(0, e), v = kv.substr(e + 1);
            if (k == "pe_orient") g_peOrient = atoi(v.c_str());
            else if (k == "rna_strandness") g_samOut.rnaStrandness = (uint32_t)atoi(v.c_str());
            else if (k == "n_ceil") {
                g_nCeilType = v[0];
                if (sscanf(v.c_str() + 1, ":%lf:%lf", &g_nCeilConst, &g_nCeilCoeff) != 2) { fprintf(stderr, "bad n_ceil %s\n", v.c_str()); return 2; }
            }
            else { fprintf(stderr, "unknown HT2_SCORE_OPTS key %s\n", k.c_str()); return 2; }
        }
    }
    return ht2_hostsim_main(argc, argv);
}
