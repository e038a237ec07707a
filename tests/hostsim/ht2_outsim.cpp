// ht2_outsim.cpp -- TEST-ONLY host build of ht2_hostsim with the SAM output settings and the alignment summary.
//
// The whole of ht2_hostsim.cpp (the per-read state machine on the CPU, results in the C ABI's batch structures,
// formatted by ht2_format_batch -- the formatter of ht2_sam.h that the device SAM kernels run) with its two SAM calls
// routed through the settings of ht2gpu_set_sam_output and the ReportingMetrics tally of the counting pass:
//   HT2_SAM_OUTPUT="no_unal=1,omit_sec_seq=1,no_sq=1,rg_id=<id>,rg=<field>,rg=<field>..."
//   HT2_SUMMARY=<file>        the run's alignment summary (ht2_format_align_summary), --no-discordant / --no-mixed
//                             from HT2_OPTS; HT2_NEW_SUMMARY=1 for the --new-summary format
// usage and every other variable as ht2_hostsim.
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <string>
#include <vector>
#include <chrono>
#include "../../hisat2_b200/csrc/ht2_host.h"
#include "../../hisat2_b200/csrc/ht2_seed.h"

static Ht2SamOutput g_samOut;
static ht2gpu_align_counts_t g_counts;
static bool g_discord = true, g_mixed = true;

static void outsimHeader(std::string& o, const Ht2Image& img) { ht2_sam_header(o, img, &g_samOut); }
static bool outsimFormat(const Ht2Image& img, const Ht2Params& P, const ht2gpu_read_batch_t* b, const char* names,
                         const ht2gpu_result_batch_t* res, char** out, size_t* out_len, unsigned nth, const uint8_t* ssT = NULL,
                         uint32_t* colCount = NULL, Ht2SsRec* colRecs = NULL, uint32_t colCap = 0)
{
    g_discord = P.discord != 0; g_mixed = P.mixed != 0;
    return ht2_format_batch(img, P, b, names, res, out, out_len, nth, ssT, colCount, colRecs, colCap, &g_samOut, &g_counts);
}

// ht2_host.h is already included (include guard), so only ht2_hostsim.cpp's own uses are renamed
#define ht2_sam_header outsimHeader
#define ht2_format_batch outsimFormat
#define main ht2_hostsim_main
#include "ht2_hostsim.cpp"
#undef main
#undef ht2_format_batch
#undef ht2_sam_header

int main(int argc, char** argv)
{
    if (const char* so = getenv("HT2_SAM_OUTPUT")) {
        std::string s(so); size_t p0 = 0;
        while (p0 < s.size()) {
            size_t c = s.find(',', p0); if (c == std::string::npos) c = s.size();
            const std::string kv = s.substr(p0, c - p0); p0 = c + 1;
            const size_t e = kv.find('=');
            if (e == std::string::npos) { fprintf(stderr, "bad HT2_SAM_OUTPUT entry %s\n", kv.c_str()); return 2; }
            const std::string k = kv.substr(0, e), v = kv.substr(e + 1);
            if (k == "no_unal") g_samOut.noUnal = atoi(v.c_str()) != 0;
            else if (k == "omit_sec_seq") g_samOut.omitSecSeq = atoi(v.c_str()) != 0;
            else if (k == "no_sq") g_samOut.noSq = atoi(v.c_str()) != 0;
            else if (k == "rg_id") g_samOut.rgId = v;
            else if (k == "rg") g_samOut.rg.push_back(v);
            else { fprintf(stderr, "unknown HT2_SAM_OUTPUT key %s\n", k.c_str()); return 2; }
        }
    }
    memset(&g_counts, 0, sizeof(g_counts));
    const int rc = ht2_hostsim_main(argc, argv);
    const char* sumOut = getenv("HT2_SUMMARY");
    if (rc != 0 || !sumOut) return rc;
    const char* ns = getenv("HT2_NEW_SUMMARY");
    std::string txt;
    ht2_format_align_summary(txt, g_counts, ns && atoi(ns) != 0, g_discord, g_mixed);
    FILE* f = fopen(sumOut, "wb");
    if (!f) { fprintf(stderr, "cannot write %s\n", sumOut); return 1; }
    fwrite(txt.data(), 1, txt.size(), f);
    fclose(f);
    return 0;
}
