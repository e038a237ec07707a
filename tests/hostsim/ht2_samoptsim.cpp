// ht2_samoptsim.cpp -- TEST-ONLY host build of ht2_hostsim with every SAM output setting and the reference-name table.
//
// The whole of ht2_hostsim.cpp (the per-read state machine on the CPU, results in the C ABI's batch structures,
// formatted by ht2_format_batch -- the formatter of ht2_sam.h that the device SAM kernels run) with its header,
// formatter, splice-site DB and novel-splice-site calls routed through the settings of ht2gpu_set_sam_output and the
// reference names of ht2gpu_options_t::chr_names, as a handle runs them:
//   HT2_SAM_OUTPUT="no_unal=1,omit_sec_seq=1,no_sq=1,rg_id=<id>,rg=<field>,...,rna_strandness=<0..4>,
//                   no_qname_trunc=1,no_templatelen_adjustment=1,chr_names=<0..2>"
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

static Ht2SamOutput g_samOut;
static int g_chrNames = 0;
static Ht2RefNames g_names;
static bool g_namesBuilt = false;

static const Ht2RefNames* samoptNames(const Ht2Image& img)
{
    if (!g_namesBuilt) { g_names.build(img, g_chrNames); g_namesBuilt = true; }
    return &g_names;
}
static void samoptHeader(std::string& o, const Ht2Image& img) { ht2_sam_header(o, img, &g_samOut, samoptNames(img)); }
static bool samoptFormat(const Ht2Image& img, const Ht2Params& P, const ht2gpu_read_batch_t* b, const char* nm,
                         const ht2gpu_result_batch_t* res, char** out, size_t* out_len, unsigned nth, const uint8_t* ssT = NULL,
                         uint32_t* colCount = NULL, Ht2SsRec* colRecs = NULL, uint32_t colCap = 0)
{
    return ht2_format_batch(img, P, b, nm, res, out, out_len, nth, ssT, colCount, colRecs, colCap, &g_samOut, NULL, NULL, samoptNames(img));
}
static bool samoptSsdbBuild(const Ht2Image& img, const std::vector<Ht2SsFile>& files, std::vector<uint8_t>& blob, uint32_t& nSites,
                            std::string& err)
{
    return ht2_ssdb_build(img, files, blob, nSites, err, samoptNames(img));
}

// ht2_host.h and ht2_index.h are already included (include guards), so only ht2_hostsim.cpp's own uses are renamed.
// Its one call of Ht2NovelSites::write gets the table as the last argument.
#define ht2_sam_header samoptHeader
#define ht2_format_batch samoptFormat
#define ht2_ssdb_build samoptSsdbBuild
#define write(img, path, nw, err) write(img, path, nw, err, samoptNames(img))
#define main ht2_hostsim_main
#include "ht2_hostsim.cpp"
#undef main
#undef write
#undef ht2_ssdb_build
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
            const int n = atoi(v.c_str());
            if (k == "no_unal") g_samOut.noUnal = n != 0;
            else if (k == "omit_sec_seq") g_samOut.omitSecSeq = n != 0;
            else if (k == "no_sq") g_samOut.noSq = n != 0;
            else if (k == "rg_id") g_samOut.rgId = v;
            else if (k == "rg") g_samOut.rg.push_back(v);
            else if (k == "rna_strandness") g_samOut.rnaStrandness = (uint32_t)n;
            else if (k == "no_qname_trunc") g_samOut.noQnameTrunc = n != 0;
            else if (k == "no_templatelen_adjustment") g_samOut.noTlenAdj = n != 0;
            else if (k == "chr_names") g_chrNames = n;
            else { fprintf(stderr, "unknown HT2_SAM_OUTPUT key %s\n", k.c_str()); return 2; }
        }
    }
    return ht2_hostsim_main(argc, argv);
}
