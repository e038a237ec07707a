// ht2_readsim.cpp -- TEST-ONLY host build of ht2_hostsim that also writes the units' outcome bytes.
//
// The whole of ht2_hostsim.cpp with its SAM formatting routed through ht2_format_batch's outcome output: the counting
// pass of the formatter in ht2_sam.h (the one the device SAM kernels run) stores one HT2GPU_OUTCOME_* byte per read
// or pair, exactly what ht2gpu_unit_outcomes hands back on the device.
//   HT2_OUTCOMES=<file>   the outcome bytes of every unit, in read order
// usage and every other variable as ht2_hostsim.
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <string>
#include <vector>
#include "../../hisat2_b200/csrc/ht2_host.h"

static std::vector<uint8_t> g_outcomes;

static bool readsimFormat(const Ht2Image& img, const Ht2Params& P, const ht2gpu_read_batch_t* b, const char* names,
                          const ht2gpu_result_batch_t* res, char** out, size_t* out_len, unsigned nth, const uint8_t* ssT = NULL,
                          uint32_t* colCount = NULL, Ht2SsRec* colRecs = NULL, uint32_t colCap = 0)
{
    const size_t at = g_outcomes.size();
    g_outcomes.resize(at + (b->paired ? b->n_reads / 2 : b->n_reads));
    return ht2_format_batch(img, P, b, names, res, out, out_len, nth, ssT, colCount, colRecs, colCap, NULL, NULL, g_outcomes.data() + at);
}

// ht2_host.h is already included (include guard), so only ht2_hostsim.cpp's own uses are renamed
#define ht2_format_batch readsimFormat
#define main ht2_hostsim_main
#include "ht2_hostsim.cpp"
#undef main
#undef ht2_format_batch

int main(int argc, char** argv)
{
    const int rc = ht2_hostsim_main(argc, argv);
    const char* path = getenv("HT2_OUTCOMES");
    if (rc != 0 || !path) return rc;
    FILE* f = fopen(path, "wb");
    if (!f) { fprintf(stderr, "cannot write %s\n", path); return 1; }
    if (!g_outcomes.empty()) fwrite(g_outcomes.data(), 1, g_outcomes.size(), f);
    fclose(f);
    return 0;
}
