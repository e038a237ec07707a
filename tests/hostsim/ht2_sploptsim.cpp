// ht2_sploptsim.cpp -- TEST-ONLY host build of ht2_hostsim with the spliced-alignment options of ht2gpu_options_t,
// applied by the library's ht2_apply_spliced_options, as ht2gpu_open applies them:
//   HT2_SPL_OPTS="pen_cansplice=N,pen_noncansplice=N,pen_conflictsplice=N,can=<C|L|S|G>:<const>:<coeff>,
//                 noncan=<C|L|S|G>:<const>:<coeff>,min_intronlen=N,max_intronlen=N,dta=<0|1|2>,no_anchorstop=1,tmo=1,
//                 avoid_pseudogene=1"
//   --seed-dump <index> <reads.fa> <no_spliced> (ht2_hostsim's) honours no_anchorstop.
//   --intron-pen <type> <const> <coeff> <max_len>: prints the runs ht2_set_intron_pen builds, one "start pen" line
//     each, or exits with status 3 when the function has too many runs.
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

static ht2gpu_options_t g_so;   // only the spliced-alignment fields are read
static int g_spliced = 0;       // HT2_OPTS spliced=1, which ht2_hostsim applies only after its parameters are made

// ht2_hostsim's parameters, then the spliced-alignment options through the library's own mapping
static void sploptDefaultParams(Ht2Params& P, const Ht2Image& img, bool noSplicedAlignment)
{
    ht2_default_params(P, img, noSplicedAlignment && !g_spliced);
    if (const char* why = ht2_apply_spliced_options(P, g_so)) { fprintf(stderr, "%s\n", why); exit(3); }
}
// the seed dump's partial searches stop at unique anchors only when the options let them, as ht2gpu_seed_search's do
template <bool GRAPH>
static bool sploptSeedPartial(const Ht2Fm<uint32_t>& fm, const Ht2Params& P, const uint8_t* seq, Ht2SeedState& st,
                              Ht2SeedHit& ph, bool& pseudogeneStop, bool& anchorStop)
{
    anchorStop = anchorStop && P.anchorStop != 0;
    return ht2_seed_partial<GRAPH>(fm, P, seq, st, ph, pseudogeneStop, anchorStop);
}

// ht2_hostsim.cpp's headers are already included (include guards), so only its own calls are renamed
#define ht2_default_params sploptDefaultParams
#define ht2_seed_partial sploptSeedPartial
#define main ht2_hostsim_main
#include "ht2_hostsim.cpp"
#undef main
#undef ht2_seed_partial
#undef ht2_default_params

static bool func(const std::string& v, int32_t& t, double& C, double& L)
{
    t = v[0];
    return sscanf(v.c_str() + 1, ":%lf:%lf", &C, &L) == 2;
}

int main(int argc, char** argv)
{
    if (argc == 6 && !strcmp(argv[1], "--intron-pen")) {
        static Ht2Params P;
        if (!ht2_set_intron_pen(P, 0, argv[2][0], atof(argv[3]), atof(argv[4]), (uint32_t)atoll(argv[5]))) return 3;
        for (uint32_t k = 0; k < P.intronPen[0].n; k++) printf("%u %d\n", P.intronPen[0].start[k], P.intronPen[0].pen[k]);
        return 0;
    }
    // ht2gpu_default_options' spliced-alignment values (hisat2.cpp:493-499)
    memset(&g_so, 0, sizeof(g_so));
    g_so.pen_noncansplice = 12; g_so.pen_conflictsplice = 1000000; g_so.min_intronlen = 20; g_so.max_intronlen = 500000;
    if (const char* so = getenv("HT2_SPL_OPTS")) {
        std::string s(so); size_t p0 = 0;
        while (p0 < s.size()) {
            size_t c = s.find(',', p0); if (c == std::string::npos) c = s.size();
            const std::string kv = s.substr(p0, c - p0); p0 = c + 1;
            const size_t e = kv.find('=');
            if (e == std::string::npos) { fprintf(stderr, "bad HT2_SPL_OPTS entry %s\n", kv.c_str()); return 2; }
            const std::string k = kv.substr(0, e), v = kv.substr(e + 1);
            const int32_t n = atoi(v.c_str());
            if (k == "pen_cansplice") g_so.pen_cansplice = n; else if (k == "pen_noncansplice") g_so.pen_noncansplice = n;
            else if (k == "pen_conflictsplice") g_so.pen_conflictsplice = n;
            else if (k == "min_intronlen") g_so.min_intronlen = n; else if (k == "max_intronlen") g_so.max_intronlen = n;
            else if (k == "dta") g_so.dta = n; else if (k == "no_anchorstop") g_so.no_anchorstop = n; else if (k == "tmo") g_so.tmo = n;
            else if (k == "avoid_pseudogene") g_so.avoid_pseudogene = n;
            else if (k == "can" && func(v, g_so.can_intronlen_type, g_so.can_intronlen_const, g_so.can_intronlen_coeff)) {}
            else if (k == "noncan" && func(v, g_so.noncan_intronlen_type, g_so.noncan_intronlen_const, g_so.noncan_intronlen_coeff)) {}
            else { fprintf(stderr, "bad HT2_SPL_OPTS entry %s\n", kv.c_str()); return 2; }
        }
    }
    if (const char* os = getenv("HT2_OPTS")) g_spliced = strstr(os, "spliced=1") != NULL;
    return ht2_hostsim_main(argc, argv);
}
