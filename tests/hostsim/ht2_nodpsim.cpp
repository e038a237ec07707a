// ht2_nodpsim.cpp -- TEST-ONLY host build: the aligner compiled without the --bowtie2-dp extension
// (Ht2AlignerT<.., .., DP = false>, what the pool kernel runs when the option is off) against the one that reads the
// option (DP = true).
//
//   ht2_nodpsim <index_base> <reads_1.fq> <reads_2.fq> <bowtie2_dp>
//       Runs every pair through both instantiations with --no-spliced-alignment and the given --bowtie2-dp mode and
//       compares everything a read hands on: reported alignments and their edits, pairs, RNG state, LF steps,
//       algorithmic bytes, error bits.  Prints "<pairs> <pairs that differ> <alignments> <pairs whose DP = true run
//       entered the extension>".  With mode 0 the two must agree on every pair; with mode 1 / 2 the DP = true side
//       runs the extension and the DP = false side must not.
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <string>
#include <vector>
#include "../../hisat2_b200/csrc/ht2_host.h"

template <typename ALIGNER>
static void runPair(ALIGNER& A, const Ht2Image* img, Ht2Params& P, Ht2Work* W, Ht2SwScratch* sw, uint32_t* swPool, Ht2HostRead& r1, Ht2HostRead& r2)
{
    memset(W, 0, sizeof(Ht2Work));
    r1.seed = ht2_gen_rand_seed(r1, 0); r2.seed = ht2_gen_rand_seed(r2, 0);
    const int64_t ms1 = ht2_minsc(P, (uint32_t)r1.seq.size()), ms2 = ht2_minsc(P, (uint32_t)r2.seq.size());
    const bool p1 = ht2_filters(r1, ms1).pass(), p2 = ht2_filters(r2, ms2).pass();
    A.bind(img->blob.data(), &P, W); A.sw = sw; A.swPl = swPool; A.swStride = 1;
    W->rnd.init((p1 && p2) ? (r1.seed ^ r2.seed) : r1.seed);
    A.nofw[0] = P.gMate1fw ? P.nofw : P.norc; A.norc[0] = P.gMate1fw ? P.norc : P.nofw;
    A.nofw[1] = P.gMate2fw ? P.nofw : P.norc; A.norc[1] = P.gMate2fw ? P.norc : P.nofw;
    A.sinkReset(true);
    if (!(p1 && p2)) return;            // the fixture's pairs all pass the filters; a pair that does not is not aligned here
    A.paired = true; A.rightendonly = false; A.minsc[0] = ms1; A.minsc[1] = ms2;
    ht2_fill_read(W->rd[0], r1); ht2_fill_read(W->rd[1], r2);
    A.machineStart();
    while (!A.machineDone()) A.machineStep();
}

static bool sameResults(const Ht2Work* a, const Ht2Work* b)
{
    if (a->err != b->err || a->rnd.last != b->rnd.last || a->nLF != b->nLF || a->algBytes != b->algBytes) return false;
    if (a->nRes[0] != b->nRes[0] || a->nRes[1] != b->nRes[1] || a->nPairs != b->nPairs || a->nResEdits != b->nResEdits) return false;
    for (uint32_t m = 0; m < 2; m++) if (memcmp(a->res[m], b->res[m], a->nRes[m] * sizeof(Ht2Res))) return false;
    if (memcmp(a->resEdits, b->resEdits, a->nResEdits * sizeof(Ht2Edit))) return false;
    return memcmp(a->pairs, b->pairs, a->nPairs * sizeof(a->pairs[0])) == 0;
}

int main(int argc, char** argv)
{
    if (argc != 5) { fprintf(stderr, "usage: %s <index_base> <reads_1.fq> <reads_2.fq> <bowtie2_dp>\n", argv[0]); return 2; }
    std::string err;
    Ht2Image* img = ht2_image_load(argv[1], err);
    if (!img) { fprintf(stderr, "%s\n", err.c_str()); return 1; }
    std::vector<Ht2HostRead> reads1, reads2;
    if (!ht2_read_reads(argv[2], reads1, 1, err) || !ht2_read_reads(argv[3], reads2, 2, err)) { fprintf(stderr, "%s\n", err.c_str()); return 1; }
    Ht2Params P;
    ht2_default_params(P, *img, true);
    P.bowtie2Dp = (uint32_t)atoi(argv[4]);
    Ht2Work* Wn = (Ht2Work*)aligned_alloc(128, sizeof(Ht2Work));
    Ht2Work* Wd = (Ht2Work*)aligned_alloc(128, sizeof(Ht2Work));
    Ht2SwScratch* sw = new Ht2SwScratch();
    uint32_t* swPool = new uint32_t[HT2_SW_POOL_WORDS];
    Ht2AlignerT<false, true, false> An;
    Ht2AlignerT<false, true, true> Ad;
    size_t differ = 0, alns = 0, ranDp = 0;
    for (size_t i = 0; i < reads1.size(); i++) {
        sw->jbest = HT2_MIN_I64 + 1; sw->nrow = 0;
        runPair(An, img, P, Wn, sw, swPool, reads1[i], reads2[i]);
        const bool untouched = sw->nrow == 0 && sw->jbest == HT2_MIN_I64 + 1;
        if (!untouched) { fprintf(stderr, "pair %zu: the DP-free aligner wrote the DP scratch\n", i); return 1; }
        runPair(Ad, img, P, Wd, sw, swPool, reads1[i], reads2[i]);
        if (!(sw->nrow == 0 && sw->jbest == HT2_MIN_I64 + 1)) ranDp++;
        if (!sameResults(Wn, Wd)) differ++;
        alns += Wd->nRes[0] + Wd->nRes[1];
    }
    printf("%zu %zu %zu %zu\n", reads1.size(), differ, alns, ranDp);
    return 0;
}
