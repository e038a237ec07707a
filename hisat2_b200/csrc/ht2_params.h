// ht2_params.h -- alignment parameters shared by host and device code.
//
// Mirrors the option statics the reference hands to the hot path
// (hisat2.cpp:305-544 resetOptions; Scoring scoring.h:96-226; ReportingParams
// hisat2.cpp:3177-3189; TranscriptomePolicy hisat2.cpp:4076-4084; GraphPolicy
// :4086-4089).  Plain data so it can sit in __constant__ memory.
#ifndef HT2_PARAMS_H_
#define HT2_PARAMS_H_

#include <stdint.h>

#define HT2_PARAMS_MAX_RDLEN 1024

// The part the kernels receive BY VALUE (kernel parameter space, read through the constant cache).
struct Ht2ParamsCore {
    // Scoring
    int32_t mmpMax;        // --mp max (6)
    int32_t mmpMin;        // --mp min (2)
    int32_t scpMax;        // --sp max (2)
    int32_t scpMin;        // --sp min (1)
    int32_t npen;          // --np (1)
    int32_t rdGapConst;    // --rdg (5)
    int32_t rdGapLinear;   // --rdg (3)
    int32_t rfGapConst;    // --rfg (5)
    int32_t rfGapLinear;   // --rfg (3)
    int32_t mmcostConstant;// 1 = --ignore-quals (COST_MODEL_CONSTANT)
    int32_t canSplPen;     // --pen-cansplice (0)
    // Reporting
    uint32_t khits;        // -k (5 linear / 10 graph unless given)
    uint32_t kseeds;       // --max-seeds (max(5, 2k))
    uint32_t secondary;    // --secondary
    // Transcriptome policy
    uint32_t minIntronLen; // 20
    uint32_t maxIntronLen; // 500000
    uint32_t minAnchorLen; // 7
    uint32_t minAnchorLenNoncan; // 14
    uint32_t noSplicedAlignment; // --no-spliced-alignment
    // Graph policy
    uint32_t maxAltsTried; // 16
    // Search
    uint32_t anchorStop;   // 1
    uint32_t minK;         // ceil(log4(genome len)) (hi_aligner.h:3979-3984)
    uint32_t minKLocal;    // 8
    // Paired-end policy (pe.h): --fr, -I, -X
    int32_t  pePolicy;     // 0=FF 1=RR 2=FR 3=RF
    uint32_t minFrag;      // -I (0)
    uint32_t maxFrag;      // -X (1000)
    uint32_t gMate1fw;     // 1
    uint32_t gMate2fw;     // 0
    uint32_t nofw;         // --nofw
    uint32_t norc;         // --norc
    uint32_t mixed;        // !--no-mixed
    uint32_t discord;      // !--no-discordant
    // --bowtie2-dp (hisat2.cpp:293, 1770): 0 off, 1 when the anchor search found nothing >= minsc, 2 always
    uint32_t bowtie2Dp;
    int32_t  gapbar;       // --gbar (4): no gaps within this many rows of either read end (DP only)
    uint32_t tranFilter;   // the transcriptome policy (HT2_TRAN_*), 0 = none
#ifdef HT2_ENABLE_SPLICED
    int32_t  noncanSplPen; // --pen-noncansplice (12); --pen-cansplice is canSplPen above
    int32_t  conflictSplPen; // --pen-conflictsplice (1000000)
#endif
};
#define HT2_TRAN_XS_ONLY 1u   // --dta-cufflinks: reportHit drops spliced hits of unknown sense (hi_aligner.h:6101-6104)
#define HT2_TRAN_TMO     2u   // --tmo: reportHit drops hits not spliced through known sites only (hi_aligner.h:6126-6127)
#define HT2_TRAN_FILTERS (HT2_TRAN_XS_ONLY | HT2_TRAN_TMO)
#define HT2_TRAN_AVOID_PSEUDOGENE 4u   // --avoid-pseudogene: unspliced alignments near listed sites rank as spliced ones
                                       // (hi_aligner.h:6105-6125); read by the SAM formatter's selection key only

// An intron-length penalty function (--pen-canintronlen / --pen-noncanintronlen) as the runs of its integer value:
// the penalty of an intron of x bases is pen[k] for the last k with start[k] <= x.  The host evaluates
// max(0, SimpleFunc::f<int>(x)) for every length a kernel can score (ht2_set_intron_pen), so no device libm call
// is involved.  A function with more runs than HT2_INTRON_RUNS over that range is refused.
#define HT2_INTRON_RUNS 1024
struct Ht2IntronPen {
    uint32_t n;
    uint32_t start[HT2_INTRON_RUNS];
    int32_t  pen[HT2_INTRON_RUNS];
};

// Host-side parameters = the core + the --score-min table.  The table reaches the device as a
// separate 1 KB buffer (DevBatch::minscTab): keeping it out of the by-value kernel parameter keeps
// every Ht2ParamsCore field a constant-bank read (a 1.2 KB parameter indexed dynamically, or the
// whole struct behind a global pointer, cost 6 % of the aligner's throughput).
struct Ht2Params : Ht2ParamsCore {
    // --score-min as a table: SimpleFunc::f<TAlScore>(len) for every read length (hisat2.cpp:3380,
    // simple_func.h:86-108), computed once on the host so that host and device agree for every
    // function type (C, L, S = sqrt, G = log).  NOT yet clamped to <= 0.
    int32_t  minscTab[HT2_PARAMS_MAX_RDLEN + 1];
    // --n-ceil as a table, SimpleFunc::f<int>(len) with min 0 and max DBL_MAX (aligner_seed_policy.cpp:293-296, 547-549;
    // default L,0,0.15): the most Ns a read of that length may hold (Scoring::nFilter) and the DP's N ceiling
    // (SwAligner::initRead).  Read lengths above the table take its last entry.  It directly follows minscTab, and the
    // two travel as one buffer: the device's (DevBatch::minscTab) and the formatter's (Ht2SamIn::minscTab) hold the
    // N ceilings from HT2_PARAMS_NCEIL on, so no kernel parameter grows.
    int32_t  nCeilTab[HT2_PARAMS_MAX_RDLEN + 1];
    // The intron-length penalties, canonical ([0]) and non-canonical ([1]), as runs.  They follow nCeilTab in the same
    // buffer (the device reads them at nCeilTab + HT2_PARAMS_NCEIL); the spliced scorer is their only reader.
    Ht2IntronPen intronPen[2];
};
#define HT2_PARAMS_NCEIL (HT2_PARAMS_MAX_RDLEN + 1)
// the tables after the core, in int32 words: the size of the device buffer (DevBatch::minscTab)
#define HT2_PARAMS_TABLE_WORDS (2 * HT2_PARAMS_NCEIL + 2 * (sizeof(Ht2IntronPen) / sizeof(int32_t)))
static_assert(sizeof(Ht2Params) == sizeof(Ht2ParamsCore) + sizeof(int32_t) * HT2_PARAMS_TABLE_WORDS,
              "minscTab, nCeilTab and intronPen must be adjacent");

#endif
