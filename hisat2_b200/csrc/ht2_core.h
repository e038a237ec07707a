// ht2_core.h -- per-read HISAT2 alignment state machine (host+device).
//
// This is the GPU re-implementation of the reference's per-read hot path
// HI_Aligner::go (hi_aligner.h:4048) and everything below it, written as a
// self-contained, allocation-free state machine over a fixed-size per-read
// workspace so that one GPU thread can run one read (pair) to completion.
// Every function cites the reference lines whose behaviour it reproduces;
// results (the ordered list of reported alignments and the RNG state) must be
// identical to the reference's.
//
// The same source compiles for the device (the product) and for the host
// (tests/hostsim only: used to debug parity against oracle/_ref on machines
// without a GPU; the shipped library never runs it).
#ifndef HT2_CORE_H_
#define HT2_CORE_H_

#include "ht2_image.h"
#include "ht2_fm.h"
#include "ht2_seed.h"
#include "ht2_gwalk.h"
#include "ht2_params.h"
#include "ht2_ssdb.h"

#ifndef HT2_MAX_RDLEN
#define HT2_MAX_RDLEN 1024
#endif
#define HT2_SW_MAX_RDLEN 256   /* --bowtie2-dp: the score planes are quadratic in the read length; longer reads skip the DP and are flagged */
#define HT2_MAX_EDITS 128  /* edits of one (trial) hit: a 250-bp read at --very-sensitive scores admits ~80 deleted bases, a 1 000-base read ~100 mismatches */
#define HT2_MAX_PHITS 160   /* partial searches per strand: a 1 000-base read makes ~70 */
#ifndef HT2_MAX_GHITS
#define HT2_MAX_GHITS 64   /* max(khits, kseeds) anchors: --very-sensitive runs -k 30, i.e. 60 seeds */
#endif
#define HT2_POOL 64
#define HT2_IE_POOL 96           /* in-edge entries per strand (graph indexes) */
#define HT2_SEARCHED_BYTES 24576   /* ~600 searched hits (40 B typical) for both mates */

#define HT2_MAX_RES 128          /* reported alignments per mate (rs1u_ / rs2u_) */
#define HT2_MAX_PAIRS 256
#define HT2_RES_EDITS 2048        /* edits of ALL reported alignments of a read (pair): one arena instead of a fixed array per alignment */
#ifndef HT2_MAX_COORDS
#define HT2_MAX_COORDS 64
#endif
#define HT2_MAX_DEPTH 128
#ifndef HT2_DEPTH_CAP
#define HT2_DEPTH_CAP 48   /* recursion depth the workspace/stack is sized for */
#endif
#ifndef HT2_REFBUF
#define HT2_REFBUF (HT2_MAX_RDLEN + 128)   /* read + the read gaps minsc allows (combineWith window): 83 at minsc -256 with the default --rdg */
#endif

#define HT2_MIN_I64 ((int64_t)0x8000000000000000ll)
#define HT2_MIN_SCORE (HT2_MIN_I64 / 2)   /* getMinScore(), aln_sink.h:34 */

// error bits (per read); any bit set => results for the read are unreliable
#define HT2_ERR_EDITS     1u
#define HT2_ERR_PHITS     2u
#define HT2_ERR_GHITS     4u
#define HT2_ERR_POOL      8u
#define HT2_ERR_SEARCHED 16u
#define HT2_ERR_RES      32u
#define HT2_ERR_PAIRS    64u
#define HT2_ERR_COORDS  128u
#define HT2_ERR_RDLEN   256u
#define HT2_ERR_GRAPH   512u
#define HT2_ERR_DEPTH  1024u
#define HT2_ERR_OUTPUT 2048u
#define HT2_ERR_SPLICE 8192u   /* spliced mode (test build only): a spliced join was needed; that branch is not built yet */
#define HT2_ERR_SW     4096u   /* --bowtie2-dp scratch missing / rectangle wider than the scratch */

enum { HT2_EDIT_READ_GAP = 1, HT2_EDIT_REF_GAP, HT2_EDIT_MM, HT2_EDIT_SNP, HT2_EDIT_SPL };
enum { HT2_CANDIDATE_HIT = 1, HT2_PSEUDOGENE_HIT, HT2_ANCHOR_HIT }; // hi_aligner.h:96-100

struct Ht2Edit {          // edit.h:41-330
    uint32_t pos;
    uint8_t  chr;         // reference char ('A','C','G','T','N','-')
    uint8_t  qchr;        // read char
    uint8_t  type;
    uint8_t  pad;
    uint32_t snpID;
};
// HT2_SPL_* direction codes: ht2_ssdb.h (splice_site.h:37-43)
// A splice edit (type HT2_EDIT_SPL; spliced alignment, host test build only for now, DESIGN.md 8.2) keeps the
// same 12 bytes: intron length (20 bits) in chr | qchr << 8 | (pad & 15) << 16, direction in pad bits 4-6,
// "known site" in pad bit 7, and -- instead of the reference's donor / acceptor context words, whose only
// consumer is SpliceSiteDB::probscore in calculateScore -- that probability itself (float bits) in snpID.
HT2_HD uint32_t ht2_spl_len(const Ht2Edit& e) { return (uint32_t)e.chr | ((uint32_t)e.qchr << 8) | ((uint32_t)(e.pad & 15) << 16); }
HT2_HD uint32_t ht2_spl_dir(const Ht2Edit& e) { return (e.pad >> 4) & 7u; }
HT2_HD bool ht2_spl_known(const Ht2Edit& e) { return (e.pad >> 7) != 0; }
HT2_HD float ht2_spl_prob(const Ht2Edit& e) { union { uint32_t u; float f; } c; c.u = e.snpID; return c.f; }
HT2_HD void ht2_spl_set(Ht2Edit& e, uint32_t len, uint32_t dir, bool known, float prob) {
    e.chr = (uint8_t)len; e.qchr = (uint8_t)(len >> 8); e.pad = (uint8_t)(((len >> 16) & 15u) | ((dir & 7u) << 4) | (known ? 128u : 0u));
    union { uint32_t u; float f; } c; c.f = prob; e.snpID = c.u;
}
#define HT2_MAX_SPL_LEN 0xfffffu

struct Ht2Hit {           // GenomeHit, hi_aligner.h:431-1369
    uint32_t fw;
    uint32_t rdoff, len, trim5, trim3;
    uint32_t tidx, toff, joinedOff;
    int64_t  score;
    uint32_t hitcount;
    uint32_t nedits;
#ifdef HT2_ENABLE_SPLICED
    double   splicescore;
#endif
    Ht2Edit  edits[HT2_MAX_EDITS];
};

struct Ht2SearchedRec {   // what GenomeHit::operator== (hi_aligner.h:1156-1183) looks at
    uint32_t tidx, toff;
    uint16_t rdoff, len, trim5, trim3;
    uint8_t  fw, rdi;
    uint16_t nedits;
};
struct Ht2SearchedEdit { uint32_t pos; uint8_t type, chr, qchr, pad; };

struct Ht2BwtHit {        // BWTHit, hi_aligner.h:108-208
    uint32_t top, bot, node_top, node_bot;
    uint32_t bwoff, len;
    uint8_t  hit_type, hasCoords;
    uint8_t  ieOff, ieN;   // graph indexes: in-edge list of the hit inside Ht2ReadHits::ie
};

struct Ht2ReadHits {      // ReadBWTHit, hi_aligner.h:216-389
    uint32_t len, cur, done;
    uint32_t numPartialSearch, numUniqueSearch;
    uint32_t nhits;
    Ht2BwtHit hits[HT2_MAX_PHITS];
    uint16_t ie[HT2_IE_POOL][2];   // graph indexes: (node index in range, # extra incoming edges) of the hits
    uint32_t nie;
};

struct Ht2Coord {         // Coord, ref_coord.h:35
    uint32_t ref;
    uint32_t off;
    uint32_t fw;
    uint32_t joinedOff;
};

// One reported alignment == the fields reportHit hands to AlnRes::init
// (hi_aligner.h:6129-6166; AlnRes::setShape aligner_result.cpp:77-132).
struct Ht2Res {
    uint32_t tidx, toff;
    uint32_t fw;
    uint32_t rdlen;
    int64_t  score;
    uint32_t trim5p, trim3p;  // 5'/3' soft trimming in read orientation
    uint32_t rfextent;        // # reference chars covered
    uint32_t nedits;
    uint32_t editOff;         // AlnRes::ned() = Ht2Work::resEdits[editOff .. editOff + nedits): 5'->3', relative to trim5p
#ifdef HT2_ENABLE_SPLICED
    double   splicescore;     // AlnScore::splicescore_
    uint32_t spliced;         // GenomeHit::spliced().first (also "near splice sites")
    uint32_t knownTranscripts;
#endif
};

struct Ht2Read {
    uint32_t len;
    uint8_t  seq[2][HT2_MAX_RDLEN];   // [0]=fw, [1]=revcomp; codes 0..4
    uint8_t  qual[2][HT2_MAX_RDLEN];  // [0]=fw, [1]=reversed; raw ASCII
};

struct Ht2Rng {           // RandomSource, random_source.h:30-110
    uint32_t last;
    HT2_HD void init(uint32_t seed) { last = seed; }
    HT2_HD uint32_t nextU32() {
#if !defined(__CUDA_ARCH__) && defined(HT2_TRACE)
        fprintf(stderr, "RNG draw (state %u)\n", last);
#endif
        uint32_t ret;
        last = 1664525u * last + 1013904223u;
        ret = last >> 16;
        last = 1664525u * last + 1013904223u;
        ret ^= last;
        return ret;
    }
};

// One activation of hybridSearch_recur in the explicit-stack formulation
// (ht2_machine.h): the locals that must survive a "recursive call".
struct Ht2Frame {
    uint16_t pc;
    uint8_t  rdi, alignMate, use_localindex, success, first, uniqueStop;
    const Ht2Hit* hit;
    Ht2Hit*  tempHit;
    uint32_t hitoff, hitlen, dep, count, extoff, extlen, ncoords, nLocalHits, ti, poolMark;
    uint32_t ssi, ssHi;       // cursor over the splice-site DB's sites of this activation (ssi == 0xffffffff: range not computed yet)
    int32_t  lid, ri;
    int64_t  maxsc, prev_score, cushion;
    Ht2Coord coords[8];
    uint16_t localHits[16];
};

// Scratch of one alignWithALTs call (graph indexes; ht2_alt.h)
#define HT2_ALT_TMP_EDITS 72     /* trial edit list of the ALT recursion: a 27-base deletion ALT alone is 27 read-gap edits */
#define HT2_ALT_CANDS 4
#define HT2_ALT_BUFS 4
#define HT2_ALT_MAXDEP 24
struct Ht2AltScratch {
    Ht2Edit  tmp[HT2_ALT_TMP_EDITS];        // tmp_edits
    uint32_t ntmp;
    int32_t  best_rdoff;
    uint32_t numALTsTried;
    uint32_t nbuf;                          // reference-window buffers in use (stack discipline)
    uint8_t  wantCands, ncand, candN[HT2_ALT_CANDS], pad[2];
    Ht2Edit  cand[HT2_ALT_CANDS][HT2_MAX_EDITS];   // candidate_edits: equally long alternatives (adjustWithALT)
    alignas(8) uint8_t ref[HT2_ALT_BUFS][HT2_REFBUF + 16];
};

// Scratch of one --bowtie2-dp problem (ht2_sw.h).  One per EXECUTING lane (a
// problem starts and ends inside one state-machine segment), not per read slot,
// and only allocated when --bowtie2-dp is on.
#define HT2_SW_MAXGAP 10
#define HT2_SW_MAXCOLS (HT2_SW_MAX_RDLEN + 4 * HT2_SW_MAXGAP)
#define HT2_SW_MAX_EDITS 160
#define HT2_SW_SEG ((HT2_SW_MAX_RDLEN + 1) / 2)     /* words per column: 2 rows (s16 halves) per 32-bit word */
// The three score matrices H, E, F (column-major, one spare column) live OUTSIDE the scratch struct, in a plane pool of
// HT2_SW_POOL_WORDS words per executing lane.  Two stripings of a column share that space (ht2_sw.h):
//   lane fill (swFill, host and single-lane device path): 2 rows per word -- row i = half i / seg of word i % seg,
//     seg = ceil(nrow / 2);
//   warp fill (swFillCoop, the pool kernel's DP rounds): an anti-diagonal wavefront, lane L owning the R = ceil(nrow / 32)
//     rows L*R .., stored step-major: ncol + 31 steps of 32 * ceil(R / 2) words.
#define HT2_SW_PLANE_WORDS ((HT2_SW_MAXCOLS + 32) * HT2_SW_SEG)
#define HT2_SW_POOL_WORDS (3 * HT2_SW_PLANE_WORDS + 7 * HT2_SW_SEG)   /* per lane: H, E, F + query profile (5) + gap barrier + barrier/read-gap-open words */
struct Ht2SwRect { int64_t refl, refr; uint32_t triml, trimr, corel, corer; };
struct Ht2SwScratch {
    uint32_t rep[((size_t)HT2_SW_MAXCOLS * HT2_SW_MAX_RDLEN + 31) / 32];   // reported-through bit per cell (col * nrow + row)
    uint32_t nrow, seg;
    uint32_t coop, rcp;                                      // layout of the planes: 0 = lane fill (striped), 1 = warp fill (seg = rows per lane, rcp = ceil(65536 / seg))
    // the framed problem (swPrepare -> swFill / swFillCoop -> swFinish)
    const uint8_t* jrd; const uint8_t* jqu; const uint8_t* jrf;
    uint32_t jncol, jfw;
    int64_t  jmsc, jbest;
    Ht2SwRect jrect;
    int32_t  lastH[HT2_SW_MAXCOLS];                          // last-row H per column (the candidates)
    uint8_t  rowPen[HT2_SW_MAX_RDLEN];                          // mismatch penalty of each read row
    alignas(8) uint8_t rf[HT2_SW_MAXCOLS + 16];              // reference window, codes 0..4
    Ht2Edit  ned[HT2_SW_MAX_EDITS];
};
static_assert(HT2_SW_SEG >= 32 * ((((HT2_SW_MAX_RDLEN + 31) / 32) + 1) / 2), "warp fill: 32 lanes x ceil(R / 2) words per step fit a column of the pool");

// Per-read (pair) workspace.  One per in-flight GPU thread.
struct alignas(128) Ht2Work {
    // ---- scalars first: every segment of the state machine starts by reading a handful of them, and a slot's
    // workspace is cold (evicted from L1, often from L2) when its next round begins -- three adjacent 128-byte
    // lines instead of twenty scattered over 240 kB
    // explicit-stack state machine (ht2_machine.h)
    int64_t     childRet;
    uint32_t    st, nFrames;
    uint8_t     curRdi, curFw, alignRet, pad8;
    uint8_t     found[2][2];
    uint32_t    err;
    uint32_t    nGenomeHits, poolTop;
    uint32_t    searchedTop;                // bytes used
    uint32_t    nSearched[2];
    uint32_t    nRes[2], nResEdits, nPairs, nCoords, nCurIe, nOffDiffs;
    // AlnSinkWrap best-score tracking (aln_sink.h:2600-2655)
    int64_t     bestPair, best2Pair, bestUnp[2], best2Unp[2];
#ifdef HT2_ENABLE_SPLICED
    uint32_t    bestSplicedUnp[2];          // # splice edits of the best unpaired alignment (aln_sink.h:2610-2640)
#endif
    // ReportingState (aln_sink.cpp:33-340), reduced to what the path reads back
    uint32_t    nconcord, nunpair[2];
    uint32_t    doneConcord, doneUnpair[2], stDone;
    int64_t     concordBest;
    uint32_t    concordInspected[2];        // _concordantIdxInspected
    Ht2Rng      rnd;
    // work counters (HIMetrics hi_aligner.h:3897 + roofline accounting)
    uint32_t    localindexatts;
    uint32_t    maxLocalindexatts;
    uint32_t    nLF;      // LF steps (boundary ranks) executed
    uint32_t    nSides;   // sides touched
    uint32_t    algBytes; // algorithmic bytes: sides*sideSz + ftab/eftab entries + SA samples + 2-bit ref bytes
    uint32_t    maxPool, maxDepth, maxEdits; // high-water marks (sizing evidence)
    // per-read configuration (so a workspace can be resumed by any lane)
    int64_t     cfgMinsc[2];
    uint8_t     cfgPaired, cfgRightendonly, cfgNofw[2], cfgNorc[2], cfgPad[2];
    uint32_t    unit, filtBits;
    uint32_t    hybIter, hybHj, mateI, mateJ, mateSize[2];
    // partialSearch continuation (time slicing, HT2_PS_SLICE): a search that has not finished after a slice of LF
    // steps parks its loop state here and the slot stays in TS_PS, so that a round never lasts longer than one slice
    // while most lanes of the group have long finished (a partial search of a 101-bp read is ~12 steps on average,
    // ~90 at most; the searches of 1 000-base reads run to hundreds)
    uint32_t    psCont, psTop, psBot, psNtop, psNbot, psDep, psSame, psSimilar;
    uint8_t     psPseudo, psAnchor, psPad[2];
    // ---- arrays
    Ht2SeedResume psG;                      // the same for graph indexes (ht2_seed_partial)
    Ht2Read     rd[2];
    Ht2ReadHits hits[2][2];                 // [mate][fw=0/rc=1]
    Ht2Frame    frames[HT2_DEPTH_CAP];
    Ht2Hit      genomeHits[HT2_MAX_GHITS];  // _genomeHits
    uint8_t     genomeHitsDone[HT2_MAX_GHITS];
    Ht2Hit      pool[HT2_POOL];             // GenomeHit temporaries (stack)
    // _hits_searched (hi_aligner.h:6898-6922) as compact records in one arena shared by both
    // mates: exactly the fields GenomeHit::operator== compares (Ht2SearchedRec + 8 B per edit)
    alignas(8) uint8_t searched[HT2_SEARCHED_BYTES];
    Ht2Res      res[2][HT2_MAX_RES];        // rs1u_/rs2u_ of AlnSinkWrap
    Ht2Edit     resEdits[HT2_RES_EDITS];    // their edits, appended in report order
    uint16_t    pairs[HT2_MAX_PAIRS][2];    // rs1_/rs2_ as indexes into res
    Ht2Coord    coords[HT2_MAX_COORDS];     // BWTHit::_coords scratch
    alignas(8) uint8_t refbuf[HT2_REFBUF + 16];   // getStretch stores 32-bit words
    alignas(8) uint8_t refbuf2[HT2_REFBUF + 16];
    int64_t     tscores[HT2_MAX_RDLEN];
    int64_t     tscores2[HT2_MAX_RDLEN];
    Ht2AltScratch alt;                      // graph indexes only
    Ht2GWalk    gw;                         // group walk over graph indexes (ht2_gwalk.h)
    uint16_t    curIe[24][2];               // in-edge list of the most recent global/local GFM search (graph)
    uint32_t    offDiffs[40][2];            // findOffDiffs scratch: (|diff|, sign as 0/1/2 = -1/0/+1)
};

// ------------------------------------------------------------------------
// Scoring helpers (scoring.h:259-318, 96-130)
// ------------------------------------------------------------------------
HT2_HD int ht2_mmpen(const Ht2ParamsCore& P, int q) {
    if (P.mmcostConstant) return P.mmpMax;
    if (q < 0) q = 0;
    int ii = q < 40 ? q : 40;
    float frac = (float)ii / 40.0f;
    return P.mmpMin + (int)(frac * (float)(P.mmpMax - P.mmpMin));
}
// Scoring::score(rdc, refm, q)
HT2_HD int ht2_score(const Ht2ParamsCore& P, int rdc, int refm, int q) {
    if (rdc > 3 || refm > 15) return -P.npen;
    if ((refm & (1 << rdc)) != 0) return 0;
    return -ht2_mmpen(P, q);
}
// Scoring::sc(q) soft-clip penalty (scoring.h:312-318)
HT2_HD int ht2_scpen(const Ht2ParamsCore& P, int q) {
    if (q <= 33) return P.scpMin;
    q -= 33;
    if (q > 40) q = 40;
    return (int)(((float)q / 40.0f) * (float)(P.scpMax - P.scpMin) + (float)P.scpMin);
}
HT2_HD int ht2_asc2code(uint8_t ch) { // dna2col[ch]-'0'
    switch (ch) { case 'A': return 0; case 'C': return 1; case 'G': return 2; case 'T': return 3; default: return 4; }
}
HT2_HD int ht2_asc2mask(uint8_t ch) { // asc2dnamask[ch]
    switch (ch) { case 'A': return 1; case 'C': return 2; case 'G': return 4; case 'T': return 8; case 'N': return 15; default: return 0; }
}
HT2_HD uint8_t ht2_code2asc(int c) { return (uint8_t)("ACGTN"[c]); }
// Scoring::maxReadGaps / maxRefGaps (scoring.cpp:42-98); match bonus is 0.
HT2_HD int ht2_max_gaps(int64_t minsc, int open, int ext) {
    int64_t sc = 0;
    bool first = true;
    int num = 0;
    while (sc >= minsc) {
        if (first) { first = false; sc -= open; }
        else sc -= ext;
        num++;
    }
    return num - 1;
}

// ------------------------------------------------------------------------
// 2 x s16 SIMD-in-word: the DPX instructions of sm_90 (VIADDMNMX / VIMNMX3 .S16x2), with
// portable forms for the host test build
// ------------------------------------------------------------------------
HT2_HD uint32_t ht2_v2_addmax(uint32_t a, uint32_t b, uint32_t c) {   // per half: max(a + b, c), signed
#ifdef __CUDA_ARCH__
    return __viaddmax_s16x2(a, b, c);
#else
    uint32_t r = 0;
    for (int k = 0; k < 32; k += 16) {
        int x = (int16_t)(a >> k) + (int16_t)(b >> k), y = (int16_t)(c >> k);
        r |= (uint32_t)(uint16_t)(x > y ? x : y) << k;
    }
    return r;
#endif
}
HT2_HD uint32_t ht2_v2_max(uint32_t a, uint32_t b) {                  // per half: signed max
#ifdef __CUDA_ARCH__
    return __vmaxs2(a, b);
#else
    uint32_t r = 0;
    for (int k = 0; k < 32; k += 16) { int x = (int16_t)(a >> k), y = (int16_t)(b >> k); r |= (uint32_t)(uint16_t)(x > y ? x : y) << k; }
    return r;
#endif
}
HT2_HD uint32_t ht2_v2_max3(uint32_t a, uint32_t b, uint32_t c) {
#ifdef __CUDA_ARCH__
    return __vimax3_s16x2(a, b, c);
#else
    return ht2_v2_max(ht2_v2_max(a, b), c);
#endif
}
HT2_HD uint32_t ht2_v2_splat(int v) { return (uint32_t)(uint16_t)v * 0x00010001u; }

#ifdef HT2_ENABLE_SPLICED
#include <math.h>
// ------------------------------------------------------------------------
// Spliced alignment (host test build only for now; DESIGN.md 8.2).
// Splice-site probability model (splice_site.cpp:30-111, 788-850, the model compiled in by default):
// position weight matrices for the donor (3 exonic + 6 intronic bases, Yeo & Burge 2004) and the acceptor
// (14 intronic + 1 exonic bases, Solovyev), turned into exp(-sum log(p / background)) tables exactly
// like init_junction_prob (float logf / expf: bit-identical to the reference's tables, checked against
// a dump of the compiled reference).
// ------------------------------------------------------------------------
struct Ht2SplTables { float donor[1 << 18], acc1[1 << 14], acc2[1 << 16]; };
inline const Ht2SplTables& ht2_spl_tables() {   // host function: a device build receives the tables as a buffer
    static Ht2SplTables* T = NULL;
    if (T) return *T;
    static const float bg[4] = {0.27f, 0.23f, 0.23f, 0.27f};
    static const float donorP[4][9] = {
        {0.340f, 0.604f, 0.092f, 0.001f, 0.001f, 0.526f, 0.713f, 0.071f, 0.160f},
        {0.363f, 0.129f, 0.033f, 0.001f, 0.001f, 0.028f, 0.076f, 0.055f, 0.165f},
        {0.183f, 0.125f, 0.803f, 1.000f, 0.001f, 0.419f, 0.118f, 0.814f, 0.209f},
        {0.114f, 0.142f, 0.073f, 0.001f, 1.000f, 0.025f, 0.093f, 0.059f, 0.462f}};
    static const float accP[4][15] = {
        {0.090f, 0.084f, 0.075f, 0.068f, 0.076f, 0.080f, 0.097f, 0.092f, 0.076f, 0.078f, 0.237f, 0.042f, 1.000f, 0.001f, 0.239f},
        {0.310f, 0.310f, 0.307f, 0.293f, 0.326f, 0.330f, 0.373f, 0.385f, 0.410f, 0.352f, 0.309f, 0.708f, 0.001f, 0.001f, 0.138f},
        {0.125f, 0.115f, 0.106f, 0.104f, 0.110f, 0.113f, 0.113f, 0.085f, 0.066f, 0.064f, 0.212f, 0.003f, 0.001f, 1.000f, 0.520f},
        {0.463f, 0.440f, 0.470f, 0.494f, 0.471f, 0.463f, 0.408f, 0.429f, 0.445f, 0.504f, 0.240f, 0.246f, 0.001f, 0.001f, 0.104f}};
    Ht2SplTables* t = new Ht2SplTables();
    float d[4][9], a[4][15];
    for (int i = 0; i < 9; i++) for (int j = 0; j < 4; j++) d[j][i] = logf(donorP[j][i] / bg[j]);
    for (int i = 0; i < 15; i++) for (int j = 0; j < 4; j++) a[j][i] = logf(accP[j][i] / bg[j]);
    for (uint32_t i = 0; i < (1u << 18); i++) { float sum = 0.0f; for (int j = 0; j < 9; j++) sum += d[(i >> (j << 1)) & 3][9 - j - 1]; t->donor[i] = expf(-sum); }
    for (uint32_t i = 0; i < (1u << 14); i++) { float sum = 0.0f; for (int j = 0; j < 7; j++) sum += a[(i >> (j << 1)) & 3][7 - j - 1]; t->acc1[i] = expf(-sum); }
    for (uint32_t i = 0; i < (1u << 16); i++) { float sum = 0.0f; for (int j = 0; j < 8; j++) sum += a[(i >> (j << 1)) & 3][15 - j - 1]; t->acc2[i] = expf(-sum); }
    T = t;
    return *T;
}
// SpliceSiteDB::probscore (splice_site.cpp:832-850)
HT2_HD float ht2_spl_probscore(const Ht2SplTables& T, int64_t donor_seq, int64_t acceptor_seq) {
    float probscore = T.donor[donor_seq & 0x3ffff];
    probscore *= T.acc1[(acceptor_seq >> 16) & 0x3fff];
    probscore *= T.acc2[acceptor_seq % (1 << 16)];
    probscore = (float)(1.0 / (1.0 + probscore));
    return probscore;
}
// MaxIntronLen / intronLen_prob (hi_aligner.h:48-89)
HT2_HD uint32_t ht2_max_intron_len(uint32_t anchor, uint32_t minAnchorLen) {
    uint32_t intronLen = 0;
    if (anchor >= minAnchorLen) { if (anchor < 2) anchor = 2; uint32_t shift = (anchor << 1) - 4; shift = shift < 13 ? 13 : shift; shift = shift > 30 ? 30 : shift; intronLen = 1u << shift; }
    return intronLen;
}
HT2_HD uint32_t ht2_max_intron_len_noncan(uint32_t anchor, uint32_t minAnchorLenNoncan) {
    uint32_t intronLen = 0;
    if (anchor >= minAnchorLenNoncan) { if (anchor < 5) anchor = 5; uint32_t shift = (anchor << 1) - 10; shift = shift > 30 ? 30 : shift; intronLen = 1u << shift; }
    return intronLen;
}
HT2_HD float ht2_intron_len_prob(uint32_t anchor, uint32_t intronLen, uint32_t maxIntronLen) {
    uint32_t expected = maxIntronLen;
    if (anchor < 14) expected = 1u << ((anchor << 1) + 4);
    if (expected > maxIntronLen) expected = maxIntronLen;
    float result = ((float)intronLen) / ((float)expected);
    if (result > 1.0f) result = 1.0f;
    return result;
}
HT2_HD float ht2_intron_len_prob_noncan(uint32_t anchor, uint32_t intronLen, uint32_t maxIntronLen) {
    uint32_t expected = maxIntronLen;
    if (anchor < 16) expected = 1u << (anchor << 1);
    if (expected > maxIntronLen) expected = maxIntronLen;
    float result = ((float)intronLen) / ((float)expected);
    if (result > 1.0f) result = 1.0f;
    return result;
}
// Scoring::canSpl / noncanSpl (scoring.h:473-487) with the default penalty functions
// (--pen-cansplice 0, --pen-noncansplice 12, --pen-canintronlen / --pen-noncanintronlen G,-8,1; hisat2.cpp:493-497)
#define HT2_PEN_CONFLICTSPLICE 1000000
// max(0, (int)(-8 + ln(x))) as integer breakpoints (the first x at which the value becomes k, found by
// scanning the double-precision expression; exhaustively equal to it for x <= 2e6): no libm call, so the
// device build will agree with the host bit for bit
HT2_HD int64_t ht2_intron_pen(int intronlen) {
    const uint32_t bp[13] = {8104u, 22027u, 59875u, 162755u, 442414u, 1202605u, 3269018u, 8886111u, 24154953u,
                                    65659970u, 178482301u, 485165196u, 1318815735u};
    int pen = 0;
    if (intronlen > 0) for (int k = 0; k < 13 && (uint32_t)intronlen >= bp[k]; k++) pen = k + 1;
    return pen;
}
#endif // HT2_ENABLE_SPLICED

// ------------------------------------------------------------------------
// The aligner
// ------------------------------------------------------------------------
// NOSPL = true compiles the aligner for --no-spliced-alignment only: every spliced branch (the spliced join of
// combineWith, splice scoring, intron windows) becomes dead code.  The pool kernel is bound by instruction fetch
// (DESIGN.md 4.1), so the DNA configuration gets its own, smaller instantiation; NOSPL = false reads the option.
template <bool GRAPH, bool NOSPL = false>
struct Ht2AlignerT {
    HT2_HD bool noSpl() const { return NOSPL ? true : (P->noSplicedAlignment != 0); }
    const uint8_t*        blob;
    const Ht2ImageHeader* H;
    Ht2Fm<uint32_t>       gfm;
    const Ht2ParamsCore*  P;
    Ht2Work*              W;
    Ht2SwScratch*         sw;      // --bowtie2-dp scratch of this lane (NULL when dp is off)
    uint32_t*             swPl;    // the lane's first word in the H / E / F plane pool
    uint32_t              swStride;
    uint32_t              swStage; // 0, or set by the pool kernel's DP round: 1 = problem framed and filled by the warp, 2 = nothing to fill (answer in swRetv)
    bool                  swRetv;
#ifdef HT2_ENABLE_SPLICED
    const Ht2SplTables*   splT;    // donor / acceptor probability tables (spliced mode)
    const uint8_t*        ssT;     // read-only splice-site DB of the run (ht2_ssdb.h), NULL = empty (SpliceSiteDB::empty())
#endif
    bool     paired;
    bool     rightendonly;
    bool     nofw[2], norc[2];
    int64_t  minsc[2];

    // save / restore the per-read configuration in the workspace
    HT2_HD void saveCfg() {
        W->cfgPaired = paired; W->cfgRightendonly = rightendonly;
        W->cfgNofw[0] = nofw[0]; W->cfgNofw[1] = nofw[1]; W->cfgNorc[0] = norc[0]; W->cfgNorc[1] = norc[1];
        W->cfgMinsc[0] = minsc[0]; W->cfgMinsc[1] = minsc[1];
    }
    HT2_HD void attach(Ht2Work* W_) {
        W = W_;
        paired = W->cfgPaired != 0; rightendonly = W->cfgRightendonly != 0;
        nofw[0] = W->cfgNofw[0] != 0; nofw[1] = W->cfgNofw[1] != 0; norc[0] = W->cfgNorc[0] != 0; norc[1] = W->cfgNorc[1] != 0;
        minsc[0] = W->cfgMinsc[0]; minsc[1] = W->cfgMinsc[1];
    }
    HT2_HD void bind(const uint8_t* blob_, const Ht2ParamsCore* P_, Ht2Work* W_) {
        blob = blob_;
        H = (const Ht2ImageHeader*)blob_;
        gfm.init(blob_, &H->global);
        P = P_;
        W = W_;
        sw = NULL; swPl = NULL; swStride = 1; swStage = 0; swRetv = false;
#ifdef HT2_ENABLE_SPLICED
        splT = NULL; ssT = NULL;
#endif
    }

    // ---- edits / hits ---------------------------------------------------
    HT2_NI static void copyHit(Ht2Hit& d, const Ht2Hit& s) {
        d.fw = s.fw; d.rdoff = s.rdoff; d.len = s.len; d.trim5 = s.trim5; d.trim3 = s.trim3;
        d.tidx = s.tidx; d.toff = s.toff; d.joinedOff = s.joinedOff; d.score = s.score;
        d.hitcount = 1; // GenomeHit::init resets _hitcount (hi_aligner.h:569)
#ifdef HT2_ENABLE_SPLICED
        d.splicescore = s.splicescore;
#endif
        d.nedits = s.nedits;
        for (uint32_t i = 0; i < s.nedits; i++) d.edits[i] = s.edits[i];
    }
    HT2_HD static void initHit(Ht2Hit& h, bool fw, uint32_t rdoff, uint32_t len, uint32_t trim5, uint32_t trim3,
                               uint32_t tidx, uint32_t toff, uint32_t joinedOff) {
        h.fw = fw ? 1 : 0; h.rdoff = rdoff; h.len = len; h.trim5 = trim5; h.trim3 = trim3;
        h.tidx = tidx; h.toff = toff; h.joinedOff = joinedOff; h.score = 0; h.hitcount = 1; h.nedits = 0;
#ifdef HT2_ENABLE_SPLICED
        h.splicescore = 0.0;
#endif
    }
    HT2_HD static Ht2Edit mkEdit(uint32_t pos, uint8_t chr, uint8_t qchr, uint8_t type) {
        Ht2Edit e; e.pos = pos; e.chr = chr; e.qchr = qchr; e.type = type; e.pad = 0; e.snpID = HT2_IDX_MAX32; return e;
    }
    HT2_HD bool pushEdit(Ht2Hit& h, const Ht2Edit& e) {
        if (h.nedits >= HT2_MAX_EDITS) { W->err |= HT2_ERR_EDITS; return false; }
        h.edits[h.nedits++] = e; if (h.nedits > W->maxEdits) W->maxEdits = h.nedits; return true;
    }
    HT2_NI bool insertEditFront(Ht2Hit& h, const Ht2Edit& e) {
        if (h.nedits >= HT2_MAX_EDITS) { W->err |= HT2_ERR_EDITS; return false; }
        for (uint32_t i = h.nedits; i > 0; i--) h.edits[i] = h.edits[i - 1];
        h.edits[0] = e; h.nedits++; if (h.nedits > W->maxEdits) W->maxEdits = h.nedits; return true;
    }
    HT2_HD static bool editEq(const Ht2Edit& a, const Ht2Edit& b) { // Edit::operator== (edit.h)
        if (a.type != b.type) return false;
        if (a.pos != b.pos) return false;
#ifdef HT2_ENABLE_SPLICED
        if (a.type == HT2_EDIT_SPL) return ht2_spl_len(a) == ht2_spl_len(b) && ht2_spl_dir(a) == ht2_spl_dir(b);
#endif
        return a.chr == b.chr && a.qchr == b.qchr;
    }
    HT2_HD static bool isGapOrSnp(const Ht2Edit& e) {
        return e.type == HT2_EDIT_SPL || e.type == HT2_EDIT_READ_GAP || e.type == HT2_EDIT_REF_GAP ||
               (e.type == HT2_EDIT_MM && e.snpID != HT2_IDX_MAX32);
    }
    // GenomeHit::operator== (hi_aligner.h:1156-1183)
    HT2_HD static bool hitEq(const Ht2Hit& a, const Ht2Hit& b) {
        if (a.fw != b.fw || a.rdoff != b.rdoff || a.len != b.len || a.tidx != b.tidx || a.toff != b.toff ||
            a.trim5 != b.trim5 || a.trim3 != b.trim3) return false;
        if (a.nedits != b.nedits) return false;
        for (uint32_t i = 0; i < a.nedits; i++) {
            const Ht2Edit& e = a.edits[i]; const Ht2Edit& oe = b.edits[i];
            if (e.type == HT2_EDIT_READ_GAP) { if (oe.type != HT2_EDIT_READ_GAP) return false; }
            else if (e.type == HT2_EDIT_REF_GAP) { if (oe.type != HT2_EDIT_REF_GAP) return false; }
            else if (!editEq(e, oe)) return false;
        }
        return true;
    }
    // Edit::invertPoss (edit.cpp:70-111), sort=false
    HT2_HD static void invertPoss(Ht2Edit* ed, uint32_t n, uint32_t sz) {
        for (uint32_t i = 0; i < n / 2; i++) { Ht2Edit t = ed[i]; ed[i] = ed[n - i - 1]; ed[n - i - 1] = t; }
        for (uint32_t i = 0; i < n; i++) {
            if (ed[i].type == HT2_EDIT_READ_GAP || ed[i].type == HT2_EDIT_SPL) ed[i].pos = (uint32_t)(sz - ed[i].pos);
            else ed[i].pos = (uint32_t)(sz - ed[i].pos - 1);
        }
    }
    HT2_HD Ht2Hit* poolAlloc() {
        if (W->poolTop >= HT2_POOL) { W->err |= HT2_ERR_POOL; return &W->pool[HT2_POOL - 1]; }
        if (W->poolTop + 1 > W->maxPool) W->maxPool = W->poolTop + 1;
        return &W->pool[W->poolTop++];
    }


#ifdef HT2_ENABLE_SPLICED
    // ---- the run's splice-site DB (ht2_ssdb.h) ---------------------------------
    HT2_HD bool ssdbEmpty() const { return ssT == NULL; }   // SpliceSiteDB::empty(): false once a file was read, even one without sites
    // GenomeHit::getLeftAnchor / getRightAnchor (hi_aligner.h:1040-1079)
    HT2_HD static void getLeftAnchor(const Ht2Hit& h, uint32_t& anchor, uint32_t& nedits) {
        anchor = h.len; nedits = 0;
        for (uint32_t i = 0; i < h.nedits; i++) {
            const Ht2Edit& e = h.edits[i];
            if (e.type == HT2_EDIT_SPL) { anchor = e.pos; break; }
            else if (e.type == HT2_EDIT_MM || e.type == HT2_EDIT_READ_GAP || e.type == HT2_EDIT_REF_GAP) nedits++;
        }
    }
    HT2_HD static void getRightAnchor(const Ht2Hit& h, uint32_t& anchor, uint32_t& nedits) {
        anchor = h.len; nedits = 0;
        for (int i = (int)h.nedits - 1; i >= 0; i--) {
            const Ht2Edit& e = h.edits[i];
            if (e.type == HT2_EDIT_SPL) { anchor = h.len - e.pos - 1; break; }
            else if (e.type == HT2_EDIT_MM || e.type == HT2_EDIT_READ_GAP || e.type == HT2_EDIT_REF_GAP) nedits++;
        }
    }
    // GFM::textOffToJoined (gfm.h:5603-5650): (reference, offset) -> offset in the joined text; false inside an N gap
    HT2_NI bool textOffToJoined(uint32_t tid, uint32_t textoff, uint32_t& off) const {
        const uint32_t nFrag = gfm.g->nFrag;
        const uint32_t* rs = gfm.rstarts;
        uint32_t top = 0, bot = nFrag, elt = HT2_IDX_MAX32;
        while (true) {
            const uint32_t oldelt = elt;
            elt = top + ((bot - top) >> 1);
            if (oldelt == elt) return false;
            const uint32_t elt_tid = rs[elt * 3 + 1];
            if (elt_tid == tid) {
                while (true) {
                    if (tid != rs[elt * 3 + 1]) return false;
                    if (rs[elt * 3 + 2] <= textoff) break;
                    if (elt == 0) return false;
                    elt--;
                }
                while (true) {
                    if (elt + 1 == nFrag || tid + 1 == rs[(elt + 1) * 3 + 1] || textoff < rs[(elt + 1) * 3 + 2]) {
                        off = rs[elt * 3] + (textoff - rs[elt * 3 + 2]);
                        if (elt + 1 < nFrag && tid == rs[(elt + 1) * 3 + 1] && off >= rs[(elt + 1) * 3]) return false;
                        break;
                    }
                    elt++;
                }
                break;
            } else if (elt_tid < tid) top = elt;
            else bot = elt;
        }
        return true;
    }
#else
    HT2_HD bool ssdbEmpty() const { return true; }
#endif

    // GenomeHit::getLeft (hi_aligner.h:919-957)
    HT2_NI void getLeft(const Ht2Hit& h, uint32_t& rdoff, uint32_t& len, uint32_t& toff, int64_t* score, uint32_t rdi) const {
        toff = h.toff; rdoff = h.rdoff; len = h.len;
        if (score) *score = 0;
        const uint8_t* qual = W->rd[rdi].qual[h.fw ? 0 : 1];
        for (uint32_t i = 0; i < h.nedits; i++) {
            const Ht2Edit& e = h.edits[i];
            if (isGapOrSnp(e)) { len = e.pos; break; }
            if (score && e.type == HT2_EDIT_MM && e.snpID == HT2_IDX_MAX32)
                *score += ht2_score(*P, ht2_asc2code(e.qchr), ht2_asc2mask(e.chr), (int)qual[h.rdoff + e.pos] - 33);
        }
    }
    // GenomeHit::getRightOff (hi_aligner.h:1020-1035)
    HT2_HD static uint32_t getRightOff(const Ht2Hit& h) {
        uint32_t toff = h.toff + h.len;
        for (uint32_t i = 0; i < h.nedits; i++) {
            if (h.edits[i].type == HT2_EDIT_READ_GAP) toff++;
            else if (h.edits[i].type == HT2_EDIT_REF_GAP) toff--;
#ifdef HT2_ENABLE_SPLICED
            else if (h.edits[i].type == HT2_EDIT_SPL) toff += ht2_spl_len(h.edits[i]);
#endif
        }
        return toff;
    }
    // GenomeHit::getRight (hi_aligner.h:962-1015)
    HT2_NI void getRight(const Ht2Hit& h, uint32_t& rdoff, uint32_t& len, uint32_t& toff, int64_t* score, uint32_t rdi) const {
        toff = h.toff; rdoff = h.rdoff; len = h.len;
        if (score) *score = 0;
        if (h.nedits == 0) return;
        const uint8_t* qual = W->rd[rdi].qual[h.fw ? 0 : 1];
        for (int i = (int)h.nedits - 1; i >= 0; i--) {
            const Ht2Edit& e = h.edits[i];
            if (isGapOrSnp(e)) {
                rdoff = h.rdoff + e.pos;
                len = h.len - e.pos;
                if (e.type == HT2_EDIT_REF_GAP) { rdoff++; len--; }
                else if (e.type == HT2_EDIT_MM) { rdoff++; len--; }
                toff = getRightOff(h) - len;
                break;
            }
            if (score && e.type == HT2_EDIT_MM && e.snpID == HT2_IDX_MAX32)
                *score += ht2_score(*P, ht2_asc2code(e.qchr), ht2_asc2mask(e.chr), (int)qual[h.rdoff + e.pos] - 33);
        }
    }

    // GenomeHit::calculateScore (hi_aligner.h:3711-3891); splice edits in the HT2_ENABLE_SPLICED build.
    HT2_NI int64_t calculateScore(Ht2Hit& h, uint32_t rdi) const {
        int64_t score = 0;
        const uint8_t* qual = W->rd[rdi].qual[h.fw ? 0 : 1];
#ifdef HT2_ENABLE_SPLICED
        double splicescore = 0; uint32_t numsplices = 0, mm = 0;
        bool conflict_splicesites = false; uint8_t whichsense = HT2_SPL_UNKNOWN;
        const uint32_t rdlenS = W->rd[rdi].len;
#endif
        for (uint32_t i = 0; i < h.nedits; i++) {
            const Ht2Edit& e = h.edits[i];
            if (e.type == HT2_EDIT_MM) {
                if (e.snpID == HT2_IDX_MAX32) {
                    score += ht2_score(*P, ht2_asc2code(e.qchr), ht2_asc2mask(e.chr), (int)qual[h.rdoff + e.pos] - 33);
#ifdef HT2_ENABLE_SPLICED
                    mm++;
#endif
                }
            } else if (e.type == HT2_EDIT_READ_GAP) {
                bool open = true;
                if (i > 0 && h.edits[i - 1].type == HT2_EDIT_READ_GAP && h.edits[i - 1].pos == e.pos) open = false;
                if (e.snpID == HT2_IDX_MAX32) score -= open ? (P->rdGapConst + P->rdGapLinear) : P->rdGapLinear;
            } else if (e.type == HT2_EDIT_REF_GAP) {
                bool open = true;
                if (i > 0 && h.edits[i - 1].type == HT2_EDIT_REF_GAP && h.edits[i - 1].pos + 1 == e.pos) open = false;
                if (e.snpID == HT2_IDX_MAX32) score -= open ? (P->rfGapConst + P->rfGapLinear) : P->rfGapLinear;
            }
#ifdef HT2_ENABLE_SPLICED
            else if (e.type == HT2_EDIT_SPL) {   // hi_aligner.h:3745-3838
                const uint32_t eDir = ht2_spl_dir(e), eLen = ht2_spl_len(e);
                const bool canon = (eDir == HT2_SPL_FW || eDir == HT2_SPL_RC);
                if (!ht2_spl_known(e)) {
                    int left_anchor_len = (int)(h.rdoff + e.pos);
                    int right_anchor_len = (int)rdlenS - left_anchor_len;
                    uint32_t mm2 = 0;
                    for (uint32_t j = i + 1; j < h.nedits; j++) {
                        const uint8_t t2 = h.edits[j].type;
                        if (t2 == HT2_EDIT_MM || t2 == HT2_EDIT_READ_GAP || t2 == HT2_EDIT_REF_GAP) mm2++;
                    }
                    left_anchor_len -= (int)(mm * 2);
                    right_anchor_len -= (int)(mm2 * 2);
                    int shorter_anchor_len = left_anchor_len < right_anchor_len ? left_anchor_len : right_anchor_len;
                    if (shorter_anchor_len <= 0) shorter_anchor_len = 1;
                    const uint32_t intronLen_thresh = canon ? ht2_max_intron_len((uint32_t)shorter_anchor_len, P->minAnchorLen)
                                                            : ht2_max_intron_len_noncan((uint32_t)shorter_anchor_len, P->minAnchorLenNoncan);
                    if (intronLen_thresh < P->maxIntronLen) {
                        if (eLen > intronLen_thresh) score += (int64_t)INT32_MIN;
                        if (canon) {
                            const float probscore = ht2_spl_prob(e);   // SpliceSiteDB::probscore of the site, taken when the edit was made
                            float thresh = 0.8f;
                            if (eLen >> 16) thresh = 0.99f;
                            else if (eLen >> 15) thresh = 0.97f;
                            else if (eLen >> 14) thresh = 0.94f;
                            else if (eLen >> 13) thresh = 0.91f;
                            else if (eLen >> 12) thresh = 0.88f;
                            if (probscore < thresh) score += (int64_t)INT32_MIN;
                        }
                        if (shorter_anchor_len == left_anchor_len) {
                            if (h.trim5 > 0) score += (int64_t)INT32_MIN;
                            for (int j = (int)i - 1; j >= 0; j--) {
                                const uint8_t t2 = h.edits[j].type;
                                if (t2 == HT2_EDIT_MM || t2 == HT2_EDIT_READ_GAP || t2 == HT2_EDIT_REF_GAP) score += (int64_t)INT32_MIN;
                            }
                        } else {
                            if (h.trim3 > 0) score += (int64_t)INT32_MIN;
                            for (uint32_t j = i + 1; j < h.nedits; j++) {
                                const uint8_t t2 = h.edits[j].type;
                                if (t2 == HT2_EDIT_MM || t2 == HT2_EDIT_READ_GAP || t2 == HT2_EDIT_REF_GAP) score += (int64_t)INT32_MIN;
                            }
                        }
                    }
                    {   // (edit.snpID is always "none" here: splice-site ALTs are not built)
                        if (canon) score -= ht2_intron_pen((int)eLen) + P->canSplPen;
                        else score -= ht2_intron_pen((int)eLen) + P->noncanSplPen;
                    }
                    if (shorter_anchor_len <= 15) { numsplices += 1; splicescore += (double)eLen; }
                }
                if (!conflict_splicesites) {
                    if (whichsense == HT2_SPL_UNKNOWN) whichsense = (uint8_t)eDir;
                    else if (eDir != HT2_SPL_UNKNOWN) {
                        if (eDir == HT2_SPL_FW || eDir == HT2_SPL_SEMI_FW) { if (whichsense != HT2_SPL_FW && whichsense != HT2_SPL_SEMI_FW) conflict_splicesites = true; }
                        if (eDir == HT2_SPL_RC || eDir == HT2_SPL_SEMI_RC) { if (whichsense != HT2_SPL_RC && whichsense != HT2_SPL_SEMI_RC) conflict_splicesites = true; }
                    }
                }
            }
#endif
        }
        // soft-clip penalty indexes qual[i], not the clipped position (hi_aligner.h:3872-3878)
        for (uint32_t i = 0; i < h.trim5; i++) score -= ht2_scpen(*P, qual[i]);
        for (uint32_t i = 0; i < h.trim3; i++) score -= ht2_scpen(*P, qual[i]);
#ifdef HT2_ENABLE_SPLICED
        if (conflict_splicesites) score -= HT2_PEN_CONFLICTSPLICE;
        if (numsplices > 1) splicescore /= (double)numsplices;
        h.splicescore = splicescore;
#endif
        h.score = score;
        return score;
    }

    // ---- 2-bit reference (reference.cpp:396-430, 486-640) ------------------
    HT2_HD uint32_t refLen(uint32_t tidx) const { return ((const uint32_t*)(blob + H->o_refLens))[tidx]; }
    // Decodes count bases starting at toff: 0-3, or 4 inside N gaps / past the
    // end.  Returns the address of the first base, dest + skip with skip < 4:
    // when the window lies inside one unambiguous stretch and dest is 4-byte
    // aligned, whole bytes of the 2-bit buffer are expanded with one 32-bit
    // store each (the reference's getStretch also returns such an offset,
    // reference.cpp:486-640).  dest needs room for count + 7 bytes.  With
    // allowSkip == false the bases always start at dest.
    HT2_NI const uint8_t* getStretch(uint8_t* dest, uint32_t tidx, uint32_t toff, uint32_t count, bool allowSkip = true) const {
        W->algBytes += (count + 3) >> 2;
        const Ht2RefRecord* recs = (const Ht2RefRecord*)(blob + H->o_recs);
        const uint32_t* recOffs = (const uint32_t*)(blob + H->o_refRecOffs);
        const uint64_t* refOffs = (const uint64_t*)(blob + H->o_refOffs);
        const uint8_t* buf = blob + H->o_refBuf;
        uint32_t reci = recOffs[tidx], recf = recOffs[tidx + 1];
        uint64_t bufOff = refOffs[tidx];
        uint64_t off = 0, t = toff;
        uint32_t cur = 0;
        for (uint32_t i = reci; i < recf && count > 0; i++) {
            off += recs[i].off;
            const uint32_t rlen = recs[i].len;
            if (allowSkip && cur == 0 && t >= off && t + count <= off + rlen && (((uintptr_t)dest) & 3) == 0) {
                bufOff += (t - off);
                const uint32_t skip = (uint32_t)(bufOff & 3);
                const uint8_t* src = buf + (bufOff >> 2);
                uint32_t* d32 = (uint32_t*)dest;
                const uint32_t nb = (skip + count + 3) >> 2;
                for (uint32_t k = 0; k < nb; k++) {
                    uint32_t x = src[k];
                    x = (x | (x << 12)) & 0x000f000fu;
                    x = (x | (x << 6)) & 0x03030303u;
                    d32[k] = x;
                }
                return dest + skip;
            }
            while (t < off && count > 0) { dest[cur++] = 4; t++; count--; }
            if (count == 0) break;
            if (t < off + rlen) bufOff += (t - off);
            else bufOff += rlen;
            off += rlen;
            while (t < off && count > 0) {
                dest[cur++] = (buf[bufOff >> 2] >> ((bufOff & 3) << 1)) & 3;
                bufOff++; t++; count--;
            }
        }
        while (count > 0) { dest[cur++] = 4; count--; }
        return dest;
    }
    HT2_HD int getBase(uint32_t tidx, uint32_t toff) const {
        uint8_t b[8]; return *getStretch(b + 1, tidx, toff, 1);
    }

    // ---- joined <-> text coordinates (gfm.h:5527-5600) ---------------------
    template <typename IT>
    HT2_NI bool joinedToTextOff(const Ht2Fm<IT>& fm, uint32_t qlen, uint32_t off, uint32_t& tidx, uint32_t& textoff,
                                bool rejectStraddle, bool& straddled) const {
        const uint32_t nFrag = fm.g->nFrag;
        uint32_t top = 0, bot = nFrag;
        uint32_t elt = (uint32_t)Ht2Fm<IT>::imax();
        while (true) {
            uint32_t oldelt = elt;
            elt = top + ((bot - top) >> 1);
            if (oldelt == elt) { tidx = HT2_IDX_MAX32; return false; }
            uint32_t lower = fm.rstarts[elt * 3];
            uint32_t upper = (elt == nFrag - 1) ? fm.g->len : fm.rstarts[(elt + 1) * 3];
            if (lower <= off) {
                if (upper > off) {
                    if (off + qlen > upper) {
                        straddled = true;
                        if (rejectStraddle) { tidx = HT2_IDX_MAX32; return false; }
                    }
                    tidx = fm.rstarts[elt * 3 + 1];
                    uint32_t fragoff = off - fm.rstarts[elt * 3];
                    textoff = (uint32_t)(IT)(fragoff + fm.rstarts[elt * 3 + 2]);
                    break;
                } else top = elt;
            } else bot = elt;
        }
        return true;
    }

    // ---- one backward-search step --------------------------------------
    // Returns new [top,bot) and node range for extending with base c
    // (partialSearch inner step, hi_aligner.h:6466-6484; mapLF gfm.h:3739,
    // mapGLF1 gfm.h:3957, mapLF1 gfm.h:3889).  Linear indexes only here;
    // graph indexes are dispatched in lfStepGraph.
    // nlf / bytes accumulate the work counters in registers (written back once per search).
    template <typename IT>
    HT2_HD void lfStep(const Ht2Fm<IT>& fm, uint32_t top, uint32_t bot, int c,
                       uint32_t& ntop, uint32_t& nbot, uint32_t& nlf, uint32_t& bytes) {
        const bool one = (bot - top == 1);
        nlf += one ? 1u : 2u;
        bytes += (one || (top >> HT2_SIDE_SHIFT) == (bot >> HT2_SIDE_SHIFT)) ? HT2_SIDE_BYTES : 2u * HT2_SIDE_BYTES;
        ht2_lf2(fm, top, bot, c, ntop, nbot);
    }

    // HI_Aligner::partialSearch (hi_aligner.h:6361-6600).  Returns stop
    // flags through pseudogeneStop/anchorStop like the reference.  Returns false when the search was parked after a
    // slice of LF steps (W->psCont): the caller calls again, with the same arguments, to continue it.
// 128 steps: short-read searches finish in the round that starts them.  Parking costs a round of its own -- a
// re-claim of the slot and a cold workspace -- so shorter slices cost more than the long lanes they cut: on an H100
// (400 W), the pool kernel of a 2 M-pair bench-shaped batch takes 156.5 ms at 8 steps, 149.5 ms at 16, 148.3 ms at
// 32, 146.9 ms at 64, and 143.5 +- 0.4 ms at 128, 256 and 1024 (DESIGN.md 4.1).
#ifndef HT2_PS_SLICE
#define HT2_PS_SLICE 128
#endif
    HT2_NI bool partialSearch(uint32_t rdi, bool fw, bool& pseudogeneStop, bool& anchorStop) {
        if (GRAPH) return partialSearchGraph(rdi, fw, pseudogeneStop, anchorStop);
        bool pseudogeneStop_ = pseudogeneStop, anchorStop_ = anchorStop;
        pseudogeneStop = anchorStop = false;
        Ht2ReadHits& hit = W->hits[rdi][fw ? 0 : 1];
        const uint32_t ftabLen = gfm.g->ftabChars;
        const uint32_t len = W->rd[rdi].len;
        const uint8_t* seq = W->rd[rdi].seq[fw ? 0 : 1];
        const uint32_t minK = P->minK;
        const bool resume = W->psCont != 0;
        if (!resume) hit.numPartialSearch++;
        uint32_t offset = hit.cur;
        uint32_t dep = offset;
        uint32_t left = len - dep;
        if (!resume && hit.nhits >= HT2_MAX_PHITS) { W->err |= HT2_ERR_PHITS; hit.cur = len; hit.done = 1; return true; }
        Ht2BwtHit& ph = hit.hits[hit.nhits];
        uint32_t top = 0, bot = 0, ntop = 0, nbot = 0;
        uint32_t same_range = 0, similar_range = 0;
        if (resume) {
            top = W->psTop; bot = W->psBot; ntop = W->psNtop; nbot = W->psNbot; dep = W->psDep;
            same_range = W->psSame; similar_range = W->psSimilar;
            pseudogeneStop_ = W->psPseudo != 0; anchorStop_ = W->psAnchor != 0;
            W->psCont = 0;
        } else {
        ph.top = ph.bot = ph.node_top = ph.node_bot = HT2_IDX_MAX32;
        ph.bwoff = offset; ph.hit_type = HT2_CANDIDATE_HIT; ph.hasCoords = 0;
        if (left < ftabLen + 1) {
            hit.cur = len;
            ph.len = hit.cur - offset; hit.nhits++;
            hit.done = 1;
            return true;
        }
        for (uint32_t i = 0; i < ftabLen; i++) {
            int c = seq[len - dep - 1 - i];
            if (c > 3) {
                hit.cur += (i + 1);
                ph.len = hit.cur - offset; hit.nhits++;
                if (hit.cur >= len) hit.done = 1;
                return true;
            }
        }
        ht2_ftab_lohi(gfm, seq, len - dep - ftabLen, top, bot);
        W->algBytes += 8;
        dep += ftabLen;
        if (top >= bot) {
            hit.cur = dep;
            ph.len = hit.cur - offset; hit.nhits++;
            if (hit.cur >= len) hit.done = 1;
            return true;
        }
        }
        uint32_t khits5 = P->khits < 5 ? P->khits : 5;
        uint32_t nlf = 0, lfBytes = 0;
        uint32_t budget = HT2_PS_SLICE;
        // node_range starts as (0,0) in the reference (hi_aligner.h:6396)
        while (dep < len) {
            if (budget-- == 0) {   // park: the slot stays in TS_PS and is regrouped with other searches
                W->psCont = 1; W->psTop = top; W->psBot = bot; W->psNtop = ntop; W->psNbot = nbot; W->psDep = dep;
                W->psSame = same_range; W->psSimilar = similar_range;
                W->psPseudo = pseudogeneStop_ ? 1 : 0; W->psAnchor = anchorStop_ ? 1 : 0;
                W->nLF += nlf; W->algBytes += lfBytes;
                return false;
            }
            int c = seq[len - dep - 1];
            uint32_t ttop = 0, tbot = 0;
            if (c <= 3) lfStep(gfm, top, bot, c, ttop, tbot, nlf, lfBytes);
            if (ttop >= tbot) break;
            const uint32_t tntop = ttop, tnbot = tbot;   // linear index: node range == row range
            uint32_t nw = tnbot - tntop, ow = nbot - ntop;
            if (pseudogeneStop_) {
                if (nw < ow && ow <= khits5) {
                    if (dep - offset >= minK + 6 && similar_range >= 5) {
                        hit.numUniqueSearch++;
                        pseudogeneStop = true;
                        break;
                    }
                }
                if (nw != 1) {
                    if (nw + 2 >= ow) similar_range++;
                    else if (nw + 4 < ow) similar_range = 0;
                } else pseudogeneStop_ = false;
            }
            if (anchorStop_) {
                if (nw != 1 && ow == nw) {
                    same_range++;
                    if (same_range >= 5) anchorStop_ = false;
                } else same_range = 0;
                if (dep - offset >= minK + 8 && nw >= 4) anchorStop_ = false;
            }
            top = ttop; bot = tbot; ntop = tntop; nbot = tnbot;
            dep++;
            if (anchorStop_) {
                if (dep - offset >= minK + 12 && bot - top == 1) {
                    hit.numUniqueSearch++;
                    anchorStop = true;
                    break;
                }
            }
        }
        W->nLF += nlf; W->algBytes += lfBytes;
        if (top < bot) {
            uint8_t hit_type = HT2_CANDIDATE_HIT;
            if (anchorStop) hit_type = HT2_ANCHOR_HIT;
            else if (pseudogeneStop) hit_type = HT2_PSEUDOGENE_HIT;
            bool report = ntop < nbot;
            if (nbot - ntop < bot - top) report = false; // no in-edge list on linear indexes
            if (report) { ph.top = top; ph.bot = bot; ph.node_top = ntop; ph.node_bot = nbot; }
            ph.len = dep - offset;
            ph.hit_type = hit_type;
            hit.nhits++;
            hit.cur = dep;
            if (hit.cur >= len) {
                if (hit_type == HT2_CANDIDATE_HIT) hit.numUniqueSearch++;
                hit.done = 1;
            }
        }
        return true;
    }

    // HI_Aligner::globalGFMSearch / localGFMSearch (hi_aligner.h:6606-6744,
    // 6751-6892) share one body; 'local' picks minUniqueLen/maxHitLen/maxHits.
    template <typename IT>
    HT2_NI uint32_t gfmSearch(const Ht2Fm<IT>& fm, uint32_t rdi, bool fw, uint32_t rdoff, uint32_t& hitlen,
                              uint32_t& top, uint32_t& bot, uint32_t& node_top, uint32_t& node_bot,
                              bool& uniqueStop, uint32_t minUniqueLen, uint32_t maxHitLen, uint32_t maxHits, bool local) {
        // a graph index may hold LINEAR local indexes (windows without ALTs, or whose local graph exploded at build time)
        if (GRAPH) { W->nCurIe = 0; if (!fm.g->linearFM) return gfmSearchGraph(fm, rdi, fw, rdoff, hitlen, top, bot, node_top, node_bot, uniqueStop, minUniqueLen, maxHitLen, maxHits, local); }
        bool uniqueStop_ = uniqueStop;
        uniqueStop = false;
        const uint32_t ftabLen = fm.g->ftabChars;
        const uint32_t len = W->rd[rdi].len;
        const uint8_t* seq = W->rd[rdi].seq[fw ? 0 : 1];
        uint32_t offset = len - rdoff - 1;
        uint32_t dep = offset;
        if (local) top = bot = node_top = node_bot = 0;
        uint32_t left = len - dep;
        if (left < ftabLen + 1) { hitlen = left; return 0; }
        for (uint32_t i = 0; i < ftabLen; i++) {
            int c = seq[len - dep - 1 - i];
            if (c > 3) { hitlen = i + 1; return 0; }
        }
        uint32_t rtop = 0, rbot = 0, ntop = 0, nbot = 0;
        ht2_ftab_lohi(fm, seq, len - dep - ftabLen, rtop, rbot);
        W->algBytes += 2 * (uint32_t)sizeof(IT);
        dep += ftabLen;
        if (rtop >= rbot) { hitlen = ftabLen; return 0; }
        uint32_t nlf = 0, lfBytes = 0;
        while (dep < len) {
            int c = seq[len - dep - 1];
            uint32_t ttop = 0, tbot = 0;
            if (c <= 3) lfStep(fm, rtop, rbot, c, ttop, tbot, nlf, lfBytes);
            if (ttop >= tbot) break;
            rtop = ttop; rbot = tbot; ntop = ttop; nbot = tbot;
            dep++;
            if (uniqueStop_) {
                if (rbot - rtop == 1 && dep - offset >= minUniqueLen) { uniqueStop = true; break; }
            }
            if (local && dep - offset >= maxHitLen) break;
        }
        W->nLF += nlf; W->algBytes += lfBytes;
        uint32_t nelt = 0;
        if (ntop < nbot && nbot - ntop <= maxHits) {
            top = rtop; bot = rbot; node_top = ntop; node_bot = nbot;
            nelt = nbot - ntop;
            hitlen = dep - offset;
        }
        return nelt;
    }

    // ---- SA-offset resolution (group_walk.h GWState::init/advance,
    // GroupWalk2S::advanceElement :1491; gfm.h tryOffset :2719) -------------
    // Walk row left until a sampled row (or '$') is met; joined offset =
    // sample + #steps.  Linear indexes: node == row.
    template <typename IT>
    HT2_NI uint32_t resolveRow(const Ht2Fm<IT>& fm, uint32_t row) {
        uint32_t steps = 0;
        const uint32_t offMask = fm.offMask, z0 = fm.z0;
        uint32_t res;
        while (true) {
            if (row == z0) { res = (uint32_t)(IT)(0 + steps); break; }
            if ((row & offMask) == row) {
                W->algBytes += (uint32_t)sizeof(IT);
                res = (uint32_t)(IT)(fm.offs[row >> fm.offRate] + steps);
                break;
            }
            int c;
            row = ht2_lf_own(fm, row, c);
            steps++;
        }
        W->nLF += steps;
        W->algBytes += steps * HT2_SIDE_BYTES;
        return res;
    }

    // HI_Aligner::getGenomeCoords (hi_aligner.h:5774-5855); appends to W->coords.
    HT2_NI bool getGenomeCoords(uint32_t top, uint32_t bot, uint32_t node_top, uint32_t node_bot, bool fw,
                                uint32_t maxelt, uint32_t rdlen, bool rejectStraddle, bool& straddled) {
        if (GRAPH) return getGenomeCoordsGraph(top, bot, node_top, node_bot, W->curIe, W->nCurIe, fw, maxelt, rdlen, rejectStraddle, straddled);
        straddled = false;
        uint32_t nelt = node_bot - node_top;
        if (nelt > maxelt) nelt = maxelt;
        for (uint32_t i = 0; i < nelt; i++) {
            uint32_t joff = resolveRow(gfm, top + i);
            uint32_t tidx = 0, toff = 0;
            bool straddled2 = false;
            joinedToTextOff(gfm, rdlen, joff, tidx, toff, rejectStraddle, straddled2);
            straddled |= straddled2;
            if (tidx == HT2_IDX_MAX32) return false;
            if (W->nCoords >= HT2_MAX_COORDS) { W->err |= HT2_ERR_COORDS; return false; }
            Ht2Coord& c = W->coords[W->nCoords++];
            c.ref = straddled2 ? HT2_IDX_MAX32 : tidx;
            c.off = toff; c.fw = fw ? 1 : 0; c.joinedOff = joff;
        }
        return true;
    }

    // HI_Aligner::getGenomeCoords_local (hi_aligner.h:5861-5941); fills out[].
    HT2_NI bool getGenomeCoordsLocal(const Ht2Fm<uint16_t>& lfm, uint32_t top, uint32_t bot, uint32_t node_top,
                                     uint32_t node_bot, bool fw, uint32_t rdoff, uint32_t rdlen,
                                     Ht2Coord* out, uint32_t& nout, uint32_t cap) {
        if (GRAPH && !lfm.g->linearFM) return getGenomeCoordsLocalGraph(lfm, top, bot, node_top, node_bot, fw, rdoff, rdlen, out, nout, cap);
        uint32_t nelt = node_bot - node_top;
        for (uint32_t i = 0; i < nelt; i++) {
            uint32_t joff = resolveRow(lfm, top + i);
            uint32_t tidx = 0, toff = 0;
            bool straddled2 = false;
            bool ok = joinedToTextOff(lfm, rdlen, joff, tidx, toff, true, straddled2);
            if (!ok) continue;
            uint32_t global_toff = toff + lfm.g->localOffset;
            uint32_t joinedOff = joff + lfm.g->joinedOffset;
            if (global_toff < rdoff) continue;
            if (nout >= cap) { W->err |= HT2_ERR_COORDS; return false; }
            Ht2Coord& c = out[nout++];
            c.ref = lfm.g->tidx; c.off = global_toff; c.fw = fw ? 1 : 0; c.joinedOff = joinedOff;
        }
        return true;
    }
    HT2_HD static bool coordLess(const Ht2Coord& a, const Ht2Coord& b) { // ref_coord.h:79-87
        if (a.ref != b.ref) return a.ref < b.ref;
        if (a.fw != b.fw) return a.fw < b.fw;
        return a.off < b.off;
    }
    HT2_HD static void sortCoords(Ht2Coord* c, uint32_t n) {
        for (uint32_t i = 1; i < n; i++) {
            Ht2Coord t = c[i]; uint32_t j = i;
            while (j > 0 && coordLess(t, c[j - 1])) { c[j] = c[j - 1]; j--; }
            c[j] = t;
        }
    }

    // ---- local index dispatch (hgfm.h:1713-1740) ------------------------------
    HT2_HD int localIndexId(uint32_t tidx, uint32_t offset) const {
        const uint32_t* first = (const uint32_t*)(blob + H->o_localFirst);
        uint32_t idx = offset / HT2_LOCAL_INDEX_INTERVAL;
        uint32_t n = first[tidx + 1] - first[tidx];
        if (idx >= n) return -1;
        return (int)(first[tidx] + idx);
    }
    HT2_HD const Ht2Gfm* localGeom(int id) const { return ((const Ht2Gfm*)(blob + H->o_localGfm)) + id; }
    HT2_HD int prevLocal(int id) const {
        const Ht2Gfm* g = localGeom(id);
        if (g->localOffset < HT2_LOCAL_INDEX_INTERVAL) return -1;
        return localIndexId(g->tidx, g->localOffset - HT2_LOCAL_INDEX_INTERVAL);
    }
    HT2_HD int nextLocal(int id) const {
        const Ht2Gfm* g = localGeom(id);
        return localIndexId(g->tidx, g->localOffset + HT2_LOCAL_INDEX_INTERVAL);
    }

    // ---- extension against the reference -------------------------------------
    // GenomeHit::alignWithALTs + alignWithALTs_recur restricted to an empty ALT
    // list (hi_aligner.h:683-783, 2763-2860, 3168-3223): mismatch-bounded scan.
    // Left: scans read positions rdoff, rdoff-1, ... against rfseq[rflen-1], ...
    // Returns the extension length; new edits are inserted at the front of h.
    HT2_NI uint32_t alignLeft(Ht2Hit& h, const uint8_t* seq, uint32_t base_rdoff, uint32_t rdoff, uint32_t rdlen,
                              uint32_t tidx, int rfoff, uint32_t rflen, uint32_t mm, uint32_t* numNs) {
        if (numNs) *numNs = 0;
        const uint32_t nedits0 = h.nedits;
        int best_rdoff = (int)rdoff;
        if (rfoff < -16) return 0;
        uint32_t contig_len = refLen(tidx);
        if (rfoff >= 0 && (uint32_t)rfoff >= contig_len) return 0;
        if (rfoff >= 0 && (uint32_t)rfoff + rflen > contig_len) rflen = contig_len - (uint32_t)rfoff;
        else if (rfoff < 0 && rflen > contig_len) rflen = contig_len;
        if (rflen == 0) return 0;
        if (rflen > HT2_REFBUF) { W->err |= HT2_ERR_RDLEN; return 0; }
        const uint8_t* rfseq = W->refbuf;
        {
            uint32_t lead = rfoff < 0 ? (uint32_t)(-rfoff) : 0;
            if (lead == 0) rfseq = getStretch(W->refbuf, tidx, (uint32_t)rfoff, rflen);
            else {
                // window starts before the reference: unaligned destination takes the generic path (skip 0)
                for (uint32_t i = 0; i < lead && i < rflen; i++) W->refbuf[i] = 4;
                if (rflen > lead) getStretch(W->refbuf + lead, tidx, 0, rflen - lead, false);
            }
        }
        uint32_t tmp_mm = 0;
        int mm_min_rd_i = (int)rdoff;
        uint32_t mm_tmp_numNs = 0;
        for (int rf_i = (int)rflen - 1; rf_i >= 0 && mm_min_rd_i >= 0; rf_i--, mm_min_rd_i--) {
            int rf_bp = rfseq[rf_i];
            int rd_bp = seq[mm_min_rd_i];
            if (rf_bp != rd_bp || rd_bp == 4) {
                if (tmp_mm >= mm) break;
                tmp_mm++;
                insertEditFront(h, mkEdit((uint32_t)mm_min_rd_i, ht2_code2asc(rf_bp), ht2_code2asc(rd_bp), HT2_EDIT_MM));
            }
            if (rf_bp == 4) mm_tmp_numNs++;
        }
        if (mm_min_rd_i < best_rdoff) {
            best_rdoff = mm_min_rd_i;
            if (numNs) *numNs = mm_tmp_numNs;
        } else {
            // edits are only committed when the scan improved on best_rdoff
            if (h.nedits > nedits0) {
                uint32_t added = h.nedits - nedits0;
                for (uint32_t i = 0; i + added < h.nedits; i++) h.edits[i] = h.edits[i + added];
                h.nedits = nedits0;
            }
        }
        uint32_t extlen = rdoff - (uint32_t)best_rdoff;
        return fixupExt(h, extlen, nedits0, base_rdoff, rdoff, true);
    }
    // Right: scans read positions rdoff.. against rfseq[0..).
    HT2_NI uint32_t alignRight(Ht2Hit& h, const uint8_t* seq, uint32_t base_rdoff, uint32_t rdoff, uint32_t rdlen,
                               uint32_t tidx, int rfoff, uint32_t rflen, uint32_t mm) {
        const uint32_t nedits0 = h.nedits;
        if (rfoff < -16) return 0;
        uint32_t contig_len = refLen(tidx);
        if (rfoff >= 0 && (uint32_t)rfoff >= contig_len) return 0;
        if (rfoff >= 0 && (uint32_t)rfoff + rflen > contig_len) rflen = contig_len - (uint32_t)rfoff;
        else if (rfoff < 0 && rflen > contig_len) rflen = contig_len;
        if (rflen == 0) return 0;
        if (rflen > HT2_REFBUF) { W->err |= HT2_ERR_RDLEN; return 0; }
        const uint8_t* rfseq = W->refbuf;
        {
            uint32_t lead = rfoff < 0 ? (uint32_t)(-rfoff) : 0;
            if (lead == 0) rfseq = getStretch(W->refbuf, tidx, (uint32_t)rfoff, rflen);
            else {
                // window starts before the reference: unaligned destination takes the generic path (skip 0)
                for (uint32_t i = 0; i < lead && i < rflen; i++) W->refbuf[i] = 4;
                if (rflen > lead) getStretch(W->refbuf + lead, tidx, 0, rflen - lead, false);
            }
        }
        const uint32_t rdoff_add = rdoff - base_rdoff;
        uint32_t tmp_mm = 0;
        uint32_t mm_max_rd_i = 0;
        for (uint32_t rf_i = 0; rf_i < rflen && mm_max_rd_i < rdlen; rf_i++, mm_max_rd_i++) {
            int rf_bp = rfseq[rf_i];
            int rd_bp = seq[rdoff + mm_max_rd_i];
            if (rf_bp != rd_bp || rd_bp == 4) {
                if (tmp_mm >= mm) break;
                tmp_mm++;
                pushEdit(h, mkEdit(mm_max_rd_i + rdoff_add, ht2_code2asc(rf_bp), ht2_code2asc(rd_bp), HT2_EDIT_MM));
            }
        }
        int best_rdoff = (int)rdoff;
        if ((int)(mm_max_rd_i + rdoff) > best_rdoff) best_rdoff = (int)(mm_max_rd_i + rdoff);
        else h.nedits = nedits0;
        uint32_t extlen = (uint32_t)best_rdoff - rdoff;
        return fixupExt(h, extlen, nedits0, base_rdoff, rdoff, false);
    }
    // tail of alignWithALTs (hi_aligner.h:756-783)
    HT2_NI uint32_t fixupExt(Ht2Hit& h, uint32_t extlen, uint32_t nedits0, uint32_t base_rdoff, uint32_t rdoff, bool left) {
        if (extlen > 0 && h.nedits > 0) {
            const Ht2Edit& f = h.edits[0];
            if (f.pos + extlen == base_rdoff + 1) {
                if (f.type == HT2_EDIT_READ_GAP || f.type == HT2_EDIT_REF_GAP || f.type == HT2_EDIT_SPL) extlen = 0;
                if (f.type == HT2_EDIT_MM && f.chr == 'N') extlen = 0;
            }
            const Ht2Edit& b = h.edits[h.nedits - 1];
            if (extlen > 0 && b.pos == rdoff - base_rdoff + extlen - 1) {
                if (b.type == HT2_EDIT_READ_GAP || b.type == HT2_EDIT_REF_GAP) extlen = 0;
            }
            if (extlen == 0 && h.nedits > nedits0) {
                if (left) {
                    uint32_t added = h.nedits - nedits0;
                    for (uint32_t i = 0; i + added < h.nedits; i++) h.edits[i] = h.edits[i + added];
                    h.nedits = nedits0;
                } else h.nedits = nedits0;
            }
        }
        return extlen;
    }

    // GenomeHit::extend (hi_aligner.h:2031-2232)
    HT2_NI bool extend(Ht2Hit& h, uint32_t rdi, uint32_t& leftext, uint32_t& rightext, uint32_t mm) {
        uint32_t max_leftext = leftext, max_rightext = rightext;
        leftext = 0; rightext = 0;
        const uint32_t rdlen = W->rd[rdi].len;
        const uint8_t* seq = W->rd[rdi].seq[h.fw ? 0 : 1];
        if (max_leftext > 0 && h.rdoff > 0) {
            if (h.toff <= 0) return false;
            int rl = (int)h.toff - (int)h.rdoff;
            uint32_t reflen = h.rdoff + 10;
            rl -= (int)(reflen - h.rdoff);
            if (rl < 0) { reflen += rl; rl = 0; }
            uint32_t numNs = 0;
            uint32_t num_prev_edits = h.nedits;
            uint32_t best_ext = GRAPH ? alignWithALTs(h, seq, h.joinedOff, h.rdoff - 1, h.rdoff - 1, h.rdoff, h.tidx, rl, reflen, true, false, mm, &numNs)
                                      : alignLeft(h, seq, h.rdoff - 1, h.rdoff - 1, h.rdoff, h.tidx, rl, reflen, mm, &numNs);
            if (h.len == 0 && mm == 0 && h.nedits > 0) { h.nedits = 0; return false; }
            if (best_ext > 0) {
                leftext = best_ext;
                uint32_t added_edits = h.nedits - num_prev_edits;
                int ref_ext = (int)best_ext;
                for (uint32_t i = 0; i < added_edits; i++) {
                    if (h.edits[i].type == HT2_EDIT_REF_GAP) ref_ext--;
                    else if (h.edits[i].type == HT2_EDIT_READ_GAP) ref_ext++;
                }
                h.rdoff -= best_ext;
                h.toff -= (uint32_t)ref_ext;
                h.len += best_ext;
                h.joinedOff -= (uint32_t)(ref_ext - (int)numNs);
                for (uint32_t i = 0; i < h.nedits; i++) {
                    if (i < added_edits) h.edits[i].pos -= h.rdoff;
                    else h.edits[i].pos += best_ext;
                }
            }
        }
        if (max_rightext > 0 && h.rdoff + h.len < rdlen) {
            uint32_t right_rdoff, right_len, right_toff;
            getRight(h, right_rdoff, right_len, right_toff, NULL, rdi);
            uint32_t rl = right_toff + right_len;
            uint32_t rr = rdlen - (right_rdoff + right_len);
            uint32_t tlen = refLen(h.tidx);
            if (rl < tlen) {
                uint32_t reflen = rr + 10;
                if (rl + reflen > tlen) reflen = tlen - rl;
                uint32_t best_ext;
                if (GRAPH) {
                    int ref_ext = (int)h.len;      // joined offset of the base right after the hit (hi_aligner.h:2152-2159)
                    for (uint32_t ei = 0; ei < h.nedits; ei++) {
                        const Ht2Edit& e = h.edits[ei];
                        if (e.type == HT2_EDIT_REF_GAP) ref_ext--;
                        else if (e.type == HT2_EDIT_READ_GAP) ref_ext++;
#ifdef HT2_ENABLE_SPLICED
                        else if (e.type == HT2_EDIT_SPL) ref_ext += (int)ht2_spl_len(e);
#endif
                        else if (e.type == HT2_EDIT_MM && e.chr == 'N') ref_ext--;
                    }
                    best_ext = alignWithALTs(h, seq, h.joinedOff + (uint32_t)ref_ext, h.rdoff, h.rdoff + h.len, rdlen - (h.rdoff + h.len),
                                             h.tidx, (int)rl, reflen, false, false, mm, NULL);
                } else best_ext = alignRight(h, seq, h.rdoff, h.rdoff + h.len, rdlen - (h.rdoff + h.len),
                                             h.tidx, (int)rl, reflen, mm);
                if (h.len == 0 && mm == 0 && h.nedits > 0) { h.nedits = 0; return false; }
                if (best_ext > 0) { rightext = best_ext; h.len += best_ext; }
            }
        }
        calculateScore(h, rdi);
        return leftext > 0 || rightext > 0;
    }

    // GenomeHit::compatibleWith (hi_aligner.h:1375-1413)
    HT2_NI bool compatibleWith(const Ht2Hit& a, const Ht2Hit& o, uint32_t rdi) const {
        if (&a == &o) return false;
        if (a.fw != o.fw || a.tidx != o.tidx) return false;
        if (a.rdoff > o.rdoff) return false;
        if (a.rdoff + a.len > o.rdoff + o.len) return false;
        if (a.toff > o.toff) return false;
        uint32_t this_rdoff, this_len, this_toff, other_rdoff, other_len, other_toff;
        getRight(a, this_rdoff, this_len, this_toff, NULL, rdi);
        getLeft(o, other_rdoff, other_len, other_toff, NULL, rdi);
        if (this_rdoff > other_rdoff) return false;
        if (this_rdoff + this_len > other_rdoff + other_len) return false;
        if (this_toff > other_toff) return false;
        uint32_t refdif = other_toff - this_toff;
        uint32_t rddif = other_rdoff - this_rdoff;
        if (!noSpl()) {
            if (refdif > rddif + P->maxIntronLen) return false;
        }
        return true;
    }

    // GenomeHit::leftAlign (hi_aligner.h:3554-3610)
    HT2_NI void leftAlign(Ht2Hit& h, uint32_t rdi) const {
        const uint8_t* seq = W->rd[rdi].seq[h.fw ? 0 : 1];
        for (uint32_t ei = 0; ei < h.nedits; ei++) {
            Ht2Edit& edit = h.edits[ei];
            if (edit.type != HT2_EDIT_READ_GAP && edit.type != HT2_EDIT_REF_GAP) continue;
            if (edit.snpID != HT2_IDX_MAX32) continue;
            uint32_t ei2 = ei + 1;
            for (; ei2 < h.nedits; ei2++) {
                const Ht2Edit& edit2 = h.edits[ei2];
                if (edit2.type != edit.type) break;
                if (edit.type == HT2_EDIT_READ_GAP) { if (edit.pos != edit2.pos) break; }
                else { if (edit.pos + ei2 - ei != edit2.pos) break; }
            }
            ei2 -= 1;
            Ht2Edit& edit2 = h.edits[ei2];
            int b = 0;
            if (ei > 0) b = (int)h.edits[ei - 1].pos;
            int l = (int)edit.pos - 1;
            while (l > b) {
                int rdc = seq[h.rdoff + l];
                uint8_t rfc = (edit.type == HT2_EDIT_READ_GAP ? edit2.chr : edit2.qchr);
                if (rfc != ht2_code2asc(rdc)) break;
                for (int ei3 = (int)ei2; ei3 > (int)ei; ei3--) {
                    if (edit.type == HT2_EDIT_READ_GAP) h.edits[ei3].chr = h.edits[ei3 - 1].chr;
                    else h.edits[ei3].qchr = h.edits[ei3 - 1].qchr;
                    h.edits[ei3].pos -= 1;
                }
                if (edit.type == HT2_EDIT_READ_GAP) edit.chr = ht2_code2asc(rdc);
                else edit.qchr = ht2_code2asc(rdc);
                edit.pos -= 1;
                l--;
            }
            ei = ei2;
        }
    }

    // GenomeHit::combineWith (hi_aligner.h:1420-2025), non-spliced paths
    // (splicing is rejected under --no-spliced-alignment, :1500-1502).
    HT2_NI bool combineWith(Ht2Hit& a, const Ht2Hit& o, uint32_t rdi, int64_t minsc_, const Ht2SsSite* spliceSite = NULL) {
        if (&a == &o) return false;
        uint32_t this_rdoff, this_len, this_toff, other_rdoff, other_len, other_toff;
        int64_t this_score, other_score;
        getRight(a, this_rdoff, this_len, this_toff, &this_score, rdi);
        getLeft(o, other_rdoff, other_len, other_toff, &other_score, rdi);
        if (this_len != 0 && other_len != 0 && this_rdoff + this_len > other_rdoff + other_len) return false;
        uint32_t len = other_rdoff - this_rdoff + other_len;
        const uint32_t reflen = refLen(a.tidx);
        if (this_toff + len > reflen) return false;
        uint32_t refdif = other_toff - this_toff;
        uint32_t rddif = other_rdoff - this_rdoff;
        bool spliced = false, ins = false, del = false;
        if (refdif != rddif) {
            if (refdif > rddif) {
                if (!noSpl() && refdif - rddif >= P->minIntronLen) spliced = true;
                else del = true;
            } else ins = true;
        }
#ifndef HT2_ENABLE_SPLICED
        if (spliced) { W->err |= HT2_ERR_SPLICE; return false; } // spliced joins exist in the host test build only (DESIGN.md 8.2); the C ABI refuses spliced mode
#endif
        if (!spliced && !ins && !del && this_rdoff + this_len == other_rdoff) {
            uint32_t addoff = o.rdoff - a.rdoff;
            for (uint32_t i = 0; i < o.nedits; i++) {
                if (!pushEdit(a, o.edits[i])) return false;
                a.edits[a.nedits - 1].pos += addoff;
            }
            a.len += o.len;
            calculateScore(a, rdi);
            return true;
        }
        const uint8_t* seq = W->rd[rdi].seq[a.fw ? 0 : 1];
        const uint8_t* qual = W->rd[rdi].qual[a.fw ? 0 : 1];
        const uint32_t rdlen = W->rd[rdi].len;
        int64_t remainsc = minsc_ - (a.score - this_score) - (o.score - other_score);
        if (remainsc > 0) remainsc = 0;
        int read_gaps = 0, ref_gaps = 0;
        if (!spliced) {
            read_gaps = ht2_max_gaps(remainsc + P->canSplPen, P->rdGapConst + P->rdGapLinear, P->rdGapLinear);
            ref_gaps = ht2_max_gaps(remainsc + P->canSplPen, P->rfGapConst + P->rfGapLinear, P->rfGapLinear);
        }
        (void)rdlen;
        if (ins) { if (refdif + (uint32_t)ref_gaps < rddif) return false; }
        else if (del) { if (rddif + (uint32_t)read_gaps < refdif) return false; }
        int this_ref_ext = read_gaps;
#ifdef HT2_ENABLE_SPLICED
        const int intronic_len = 14;   // max(donor_intronic_len 6, acceptor_intronic_len 14), splice_site.h:76
        if (spliced) this_ref_ext += intronic_len;
#endif
        if (this_toff + len > reflen) return false;
        if (this_toff + len + (uint32_t)this_ref_ext > reflen) this_ref_ext = (int)(reflen - (this_toff + len));
        if (len + (uint32_t)this_ref_ext > HT2_REFBUF || len > HT2_MAX_RDLEN) { W->err |= HT2_ERR_RDLEN; return false; }
        const uint8_t* refbuf = getStretch(W->refbuf, a.tidx, this_toff, len + (uint32_t)this_ref_ext);
        const uint8_t* refbuf2 = NULL;
        uint32_t maxscorei = HT2_IDX_MAX32;
        int64_t maxscore = HT2_MIN_I64;
#ifdef HT2_ENABLE_SPLICED
        uint32_t maxspldir = HT2_SPL_UNKNOWN; float maxsplscore = 0.0f; int64_t donor_seq = 0, acceptor_seq = 0;
        if (spliced) {   // hi_aligner.h:1576-1758, 1796-1816
            int other_ref_ext = read_gaps + intronic_len;
            { int lim = (int)(other_toff + other_len - len); if (lim < other_ref_ext) other_ref_ext = lim; }
            if ((int)len + other_ref_ext > (int)HT2_REFBUF || other_ref_ext < 0) { W->err |= HT2_ERR_RDLEN; return false; }
            refbuf2 = getStretch(W->refbuf2, o.tidx, other_toff + other_len - len - (uint32_t)other_ref_ext, len + (uint32_t)other_ref_ext)
                      + other_ref_ext;
            int64_t* ts = W->tscores; int64_t* ts2 = W->tscores2;
            const int GT = 0x23, AG = 0x02, GTrc = 0x01, AGrc = 0x13, GC = 0x21, GCrc = 0x21, AT = 0x03, AC = 0x01, ATrc = 0x03, ACrc = 0x20;
            const int donor_exonic_len = 3, donor_intronic_len = 6, acceptor_intronic_len = 14, acceptor_exonic_len = 1;
            int i;
            for (i = 0; i < (int)len; i++) {
                int rdc = seq[this_rdoff + i], rfc = refbuf[i];
                ts[i] = i > 0 ? ts[i - 1] : 0;
                if (rdc != rfc) ts[i] += ht2_score(*P, rdc, 1 << rfc, (int)qual[this_rdoff + i] - 33);
                if (ts[i] < remainsc) break;
            }
            int i_limit = i < (int)len ? i : (int)len;
            int i2;
            for (i2 = (int)len - 1; i2 >= 0; i2--) {
                int rdc = seq[this_rdoff + i2], rfc = refbuf2[i2];
                ts2[i2] = ((uint32_t)(i2 + 1) < len) ? ts2[i2 + 1] : 0;
                if (rdc != rfc) ts2[i2] += ht2_score(*P, rdc, 1 << rfc, (int)qual[this_rdoff + i2] - 33);
                if (ts2[i2] < remainsc) break;
            }
            int i2_limit = i2 > 0 ? i2 : 0;
            if (spliceSite != NULL) {   // a site of the splice-site DB: only its own split point is tried (hi_aligner.h:1626-1634)
                if (i2_limit <= (int)(spliceSite->left - this_toff)) { i2_limit = (int)(spliceSite->left - this_toff); i_limit = i2_limit + 1; }
                else i_limit = i2_limit;
            }
            for (i = i2_limit, i2 = i2_limit + 1; i < i_limit && i2 < (int)len; i++, i2++) {
                int64_t tempscore = ts[i] + ts2[i2];
                int donor = 0xff, acceptor = 0xff;   // (char)0xff in the reference: compares unequal to every motif
                if ((uint32_t)(i + 2) < len + (uint32_t)this_ref_ext) donor = (int)(int8_t)(uint8_t)(((uint8_t)refbuf[i + 1] << 4) | (uint8_t)refbuf[i + 2]);
                if (i2 - 2 >= -other_ref_ext) acceptor = (int)(int8_t)(uint8_t)(((uint8_t)refbuf2[i2 - 2] << 4) | (uint8_t)refbuf2[i2 - 1]);
                bool canonical = false, semi_canonical = false;
                uint32_t spldir = HT2_SPL_UNKNOWN;
                if (donor == GT && acceptor == AG) { spldir = HT2_SPL_FW; canonical = true; }
                else if (donor == AGrc && acceptor == GTrc) { spldir = HT2_SPL_RC; canonical = true; }
                else if ((donor == GC && acceptor == AG) || (donor == AT && acceptor == AC)) { spldir = HT2_SPL_SEMI_FW; semi_canonical = true; }
                else if ((donor == AGrc && acceptor == GCrc) || (donor == ACrc && acceptor == ATrc)) { spldir = HT2_SPL_SEMI_RC; semi_canonical = true; }
                tempscore -= (canonical ? (int64_t)P->canSplPen : (int64_t)P->noncanSplPen);
                int64_t temp_donor_seq = 0, temp_acceptor_seq = 0;
                float splscore = 0.0f;
                if (canonical) {
                    if (spldir == HT2_SPL_FW) {
                        if (i + 1 >= donor_exonic_len && (int)(len + (uint32_t)this_ref_ext) > i + donor_intronic_len &&
                            i2 + other_ref_ext >= acceptor_intronic_len && (int)len > i2 + acceptor_exonic_len - 1) {
                            int from = i + 1 - donor_exonic_len, to = i + donor_intronic_len;
                            for (int j = from; j <= to; j++) { int base = refbuf[j]; if (base > 3) base = 0; temp_donor_seq = temp_donor_seq << 2 | base; }
                            from = i2 - acceptor_intronic_len; to = i2 + acceptor_exonic_len - 1;
                            for (int j = from; j <= to; j++) { int base = refbuf2[j]; if (base > 3) base = 0; temp_acceptor_seq = temp_acceptor_seq << 2 | base; }
                        }
                    } else {
                        if (i + 1 >= acceptor_exonic_len && (int)(len + (uint32_t)this_ref_ext) > i + acceptor_intronic_len &&
                            i2 + other_ref_ext >= donor_intronic_len && (int)len > i2 + donor_exonic_len - 1) {
                            int from = i + 1 - acceptor_exonic_len, to = i + acceptor_intronic_len;
                            for (int j = to; j >= from; j--) { int base = refbuf[j]; if (base > 3) base = 0; temp_acceptor_seq = temp_acceptor_seq << 2 | (base ^ 0x3); }
                            from = i2 - donor_intronic_len; to = i2 + donor_exonic_len - 1;
                            for (int j = to; j >= from; j--) { int base = refbuf2[j]; if (base > 3) base = 0; temp_donor_seq = temp_donor_seq << 2 | (base ^ 0x3); }
                        }
                    }
                    splscore = ht2_spl_probscore(*splT, temp_donor_seq, temp_acceptor_seq);
                }
                const bool mu = (maxspldir == HT2_SPL_UNKNOWN), su = (spldir == HT2_SPL_UNKNOWN);
                if ((mu && su && maxscore < tempscore) || (mu && su && maxscore == tempscore && semi_canonical) ||
                    (!mu && !su && (maxscore < tempscore || (maxscore == tempscore && maxsplscore < splscore))) || (mu && !su)) {
                    maxscore = tempscore; maxscorei = (uint32_t)i; maxspldir = spldir; maxsplscore = splscore;
                    if (maxspldir != HT2_SPL_UNKNOWN) { donor_seq = temp_donor_seq; acceptor_seq = temp_acceptor_seq; }
                    else { donor_seq = 0; acceptor_seq = 0; }
                }
            }
            if (maxscore == HT2_MIN_I64) return false;
            if (spliceSite == NULL) {   // hi_aligner.h:1797
                uint32_t shorter_anchor_len = maxscorei + 1 < len - maxscorei - 1 ? maxscorei + 1 : len - maxscorei - 1;
                if (maxspldir == HT2_SPL_SEMI_FW || maxspldir == HT2_SPL_SEMI_RC || maxspldir == HT2_SPL_UNKNOWN) {
                    if (shorter_anchor_len < P->minAnchorLenNoncan) {
                        if (ht2_intron_len_prob_noncan(shorter_anchor_len, other_toff - this_toff, P->maxIntronLen) > 0.01f) return false;
                    }
                } else if (shorter_anchor_len < P->minAnchorLen) {
                    if (ht2_intron_len_prob(shorter_anchor_len, other_toff - this_toff, P->maxIntronLen) > 0.01f) return false;
                }
            }
            if (maxscore < remainsc) return false;
        }
#endif
        if (ins || del) {
            int other_ref_ext = read_gaps;
            int lim = (int)(other_toff + other_len - len);
            if (lim < other_ref_ext) other_ref_ext = lim;
            if ((int)len + other_ref_ext > (int)HT2_REFBUF || other_ref_ext < 0) { W->err |= HT2_ERR_RDLEN; return false; }
            refbuf2 = getStretch(W->refbuf2, o.tidx, other_toff + other_len - len - (uint32_t)other_ref_ext, len + (uint32_t)other_ref_ext)
                      + other_ref_ext;
            int64_t* ts = W->tscores; int64_t* ts2 = W->tscores2;
            int inslen = (ins ? (int)(rddif - refdif) : 0);
            int dellen = (del ? (int)(refdif - rddif) : 0);
            int64_t gap_penalty;
            if (ins) gap_penalty = -((int64_t)(P->rfGapConst + P->rfGapLinear) + (int64_t)P->rfGapLinear * (inslen - 1));
            else gap_penalty = -((int64_t)(P->rdGapConst + P->rdGapLinear) + (int64_t)P->rdGapLinear * (dellen - 1));
            if (gap_penalty < remainsc) return false;
            int i;
            for (i = 0; i < (int)len; i++) {
                int rdc = seq[this_rdoff + i], rfc = refbuf[i];
                ts[i] = i > 0 ? ts[i - 1] : 0;
                if (rdc != rfc) ts[i] += ht2_score(*P, rdc, 1 << rfc, (int)qual[this_rdoff + i] - 33);
                if (ts[i] + gap_penalty < remainsc) break;
            }
            int i_limit = i < (int)len ? i : (int)len;
            int i2;
            for (i2 = (int)len - 1; i2 >= 0; i2--) {
                int rdc = seq[this_rdoff + i2], rfc = refbuf2[i2];
                ts2[i2] = ((uint32_t)(i2 + 1) < len) ? ts2[i2 + 1] : 0;
                if (rdc != rfc) ts2[i2] += ht2_score(*P, rdc, 1 << rfc, (int)qual[this_rdoff + i2] - 33);
                if (ts2[i2] + gap_penalty < remainsc) break;
            }
            int i2_limit = (i2 < inslen ? 0 : i2 - inslen);
            for (i = i2_limit, i2 = i2_limit + 1 + inslen; i < i_limit && i2 < (int)len; i++, i2++) {
                int64_t tempscore = ts[i] + ts2[i2] + gap_penalty;
                if (maxscore < tempscore) { maxscore = tempscore; maxscorei = (uint32_t)i; }
            }
            if (maxscore == HT2_MIN_I64) return false;
            if (maxscore < remainsc) return false;
        }
        // drop this hit's trailing plain mismatches (hi_aligner.h:1818-1830)
        {
            bool clear = true;
            for (int i = (int)a.nedits - 1; i >= 0; i--) {
                if (isGapOrSnp(a.edits[i])) { a.nedits = (uint32_t)i + 1; clear = false; break; }
            }
            if (clear) a.nedits = 0;
        }
#ifdef HT2_ENABLE_SPLICED
        if (spliced) {   // hi_aligner.h:1832-1880 (splice_gap_off is always 0 there)
            const uint32_t addoff = this_rdoff - a.rdoff;
            for (uint32_t i = 0; i < len; i++) {
                int rdc = seq[this_rdoff + i];
                int rfc = (i <= maxscorei ? refbuf[i] : refbuf2[i]);
                if (rdc != rfc) { if (!pushEdit(a, mkEdit(i + addoff, ht2_code2asc(rfc), ht2_code2asc(rdc), HT2_EDIT_MM))) return false; }
                if (i == maxscorei) {
                    uint32_t left = this_toff + i + 1;
                    uint32_t right = other_toff + other_len - (len - i - 1);
                    Ht2Edit e = mkEdit(i + 1 + addoff, 'A', 'A', HT2_EDIT_SPL);
                    if (right - left > HT2_MAX_SPL_LEN) { W->err |= HT2_ERR_SPLICE; return false; }
                    ht2_spl_set(e, right - left, maxspldir, spliceSite != NULL, ht2_spl_probscore(*splT, donor_seq, acceptor_seq));
                    if (!pushEdit(a, e)) return false;
                }
            }
        } else
#endif
        {
            uint32_t ins_len = 0;
            for (uint32_t i = 0; i < len; i++) {
                int rdc = seq[this_rdoff + i];
                int rfc = (i <= maxscorei ? refbuf[i] : refbuf2[i]);
                uint32_t addoff = this_rdoff - a.rdoff;
                if (rdc != rfc) {
                    Ht2Edit me = mkEdit(i + addoff, ht2_code2asc(rfc), ht2_code2asc(rdc), HT2_EDIT_MM);
                    if (GRAPH) {
                        // a mismatch that is a known single-base ALT carries its id (hi_aligner.h:1917-1933)
                        const uint32_t key = a.joinedOff + i + (this_toff - a.toff) - ins_len;
                        const Ht2Alt* alts = altTable();
                        for (uint32_t ai = altLoBound(key); ai < numAlts(); ai++) {
                            if (alts[ai].pos > key) break;
                            if (alts[ai].type != HT2_ALT_SNP_SGL) continue;
                            if (alts[ai].seq == (uint64_t)rdc) { me.snpID = ai; break; }
                        }
                    }
                    if (!pushEdit(a, me)) return false;
                }
                if (i == maxscorei) {
                    uint32_t left = this_toff + i + 1;
                    if (other_toff + other_len < len - i - 1) return false;
                    uint32_t right = other_toff + other_len - (len - i - 1);
                    if (del) {
                        uint32_t skipLen = right - left;
                        for (uint32_t j = 0; j < skipLen; j++) {
                            int temp_rfc;
                            if (i + 1 + j < len) temp_rfc = refbuf[i + 1 + j];
                            else temp_rfc = getBase(a.tidx, this_toff + i + 1 + j);
                            if (!pushEdit(a, mkEdit(i + 1 + addoff, ht2_code2asc(temp_rfc), '-', HT2_EDIT_READ_GAP))) return false;
                        }
                    } else {
                        uint32_t skipLen = left - right;
                        for (uint32_t j = 0; j < skipLen; j++) {
                            int temp_rdc = seq[this_rdoff + i + 1 + j];
                            if (!pushEdit(a, mkEdit(i + 1 + j + addoff, '-', ht2_code2asc(temp_rdc), HT2_EDIT_REF_GAP))) return false;
                        }
                        i += skipLen;
                        ins_len += skipLen;
                    }
                }
            }
            (void)ins_len;
        }
        uint32_t fsi = o.nedits;
        for (uint32_t i = 0; i < o.nedits; i++) {
            if (isGapOrSnp(o.edits[i])) { fsi = i; break; }
        }
        uint32_t addoff = o.rdoff - a.rdoff;
        for (uint32_t i = fsi; i < o.nedits; i++) {
            if (!pushEdit(a, o.edits[i])) return false;
            a.edits[a.nedits - 1].pos += addoff;
        }
        if (ins || del) leftAlign(a, rdi);
        a.len = o.rdoff + o.len - a.rdoff;
        a.trim3 += o.trim3;
        calculateScore(a, rdi);
        return true;
    }

    // ---- sink: AlnSinkWrap::report (aln_sink.h:2565-2655) + ReportingState ----
    HT2_NI void sinkReset(bool paired_) {
        W->nRes[0] = W->nRes[1] = 0; W->nPairs = 0; W->nResEdits = 0;
        // AlnSinkWrap::nextRead starts these at numeric_limits<THitInt>::min() (aln_sink.h:1896-1898)
        W->bestPair = W->best2Pair = HT2_MIN_I64;
        W->bestUnp[0] = W->best2Unp[0] = W->bestUnp[1] = W->best2Unp[1] = HT2_MIN_I64;
#ifdef HT2_ENABLE_SPLICED
        W->bestSplicedUnp[0] = W->bestSplicedUnp[1] = 0;
#endif
        W->nconcord = 0; W->nunpair[0] = W->nunpair[1] = 0;
        // ReportingState::nextRead (aln_sink.cpp:33-66)
        if (paired_) {
            W->doneConcord = 0;
            W->doneUnpair[0] = P->mixed ? 0 : 1;
            W->doneUnpair[1] = P->mixed ? 0 : 1;
        } else {
            W->doneConcord = 1; W->doneUnpair[0] = 0; W->doneUnpair[1] = 1;
        }
        W->stDone = 0;
        W->concordBest = HT2_MIN_SCORE;
    }
    HT2_HD uint32_t bestSpliced(uint32_t mate) const {
#ifdef HT2_ENABLE_SPLICED
        return W->bestSplicedUnp[mate];
#else
        (void)mate; return 0;   // no splice edits without spliced alignment
#endif
    }
    HT2_HD void reportUnpaired(uint32_t mate /*0 or 1 == rs1/rs2*/, int64_t score, uint32_t numSpliced = 0) {
        // ReportingState::foundUnpaired (aln_sink.cpp:96-132), -k mode (mhits unset)
        W->nunpair[mate]++;
        if (!W->doneUnpair[mate]) {
            if (W->nunpair[mate] >= P->khits) {
                W->doneUnpair[mate] = 1;
                if (W->doneUnpair[0] && W->doneUnpair[1]) { /* updateDone */ }
            }
        }
        if (score > W->bestUnp[mate]) {
            W->best2Unp[mate] = W->bestUnp[mate]; W->bestUnp[mate] = score;
#ifdef HT2_ENABLE_SPLICED
            W->bestSplicedUnp[mate] = numSpliced;
#endif
        }
        else if (score > W->best2Unp[mate]) W->best2Unp[mate] = score;
        (void)numSpliced;
    }

    // HI_Aligner::reportHit (hi_aligner.h:6064-6198), unpaired form.
    HT2_NI bool reportHit(uint32_t rdi, const Ht2Hit& hit) {
#if !defined(__CUDA_ARCH__) && defined(HT2_TRACE)
        fprintf(stderr, "reportHit rdi %u fw %u toff %u score %lld ned %u\n", rdi, hit.fw, hit.toff, (long long)hit.score, hit.nedits);
#endif
        const uint32_t rdlen = W->rd[rdi].len;
        if (hit.rdoff - hit.trim5 > 0 || hit.len + hit.trim5 + hit.trim3 < rdlen) return false;
        if (hit.score < minsc[rdi]) return false;
        uint32_t slot = (rdi == 0 && !rightendonly) ? 0 : 1;
        if (W->nRes[slot] >= HT2_MAX_RES) { W->err |= HT2_ERR_RES; return false; }
        if (W->nResEdits + hit.nedits > HT2_RES_EDITS) { W->err |= HT2_ERR_RES; return false; }
        Ht2Res& r = W->res[slot][W->nRes[slot]++];
        r.tidx = hit.tidx; r.toff = hit.toff; r.fw = hit.fw; r.rdlen = rdlen; r.score = hit.score;
        r.trim5p = hit.fw ? hit.trim5 : hit.trim3;
        r.trim3p = hit.fw ? hit.trim3 : hit.trim5;
        r.nedits = hit.nedits;
        r.editOff = W->nResEdits;
        W->nResEdits += hit.nedits;
        Ht2Edit* red = W->resEdits + r.editOff;
        for (uint32_t i = 0; i < hit.nedits; i++) { red[i] = hit.edits[i]; red[i].pos += hit.trim5; }
        if (!hit.fw) invertPoss(red, r.nedits, rdlen);
        // AlnRes::setShape (aligner_result.cpp:111-129)
        for (uint32_t i = 0; i < r.nedits; i++) red[i].pos -= r.trim5p;
        uint32_t rfextent = rdlen - r.trim5p - r.trim3p;
        for (uint32_t i = 0; i < r.nedits; i++) {
            if (red[i].type == HT2_EDIT_REF_GAP) rfextent--;
            else if (red[i].type == HT2_EDIT_READ_GAP) rfextent++;
        }
        r.rfextent = rfextent;
#ifdef HT2_ENABLE_SPLICED
        {   // GenomeHit::spliced() -> AlnScore(..., splicescore, knownTranscripts, nearSpliceSites, ...) (hi_aligner.h:6100-6145)
            bool spl = false, known = true;
            for (uint32_t i = 0; i < hit.nedits; i++) if (hit.edits[i].type == HT2_EDIT_SPL) { spl = true; known = known && ht2_spl_known(hit.edits[i]); }
            r.spliced = spl ? 1 : 0; r.knownTranscripts = (spl && known) ? 1 : 0; r.splicescore = hit.splicescore;
        }
#endif
        {
            uint32_t nspl = 0;
            for (uint32_t i = 0; i < hit.nedits; i++) if (hit.edits[i].type == HT2_EDIT_SPL) nspl++;
            reportUnpaired(slot, hit.score, nspl);
        }
        return true;
    }

    // HI_Aligner::redundant(sink, rdi, hit) (hi_aligner.h:6311-6351)
    HT2_NI bool redundant(uint32_t rdi, const Ht2Hit& hit) {
        const uint32_t rdlen = W->rd[rdi].len;
        for (uint32_t i = 0; i < W->nRes[rdi]; i++) {
            const Ht2Res& rsi = W->res[rdi][i];
            if (rsi.tidx == hit.tidx && rsi.toff == hit.toff && rsi.fw == hit.fw) {
                if (rsi.nedits == hit.nedits) {
                    uint32_t eidx = 0;
                    for (; eidx < rsi.nedits; eidx++) {
                        // compare against hit.edits as Edit::invertPoss(edits, rdlen) would lay them out
                        Ht2Edit e = hit.fw ? hit.edits[eidx] : hit.edits[hit.nedits - eidx - 1];
                        if (!hit.fw) {
                            if (e.type == HT2_EDIT_READ_GAP || e.type == HT2_EDIT_SPL) e.pos = (uint32_t)(rdlen - e.pos);
                            else e.pos = (uint32_t)(rdlen - e.pos - 1);
                        }
                        if (!editEq(W->resEdits[rsi.editOff + eidx], e)) break;
                    }
                    if (eidx >= rsi.nedits) return true;
                }
            }
        }
        return false;
    }
    // isSearched / addSearched (hi_aligner.h:6898-6922)
    HT2_NI bool isSearched(const Ht2Hit& hit, uint32_t rdi) const {
        uint32_t off = 0;
        const uint32_t top = W->searchedTop;
        while (off < top) {
            const Ht2SearchedRec& r = *(const Ht2SearchedRec*)(W->searched + off);
            const uint32_t ne = r.nedits;
            const Ht2SearchedEdit* ed = (const Ht2SearchedEdit*)(W->searched + off + sizeof(Ht2SearchedRec));
            off += (uint32_t)sizeof(Ht2SearchedRec) + ne * (uint32_t)sizeof(Ht2SearchedEdit);
            if (r.rdi != rdi || r.toff != hit.toff || r.tidx != hit.tidx || (r.fw != 0) != (hit.fw != 0) || r.rdoff != hit.rdoff ||
                r.len != hit.len || r.trim5 != hit.trim5 || r.trim3 != hit.trim3 || ne != hit.nedits) continue;
            bool same = true;
            for (uint32_t i = 0; i < ne && same; i++) {   // GenomeHit::operator== with the stored hit on the left
                const Ht2SearchedEdit& e = ed[i]; const Ht2Edit& oe = hit.edits[i];
                if (e.type == HT2_EDIT_READ_GAP) { if (oe.type != HT2_EDIT_READ_GAP) same = false; }
                else if (e.type == HT2_EDIT_REF_GAP) { if (oe.type != HT2_EDIT_REF_GAP) same = false; }
#ifdef HT2_ENABLE_SPLICED
                else if (e.type == HT2_EDIT_SPL) {
                    const uint32_t v = (ht2_spl_len(oe) & 0xfffffu) | (ht2_spl_dir(oe) << 20);
                    if (oe.type != HT2_EDIT_SPL || e.pos != oe.pos || e.chr != (uint8_t)v || e.qchr != (uint8_t)(v >> 8) || e.pad != (uint8_t)(v >> 16)) same = false;
                }
#endif
                else if (e.type != oe.type || e.pos != oe.pos || e.chr != oe.chr || e.qchr != oe.qchr) same = false;
            }
            if (same) return true;
        }
        return false;
    }
    HT2_NI void addSearched(const Ht2Hit& hit, uint32_t rdi) {
        const uint32_t need = (uint32_t)sizeof(Ht2SearchedRec) + hit.nedits * (uint32_t)sizeof(Ht2SearchedEdit);
        if (W->searchedTop + need > HT2_SEARCHED_BYTES) { W->err |= HT2_ERR_SEARCHED; return; }
        Ht2SearchedRec& r = *(Ht2SearchedRec*)(W->searched + W->searchedTop);
        r.tidx = hit.tidx; r.toff = hit.toff; r.rdoff = (uint16_t)hit.rdoff; r.len = (uint16_t)hit.len;
        r.trim5 = (uint16_t)hit.trim5; r.trim3 = (uint16_t)hit.trim3; r.fw = hit.fw ? 1 : 0; r.rdi = (uint8_t)rdi;
        r.nedits = (uint16_t)hit.nedits;
        Ht2SearchedEdit* ed = (Ht2SearchedEdit*)(W->searched + W->searchedTop + sizeof(Ht2SearchedRec));
        for (uint32_t i = 0; i < hit.nedits; i++) {
            ed[i].pos = hit.edits[i].pos; ed[i].type = hit.edits[i].type; ed[i].chr = hit.edits[i].chr; ed[i].qchr = hit.edits[i].qchr; ed[i].pad = 0;
#ifdef HT2_ENABLE_SPLICED
            if (hit.edits[i].type == HT2_EDIT_SPL) {   // Edit::operator== compares splLen and splDir of splice edits (edit.h:195-210)
                const uint32_t v = (ht2_spl_len(hit.edits[i]) & 0xfffffu) | (ht2_spl_dir(hit.edits[i]) << 20);
                ed[i].chr = (uint8_t)v; ed[i].qchr = (uint8_t)(v >> 8); ed[i].pad = (uint8_t)(v >> 16);
            }
#endif
        }
        W->searchedTop += need;
        W->nSearched[rdi]++;
    }

    // ---- policy --------------------------------------------------------------
    // ReadBWTHit::searchScore (hi_aligner.h:321-334)
    HT2_HD int64_t searchScore(const Ht2ReadHits& h) const {
        int64_t score = 0;
        const int64_t penaltyPerOffset = (int64_t)P->minK * P->minK;
        for (uint32_t i = 0; i < h.nhits; i++) { uint32_t len = h.hits[i].len; score += (int64_t)(uint32_t)(len * len); }
        uint32_t aps = h.numPartialSearch - h.numUniqueSearch;
        score -= (int64_t)aps * penaltyPerOffset;
        // the reference computes 1 << (aps << 1) in 32-bit int (hi_aligner.h:332); from 16 partial searches on the
        // shift count is >= 32, which its x86 build executes with the count taken mod 32 (SHL) -- a GPU would
        // produce 0 instead -- and a count of 31 yields INT_MIN: reproduce exactly that, without the undefined shift
        score -= (int64_t)(int32_t)(1u << ((aps << 1) & 31u));
        return score;
    }
    // HI_Aligner::pickNextReadToSearch (hi_aligner.h:4868-4894)
    HT2_NI bool pickNextReadToSearch(uint32_t& rdi, bool& fw) {
        rdi = 0; fw = true;
        bool picked = false;
        int64_t maxScore = HT2_MIN_I64;
        for (uint32_t rdi2 = 0; rdi2 < (paired ? 2u : 1u); rdi2++) {
            for (uint32_t fwi = 0; fwi < 2; fwi++) {
                if (fwi == 0 && nofw[rdi2]) continue;
                else if (fwi == 1 && norc[rdi2]) continue;
                Ht2ReadHits& h = W->hits[rdi2][fwi];
                if (h.done) continue;
                int64_t curScore = searchScore(h);
                if (h.cur == 0) curScore = 0x7fffffffffffffffll;
                if (curScore > maxScore) { maxScore = curScore; rdi = rdi2; fw = (fwi == 0); picked = true; }
            }
        }
        return picked;
    }
    // HI_Aligner::nextBWT (hi_aligner.h:4644-4752)
    HT2_NI bool nextBWT(uint32_t& rdi, bool& fw) {
        while (pickNextReadToSearch(rdi, fw)) {
            uint32_t fwi = fw ? 0 : 1;
            Ht2ReadHits& hit = W->hits[rdi][fwi];
            bool pseudogeneStop = gfm.g->linearFM && !noSpl();
            bool anchorStop = P->anchorStop != 0;
            if (!P->secondary) {
                uint32_t numSearched = hit.numPartialSearch - hit.numUniqueSearch;
                int64_t bestScore = W->bestUnp[rdi];
                if (bestScore >= minsc[rdi]) {
                    uint32_t maxmm = (uint32_t)((-bestScore + P->mmpMax - 1) / P->mmpMax);
                    if (numSearched > maxmm + bestSpliced(rdi) + 1) {
                        hit.done = 1;
                        if (paired) {
                            if (W->bestUnp[1 - rdi] >= minsc[1 - rdi] && W->nPairs > 0) return false;
                            else continue;
                        } else return false;
                    }
                }
                Ht2ReadHits& rchit = W->hits[rdi][1 - fwi];
                if (rchit.done && bestScore < minsc[rdi]) {
                    if (numSearched > (rchit.numPartialSearch - rchit.numUniqueSearch) + (anchorStop ? 1u : 0u)) {
                        hit.done = 1;
                        return false;
                    }
                }
            }
            while (!partialSearch(rdi, fw, pseudogeneStop, anchorStop)) {}
            if (hit.done) return true;
            if (!pseudogeneStop) { if (hit.cur + 1 < hit.len) hit.cur++; }
            if (anchorStop) { hit.done = 1; return true; }
        }
        return false;
    }

    // HI_Aligner::getAnchorHits (hi_aligner.h:5007-5193), linear-index form of
    // adjustWithALT (hi_aligner.h:2251-2264).
    HT2_NI uint32_t getAnchorHits(uint32_t rdi, bool fw, uint32_t maxGenomeHitSize) {
        Ht2ReadHits& hit = W->hits[rdi][fw ? 0 : 1];
        const uint32_t offsetSize = hit.nhits;
        const uint32_t minK = P->minK;
        for (uint32_t hi = 0; hi < offsetSize; hi++) {
            uint32_t hj = 0;
            for (; hj < offsetSize; hj++) {
                Ht2BwtHit& pj = hit.hits[hj];
                if (pj.bot <= pj.top || pj.hasCoords || pj.len <= minK + 2) continue;
                else break;
            }
            if (hj >= offsetSize) break;
            for (uint32_t hk = hj + 1; hk < offsetSize; hk++) {
                Ht2BwtHit& pj = hit.hits[hj];
                Ht2BwtHit& pk = hit.hits[hk];
                if (pk.bot <= pk.top || pk.hasCoords || pk.len <= minK + 2) continue;
                if (pj.hit_type == pk.hit_type) {
                    uint32_t sj = pj.bot - pj.top, sk = pk.bot - pk.top;
                    if (sj > sk || (sj == sk && pj.len < pk.len)) hj = hk;
                } else if (pk.hit_type > pj.hit_type) hj = hk;
            }
            Ht2BwtHit& ph = hit.hits[hj];
            uint32_t remained = maxGenomeHitSize - W->nGenomeHits;
            if (remained <= 0) break;
            uint32_t expectedNumCoords = ph.node_bot - ph.node_top;
            bool straddled = false;
            W->nCoords = 0;
            if (expectedNumCoords <= remained) {
                if (GRAPH) getGenomeCoordsGraph(ph.top, ph.bot, ph.node_top, ph.node_bot, hit.ie + ph.ieOff, ph.ieN, fw, ph.bot - ph.top, ph.len, false, straddled);
                else getGenomeCoords(ph.top, ph.bot, ph.node_top, ph.node_bot, fw, ph.bot - ph.top, ph.len, false, straddled);
            } else {
                uint32_t top = ph.top;
                uint32_t added = 0;
                uint32_t edgeIdx = 0;
                for (uint32_t node = ph.node_top; node < ph.node_bot; node++, expectedNumCoords--) {
                    uint32_t bot = top + 1;
                    uint16_t oneIe[1][2]; uint32_t nOneIe = 0;
                    if (GRAPH && edgeIdx < ph.ieN && node - ph.node_top == hit.ie[ph.ieOff + edgeIdx][0]) {
                        bot += hit.ie[ph.ieOff + edgeIdx][1];      // this node has extra incoming edges (hi_aligner.h:5097-5107)
                        oneIe[0][0] = 0; oneIe[0][1] = hit.ie[ph.ieOff + edgeIdx][1]; nOneIe = 1;
                        edgeIdx++;
                    }
                    uint32_t rndi = W->rnd.nextU32() % expectedNumCoords;
                    if (rndi < remained - added) {
                        if (GRAPH) getGenomeCoordsGraph(top, bot, node, node + 1, oneIe, nOneIe, fw, ph.bot - ph.top, ph.len, false, straddled);
                        else getGenomeCoords(top, bot, node, node + 1, fw, ph.bot - ph.top, ph.len, false, straddled);
                        added++;
                        if (added >= remained) break;
                    }
                    top = bot;
                }
            }
            ph.hasCoords = W->nCoords > 0 ? 1 : 0;
            if (!ph.hasCoords) continue;
            const uint32_t genomeHit_size = W->nGenomeHits;
            if (genomeHit_size + W->nCoords > maxGenomeHitSize) {
                // EList::shufflePortion (ds.h:836-847)
                uint32_t left = W->nCoords;
                for (uint32_t i = 0; i + 1 < W->nCoords; i++) {
                    uint32_t rndi = W->rnd.nextU32() % left;
                    if (rndi > 0) { Ht2Coord t = W->coords[i]; W->coords[i] = W->coords[i + rndi]; W->coords[i + rndi] = t; }
                    left--;
                }
            }
#if !defined(__CUDA_ARCH__) && defined(HT2_TRACE)
            fprintf(stderr, "partial hj %u bwoff %u len %u top %u bot %u ntop %u nbot %u ncoords %u\n", hj, ph.bwoff, ph.len, ph.top, ph.bot, ph.node_top, ph.node_bot, W->nCoords);
            for (uint32_t k = 0; k < W->nCoords; k++) fprintf(stderr, "  coord ref %u off %u joined %u\n", W->coords[k].ref, W->coords[k].off, W->coords[k].joinedOff);
#endif
            for (uint32_t k = 0; k < W->nCoords; k++) {
                const Ht2Coord& coord = W->coords[k];
                if (coord.ref == HT2_IDX_MAX32) continue;
                uint32_t len = ph.len;
                uint32_t rdoff = hit.len - ph.bwoff - len;
                bool overlapped = false;
                for (uint32_t l = 0; l < genomeHit_size; l++) {
                    Ht2Hit& gh = W->genomeHits[l];
                    if (gh.tidx != coord.ref || gh.fw != coord.fw) continue;
                    uint32_t hitoff = gh.toff + hit.len - gh.rdoff;
                    uint32_t hitoff2 = coord.off + hit.len - rdoff;
                    int64_t hitoff_diff = (noSpl() ? 0 : (int64_t)P->maxIntronLen);
                    int64_t d = (int64_t)hitoff - (int64_t)hitoff2;
                    if (d < 0) d = -d;
                    if (d <= hitoff_diff) { overlapped = true; gh.hitcount++; break; }
                }
                if (!overlapped) {
                    if (W->nGenomeHits >= HT2_MAX_GHITS) { W->err |= HT2_ERR_GHITS; break; }
                    adjustWithALTCoord(rdoff, len, coord, rdi);     // plain init on linear indexes (hi_aligner.h:2251-2264)
                }
                if (ph.hit_type == HT2_CANDIDATE_HIT && W->nGenomeHits >= maxGenomeHitSize) break;
            }
            if (ph.hit_type == HT2_CANDIDATE_HIT && W->nGenomeHits >= maxGenomeHitSize) break;
        }
#if !defined(__CUDA_ARCH__) && defined(HT2_TRACE)
        for (uint32_t gi = 0; gi < W->nGenomeHits; gi++) fprintf(stderr, "anchor %u fw %u rdoff %u len %u toff %u ned %u\n", gi, W->genomeHits[gi].fw, W->genomeHits[gi].rdoff, W->genomeHits[gi].len, W->genomeHits[gi].toff, W->genomeHits[gi].nedits);
#endif
        return W->nGenomeHits;
    }

    HT2_HD int64_t sinkFloor(uint32_t rdi, int64_t cushion) const {
        int64_t m = minsc[rdi];
        if (!P->secondary) {
            // the reference computes sink.bestUnpN() - cushion in int64; with no alignment yet
            // (INT64_MIN) and a non-zero cushion this wraps to a huge positive floor
            int64_t b = (int64_t)((uint64_t)W->bestUnp[rdi] - (uint64_t)cushion);
            if (b > m) m = b;
        }
        return m;
    }

    // HI_Aligner::pairReads / alignMate anchors (hi_aligner.h:5948, 5600-5717); the control flow of go() /
    // hybridSearch_recur / alignMate is the explicit-stack machine below (ht2_machine.h)
    HT2_NI void pairReads();
    HT2_NI bool peConcordant(int64_t off1, uint32_t len1, bool fw1, int64_t off2, uint32_t len2, bool fw2) const;
    HT2_NI void alignMateAnchors(uint32_t rdi, bool fw, uint32_t tidx, uint32_t toff);
    // explicit-stack formulation (ht2_machine.h)
    HT2_HD void pushFrame(uint32_t rdi, const Ht2Hit* hit, uint32_t hitoff, uint32_t hitlen, bool alignMate, uint32_t dep);
    HT2_NI void runFrame();
    HT2_NI void runTop();
    HT2_HD void machineStart();
    HT2_HD bool machineDone() const;
    HT2_HD void machineStep();
    HT2_HD bool machineAtHeavyState() const;
    HT2_HD void machineRun();

#include "ht2_alt.h"
#include "ht2_sw.h"
};
typedef Ht2AlignerT<false> Ht2Aligner;        // linear indexes
typedef Ht2AlignerT<true>  Ht2GraphAligner;   // graph (SNP) indexes

#include "ht2_pair.h"
#include "ht2_machine.h"

#endif // HT2_CORE_H_
