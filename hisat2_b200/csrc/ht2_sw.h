// ht2_sw.h -- the --bowtie2-dp seed extension: end-to-end dynamic programming
// around an anchor, then a deterministic backtrace.  Textually included inside
// Ht2AlignerT (ht2_core.h).
//
// What the reference does (SplicedAligner::hybridSearch, spliced_aligner.h:209-297):
// after the first hybridSearch_recur on an anchor, when --bowtie2-dp is 2, or 1
// and the recursion found nothing >= minsc, it frames a rectangle of
// rdlen x (rdlen + 40) cells around the anchor's diagonal
// (DynProgFramer::frameSeedExtensionRect, dp_framer.cpp:81-132), fills E/F/H
// with the striped 8-bit (or 16-bit when minsc < -254) SSE kernel
// (aligner_swsse_ee_u8.cpp:791-1163 / _i16.cpp), gathers the last-row cells
// >= minsc as candidates (aligner_swsse_ee_u8.cpp:1202-1233), sorted by
// (score desc, col desc) (aligner_sw_nuc.h:149-157), and backtraces from the first
// candidate that succeeds (SwAligner::nextAlignment aligner_sw.cpp:709-1122,
// backtraceNucleotidesEnd2EndSseU8 aligner_swsse_ee_u8.cpp:1309-1902).  The
// result replaces the anchor with a full-length hit.
//
// Restated here: swFill IS the striped kernel, two rows per 32-bit word as signed 16-bit halves instead of
// 16 (or 8) per SSE register, because sm_90a executes max(a + b, c) on s16x2 and the 3-input max in ONE
// instruction each (the DPX family: __viaddmax_s16x2, __vimax3_s16x2) while the byte-wise video
// instructions (__vsubus4, __vmaxu4) are emulated (about 6 and 4 instructions, measured in the SASS): a
// column costs 8 SIMD instructions per word = 4 per cell.  Saturating subtraction a (-) b is
// max(a + (-b), 0); the gap barrier is a penalty larger than any value.  The striped kernel plus its
// lazy-F loop computes exactly the saturating Gotoh recurrences
//     E[i][j] = max(E[i][j-1] (-) rdgape, (H[i][j-1] (-) rdgapo) (-) bar_i)
//     F[i][j] = max(F[i-1][j] (-) rfgape,  H[i-1][j] (-) rfgapo) (-) bar_i
//     H[i][j] = max(Hd (-) pen(i,j), E[i][j], F[i][j]),  Hd = top for row 0, floor for column 0
// and the same code serves the reference's 8-bit and 16-bit paths: their floors (255 resp. 65535 below
// the top) only clamp cells below minsc - 255, and such cells are never candidates, never on a path
// (scores along a backtrace only rise towards row 0), never win a max against a cell >= minsc, and never
// satisfy one of the backtrace's equality tests against a cell on the path -- so a floor 16383 below the
// top gives the same candidates, paths and edits (minsc below -15000 is refused as a capacity error).
//
// The H, E and F planes are kept (6 B/cell, one 32-bit store per 2 cells per plane).  The backtrace only
// ever compares stored cell values for equality; the move bits of a cell (the bits the reference keeps in
// SSEMatrix::masks_, sse_util.h) are derived from the planes for the ~rdlen cells a backtrace visits.
//
// The backtrace is deterministic in this reference (the randomised choices are
// compiled out, aligner_swsse_ee_u8.cpp:1405, 1461, 1532): preference diag > H up
// > F up > H left > E left.  Its backtrack stack never helps: a popped branch
// cell is already marked reported-through, so the pop cascades until the stack
// is empty (aligner_swsse_ee_u8.cpp:1353-1361, 1580-1606); a blocked cell
// therefore simply fails the candidate.  For the same reason the in-place mask updates
// (hMaskSet / eMaskSet / fMaskSet) are never observed: the only mutable per-cell state that matters is
// the reported-through bit, kept as one bit per cell for the candidates that follow.

#define HT2_SWM_H(c)      ((c) & 31u)
#define HT2_SWM_E(c)      (((c) >> 5) & 3u)
#define HT2_SWM_F(c)      (((c) >> 7) & 3u)
#define HT2_SWM_REP       (1u << 9)
#define HT2_SWM_OH        (1u << 10)
#define HT2_SWM_OE        (1u << 11)
#define HT2_SWM_OF        (1u << 12)

typedef Ht2SwRect SwRect;

// DynProgFramer::frameSeedExtensionRect with readGaps = refGaps = maxhalf = 10, nceil = 0,
// trimToRef = false (the arguments of spliced_aligner.h:226-239)
HT2_HD static bool swFrameRect(int64_t off, uint32_t rdlen, int64_t reflen, SwRect& r) {
    const int64_t maxgap = HT2_SW_MAXGAP;
    int64_t refl = off - 2 * maxgap, refr = off + ((int64_t)rdlen - 1) + 2 * maxgap;
    int64_t maxns = 0;
    if (maxns == (int64_t)rdlen) maxns--;
    uint32_t triml = 0, trimr = 0;
    if (refr >= reflen + maxns) trimr = (uint32_t)(refr - (reflen + maxns - 1));
    if (refl < -maxns) triml = (uint32_t)((-refl) - maxns);
    r.refl = refl + triml; r.refr = refr - trimr; r.triml = triml; r.trimr = trimr;
    r.corel = (uint32_t)maxgap; r.corer = r.corel + 2 * (uint32_t)maxgap;
    return r.refr >= r.refl;
}

HT2_HD static uint8_t swMask2dna(int code) { return (uint8_t)("ACGTN"[code]); }

// plane pool accessors (Ht2SwScratch, ht2_core.h): score planes 0 = H, 1 = E, 2 = F; small per-problem arrays
// 0..4 = negated query profile per reference character, 5 = gap barrier, 6 = barrier + read-gap-open
#define HT2_SWP(pl, idx) swPl[((size_t)(pl) * HT2_SW_PLANE_WORDS + (size_t)(idx)) * swStride]
#define HT2_SWQ(k, s) swPl[((size_t)3 * HT2_SW_PLANE_WORDS + (size_t)(k) * HT2_SW_SEG + (size_t)(s)) * swStride]

#define HT2_SW_TOP 16383      /* raw value of a perfect score; 0 = floor */
#define HT2_SW_BAR 16384      /* gap-barrier penalty: larger than any raw value */

// Striped fill + gather (alignNucleotidesEnd2EndSseU8 / SseI16, aligner_swsse_ee_u8.cpp:791-1163).
// Row i lives in half i / seg of word i % seg.  Returns the best last-row score (0 = perfect), or
// HT2_MIN_I64 when nothing reaches minsc.
HT2_NI int64_t swFill(const uint8_t* rd, const uint8_t* qu, uint32_t nrow, const uint8_t* rf, uint32_t ncol, int64_t minscR) {
    Ht2SwScratch& S = *sw;
    const uint32_t seg = (nrow + 1) >> 1;
    const uint32_t gapbar = (uint32_t)P->gapbar;
    const int rdgapo = P->rdGapConst + P->rdGapLinear;
    S.nrow = nrow; S.seg = seg; S.coop = 0; S.rcp = 0;
    for (uint32_t k = 0, n = (ncol * nrow + 31) >> 5; k < n; k++) S.rep[k] = 0;   // reported-through bits
    for (uint32_t i = 0; i < nrow; i++) S.rowPen[i] = (uint8_t)ht2_mmpen(*P, (int)qu[i] - 33);
    for (uint32_t s = 0; s < seg; s++) {   // negated query profile / gap-barrier words (buildQueryProfileEnd2EndSseU8, :76-140)
        uint32_t g = 0, go = 0, w[5] = {0, 0, 0, 0, 0};
        for (uint32_t k = 0; k < 2; k++) {
            const uint32_t i = k * seg + s;
            int bar = 0;
            if (i < nrow) {
                if (i < gapbar || nrow - 1 - i < gapbar) bar = HT2_SW_BAR;
                const int rdc = rd[i];
                for (int refc = 0; refc < 5; refc++) {
                    const int pen = (rdc > 3 || refc > 3) ? P->npen : (rdc == refc ? 0 : (int)S.rowPen[i]);
                    w[refc] |= (uint32_t)(uint16_t)(-pen) << (16 * k);
                }
            }
            g  |= (uint32_t)(uint16_t)(-bar) << (16 * k);
            go |= (uint32_t)(uint16_t)(-(bar + rdgapo)) << (16 * k);
        }
        HT2_SWQ(5, s) = g; HT2_SWQ(6, s) = go;
        for (int refc = 0; refc < 5; refc++) HT2_SWQ(refc, s) = w[refc];
    }
    const uint32_t nRDE = ht2_v2_splat(-P->rdGapLinear);
    const uint32_t nRFO = ht2_v2_splat(-(P->rfGapConst + P->rfGapLinear)), nRFE = ht2_v2_splat(-P->rfGapLinear);
    // plain pointers into the lane's pool (stride 1): the inner loop is latency-bound on a lone lane -- one DP problem
    // rarely has company in its warp -- so every address computation it does not do counts (the strided accessor
    // macros cost ~40 of the ~70 instructions per word in the round-2 profile)
    uint32_t* const plH = &HT2_SWP(0, 0); uint32_t* const plE = &HT2_SWP(1, 0); uint32_t* const plF = &HT2_SWP(2, 0);
    const uint32_t* const qG = &HT2_SWQ(5, 0); const uint32_t* const qR = &HT2_SWQ(6, 0);
    uint32_t* const Hzc = plH + (size_t)ncol * seg;   // an all-floor column of H standing in for column -1
    for (uint32_t s = 0; s < seg; s++) { Hzc[s] = 0; plE[s] = 0; }
    const uint32_t lastW = (nrow - 1) % seg, lastB = 16 * ((nrow - 1) / seg);
    int best = 0;
    for (uint32_t j = 0; j < ncol; j++) {
        const uint32_t pr = rf[j] > 4 ? 4u : (uint32_t)rf[j];
        const uint32_t* const qP = &HT2_SWQ(pr, 0);
        uint32_t* const Hc = plH + (size_t)j * seg; uint32_t* const Fc = plF + (size_t)j * seg;
        uint32_t* const Ec = plE + (size_t)j * seg; uint32_t* const En = Ec + seg;
        const uint32_t* const Hp = j ? Hc - seg : Hzc;
        uint32_t vF = 0;
        uint32_t vH = (Hp[seg - 1] << 16) | (uint32_t)HT2_SW_TOP;   // diagonal of row 0 = perfect; of row seg = last row of half 0
        // The loads of iteration s + 1 are issued before the stores of iteration s: all planes live in one pool, so
        // the compiler must assume the stores alias them and would otherwise start each iteration's loads only
        // after the previous iteration's stores.
        uint32_t nE = Ec[0], nHp = Hp[0], nG = qG[0], nP = qP[0], nR = qR[0];
        for (uint32_t s = 0; s < seg; s++) {
            uint32_t vE = nE;
            const uint32_t hp = nHp, wG = nG, wP = nP, wR = nR;
            if (s + 1 < seg) { nE = Ec[s + 1]; nHp = Hp[s + 1]; nG = qG[s + 1]; nP = qP[s + 1]; nR = qR[s + 1]; }
            vF = ht2_v2_addmax(vF, wG, 0);                                  // veto ref-gap extensions in barrier rows
            Fc[s] = vF;
            vH = ht2_v2_addmax(vH, wP, 0);                                  // match / mismatch
            vH = ht2_v2_max3(vH, vE, vF);
            Hc[s] = vH;
            vE = ht2_v2_addmax(vE, nRDE, ht2_v2_addmax(vH, wR, 0));         // E of the next column
            En[s] = vE;
            vF = ht2_v2_addmax(vF, nRFE, ht2_v2_addmax(vH, nRFO, 0));       // F of the next row
            vH = hp;
        }
        // lazy F: carry each half's last F into the other half's first rows while it still improves
        {
            uint32_t s = 0;
            vF = ht2_v2_addmax(vF << 16, qG[0], 0);
            for (;;) {
                const uint32_t old = Fc[s];
                const uint32_t nf = ht2_v2_max(old, vF);
                if (nf == old) break;
                Fc[s] = nf;
                const uint32_t vh = ht2_v2_max(Hc[s], nf);
                Hc[s] = vh;
                En[s] = ht2_v2_max(En[s], ht2_v2_addmax(vh, qR[s], 0));
                vF = nf;
                if (++s == seg) { s = 0; vF <<= 16; }
                vF = ht2_v2_addmax(ht2_v2_addmax(vF, nRFE, 0), qG[s], 0);
            }
        }
        const int lr = (int)((Hc[lastW] >> lastB) & 0xffffu);
        S.lastH[j] = lr - HT2_SW_TOP;
        if (lr > best) best = lr;
    }
    if ((int64_t)(best - HT2_SW_TOP) < minscR) return HT2_MIN_I64;
    return best - HT2_SW_TOP;
}

#if defined(__CUDACC__)
// One vector position down: element p of the warp-wide vector (lane p % 32, half p / 32) receives element p - 1;
// element 0 receives 'first'.  The s16x2 counterpart of the striped kernel's byte shift (_mm_slli_si128).
__device__ __forceinline__ static uint32_t swShift1(uint32_t w, uint32_t lane, uint32_t first) {
    const uint32_t up = __shfl_up_sync(0xffffffffu, w, 1);
    const uint32_t l31 = __shfl_sync(0xffffffffu, w, 31);
    return lane ? up : ((l31 << 16) | first);
}
// The fill run by a whole warp on ONE problem (the problem framed in *Sp by swPrepare on its owner lane; planes
// into the owner's pool), as an anti-diagonal wavefront: lane L owns the R = ceil(nrow / 32) consecutive rows
// L*R .. L*R + R - 1 and works on column t - L at step t, so that everything a cell needs is either in the lane's
// own registers (left neighbours, the rows above inside its block) or was produced by lane L - 1 one step earlier
// (H and F of its last row: two shuffles per step).  ncol + 31 steps of R cells; a cell is ~12 scalar DPX /
// integer instructions.  This evaluates the saturating recurrences at the top of this file DIRECTLY -- no lazy-F
// loop: the striped kernel's lazy-F pass, cheap with 2 (swFill) or 16 (SSE) rows per vector, degenerates when
// the vector is a warp wide, because a reference-gap chain below the read's diagonal crosses a vector position
// every R rows and each crossing costs a pass (about 20 passes per column on the --bowtie2-dp 2 fixtures).  Cell values
// are those of swFill; they are stored skewed, step-major (word q of lane L at step t), so that every store is a
// coalesced line: cell (row, col) = half k & 1 of word ((col + L) * 32 + L) * RW + k / 2, L = row / R, k = row % R,
// RW = ceil(R / 2) (swRaw).  All 32 lanes must call this with the same arguments.
__device__ __noinline__ void swFillCoop(Ht2SwScratch* Sp, uint32_t* pool, uint32_t lane) const {
    constexpr int MR = (HT2_SW_MAX_RDLEN + 31) / 32;
    Ht2SwScratch& S = *Sp;
    const uint32_t nrow = S.nrow, ncol = S.jncol;
    const uint8_t* const rd = S.jrd; const uint8_t* const qu = S.jqu; const uint8_t* const rf = S.jrf;
    const uint32_t R = (nrow + 31) >> 5, RW = (R + 1) >> 1;
    const uint32_t gapbar = (uint32_t)P->gapbar;
    const int rdo = P->rdGapConst + P->rdGapLinear, rde = P->rdGapLinear, rfo = P->rfGapConst + P->rfGapLinear, rfe = P->rfGapLinear;
    const int npen = P->npen;
    for (uint32_t k = lane, n = (ncol * nrow + 31) >> 5; k < n; k += 32) S.rep[k] = 0;
    int rdc[MR], mm[MR], nbar[MR], nbo[MR], Hl[MR], El[MR], Fk[MR];
#pragma unroll
    for (int k = 0; k < MR; k++) {
        const uint32_t i = lane * R + (uint32_t)k;
        rdc[k] = 0; mm[k] = 0; nbar[k] = 0; nbo[k] = -rdo; Hl[k] = 0; El[k] = 0; Fk[k] = 0;
        if ((uint32_t)k < R && i < nrow) {
            const int bar = (i < gapbar || nrow - 1 - i < gapbar) ? HT2_SW_BAR : 0;
            rdc[k] = rd[i];
            mm[k] = ht2_mmpen(*P, (int)qu[i] - 33);
            S.rowPen[i] = (uint8_t)mm[k];
            nbar[k] = -bar; nbo[k] = -(bar + rdo);
        }
    }
    uint32_t* const plH = pool + lane * RW; uint32_t* const plE = plH + (size_t)HT2_SW_PLANE_WORDS; uint32_t* const plF = plE + (size_t)HT2_SW_PLANE_WORDS;
    const uint32_t lastLane = ((nrow - 1) * ((65536 + R - 1) / R)) >> 16, lastK = (nrow - 1) - lastLane * R;
    int diagIn = 0, outH = 0, outF = 0, best = 0;
    const uint32_t nstep = ncol + 31;
    for (uint32_t t = 0; t < nstep; t++) {
        const int inH = __shfl_up_sync(0xffffffffu, outH, 1), inF = __shfl_up_sync(0xffffffffu, outF, 1);
        const uint32_t j = t - lane;
        if (j < ncol) {                                   // (t < lane wraps to a huge j)
            int refc = rf[j]; if (refc > 4) refc = 4;
            int hd = lane ? diagIn : HT2_SW_TOP;          // H[i-1][j-1]: row 0's diagonal is the perfect score
            int hu = inH, fu = inF;
#pragma unroll
            for (int k = 0; k < MR; k++) if ((uint32_t)k < R) {
                const int e = __viaddmax_s32(El[k], -rde, __viaddmax_s32(Hl[k], nbo[k], 0));
                int f = __viaddmax_s32(__viaddmax_s32(fu, -rfe, __viaddmax_s32(hu, -rfo, 0)), nbar[k], 0);
                if (k == 0 && lane == 0) f = 0;           // row 0 has no row above
                const int pen = (rdc[k] > 3 || refc > 3) ? npen : (rdc[k] == refc ? 0 : mm[k]);
                const int h = __vimax3_s32(__viaddmax_s32(hd, -pen, 0), e, f);
                hd = Hl[k];
                Hl[k] = h; El[k] = e; Fk[k] = f;
                hu = h; fu = f;
            }
            diagIn = inH; outH = hu; outF = fu;
            const size_t o = (size_t)t * 32 * RW;
#pragma unroll
            for (int q = 0; q < MR / 2; q++) if ((uint32_t)q < RW) {
                plH[o + q] = (uint32_t)Hl[2 * q] | ((uint32_t)Hl[2 * q + 1] << 16);
                plE[o + q] = (uint32_t)El[2 * q] | ((uint32_t)El[2 * q + 1] << 16);
                plF[o + q] = (uint32_t)Fk[2 * q] | ((uint32_t)Fk[2 * q + 1] << 16);
            }
            if (lane == lastLane) {
                int lr = 0;
#pragma unroll
                for (int k = 0; k < MR; k++) if ((uint32_t)k == lastK) lr = Hl[k];
                S.lastH[j] = lr - HT2_SW_TOP;
                if (lr > best) best = lr;
            }
        }
    }
    best = __shfl_sync(0xffffffffu, best, lastLane);
    if (lane == 0) {
        S.seg = R; S.coop = 1; S.rcp = (65536 + R - 1) / R;
        S.jbest = ((int64_t)(best - HT2_SW_TOP) < S.jmsc) ? HT2_MIN_I64 : (int64_t)(best - HT2_SW_TOP);
    }
    __syncwarp();
}
#endif

HT2_HD int swRaw(int plane, uint32_t seg, uint32_t row, uint32_t col) const {
    const Ht2SwScratch& S = *sw;
    if (S.coop) {   // warp fill (seg = R rows per lane; the 16-bit reciprocal is exact for row < 8192)
        const uint32_t L = (row * S.rcp) >> 16, k = row - L * seg, rw = (seg + 1) >> 1;
        return (int)((HT2_SWP(plane, ((size_t)(col + L) * 32 + L) * rw + (k >> 1)) >> (16 * (k & 1))) & 0xffffu);
    }
    return (int)((HT2_SWP(plane, (size_t)col * seg + row % seg) >> (16 * (row / seg))) & 0xffffu);
}
// Move bits of a cell from the score planes (what the reference recomputes at every visited cell,
// aligner_swsse_ee_u8.cpp:1376-1545); row > 0.
HT2_NI uint32_t swCellFromPlanes(const uint8_t* rd, const uint8_t* rf, uint32_t row, uint32_t col) const {
    const Ht2SwScratch& S = *sw;
    const uint32_t seg = S.seg, nrow = S.nrow;
    const int rdgapo = P->rdGapConst + P->rdGapLinear, rdgape = P->rdGapLinear;
    const int rfgapo = P->rfGapConst + P->rfGapLinear, rfgape = P->rfGapLinear;
    const uint32_t gapbar = (uint32_t)P->gapbar;
    const bool gb = (row < gapbar) || (nrow - 1 - row < gapbar);
    int h, e, f, hup, fup, hleft = 0, eleft = 0, hd = 0;
    if (S.coop) {
        // warp-fill layout: all eight words are addressed first and loaded side by side -- the planes were written by
        // other lanes, so every load is an L2 round trip, and a backtrace is a chain of ~nrow such cells
        const uint32_t rw = (seg + 1) >> 1;
        const uint32_t L = (row * S.rcp) >> 16, k = row - L * seg;
        const uint32_t Lu = k ? L : L - 1, ku = k ? k - 1 : seg - 1;              // row - 1
        const size_t a = ((size_t)(col + L) * 32 + L) * rw + (k >> 1), au = ((size_t)(col + Lu) * 32 + Lu) * rw + (ku >> 1);
        const size_t back = (size_t)32 * rw;                                      // one column to the left = one step earlier
        const uint32_t* const pH = swPl; const uint32_t* const pE = swPl + (size_t)HT2_SW_PLANE_WORDS; const uint32_t* const pF = pE + (size_t)HT2_SW_PLANE_WORDS;
        const bool left = col > 0;
        const uint32_t wh = pH[a], we = pE[a], wf = pF[a], whu = pH[au], wfu = pF[au];
        const uint32_t whl = left ? pH[a - back] : 0u, wel = left ? pE[a - back] : 0u, whd = left ? pH[au - back] : 0u;
        const uint32_t sh = 16 * (k & 1), su = 16 * (ku & 1);
        h = (int)((wh >> sh) & 0xffffu); e = (int)((we >> sh) & 0xffffu); f = (int)((wf >> sh) & 0xffffu);
        hup = (int)((whu >> su) & 0xffffu); fup = (int)((wfu >> su) & 0xffffu);
        hleft = (int)((whl >> sh) & 0xffffu); eleft = (int)((wel >> sh) & 0xffffu); hd = (int)((whd >> su) & 0xffffu);
    } else {
        h = swRaw(0, seg, row, col); e = swRaw(1, seg, row, col); f = swRaw(2, seg, row, col);
        hup = swRaw(0, seg, row - 1, col); fup = swRaw(2, seg, row - 1, col);
        if (col > 0) { hleft = swRaw(0, seg, row, col - 1); eleft = swRaw(1, seg, row, col - 1); hd = swRaw(0, seg, row - 1, col - 1); }
    }
    uint32_t hm = 0, em = 0, fm = 0;
    if (!gb) { if (h + rfgapo == hup) hm |= 1; if (h + rfgape == fup) hm |= 4; }
    if (col > 0) {
        const int rdc = rd[row], refc = rf[col];
        const int pen = (rdc > 3 || refc > 3) ? P->npen : (rdc == refc ? 0 : (int)S.rowPen[row]);
        if (!gb) { if (h + rdgapo == hleft) hm |= 2; if (h + rdgape == eleft) hm |= 8; }
        if (h + pen == hd) hm |= 16;
        if (hleft - rdgapo == e) em |= 1;
        if (eleft - rdgape == e) em |= 2;
    }
    if (hup - rfgapo == f) fm |= 1;
    if (fup - rfgape == f) fm |= 2;
    return hm | (em << 5) | (fm << 7) | (hm ? HT2_SWM_OH : 0) | (em ? HT2_SWM_OE : 0) | (fm ? HT2_SWM_OF : 0);
}
// One backtrace (aligner_swsse_ee_u8.cpp:1309-1902).  Edits land in S.ned (left to right).
HT2_NI bool swBacktrace(const uint8_t* rd, const uint8_t* qu, uint32_t nrow, const uint8_t* rf, const SwRect& rect, int nceil,
                        uint32_t row, uint32_t col, uint32_t& nedOut, uint32_t& offOut, int64_t& scoreOut) {
    Ht2SwScratch& S = *sw;
    const int rdgapo = P->rdGapConst + P->rdGapLinear, rdgape = P->rdGapLinear;
    const int rfgapo = P->rfGapConst + P->rfGapLinear, rfgape = P->rfGapLinear;
    enum { CT_H = 0, CT_E = 1, CT_F = 2 };
    enum { MV_DIAG, MV_REF_OPEN, MV_RFGAP_EXT, MV_READ_OPEN, MV_RDGAP_EXT };
    int ct = CT_H;
    uint32_t ned = 0;
    int64_t score = 0; int ns = 0;
    bool ovl = false;
    for (;;) {
        const uint32_t bit = col * S.nrow + row;
        const uint32_t repw = S.rep[bit >> 5];                                   // read once: reported-through test here, mark below
        const uint32_t planes = row > 0 ? swCellFromPlanes(rd, rf, row, col) : 0u;
        const uint32_t cell = ((repw >> (bit & 31)) & 1u) ? (uint32_t)HT2_SWM_REP : planes;
        bool empty = false, canMoveThru = true;
        int cur = -1;
        if (cell & HT2_SWM_REP) canMoveThru = false;
        else if (row > 0) {
            if (ct == CT_E) {
                const uint32_t m = HT2_SWM_E(cell);
                if (m == 3 || m == 1) cur = MV_READ_OPEN;          // H -> E preferred (:1405)
                else if (m == 2) cur = MV_RDGAP_EXT;
                else { empty = true; canMoveThru = (cell & HT2_SWM_OE) == 0; }
            } else if (ct == CT_F) {
                const uint32_t m = HT2_SWM_F(cell);
                if (m == 3 || m == 1) cur = MV_REF_OPEN;           // H -> F preferred (:1461)
                else if (m == 2) cur = MV_RFGAP_EXT;
                else { empty = true; canMoveThru = (cell & HT2_SWM_OF) == 0; }
            } else {
                const uint32_t m = HT2_SWM_H(cell);
                int select = -1;
                if (m != 0) {
                    if (m & 16) select = 4;        // H diag
                    else if (m & 1) select = 0;    // H up
                    else if (m & 4) select = 2;    // F up
                    else if (m & 2) select = 1;    // H left
                    else select = 3;               // E left
                    cur = select == 4 ? MV_DIAG : select == 0 ? MV_REF_OPEN : select == 1 ? MV_READ_OPEN : select == 2 ? MV_RFGAP_EXT : MV_RDGAP_EXT;
                } else { empty = true; canMoveThru = (cell & HT2_SWM_OH) == 0; }
            }
        }
        S.rep[bit >> 5] = repw | (1u << (bit & 31));
        if (!canMoveThru) return false;
        {   // the cell joins the path: does it sit on a core diagonal?
            int64_t diagi = (int64_t)col - (int64_t)row + (int64_t)rect.triml;
            if (diagi >= 0 && (uint64_t)diagi >= rect.corel && (uint64_t)diagi <= rect.corer) ovl = true;
        }
        if (empty || row == 0) break;
        const int rdc = rd[row];
        const int refc = rf[col];
        if (ned >= HT2_SW_MAX_EDITS) { W->err |= HT2_ERR_EDITS; return false; }
        switch (cur) {
        case MV_DIAG: {
            const bool amb = (rdc > 3 || refc > 3);
            if (amb || rdc != refc) {
                S.ned[ned++] = mkEdit(row, swMask2dna(refc), ht2_code2asc(rdc), HT2_EDIT_MM);
                score -= amb ? P->npen : (int)S.rowPen[row];
            }
            if (amb) ns++;
            row--; col--; ct = CT_H;
            break;
        }
        case MV_REF_OPEN: case MV_RFGAP_EXT:
            S.ned[ned++] = mkEdit(row, '-', ht2_code2asc(rdc), HT2_EDIT_REF_GAP);
            row--;
            if (cur == MV_REF_OPEN) { ct = CT_H; score -= rfgapo; } else { ct = CT_F; score -= rfgape; }
            break;
        default: // MV_READ_OPEN / MV_RDGAP_EXT
            S.ned[ned++] = mkEdit(row + 1, swMask2dna(refc), '-', HT2_EDIT_READ_GAP);
            col--;
            if (cur == MV_READ_OPEN) { ct = CT_H; score -= rdgapo; } else { ct = CT_E; score -= rdgape; }
            break;
        }
    }
    if (!ovl) return false;   // must overlap a core diagonal (aligner_swsse_ee_u8.cpp:1789-1822)
    {
        const int rdc = rd[row], refc = rf[col];
        const bool amb = (rdc > 3 || refc > 3);
        if (amb || rdc != refc) {
            if (ned >= HT2_SW_MAX_EDITS) { W->err |= HT2_ERR_EDITS; return false; }
            S.ned[ned++] = mkEdit(row, swMask2dna(refc), ht2_code2asc(rdc), HT2_EDIT_MM);
            score -= amb ? P->npen : (int)S.rowPen[row];
        }
        if (amb) ns++;
    }
    if (ns > nceil) return false;
    for (uint32_t a = 0, b = ned; a + 1 < b; a++, b--) { Ht2Edit t = S.ned[a]; S.ned[a] = S.ned[b - 1]; S.ned[b - 1] = t; }
    (void)qu;
    nedOut = ned; offOut = col; scoreOut = score;
    return true;
}

// GenomeHit::replace_edits_with_alts (hi_aligner.h:1229-1330)
HT2_NI void replaceEditsWithAlts(Ht2Hit& h, uint32_t rdi) {
    if (!GRAPH) return;
    const uint32_t nalts = numAlts();
    if (nalts == 0 || h.nedits == 0) return;
    const Ht2Alt* alts = altTable();
    int64_t offset = 0;
    uint32_t i = 0;
    while (i < h.nedits) {
        uint32_t next_i = i + 1;
        Ht2Edit& ed = h.edits[i];
        if (ed.type == HT2_EDIT_READ_GAP || ed.type == HT2_EDIT_REF_GAP)
            for (; next_i < h.nedits; next_i++) if (h.edits[next_i].type != ed.type) break;
        const uint32_t gap = next_i - i;
        if (ed.snpID == HT2_IDX_MAX32) {
            const uint32_t key = (uint32_t)((int64_t)h.joinedOff + (int64_t)ed.pos + offset);
            for (uint32_t ai = altLoBound(key); ai < nalts; ai++) {
                const Ht2Alt& alt = alts[ai];
                if (alt.pos > key) break;
                if (ed.type == HT2_EDIT_MM) {
                    if (alt.type != HT2_ALT_SNP_SGL) continue;
                    if (alt.seq < 4 && "ACGT"[alt.seq] == (char)ed.qchr) { ed.snpID = ai; break; }
                } else if (ed.type == HT2_EDIT_READ_GAP) {
                    if (alt.type != HT2_ALT_SNP_DEL) continue;
                    if (alt.len == gap) { for (uint32_t ii = i; ii < next_i; ii++) h.edits[ii].snpID = ai; break; }
                } else {
                    if (alt.type != HT2_ALT_SNP_INS) continue;
                    if (alt.len == gap) {
                        uint64_t seq = 0;
                        for (uint32_t ii = i; ii < next_i; ii++) seq = (seq << 2) | (uint64_t)(ht2_asc2code(h.edits[ii].qchr) & 3);
                        if (alt.seq == seq) { for (uint32_t ii = i; ii < next_i; ii++) h.edits[ii].snpID = ai; break; }
                    }
                }
            }
        }
        if (ed.type == HT2_EDIT_READ_GAP) offset += gap;
        else if (ed.type == HT2_EDIT_REF_GAP) offset -= gap;
        i = next_i;
    }
    calculateScore(h, rdi);
}

// The dp block of SplicedAligner::hybridSearch (spliced_aligner.h:209-297) in three steps, so that the pool kernel
// can run the middle one with a whole warp per problem: swPrepare frames the rectangle and fetches the reference
// window (returns false when there is nothing to fill: the answer is 'ret'), swFill / swFillCoop fill the planes,
// swFinish walks the candidates.
HT2_NI bool swPrepare(uint32_t rdi, Ht2Hit& gh, bool& ret) {
    ret = false;
    const Ht2Read& R = W->rd[rdi];
    const uint32_t rdlen = R.len;
    if (gh.len >= rdlen) { ret = true; return false; }
    if (sw == NULL) { W->err |= HT2_ERR_SW; return false; }
    Ht2SwScratch& S = *sw;
    const bool fw = gh.fw != 0;
    const int64_t tlen = (int64_t)refLen(gh.tidx);
    const uint32_t refoff = gh.toff > gh.rdoff ? gh.toff - gh.rdoff : 0;
    SwRect rect;
    if (!swFrameRect((int64_t)refoff, rdlen, tlen, rect)) return false;
    const uint32_t ncol = (uint32_t)(rect.refr - rect.refl + 1);
    if (ncol > HT2_SW_MAXCOLS || rdlen > HT2_SW_MAX_RDLEN) { W->err |= HT2_ERR_SW; return false; }   // the score planes are sized for reads of up to 256 bases
    const int64_t msc = minsc[rdi];
    if (msc < -15000) { W->err |= HT2_ERR_SW; return false; }
    // reference window; positions past the end of the sequence read as N (aligner_sw.cpp:160-212)
    S.jrf = getStretch(S.rf, gh.tidx, (uint32_t)rect.refl, ncol);
    S.jrd = R.seq[fw ? 0 : 1]; S.jqu = R.qual[fw ? 0 : 1];
    S.nrow = rdlen; S.jncol = ncol; S.jfw = fw ? 1u : 0u; S.jmsc = msc; S.jrect = rect; S.jbest = HT2_MIN_I64;
    return true;
}
HT2_NI bool swFinish(uint32_t rdi, Ht2Hit& gh) {
    Ht2SwScratch& S = *sw;
    const uint8_t* rd = S.jrd; const uint8_t* qu = S.jqu; const uint8_t* rf = S.jrf;
    const uint32_t rdlen = S.nrow, ncol = S.jncol;
    const bool fw = S.jfw != 0;
    const int64_t msc = S.jmsc;
    const SwRect rect = S.jrect;
    const bool use16 = !(msc >= -254);                    // the reference's 16-bit path (aligner_sw.cpp:496): only the RNG reseeding differs
    // nCeil.f<int>(rdlen) (SwAligner::initRead, aligner_sw.cpp:44)
    const int nceil = ht2_nceil(nCeilTab, rdlen);
    if (S.jbest == HT2_MIN_I64) return false;
    // SwAligner::nextAlignment: candidates in (score desc, col desc) order
    int64_t prevScore = 0; uint32_t prevCol = 0; bool havePrev = false;
    for (;;) {
        int64_t cs = HT2_MIN_I64; uint32_t cc = 0; bool got = false;
        for (uint32_t j = 0; j < ncol; j++) {
            const int64_t s = S.lastH[j];
            if (s < msc) continue;
            if (havePrev && !(s < prevScore || (s == prevScore && j < prevCol))) continue;
            if (!got || s > cs || (s == cs && j > cc)) { cs = s; cc = j; got = true; }
        }
        if (!got) return false;
        prevScore = cs; prevCol = cc; havePrev = true;
        { const uint32_t bit = cc * S.nrow + (rdlen - 1); if ((S.rep[bit >> 5] >> (bit & 31)) & 1u) continue; }   // starting cell already covered
        uint32_t reseed = W->rnd.nextU32() + 1;
        if (!use16) W->rnd.init(reseed);
        uint32_t ned = 0, off = 0; int64_t score = 0;
        const bool ok = swBacktrace(rd, qu, rdlen, rf, rect, nceil, rdlen - 1, cc, ned, off, score);
        W->rnd.init(use16 ? reseed : reseed + 1);
        if (W->err) return false;
        if (!ok) continue;
        if (ned > HT2_MAX_EDITS) { W->err |= HT2_ERR_EDITS; return false; }
        const uint32_t coordOff = (uint32_t)(rect.refl + off);
        const uint32_t joinedOff = gh.joinedOff + coordOff - gh.toff;
        initHit(gh, fw, 0, rdlen, 0, 0, gh.tidx, coordOff, joinedOff);
        gh.score = score;
        gh.nedits = ned;
        for (uint32_t k = 0; k < ned; k++) gh.edits[k] = S.ned[k];
        HT2_HIWATER(maxEdits, ned);
        replaceEditsWithAlts(gh, rdi);
        return true;
    }
}
// Returns 'found': true when the caller has to run hybridSearch_recur on gh once more.
HT2_NI bool swExtendAnchor(uint32_t rdi, Ht2Hit& gh) {
    if (swStage) {                                       // framed (and filled) by the pool kernel's warp-wide DP round
        const bool filled = swStage == 1;
        swStage = 0;
        return filled ? swFinish(rdi, gh) : swRetv;
    }
    bool ret;
    if (!swPrepare(rdi, gh, ret)) return ret;
    Ht2SwScratch& S = *sw;
    S.jbest = swFill(S.jrd, S.jqu, S.nrow, S.jrf, S.jncol, S.jmsc);
    return swFinish(rdi, gh);
}
