// ht2_gpu.cu -- CUDA kernels + C ABI (include/ht2gpu.h) of the alignment path.
//
// Kernel inventory
//   ht2_align_pool_kernel : the alignment path -- every read (pair) runs the complete HI_Aligner::go state
//                           machine (ht2_core.h, ht2_machine.h) against the HBM-resident index image and
//                           appends its alignments to the batch result pools.
//   ht2_seed_kernel       : the seed search (LF mapping) on its own.
//   ht2_sam_*_kernel      : the SAM back end on the device (ht2_sam.h): finishRead for every read of the batch.
// Host code here only moves bytes and launches; it never aligns anything.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <thread>
#include <string>
#include <vector>

#include "../../include/ht2gpu.h"
#include "ht2_core.h"
#include "ht2_seed.h"
#include "ht2_sam.h"
#include "ht2_host.h"
#include "ht2_index.h"

// ---------------------------------------------------------------------------
// device side
// ---------------------------------------------------------------------------
struct DevBatch {
    const uint8_t*  seq;
    const uint8_t*  qual;   // may be NULL
    const uint64_t* offs;
    const uint32_t* seeds;
    uint32_t        n_units;
    int32_t         paired;
    Ht2SwScratch*   sw;     // --bowtie2-dp scratch, one per launched thread (NULL when dp is off)
    uint32_t*       swPool; // ... and the H / E / F plane pool: HT2_SW_POOL_WORDS words per thread, interleaved per warp
    const int32_t*  minscTab; // --score-min per read length (Ht2Params::minscTab)
    uint32_t        elect;    // a warp stays on the block's current target state while it has at least this many claimable slots
#ifdef HT2_ENABLE_SPLICED
    const Ht2SplTables* splT; // donor / acceptor probability tables (spliced mode)
    const uint8_t*  ssT;      // the run's splice-site DB (ht2_ssdb.h) or NULL
#endif
};

struct DevOut {
    ht2gpu_read_result_t* reads;
    ht2gpu_aln_t*         alns;
    ht2gpu_edit_t*        edits;
    uint16_t*             pairs;
    uint32_t              capAlns, capEdits, capPairs;
    unsigned int*         counters; // [0] alns, [1] edits, [2] pairs
    unsigned long long*   stats;    // optional (HT2GPU_STATS=1): per state code [rounds, lanes, cycles, max cycles]
};

// Four bytes starting at any byte address, from two aligned 32-bit loads (the batch buffers have 8 bytes of slack).
__device__ __forceinline__ uint32_t ht2_ld4(const uint8_t* p)
{
    const uintptr_t a = (uintptr_t)p;
    const uint32_t sh = (uint32_t)(a & 3) * 8;
    const uint32_t* w = (const uint32_t*)(a & ~(uintptr_t)3);
    const uint32_t lo = w[0];
    return sh ? __funnelshift_r(lo, w[1], sh) : lo;
}
// complement of four base codes 0..4 (N stays N)
__device__ __forceinline__ uint32_t ht2_comp4(uint32_t x)
{
    const uint32_t n4 = x & 0x04040404u;
    return ((x ^ 0x03030303u) & ~(n4 | (n4 >> 1) | (n4 >> 2))) | n4;
}

// Read i of the batch into the workspace: forward and reverse-complement bases, forward and reversed qualities
// (Read::finalize, read.h:84-92).  Word-wise: one lane loads a whole read, so byte accesses (404 byte stores and
// 202 byte loads per 101-bp read) made this the most expensive glue state of the kernel.
__device__ __forceinline__ void ht2_load_read(Ht2Read& dst, const DevBatch& b, uint32_t ri, uint32_t& err)
{
    uint64_t o0 = b.offs[ri], o1 = b.offs[ri + 1];
    uint32_t n = (uint32_t)(o1 - o0);
    if (n > HT2_MAX_RDLEN) { err |= HT2_ERR_RDLEN; n = HT2_MAX_RDLEN; }
    dst.len = n;
    const uint8_t* s = b.seq + o0;
    const uint8_t* q = b.qual ? b.qual + o0 : NULL;
    uint32_t* f0 = (uint32_t*)dst.seq[0]; uint32_t* f1 = (uint32_t*)dst.seq[1];
    uint32_t* q0 = (uint32_t*)dst.qual[0]; uint32_t* q1 = (uint32_t*)dst.qual[1];
    for (uint32_t k = 0; k < n; k += 4) {                     // forward strand: words straight through
        f0[k >> 2] = ht2_ld4(s + k);
        q0[k >> 2] = q ? ht2_ld4(q + k) : 0x49494949u;
    }
    uint32_t m = 0;
    for (; m + 4 <= n; m += 4) {                              // reverse strand: bytes [n-4-m, n-m) reversed
        const uint32_t x = __byte_perm(ht2_ld4(s + (n - 4 - m)), 0, 0x0123);
        f1[m >> 2] = ht2_comp4(x);
        q1[m >> 2] = q ? __byte_perm(ht2_ld4(q + (n - 4 - m)), 0, 0x0123) : 0x49494949u;
    }
    for (; m < n; m++) {                                      // the last 1-3 positions = the read's first bases
        const uint8_t c = s[n - 1 - m];
        dst.seq[1][m] = c < 4 ? (uint8_t)(c ^ 3) : (uint8_t)4;
        dst.qual[1][m] = q ? q[n - 1 - m] : (uint8_t)'I';
    }
}

// Per-read filters and minimum score (hisat2.cpp:3387-3440): length filter,
// N filter (Scoring::nFilter, nCeil = L,0,0.15 -- the parseString default, aligner_seed_policy.cpp:293-296), score filter
// (minsc = --score-min(len), default L,0,-0.2, clamped to <= 0 -- hisat2.cpp:441, 3380-3402; the
// function is tabulated per read length on the host, Ht2Params::minscTab).  The N-ceiling product is
// exact in double (24-bit constant x length < 2^9), so host (ht2_host.cpp:ht2_filters) and device agree.
__device__ __forceinline__ bool ht2_dev_filter(const DevBatch& b, uint32_t ri, int64_t& minsc)
{
    const uint64_t o0 = b.offs[ri];
    const uint32_t len = (uint32_t)(b.offs[ri + 1] - o0);
    int64_t m = b.minscTab[len <= HT2_PARAMS_MAX_RDLEN ? len : HT2_PARAMS_MAX_RDLEN];   // --score-min, tabulated on the host (ht2_set_score_min)
    if (m > 0) m = 0;
    minsc = m;
    const uint32_t maxns = (uint32_t)((double)0.0f + (double)0.15f * (double)len);   // nCeil = L,0,0.15 (aligner_seed_policy.cpp:293-296)
    const uint8_t* s = b.seq + o0;
    uint32_t ns = 0;
    for (uint32_t k = 0; k < len; k += 4) {
        uint32_t x = ht2_ld4(s + k);
        if (k + 4 > len) x &= (1u << (8 * (len - k))) - 1u;
        ns += (uint32_t)__popc(x & 0x04040404u);
    }
    return ns <= maxns && len >= 2 && 0 >= m;
}

// Set up workspace W for unit u (one read or one pair): filters, seeds, reads.
// Returns true when there is something to align (machineStart() was called).
template <typename ALIGNER>
__device__ __noinline__ bool ht2_setup_unit(ALIGNER& A, const Ht2ParamsCore& P, const DevBatch& b, uint32_t u, uint32_t& filtBits)
{
    Ht2Work* W = A.W;
    W->err = 0; W->localindexatts = 0; W->maxLocalindexatts = 0; W->nLF = 0; W->nSides = 0; W->algBytes = 0;
    W->maxPool = W->maxDepth = W->maxEdits = 0;
    W->nFrames = 0; W->st = TS_DONE;
    filtBits = 0;
    bool run = false;
    if (!b.paired) {
        const uint32_t ri = u;
        A.paired = false; A.rightendonly = false;
        A.nofw[0] = P.nofw != 0; A.norc[0] = P.norc != 0; A.nofw[1] = true; A.norc[1] = true;
        int64_t ms;
        const bool f0 = ht2_dev_filter(b, ri, ms);
        A.minsc[0] = ms; A.minsc[1] = (int64_t)HT2_IDX_MAX32;
        W->rnd.init(b.seeds[ri]);
        A.sinkReset(false);
        if (f0) {
            filtBits = 1;
            ht2_load_read(W->rd[0], b, ri, W->err);
            run = !W->err;
        }
    } else {
        const uint32_t r1 = 2 * u, r2 = 2 * u + 1;
        int64_t ms1, ms2;
        const bool f1 = ht2_dev_filter(b, r1, ms1), f2 = ht2_dev_filter(b, r2, ms2);
        filtBits = (f1 ? 1u : 0u) | (f2 ? 2u : 0u);
        // nofw/norc per mate (hisat2.cpp:3444-3447)
        A.nofw[0] = P.gMate1fw ? (P.nofw != 0) : (P.norc != 0);
        A.norc[0] = P.gMate1fw ? (P.norc != 0) : (P.nofw != 0);
        A.nofw[1] = P.gMate2fw ? (P.nofw != 0) : (P.norc != 0);
        A.norc[1] = P.gMate2fw ? (P.norc != 0) : (P.nofw != 0);
        W->rnd.init((f1 && f2) ? (b.seeds[r1] ^ b.seeds[r2]) : b.seeds[r1]);
        A.sinkReset(true);
        if (f1 && f2) {
            A.paired = true; A.rightendonly = false;
            A.minsc[0] = ms1; A.minsc[1] = ms2;
            ht2_load_read(W->rd[0], b, r1, W->err);
            ht2_load_read(W->rd[1], b, r2, W->err);
            run = !W->err;
        } else if (f1 || f2) {
            A.paired = false; A.rightendonly = !f1;
            uint32_t rr = f1 ? r1 : r2;
            uint32_t m = f1 ? 0 : 1;
            bool nf = A.nofw[m], nr = A.norc[m];
            A.nofw[0] = nf; A.norc[0] = nr; A.nofw[1] = true; A.norc[1] = true;
            A.minsc[0] = f1 ? ms1 : ms2; A.minsc[1] = (int64_t)HT2_IDX_MAX32;
            ht2_load_read(W->rd[0], b, rr, W->err);
            run = !W->err;
        }
    }
    W->unit = u; W->filtBits = filtBits;
    A.saveCfg();
    if (run) A.machineStart();
    return run;
}

// Append unit u's alignments to the batch result pools.
template <int LANES>
__device__ __noinline__ void ht2_finish_unit(Ht2Work* W, const DevOut& o, uint32_t u, uint32_t filtBits, uint32_t lane)
{
    ht2gpu_read_result_t rr;
    rr.n_aln[0] = (uint16_t)W->nRes[0];
    rr.n_aln[1] = (uint16_t)W->nRes[1];
    rr.n_pairs = W->nPairs;
    rr.rng_state = W->rnd.last;
    rr.n_lf = W->nLF;
    rr.alg_bytes = W->algBytes;
    rr.filt = filtBits;
    uint32_t nal = W->nRes[0] + W->nRes[1];
    uint32_t ned = 0;
    for (uint32_t m = 0; m < 2; m++)
        for (uint32_t i = 0; i < W->nRes[m]; i++) ned += W->res[m][i].nedits;
    uint32_t aoff = 0, eoff = 0, poff = 0;
    if (lane == 0) {
        aoff = nal ? atomicAdd(&o.counters[0], nal) : 0;
        eoff = ned ? atomicAdd(&o.counters[1], ned) : 0;
        poff = W->nPairs ? atomicAdd(&o.counters[2], W->nPairs) : 0;
    }
    if (LANES > 1) {
        aoff = __shfl_sync(0xffffffffu, aoff, 0);
        eoff = __shfl_sync(0xffffffffu, eoff, 0);
        poff = __shfl_sync(0xffffffffu, poff, 0);
    }
    if (aoff + nal > o.capAlns || eoff + ned > o.capEdits || poff + W->nPairs > o.capPairs) {
        W->err |= HT2_ERR_OUTPUT;
        rr.n_aln[0] = rr.n_aln[1] = 0; rr.n_pairs = 0;
    } else if (lane == 0) {
        uint32_t a = aoff, e = eoff;
        for (uint32_t m = 0; m < 2; m++) {
            for (uint32_t i = 0; i < W->nRes[m]; i++) {
                const Ht2Res& r = W->res[m][i];
                ht2gpu_aln_t& d = o.alns[a++];
                d.tidx = r.tidx; d.toff = r.toff; d.score = (int32_t)r.score;
                d.fw = (uint8_t)r.fw; d.mate = (uint8_t)m; d.n_edits = (uint16_t)r.nedits;
                d.trim5 = (uint16_t)r.trim5p; d.trim3 = (uint16_t)r.trim3p;
                d.ref_extent = r.rfextent; d.edit_off = e;
                const Ht2Edit* red = W->resEdits + r.editOff;
                for (uint32_t k = 0; k < r.nedits; k++) {
                    ht2gpu_edit_t& de = o.edits[e++];
                    de.pos = red[k].pos; de.chr = red[k].chr; de.qchr = red[k].qchr;
                    de.type = red[k].type; de.pad = red[k].pad; de.snp_id = red[k].snpID;
                }
            }
        }
        for (uint32_t i = 0; i < W->nPairs; i++) {
            o.pairs[2 * (poff + i)] = W->pairs[i][0];
            o.pairs[2 * (poff + i) + 1] = W->pairs[i][1];
        }
    }
    rr.aln_off = aoff;
    rr.pair_off = poff;
    rr.err = W->err;
    if (lane == 0) o.reads[u] = rr;
}

// Slot state codes of the pool kernel: what a read slot has to do next.
#define RG_NEED 0u         /* empty: draw the next read */
#define RG_FINISH 1u       /* machine done: append the results */
#define RG_TOP 2u          /* + TS_* (top-level state of go()) */
#define RG_FRAME 20u       /* + F_*  (state of the innermost hybridSearch_recur frame) */
#define RG_EXIT 255u
#define RG_BINS 64

__device__ __forceinline__ uint32_t rg_code(const Ht2Work* W)
{
    if (W->nFrames > 0) return RG_FRAME + W->frames[W->nFrames - 1].pc;
    if (W->st == TS_DONE) return RG_FINISH;
    return RG_TOP + W->st;
}

// A round of DP problems (--bowtie2-dp): every lane with a slot (my >= 0: base + my) frames its own rectangle, then the WARP
// fills the score planes of one problem after the other (ht2_sw.h swFillCoop: a 64-row vector per column instead of
// a lone lane's 2), and the lanes go back to their own candidates / backtraces (swExtendAnchor -> swFinish).  Run by
// the pool kernel and by ht2gpu_sw_extend's harness; all 32 lanes must call it.
template <bool GRAPH, bool NOSPL>
__device__ __forceinline__ void ht2_dp_round(Ht2AlignerT<GRAPH, NOSPL>& A, Ht2Work* base, int my, uint32_t lane)
{
    bool fill = false;
    if (my >= 0) {
        Ht2Work* W = base + my;
        A.attach(W);
        bool ret;
        fill = A.swPrepare(W->curRdi, W->genomeHits[W->hybHj], ret);
        A.swStage = fill ? 1u : 2u; A.swRetv = ret;
    }
    __syncwarp();
    uint32_t m = __ballot_sync(0xffffffffu, fill);
    while (m) {
        const int k = __ffs((int)m) - 1;
        m &= m - 1;
        Ht2SwScratch* Sk = (Ht2SwScratch*)__shfl_sync(0xffffffffu, (unsigned long long)A.sw, k);
        uint32_t* pk = (uint32_t*)__shfl_sync(0xffffffffu, (unsigned long long)A.swPl, k);
        A.swFillCoop(Sk, pk, lane);
    }
    __syncwarp();
}

// ---------------------------------------------------------------------------
// ht2_align_pool_kernel: block-shared slot pool, warp-independent rounds, lock-free claims.
//
// The NW warps of a block share one pool of NW*32*K read slots.  What a slot has to do next (its state code)
// is kept as one BIT PER SLOT in a per-state bitmap in shared memory (a slot that is being run is in no bitmap).
// Every warp runs its own rounds: pick the block's target state, claim up to 32 of its slots straight out of the
// bitmap (lane w reads word w, a warp prefix sum decides how many bits each lane may take, atomicAnd takes them,
// the returned old word tells which ones were really won), run one segment of each claimed slot on its 32 lanes,
// and publish the new states with atomicOr.  No lock, no scan over the slot array, no waiting for another warp's
// segments (round 1 serialised the gather under a block lock: 20 % of all executed instructions were warps
// spinning on it).  The target state is a block-wide hint: warps stay on it while it has
// plenty of claimable slots and otherwise re-elect the most populous state from per-state counters, so the warps
// of an SM execute the same code most of the time (instruction fetch is the scarce resource: the L1.5 I-cache and
// the GPC instruction cache saturate when every warp walks different code) while groups are drawn from a pool
// large enough to fill all 32 lanes.
// ---------------------------------------------------------------------------
template <int NW, int K, bool GRAPH, bool NOSPL>
__global__ void __launch_bounds__(32 * NW)
ht2_align_pool_kernel(const uint8_t* __restrict__ blob, Ht2ParamsCore P, DevBatch b, DevOut o, Ht2Work* work)
{
    constexpr int S = NW * 32 * K;      // slots of this block
    constexpr int NWORD = S / 32;       // bitmap words per state; lane w owns word w during a gather
    static_assert(NWORD <= 32, "one bitmap word per lane");
    __shared__ unsigned int sBits[RG_BINS][NWORD];
    __shared__ int sCount[RG_BINS];     // claimable slots per state code (a hint: updated after the bitmaps)
    __shared__ unsigned int sTarget;
    __shared__ int sExit;
    __shared__ uint16_t sSel[NW][32];
    const uint32_t t = threadIdx.x, lane = t & 31, wib = t >> 5;
    Ht2Work* base = work + (size_t)blockIdx.x * S;
    for (int i = t; i < RG_BINS * NWORD; i += 32 * NW) sBits[i / NWORD][i % NWORD] = (i / NWORD == (int)RG_NEED) ? 0xffffffffu : 0u;
    if (t < RG_BINS) sCount[t] = (t == RG_NEED) ? S : 0;
    if (t == 0) { sTarget = RG_NEED; sExit = 0; }
    Ht2AlignerT<GRAPH, NOSPL> A;
    A.bind(blob, &P, base);
    A.sw = b.sw ? b.sw + ((size_t)blockIdx.x * blockDim.x + threadIdx.x) : NULL;
    A.swPl = b.swPool ? b.swPool + ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * (size_t)HT2_SW_POOL_WORDS : NULL;
    A.swStride = 1;
#ifdef HT2_ENABLE_SPLICED
    A.splT = b.splT; A.ssT = b.ssT;
#endif
    __syncthreads();
    volatile int* vCount = sCount;
    uint16_t* sel = sSel[wib];
    uint32_t rot = wib * (NWORD / NW > 0 ? NWORD / NW : 1);   // warps start their scans at different words
    for (;;) {
        // ---- nothing claimable at all (every remaining slot is being run by another warp, or the batch has
        // drained): wait -- spinning warps cost instruction fetch
        uint32_t T;
        {
            int c0 = vCount[lane], c1 = vCount[lane + 32];
            if (__ballot_sync(0xffffffffu, c0 > 0 || c1 > 0) == 0) {
                const bool done = __shfl_sync(0xffffffffu, *(volatile int*)&sExit >= S ? 1 : 0, 0) != 0;
                if (done) break;
                __nanosleep(1000);
                continue;
            }
            // every decision below is made warp-uniform (the counters change under our feet)
            T = __shfl_sync(0xffffffffu, *(volatile unsigned int*)&sTarget, 0);
            const int cT = __shfl_sync(0xffffffffu, vCount[T], 0);
            if (cT < (int)b.elect) {
                // elect the most populous claimable state
                if (c0 < 0) c0 = 0;
                if (c1 < 0) c1 = 0;
                uint32_t best = c0 >= c1 ? (((uint32_t)c0 << 8) | lane) : (((uint32_t)c1 << 8) | (lane + 32));
                for (int off = 16; off > 0; off >>= 1) { uint32_t v = __shfl_xor_sync(0xffffffffu, best, off); best = v > best ? v : best; }
                if ((best >> 8) == 0) { __nanosleep(200); continue; }
                T = best & 0xff;
                if (lane == 0) *(volatile unsigned int*)&sTarget = T;
            }
        }
        // ---- claim up to 32 slots in state T out of its bitmap
        uint32_t nsel;
        {
            const uint32_t w = (lane + rot) & (NWORD - 1);
            const bool mine = lane < (uint32_t)NWORD;
            const uint32_t word = mine ? *(volatile unsigned int*)&sBits[T][w] : 0u;
            const uint32_t c = (uint32_t)__popc(word);
            uint32_t incl = c;
            for (int off = 1; off < 32; off <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, incl, off); if ((int)lane >= off) incl += v; }
            const uint32_t before = incl - c;
            const uint32_t want = before >= 32u ? 0u : (c < 32u - before ? c : 32u - before);
            uint32_t got = 0;
            if (want) {
                const uint32_t last = __fns(word, 0, (int)want);            // position of the want-th set bit
                const uint32_t mask = word & (0xffffffffu >> (31u - last));
                got = atomicAnd(&sBits[T][w], ~mask) & mask;                  // the bits this lane really won
            }
            const uint32_t g = (uint32_t)__popc(got);
            uint32_t gi = g;
            for (int off = 1; off < 32; off <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, gi, off); if ((int)lane >= off) gi += v; }
            nsel = __shfl_sync(0xffffffffu, gi, 31);
            uint32_t r = gi - g;
            while (got) { const uint32_t bpos = (uint32_t)__ffs((int)got) - 1u; sel[r++] = (uint16_t)(w * 32u + bpos); got &= got - 1u; }
            if (lane == 0 && nsel) atomicSub(&sCount[T], (int)nsel);
            rot += 5;
        }
        __syncwarp();
        if (nsel == 0) continue;        // another warp took them first, or the counter was ahead of the bitmap
        const int my = lane < nsel ? (int)sel[lane] : -1;
        if (my >= 0) {   // the slot's scalars (first three lines of Ht2Work) are cold by now: fetch them side by side, not one after the other
            const char* wp = (const char*)(base + my);
            asm volatile("prefetch.global.L2 [%0];" :: "l"(wp));
            asm volatile("prefetch.global.L2 [%0];" :: "l"(wp + 128));
            asm volatile("prefetch.global.L2 [%0];" :: "l"(wp + 256));
        }
        __threadfence_block();   // acquire: the previous owner's workspace writes
        const long long t0 = o.stats ? clock64() : 0;
#ifndef HT2_NO_DP
        if (T == RG_TOP + TS_HYB_DP) ht2_dp_round(A, base, my, lane);
#endif
        if (my >= 0) {
            Ht2Work* W = base + my;
            uint32_t nc;
            if (T == RG_NEED) {
                uint32_t u = atomicAdd(&o.counters[3], 1u);
                if (u >= b.n_units) nc = RG_EXIT;
                else {
                    A.W = W;
                    uint32_t filtBits;
                    bool run = ht2_setup_unit(A, P, b, u, filtBits);
                    if (run) { while (!A.machineAtHeavyState()) A.machineStep(); }
                    nc = run ? rg_code(W) : RG_FINISH;
                }
            } else if (T == RG_FINISH) {
                ht2_finish_unit<1>(W, o, W->unit, W->filtBits, 0);
                nc = RG_NEED;
            } else {
                A.attach(W);
                A.machineRun();
                nc = rg_code(W);
            }
            __threadfence_block();   // release
            if (nc == RG_EXIT) atomicAdd(&sExit, 1);
            else { atomicOr(&sBits[nc][my >> 5], 1u << (my & 31)); atomicAdd(&sCount[nc], 1); }
        }
        __syncwarp();
        if (o.stats && lane == 0) {
            const unsigned long long dt = (unsigned long long)(clock64() - t0);
            atomicAdd(&o.stats[T * 4 + 0], 1ull);
            atomicAdd(&o.stats[T * 4 + 1], (unsigned long long)nsel);
            atomicAdd(&o.stats[T * 4 + 2], dt);
            atomicMax(&o.stats[T * 4 + 3], dt);
            const uint32_t bk = nsel >= 32 ? 5 : (nsel >= 16 ? 4 : (nsel >= 8 ? 3 : (nsel >= 4 ? 2 : (nsel >= 2 ? 1 : 0))));
            atomicAdd(&o.stats[1024 + (T * 6 + bk) * 2 + 0], 1ull);
            atomicAdd(&o.stats[1024 + (T * 6 + bk) * 2 + 1], dt);
        }
    }
}

// ---------------------------------------------------------------------------
// ht2_seed_kernel: the seed search on its own (ht2_seed.h), one lane per read,
// two passes (count, then fill at host-computed offsets) so that the output is
// laid out per read without a worst-case allocation.
// ---------------------------------------------------------------------------
struct SeedOut {
    uint32_t*            counts;     // [n][3] hits, iedges, coords            (pass 0 out)
    const uint32_t*      offs;       // [n][3] exclusive prefix of counts       (pass 1 in)
    ht2gpu_seed_hit_t*   hits;
    uint16_t*            iedges;
    ht2gpu_seed_coord_t* coords;
    unsigned long long*  totals;     // [0] nLF, [1] algBytes, [2] reads with errors
};

template <bool GRAPH, bool FILL>
__global__ void __launch_bounds__(128)
ht2_seed_kernel(const uint8_t* __restrict__ blob, Ht2ParamsCore P, DevBatch b, uint32_t nReads, uint32_t maxRange, SeedOut o)
{
    const Ht2ImageHeader* H = (const Ht2ImageHeader*)blob;
    Ht2Fm<uint32_t> fm;
    fm.init(blob, &H->global);
    const uint32_t nFrag = H->global.nFrag;
    for (uint32_t ri = blockIdx.x * blockDim.x + threadIdx.x; ri < nReads; ri += gridDim.x * blockDim.x) {
        const uint64_t o0 = b.offs[ri];
        uint32_t len = (uint32_t)(b.offs[ri + 1] - o0);
        Ht2SeedState st;
        st.err = 0; st.nLF = 0; st.algBytes = 0;
        if (len > HT2_MAX_RDLEN) { st.err = 2; len = 0; }
        uint8_t rc[HT2_MAX_RDLEN];
        const uint8_t* fwseq = b.seq + o0;
        for (uint32_t i = 0; i < len; i++) { const uint8_t c = fwseq[len - 1 - i]; rc[i] = c < 4 ? (uint8_t)(c ^ 3) : (uint8_t)4; }
        uint32_t nh = 0, ne = 0, nc = 0;
        uint32_t bh = 0, be = 0, bc = 0;
        if (FILL) { bh = o.offs[3 * ri]; be = o.offs[3 * ri + 1]; bc = o.offs[3 * ri + 2]; }
        for (int fwi = 0; fwi < 2 && len > 0; fwi++) {
            const uint8_t* seq = fwi == 0 ? fwseq : rc;
            st.len = len; st.cur = 0; st.done = 0; st.numPartialSearch = 0; st.numUniqueSearch = 0;
            while (!st.done) {
                Ht2SeedHit ph;
                bool pseudogeneStop = !GRAPH && !P.noSplicedAlignment, anchorStop = true;   // hi_aligner.h:4669-4670
                ht2_seed_partial<GRAPH>(fm, P, seq, st, ph, pseudogeneStop, anchorStop);
                const bool blank = ph.top == HT2_IDX_MAX32;
                const uint32_t nelt = blank ? 0u : ph.node_bot - ph.node_top;
                const uint32_t ncoord = (!blank && nelt <= maxRange) ? nelt : 0u;
                if (FILL) {
                    ht2gpu_seed_hit_t& out = o.hits[bh + nh];
                    out.read = ri; out.fw = fwi == 0; out.hit_type = ph.hit_type;
                    out.pseudogene_stop = ph.pseudogeneStop; out.anchor_stop = ph.anchorStop;
                    out.bwoff = ph.bwoff; out.len = ph.len; out.top = ph.top; out.bot = ph.bot;
                    out.node_top = ph.node_top; out.node_bot = ph.node_bot;
                    out.n_iedges = ph.niedges; out.iedge_off = be + ne;
                    out.n_coords = ncoord; out.coord_off = bc + nc;
                    for (uint32_t e = 0; e < ph.niedges; e++) {
                        o.iedges[2 * (size_t)(be + ne + e)] = ph.iedges[e][0];
                        o.iedges[2 * (size_t)(be + ne + e) + 1] = ph.iedges[e][1];
                    }
                    for (uint32_t i = 0; i < ncoord; i++) {
                        uint32_t row;
                        const uint32_t joff = ht2_seed_elt_offset<GRAPH>(fm, ph, i, row, st);
                        ht2gpu_seed_coord_t& cc = o.coords[bc + nc + i];
                        cc.row = row; cc.joined_off = joff; cc.tidx = HT2_IDX_MAX32; cc.toff = 0;
                        // GFM::joinedToTextOff, rejectStraddle = false (gfm.h:5527-5600)
                        uint32_t lo = 0, hi = nFrag, elt = HT2_IDX_MAX32;
                        while (true) {
                            const uint32_t old = elt;
                            elt = lo + ((hi - lo) >> 1);
                            if (old == elt) break;
                            const uint32_t lower = fm.rstarts[elt * 3];
                            const uint32_t upper = (elt == nFrag - 1) ? fm.g->len : fm.rstarts[(elt + 1) * 3];
                            if (lower <= joff) {
                                if (upper > joff) { cc.tidx = fm.rstarts[elt * 3 + 1]; cc.toff = joff - lower + fm.rstarts[elt * 3 + 2]; break; }
                                lo = elt;
                            } else hi = elt;
                        }
                    }
                }
                nh++; ne += ph.niedges; nc += ncoord;
                if (st.done) break;
                if (!pseudogeneStop) { if (st.cur + 1 < st.len) st.cur++; }
            }
        }
        if (!FILL) { o.counts[3 * ri] = nh; o.counts[3 * ri + 1] = ne; o.counts[3 * ri + 2] = nc; }
        else {
            atomicAdd(&o.totals[0], (unsigned long long)st.nLF);
            atomicAdd(&o.totals[1], (unsigned long long)st.algBytes);
            if (st.err) atomicAdd(&o.totals[2], 1ull);
        }
    }
}

// ---------------------------------------------------------------------------
// The SAM back end on the device (ht2_sam.h).  One thread formats one unit (read or pair):
//   ht2_sam_kernel<false> : counting pass -- bytes of SAM text per unit (lens) and per block (blk)
//   ht2_sam_scan_kernel   : exclusive scan of the block sums (one block), blk[nBlk] = total
//   ht2_sam_kernel<true>  : writing pass -- unit offset = block offset + in-block exclusive scan of lens
// Records land in read order (= --reorder), exactly the bytes AlnSinkWrap::finishRead prints.
//
// The block's units fill one contiguous byte range of the output, [blk[b], blk[b+1]).  The writing pass formats
// them into shared memory at their in-block offsets and then copies the range out with aligned 16-byte stores:
// one thread's text is a few hundred bytes long, so byte stores straight to global memory would have every store
// instruction touch 32 different sectors.  A block whose text does not fit the staging buffer (many multi-mapping
// records, long reads) formats straight into global memory; the bytes are the same either way.
// ---------------------------------------------------------------------------
#define HT2_SAM_TPB 128
#define HT2_SAM_STAGE_BLOCKS 2     // writing-pass blocks per SM the staging buffer leaves room for

template <bool WRITE>
__global__ void __launch_bounds__(HT2_SAM_TPB)
ht2_sam_kernel(Ht2SamIn in, uint32_t units, uint32_t* __restrict__ lens, unsigned long long* __restrict__ blk, char* __restrict__ out,
               unsigned long long cap, unsigned int* counters, unsigned long long* __restrict__ tally, uint32_t stageBytes)
{
    extern __shared__ uint4 sStage[];   // writing pass: stageBytes of dynamic shared memory
    __shared__ unsigned long long sWarp[HT2_SAM_TPB / 32];
    __shared__ uint32_t sTally[HT2_SAM_TPB / 32][HT2_T_N];
    const uint32_t u = blockIdx.x * HT2_SAM_TPB + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    Ht2SamFmt F;
    F.bind(&in);
    unsigned long long mine = 0;
    if (!WRITE) {
        Ht2SamTally t;
#pragma unroll
        for (int k = 0; k < HT2_T_N; k++) t.c[k] = 0;
        if (u < units) {
            Ht2SamOut<false> o; o.p = NULL; o.n = 0;
            F.unit(o, u, &t);
            mine = o.n;
            lens[u] = (uint32_t)o.n;
            if (in.reads[u].err) atomicAdd(&counters[4], 1u);
        }
        // ReportingMetrics of the block: warp sums, then one 64-bit atomic per counter per block
#pragma unroll
        for (int k = 0; k < HT2_T_N; k++) {
            const uint32_t s = __reduce_add_sync(0xffffffffu, t.c[k]);
            if (lane == 0) sTally[wib][k] = s;
        }
        __syncthreads();
        if (threadIdx.x < HT2_T_N) {
            unsigned long long s = 0;
            for (int w = 0; w < HT2_SAM_TPB / 32; w++) s += sTally[w][threadIdx.x];
            if (s) atomicAdd(&tally[threadIdx.x], s);
        }
    } else mine = u < units ? lens[u] : 0;
    // inclusive warp scan, then across the block's warps
    unsigned long long incl = mine;
    for (int off = 1; off < 32; off <<= 1) { const unsigned long long v = __shfl_up_sync(0xffffffffu, incl, off); if ((int)lane >= off) incl += v; }
    if (lane == 31) sWarp[wib] = incl;
    __syncthreads();
    unsigned long long base = 0;
    for (uint32_t w = 0; w < wib; w++) base += sWarp[w];
    if (!WRITE) {
        if (threadIdx.x == HT2_SAM_TPB - 1) blk[blockIdx.x] = base + incl;
        return;
    }
    // the staging buffer starts at the 16-byte boundary at or below the block's first output byte
    const unsigned long long b0 = blk[blockIdx.x], b1 = blk[blockIdx.x + 1];
    const uint32_t head = (uint32_t)(b0 & 15);
    const bool staged = b1 <= cap && b1 - b0 + head <= stageBytes;   // the same for the whole block
    char* const stage = (char*)sStage;
    if (u < units) {
        const unsigned long long at = base + incl - mine;   // in the block
        Ht2SamOut<true> o; o.n = 0;
        o.p = staged ? stage + head + at : out + b0 + at;
        if (staged || b0 + at + mine <= cap) F.unit(o, u);   // one call site: the formatter is inlined once
    }
    if (!staged) return;
    __syncthreads();
    char* const dst = out + (b0 - head);   // out is 16-byte aligned (cudaMalloc)
    const uint32_t end = head + (uint32_t)(b1 - b0);
    for (uint32_t lo = threadIdx.x * 16; lo < end; lo += HT2_SAM_TPB * 16) {
        if (lo >= head && lo + 16 <= end) *(uint4*)(dst + lo) = sStage[lo / 16];
        else for (uint32_t i = lo < head ? head : lo; i < end && i < lo + 16; i++) dst[i] = stage[i];
    }
}

__global__ void __launch_bounds__(1024)
ht2_sam_scan_kernel(unsigned long long* blk, uint32_t nBlk)
{
    __shared__ unsigned long long sPart[1024];
    const uint32_t t = threadIdx.x;
    const uint32_t per = (nBlk + 1023) / 1024;
    const uint32_t lo = t * per, hi = lo + per < nBlk ? lo + per : nBlk;
    unsigned long long sum = 0;
    for (uint32_t i = lo; i < hi; i++) sum += blk[i];
    sPart[t] = sum;
    __syncthreads();
    if (t == 0) { unsigned long long acc = 0; for (int i = 0; i < 1024; i++) { const unsigned long long v = sPart[i]; sPart[i] = acc; acc += v; } blk[nBlk] = acc; }
    __syncthreads();
    unsigned long long acc = sPart[t];
    for (uint32_t i = lo; i < hi; i++) { const unsigned long long v = blk[i]; blk[i] = acc; acc += v; }
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
// One in-flight batch of the SAM path (ht2gpu_submit_sam / ht2gpu_wait_sam): its own stream, device input
// buffers, device result pools, device SAM text and pinned host output, so that the H2D copy of batch i+1 and
// the D2H copy of batch i-1 overlap the kernels of batch i.  The alignment workspaces (dWork) are shared by all
// slots: kernels of different slots are chained through the device's WorkPool.
#define HT2GPU_N_SLOTS 3
#define HT2_META_TALLY 16
// device memory a handle leaves free beside its workspace pool: slot buffers of 4 M-read batches, the per-thread
// stack of the pool kernel, and headroom for other work on the device
#define HT2_MEM_RESERVE ((size_t)10 << 30)
struct SamSlot {
    bool         init;
    cudaStream_t stream;
    cudaEvent_t  ev[6];            // start, h2d done, kernel start, align done, sam done, d2h done
    cudaEvent_t  evSplit[3];       // HT2GPU_SAM_SPLIT=1: before the counting pass, after it, after the block scan
    uint8_t *dSeq, *dQual; uint64_t* dOffs; uint32_t* dSeeds; char* dNames; uint32_t* dNameOffs;
    size_t capSeq, capQual, capOffs, capSeeds, capNames, capNameOffs;
    ht2gpu_read_result_t* dReads; ht2gpu_aln_t* dAlns; ht2gpu_edit_t* dEdits; uint16_t* dPairs; unsigned int* dCounters;
    size_t capUnits, capAlns, capEdits, capPairs;
    uint32_t* dSamLen; size_t capSamLen;          // bytes of SAM text per unit
    unsigned long long* dBlk; size_t capBlk;      // per-block sums, then exclusive block offsets; [nBlk] = total
    char* dSam; size_t capSam;
    Ht2SsRec* dColRecs; size_t capCol;            // --novel-splicesite-outfile: junction records of the batch (count in dCounters[6])
    unsigned long long* dTally;                   // ReportingMetrics of the batch (HT2_T_N counters, ht2_sam.h), zeroed per SAM pass
    uint8_t* dOut; size_t capOut;                 // ht2gpu_record_outcomes: one HT2GPU_OUTCOME_* byte per unit (counting pass)
    uint8_t* hOut; size_t capHOut;                // ... copied back with the meta (pinned)
    bool outValid;                                // hOut holds the outcomes of the batch the last ht2gpu_wait_sam returned
    char* hSam; size_t capHSam;                   // pinned
    unsigned long long* hMeta;                    // pinned: [0] total SAM bytes, [1..4] result counters, [5] reads with errors,
                                                  //         [HT2_META_TALLY ..] the batch's ReportingMetrics
    // the submitted batch (for a re-run after a pool overflow)
    ht2gpu_read_batch_t batch; uint32_t units; size_t namesBytes; uint64_t h2dBytes; uint32_t nLaunch;
    bool pending;
};

// Alignment workspaces are a property of the DEVICE, not of an index handle: every handle of the process that runs
// the same launch geometry on a device shares one WorkPool (a test process opens a dozen handles; 38 GB each would
// not fit).  Kernels that use the workspace are chained through evDone.  (Round 2 also tried two workspaces with
// the next batch's kernel released by the previous kernel's tail flag -- cuStreamWaitValue32 -- so that the drain
// of one batch overlaps the start of the next: no gain, DESIGN.md 4.1; removed.)
struct WorkPool {
    int            device;
    size_t         nWork;
    Ht2Work*       dWork;
    cudaEvent_t    evDone;        // recorded after the latest kernels of a batch (alignment + SAM)
    Ht2SwScratch*  dSw;           // --bowtie2-dp scratch per launched thread (allocated on first use)
    uint32_t*      dSwPool;
    size_t         swThreads;     // launched threads dSw / dSwPool hold: geometries of equal nWork differ in grid size
    std::mutex     mu;            // [wait, launches, record] of one batch are one critical section
    int            refs;
};
static std::mutex gPoolMu;
static std::vector<WorkPool*> gPools;

struct ht2gpu_handle {
    WorkPool*      pool;
    Ht2Image*      img;        // host copy (may hold only the header prefix when adopting a device image)
    uint8_t*       dBlob;
    bool           ownBlob;
    size_t         blobBytes;
    Ht2Params      P;
    ht2gpu_options_t opt;
    int            device;
    int            nSM;
    int            tpb, bpsm;
    uint32_t       samStage;  // bytes of the SAM writing pass's staging buffer (dynamic shared memory per block)
    bool           graph;
    int            poolWarps;
    int            rgK;
    int32_t*       dMinsc;   // --score-min table on the device (Ht2Params::minscTab)
    void*          dSplT;    // spliced builds: Ht2SplTables on the device
    uint8_t*       dSsT;     // the run's splice-site DB on the device (ht2gpu_load_splicesites) or NULL
    bool           collectSs; // --novel-splicesite-outfile: collect the junctions of printed alignments
    bool           recordOut; // ht2gpu_record_outcomes: the SAM counting pass stores each unit's outcome byte
    Ht2NovelSites  novel;     // ... aggregated here (ht2gpu_wait_sam), written by ht2gpu_write_novel_splicesites
    std::mutex     novelMu;
    std::vector<uint8_t> ssBlob;   // ... and its host copy (host formatter)
    Ht2SamOutput   samOut;    // SAM output settings (ht2gpu_set_sam_output)
    char*          dRgTag;    // ... its "RG:Z:<id>" on the device, or NULL
    ht2gpu_align_counts_t counts;   // ReportingMetrics of every batch ht2gpu_wait_sam returned (ht2gpu_align_counts)
    std::mutex     countMu;
    size_t         nWork;
    cudaStream_t   stream;
    cudaEvent_t    ev[4];
    std::string    err;
    unsigned long long* dStats;   // HT2GPU_STATS=1: per-state round statistics of the pool kernel
    SamSlot        slots[HT2GPU_N_SLOTS];
    void*          pipeCtx;       // ht2_pipeline.cpp's per-handle context
    void         (*pipeCtxFree)(void*);
};

// Results live in ONE pinned host buffer per batch (D2H at PCIe speed instead of
// the pageable-copy path); freed buffers are cached process-wide because
// cudaHostAlloc costs milliseconds per hundred MB.
struct ResPriv {
    void*  buf;
    size_t cap;
};
static std::mutex gPinMu;
static std::vector<ResPriv> gPinFree;

static bool pinnedGet(size_t need, ResPriv& out)
{
    {
        std::lock_guard<std::mutex> lk(gPinMu);
        int best = -1;
        for (size_t i = 0; i < gPinFree.size(); i++)
            if (gPinFree[i].cap >= need && (best < 0 || gPinFree[i].cap < gPinFree[best].cap)) best = (int)i;
        if (best >= 0) { out = gPinFree[best]; gPinFree.erase(gPinFree.begin() + best); return true; }
    }
    size_t cap = need + need / 4 + 4096;
    void* p = NULL;
    if (cudaHostAlloc(&p, cap, cudaHostAllocPortable) != cudaSuccess) return false;
    out.buf = p; out.cap = cap;
    return true;
}
static void pinnedPut(const ResPriv& r)
{
    std::lock_guard<std::mutex> lk(gPinMu);
    if (gPinFree.size() >= 4) {     // keep the largest few
        size_t mi = 0;
        for (size_t i = 1; i < gPinFree.size(); i++) if (gPinFree[i].cap < gPinFree[mi].cap) mi = i;
        if (gPinFree[mi].cap < r.cap) { cudaFreeHost(gPinFree[mi].buf); gPinFree[mi] = r; }
        else cudaFreeHost(r.buf);
        return;
    }
    gPinFree.push_back(r);
}

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { h->err = std::string(#call) + ": " + cudaGetErrorString(e_); return HT2GPU_ERR_CUDA; } } while (0)

extern "C" void ht2gpu_default_options(ht2gpu_options_t* o)
{
    memset(o, 0, sizeof(*o));
    o->device = 0;
    o->no_spliced_alignment = 1;
    o->mp_max = 6; o->mp_min = 2; o->sp_max = 2; o->sp_min = 1; o->np = 1;
    o->rdg_const = 5; o->rdg_linear = 3; o->rfg_const = 5; o->rfg_linear = 3;
    o->min_frag = 0; o->max_frag = 1000;
    o->bowtie2_dp = 0; o->gbar = 4;
    o->score_min_type = 'L'; o->score_min_const = (double)0.0f; o->score_min_coeff = (double)-0.2f;   // hisat2.cpp:441
}

static void applyOptions(Ht2Params& P, const Ht2Image& img, const ht2gpu_options_t& o)
{
    ht2_default_params(P, img, o.no_spliced_alignment != 0);
    if (o.khits > 0) P.khits = (uint32_t)o.khits;
    P.kseeds = o.max_seeds > 0 ? (uint32_t)o.max_seeds : (P.khits * 2 > 5 ? P.khits * 2 : 5);
    P.secondary = o.secondary ? 1 : 0;
    P.mmpMax = o.mp_max; P.mmpMin = o.mp_min; P.scpMax = o.sp_max; P.scpMin = o.sp_min; P.npen = o.np;
    P.rdGapConst = o.rdg_const; P.rdGapLinear = o.rdg_linear; P.rfGapConst = o.rfg_const; P.rfGapLinear = o.rfg_linear;
    P.mmcostConstant = o.ignore_quals ? 1 : 0;
    P.nofw = o.nofw ? 1 : 0; P.norc = o.norc ? 1 : 0;
    P.minFrag = (uint32_t)o.min_frag; P.maxFrag = (uint32_t)o.max_frag;
    P.mixed = o.no_mixed ? 0 : 1; P.discord = o.no_discordant ? 0 : 1;
    P.bowtie2Dp = (uint32_t)o.bowtie2_dp; P.gapbar = o.gbar < 1 ? 1 : o.gbar;   // hisat2.cpp:1969-1973
    if (o.score_min_type != 0) ht2_set_score_min(P, (char)o.score_min_type, o.score_min_const, o.score_min_coeff);
}

static int finishOpen(ht2gpu_handle* h)
{
    const Ht2ImageHeader* H = h->img->header();
    if (H->magic != HT2_MAGIC || H->version != HT2_IMAGE_VERSION) { h->err = "bad index image"; return HT2GPU_ERR_INDEX; }
    if (H->totalBytes != h->blobBytes) { h->err = "index image is truncated (header.totalBytes differs from the bytes given)"; return HT2GPU_ERR_INDEX; }
#ifndef HT2_ENABLE_SPLICED
    if (!h->opt.no_spliced_alignment) { h->err = "spliced alignment is not implemented in this build; pass --no-spliced-alignment"; return HT2GPU_ERR_UNSUPPORTED; }
#else
    // spliced mode (the default build; HT2_NO_SPLICED=1 leaves it out) == the reference's --no-temp-splicesite: the
    // splice-site DB holds only the sites loaded with ht2gpu_load_splicesites, never junctions of earlier reads
    if (!h->opt.no_spliced_alignment) {
        const Ht2SplTables& T = ht2_spl_tables();
        CK(cudaMalloc(&h->dSplT, sizeof(Ht2SplTables)));
        CK(cudaMemcpy(h->dSplT, &T, sizeof(Ht2SplTables), cudaMemcpyHostToDevice));
    }
#endif
    h->graph = !H->global.linearFM;   // graph (SNP) indexes: ALT-aware aligner instantiation, graph seed kernel
    applyOptions(h->P, *h->img, h->opt);
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, h->device));
    h->nSM = prop.multiProcessorCount;
    // the pool kernel: one block of poolWarps warps per SM, rgK read slots per lane (DESIGN.md 4)
    h->poolWarps = (h->opt.threads_per_block == 128 && !h->graph) ? 4 : 8;
    h->tpb = 32 * h->poolWarps;
    h->bpsm = (h->opt.blocks_per_sm > 0 && !h->graph) ? h->opt.blocks_per_sm : 1;
    h->rgK = (h->opt.slots_per_lane > 0 && !h->graph) ? h->opt.slots_per_lane : 4;
    if (h->rgK != 2 && h->rgK != 4 && !(h->poolWarps == 4 && h->rgK == 8)) h->rgK = 4;
    if (h->poolWarps == 16) { h->poolWarps = 8; h->tpb = 256; }   // the 16-warp variant was slower and is no longer built
    h->nWork = (size_t)h->nSM * h->bpsm * h->poolWarps * 32 * h->rgK;
    CK(cudaMalloc(&h->dMinsc, sizeof(h->P.minscTab)));
    CK(cudaMemcpy(h->dMinsc, h->P.minscTab, sizeof(h->P.minscTab), cudaMemcpyHostToDevice));
    {   // the device's workspace pool for this launch geometry
        std::lock_guard<std::mutex> lk(gPoolMu);
        auto findPool = [&](size_t n) { WorkPool* r = NULL; for (WorkPool* q : gPools) if (q->device == h->device && q->nWork == n) r = q; return r; };
        const size_t nThreads = (size_t)h->nSM * h->bpsm * (size_t)h->tpb;
        const size_t dpBytes = nThreads * (sizeof(Ht2SwScratch) + (size_t)HT2_SW_POOL_WORDS * sizeof(uint32_t));
        WorkPool* wp = findPool(h->nWork);
        if (!wp && h->opt.slots_per_lane <= 0 && !h->graph && h->poolWarps == 8 && h->rgK == 4) {
            // The default geometry's workspace (368 kB per slot, ~50 GB on an H100) must leave room for what else the
            // process and the device need: the DP scratch of this handle, slot buffers, stack, other processes.  Where
            // it does not, or where the process already has the half-size pool, linear indexes run with 2 slots per
            // lane: half the memory, about 12 % less kernel throughput (DESIGN.md 3).  Graph indexes have one geometry.
            size_t freeB = 0, totalB = 0;
            CK(cudaMemGetInfo(&freeB, &totalB));
            WorkPool* half = findPool(h->nWork / 2);
            const size_t need = h->nWork * sizeof(Ht2Work) + (h->P.bowtie2Dp ? dpBytes : 0) + HT2_MEM_RESERVE;
            if (half || need > freeB) { h->rgK = 2; h->nWork /= 2; wp = half; }
        }
        if (!wp) {
            wp = new WorkPool();
            wp->device = h->device; wp->nWork = h->nWork; wp->refs = 0;
            wp->dWork = NULL; wp->dSw = NULL; wp->dSwPool = NULL; wp->swThreads = 0;
            CK(cudaMalloc(&wp->dWork, wp->nWork * sizeof(Ht2Work)));
            CK(cudaMemset(wp->dWork, 0, wp->nWork * sizeof(Ht2Work)));
            CK(cudaEventCreateWithFlags(&wp->evDone, cudaEventDisableTiming));
            CK(cudaEventRecord(wp->evDone, 0));
            CK(cudaDeviceSynchronize());
            gPools.push_back(wp);
        }
        if (h->P.bowtie2Dp && wp->swThreads < nThreads) {
            // dynamic-programming scratch (ht2_sw.h): per executing thread, not per read slot.  Geometries with the same
            // nWork share the pool but not the grid (8x4 and blocks_per_sm=2 x 2 slots: twice the threads), so the
            // scratch grows to the largest grid once the pool's kernels are done.
            std::lock_guard<std::mutex> lw(wp->mu);
            CK(cudaEventSynchronize(wp->evDone));
            cudaFree(wp->dSw); cudaFree(wp->dSwPool);
            wp->dSw = NULL; wp->dSwPool = NULL; wp->swThreads = 0;
            CK(cudaMalloc(&wp->dSw, nThreads * sizeof(Ht2SwScratch)));
            CK(cudaMalloc(&wp->dSwPool, nThreads * (size_t)HT2_SW_POOL_WORDS * sizeof(uint32_t)));
            wp->swThreads = nThreads;
        }
        wp->refs++;
        h->pool = wp;
    }
    {   // per-thread stack: what the kernels of this index type need, not a blanket value (the limit is
        // context-wide and the driver backs it for every resident thread).  Linear indexes have a statically
        // known call tree; graph indexes recurse through alignWithALTs (ht2_alt.h, depth <= HT2_ALT_MAXDEP).
        size_t need = 0;
        cudaFuncAttributes fa;
        if (h->graph) { CK(cudaFuncGetAttributes(&fa, ht2_align_pool_kernel<8, 4, true, false>)); need = fa.localSizeBytes + 36 * 1024; }
        else { CK(cudaFuncGetAttributes(&fa, ht2_align_pool_kernel<8, 4, false, false>)); need = fa.localSizeBytes + 4 * 1024; }
        CK(cudaFuncGetAttributes(&fa, ht2_sam_kernel<true>));
        if (fa.localSizeBytes + 2048 > need) need = fa.localSizeBytes + 2048;
        // the writing pass's staging buffer: what leaves room for HT2_SAM_STAGE_BLOCKS blocks per SM (1 KB of every
        // block's shared memory is reserved by the system)
        int smemSM = 0, smemBlk = 0;
        CK(cudaDeviceGetAttribute(&smemSM, cudaDevAttrMaxSharedMemoryPerMultiprocessor, h->device));
        CK(cudaDeviceGetAttribute(&smemBlk, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->device));
        size_t stage = (size_t)smemSM / HT2_SAM_STAGE_BLOCKS - 1024 - fa.sharedSizeBytes;
        if (stage > (size_t)smemBlk - fa.sharedSizeBytes) stage = (size_t)smemBlk - fa.sharedSizeBytes;
        h->samStage = (uint32_t)(stage & ~(size_t)15);
        CK(cudaFuncSetAttribute(ht2_sam_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->samStage));
        size_t cur = 0;
        CK(cudaDeviceGetLimit(&cur, cudaLimitStackSize));
        if (cur < need) CK(cudaDeviceSetLimit(cudaLimitStackSize, need));
    }
    CK(cudaStreamCreate(&h->stream));
    for (int i = 0; i < 4; i++) CK(cudaEventCreate(&h->ev[i]));
    return HT2GPU_OK;
}

static ht2gpu_handle* newHandle(const ht2gpu_options_t* opt)
{
    ht2gpu_handle* h = new ht2gpu_handle();
    h->img = NULL; h->dBlob = NULL; h->ownBlob = false; h->blobBytes = 0; h->pool = NULL; h->nWork = 0; h->dMinsc = NULL; h->dSplT = NULL; h->dSsT = NULL; h->collectSs = false; h->recordOut = false;
    h->stream = 0;
    h->dStats = NULL;
    memset((void*)h->slots, 0, sizeof(h->slots));
    h->pipeCtx = NULL; h->pipeCtxFree = NULL;
    if (opt) h->opt = *opt; else ht2gpu_default_options(&h->opt);
    h->device = h->opt.device;
    return h;
}

static int selectDevice(ht2gpu_handle* h)
{
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        h->err = std::string("no usable CUDA device (this library has no CPU path): ") + (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
        return HT2GPU_ERR_CUDA;
    }
    CK(cudaSetDevice(h->device));
    return HT2GPU_OK;
}

extern "C" int ht2gpu_build_image(const char* index_base, void** image, size_t* bytes, char* errbuf, size_t errbuf_len)
{
    std::string err;
    Ht2Image* img = ht2_image_load(index_base, err);
    if (!img) {
        if (errbuf && errbuf_len) { strncpy(errbuf, err.c_str(), errbuf_len - 1); errbuf[errbuf_len - 1] = 0; }
        return HT2GPU_ERR_INDEX;
    }
    void* p = malloc(img->blob.size());
    memcpy(p, img->blob.data(), img->blob.size());
    *image = p; *bytes = img->blob.size();
    delete img;
    return HT2GPU_OK;
}
extern "C" void ht2gpu_free_image(void* image) { free(image); }

extern "C" int ht2gpu_open_image(const void* image, size_t bytes, const ht2gpu_options_t* opt, ht2gpu_handle_t** out)
{
    if (!image || !out || bytes < sizeof(Ht2ImageHeader)) return HT2GPU_ERR_ARG;
    ht2gpu_handle* h = newHandle(opt);
    *out = h;
    int rc = selectDevice(h);
    if (rc) return rc;
    h->img = new Ht2Image();
    h->img->blob.assign((const uint8_t*)image, (const uint8_t*)image + bytes);
    h->blobBytes = bytes;
    CK(cudaMalloc(&h->dBlob, bytes));
    h->ownBlob = true;
    CK(cudaMemcpy(h->dBlob, image, bytes, cudaMemcpyHostToDevice));
    return finishOpen(h);
}

extern "C" int ht2gpu_open_device_image(const void* dev_image, size_t bytes, const void* host_prefix, size_t prefix_bytes,
                                        const ht2gpu_options_t* opt, ht2gpu_handle_t** out)
{
    if (!dev_image || !out || !host_prefix || prefix_bytes < sizeof(Ht2ImageHeader)) return HT2GPU_ERR_ARG;
    ht2gpu_handle* h = newHandle(opt);
    *out = h;
    int rc = selectDevice(h);
    if (rc) return rc;
    h->img = new Ht2Image();
    // host copy is needed for reference names / lengths (SAM) -- fetch it from the device
    h->img->blob.resize(bytes);
    CK(cudaMemcpy(h->img->blob.data(), dev_image, bytes, cudaMemcpyDeviceToHost));
    h->blobBytes = bytes;
    h->dBlob = (uint8_t*)dev_image;
    h->ownBlob = false;
    return finishOpen(h);
}

extern "C" int ht2gpu_open_peer(const ht2gpu_handle_t* src, const ht2gpu_options_t* opt, ht2gpu_handle_t** out)
{
    if (!src || !out || !src->dBlob || !src->img) return HT2GPU_ERR_ARG;
    ht2gpu_handle* h = newHandle(opt ? opt : &src->opt);
    *out = h;
    int rc = selectDevice(h);
    if (rc) return rc;
    h->img = new Ht2Image();
    h->img->blob = src->img->blob;            // host copy: reference names / lengths for SAM
    h->blobBytes = src->blobBytes;
    CK(cudaMalloc(&h->dBlob, h->blobBytes));
    h->ownBlob = true;
    if (h->device == src->device) CK(cudaMemcpy(h->dBlob, src->dBlob, h->blobBytes, cudaMemcpyDeviceToDevice));
    else {
        int can = 0;
        cudaDeviceCanAccessPeer(&can, h->device, src->device);
        if (can) { cudaError_t e = cudaDeviceEnablePeerAccess(src->device, 0); if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CK(e); cudaGetLastError(); }
        CK(cudaMemcpyPeer(h->dBlob, h->device, src->dBlob, src->device, h->blobBytes));
    }
    return finishOpen(h);
}

extern "C" int ht2gpu_open(const char* index_base, const ht2gpu_options_t* opt, ht2gpu_handle_t** out)
{
    if (!index_base || !out) return HT2GPU_ERR_ARG;
    ht2gpu_handle* h = newHandle(opt);
    *out = h;
    int rc = selectDevice(h);
    if (rc) return rc;
    h->img = ht2_image_load(index_base, h->err);
    if (!h->img) return HT2GPU_ERR_INDEX;
    h->blobBytes = h->img->blob.size();
    CK(cudaMalloc(&h->dBlob, h->blobBytes));
    h->ownBlob = true;
    CK(cudaMemcpy(h->dBlob, h->img->blob.data(), h->blobBytes, cudaMemcpyHostToDevice));
    return finishOpen(h);
}

extern "C" const void* ht2gpu_image_data(const ht2gpu_handle_t* h) { return h && h->img ? h->img->blob.data() : NULL; }
extern "C" size_t ht2gpu_image_bytes(const ht2gpu_handle_t* h) { return h ? h->blobBytes : 0; }
extern "C" const void* ht2gpu_device_image(const ht2gpu_handle_t* h) { return h ? h->dBlob : NULL; }
extern "C" const char* ht2gpu_last_error(const ht2gpu_handle_t* h) { return h ? h->err.c_str() : "null handle"; }
extern "C" int ht2gpu_launch_geometry(const ht2gpu_handle_t* h, int32_t out[3])
{
    if (!h || !out || !h->pool) return HT2GPU_ERR_ARG;
    out[0] = h->poolWarps; out[1] = h->rgK; out[2] = h->bpsm;
    return HT2GPU_OK;
}
extern "C" uint32_t ht2gpu_num_refs(const ht2gpu_handle_t* h) { return h && h->img ? h->img->header()->nRefs : 0; }
extern "C" const char* ht2gpu_ref_name(const ht2gpu_handle_t* h, uint32_t i) { return h->img->refName(i); }
extern "C" uint32_t ht2gpu_ref_len(const ht2gpu_handle_t* h, uint32_t i) { return h->img->refPlen(i); }

extern "C" int ht2gpu_close(ht2gpu_handle_t* h)
{
    if (!h) return HT2GPU_OK;
    if (h->pipeCtx && h->pipeCtxFree) h->pipeCtxFree(h->pipeCtx);
    if (h->dBlob && h->ownBlob) cudaFree(h->dBlob);
    if (h->pool) {   // the last handle of a pool frees the workspaces
        std::lock_guard<std::mutex> lk(gPoolMu);
        WorkPool* wp = h->pool;
        if (--wp->refs == 0) {
            cudaSetDevice(wp->device);
            cudaDeviceSynchronize();
            cudaFree(wp->dWork); cudaFree(wp->dSw); cudaFree(wp->dSwPool); cudaEventDestroy(wp->evDone);
            for (size_t i = 0; i < gPools.size(); i++) if (gPools[i] == wp) { gPools.erase(gPools.begin() + i); break; }
            delete wp;
        }
        h->pool = NULL;
    }
    if (h->dMinsc) cudaFree(h->dMinsc);
    if (h->dSplT) cudaFree(h->dSplT);
    if (h->dSsT) cudaFree(h->dSsT);
    if (h->dRgTag) cudaFree(h->dRgTag);
    cudaFree(h->dStats);
    for (int k = 0; k < HT2GPU_N_SLOTS; k++) {
        SamSlot& S = h->slots[k];
        if (!S.init) continue;
        cudaStreamSynchronize(S.stream);
        cudaFree(S.dSeq); cudaFree(S.dQual); cudaFree(S.dOffs); cudaFree(S.dSeeds); cudaFree(S.dNames); cudaFree(S.dNameOffs);
        cudaFree(S.dReads); cudaFree(S.dAlns); cudaFree(S.dEdits); cudaFree(S.dPairs); cudaFree(S.dCounters);
        cudaFree(S.dSamLen); cudaFree(S.dBlk); cudaFree(S.dSam); cudaFree(S.dColRecs); cudaFree(S.dTally); cudaFree(S.dOut);
        if (S.hSam) cudaFreeHost(S.hSam);
        if (S.hOut) cudaFreeHost(S.hOut);
        if (S.hMeta) cudaFreeHost(S.hMeta);
        cudaStreamDestroy(S.stream);
        for (int i = 0; i < 6; i++) cudaEventDestroy(S.ev[i]);
        for (int i = 0; i < 3; i++) if (S.evSplit[i]) cudaEventDestroy(S.evSplit[i]);
    }
    if (h->stream) { cudaStreamDestroy(h->stream); for (int i = 0; i < 4; i++) cudaEventDestroy(h->ev[i]); }
    delete h->img;
    delete h;
    return HT2GPU_OK;
}

extern "C" uint32_t ht2gpu_read_seed(const uint8_t* seq, const uint8_t* qual, uint32_t len, const char* name, uint32_t global_seed)
{
    Ht2HostRead r;
    r.seq.assign(seq, seq + len);
    if (qual) r.qual.assign(qual, qual + len); else r.qual.assign(len, (uint8_t)'I');
    r.name = name ? name : "";
    return ht2_gen_rand_seed(r, global_seed);
}

template <typename T>
static cudaError_t growBuf(T*& p, size_t& cap, size_t need, size_t slackNum = 5, size_t slackDen = 4)
{
    if (need <= cap && p) return cudaSuccess;
    if (p) cudaFree(p);
    p = NULL;
    size_t ncap = need * slackNum / slackDen + 16;
    cudaError_t e = cudaMalloc(&p, ncap * sizeof(T));
    cap = (e == cudaSuccess) ? ncap : 0;
    return e;
}

static int slotInit(ht2gpu_handle* h, SamSlot& S)
{
    if (S.init) return HT2GPU_OK;
    CK(cudaStreamCreateWithFlags(&S.stream, cudaStreamNonBlocking));
    for (int i = 0; i < 6; i++) CK(cudaEventCreate(&S.ev[i]));
    if (getenv("HT2GPU_SAM_SPLIT")) for (int i = 0; i < 3; i++) CK(cudaEventCreate(&S.evSplit[i]));
    CK(cudaMalloc(&S.dCounters, 8 * sizeof(unsigned int)));
    CK(cudaMalloc(&S.dTally, HT2_T_N * sizeof(unsigned long long)));
    CK(cudaHostAlloc(&S.hMeta, (HT2_META_TALLY + HT2_T_N) * sizeof(unsigned long long), cudaHostAllocPortable));
    S.init = true;
    return HT2GPU_OK;
}

// Stage a batch in a slot: H2D copies only (the per-read filters run on the device, ht2_dev_filter).
// Every buffer has its own capacity (a FASTA batch leaves dQual untouched).
static int uploadBatch(ht2gpu_handle* h, SamSlot& S, const ht2gpu_read_batch_t* b, const char* names, const uint32_t* nameOffs,
                       size_t namesBytes, uint64_t& h2dBytes)
{
    const uint32_t n = b->n_reads;
    const uint64_t nb = b->offs[n];
    CK(growBuf(S.dSeq, S.capSeq, nb + 8));
    if (b->qual) CK(growBuf(S.dQual, S.capQual, nb + 8));
    CK(growBuf(S.dOffs, S.capOffs, (size_t)n + 1));
    CK(growBuf(S.dSeeds, S.capSeeds, (size_t)n + 1));
    CK(cudaMemcpyAsync(S.dSeq, b->seq, nb, cudaMemcpyHostToDevice, S.stream));
    if (b->qual) CK(cudaMemcpyAsync(S.dQual, b->qual, nb, cudaMemcpyHostToDevice, S.stream));
    CK(cudaMemcpyAsync(S.dOffs, b->offs, ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, S.stream));
    CK(cudaMemcpyAsync(S.dSeeds, b->seeds, (size_t)n * 4, cudaMemcpyHostToDevice, S.stream));
    h2dBytes = nb * (b->qual ? 2 : 1) + ((size_t)n + 1) * 8 + (size_t)n * 4;
    if (names) {
        CK(growBuf(S.dNames, S.capNames, namesBytes + 8));
        CK(growBuf(S.dNameOffs, S.capNameOffs, (size_t)n + 1));
        CK(cudaMemcpyAsync(S.dNames, names, namesBytes, cudaMemcpyHostToDevice, S.stream));
        CK(cudaMemcpyAsync(S.dNameOffs, nameOffs, ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, S.stream));
        h2dBytes += namesBytes + ((size_t)n + 1) * 4;
    }
    return HT2GPU_OK;
}

static int ensureOut(ht2gpu_handle* h, SamSlot& S, uint32_t units, size_t alns, size_t edits, size_t pairs)
{
    CK(growBuf(S.dReads, S.capUnits, units));
    CK(growBuf(S.dAlns, S.capAlns, alns));
    CK(growBuf(S.dEdits, S.capEdits, edits));
    size_t pc = S.capPairs * 2, need = pairs * 2;
    if (need > pc || !S.dPairs) { CK(growBuf(S.dPairs, pc, need)); S.capPairs = pc / 2; }
    if (!h->dStats && getenv("HT2GPU_STATS")) {
        CK(cudaMalloc(&h->dStats, (1024 + 256 * 12) * sizeof(unsigned long long)));
        CK(cudaMemset(h->dStats, 0, (1024 + 256 * 12) * sizeof(unsigned long long)));
    }
    return HT2GPU_OK;
}

// Enqueue the alignment kernel of the slot's batch on the slot's stream.  The caller holds the pool's mutex and has
// made the stream wait for the pool's evDone (the workspaces are shared by every slot of every handle).
static int launchAlign(ht2gpu_handle* h, SamSlot& S, const ht2gpu_read_batch_t* b, uint32_t units, cudaEvent_t evStart = NULL)
{
    WorkPool* wp = h->pool;
    const uint32_t grid = (uint32_t)(h->nSM * h->bpsm);
    if (h->P.bowtie2Dp && wp->swThreads < (size_t)grid * h->tpb) {   // every launched thread indexes its own DP scratch
        h->err = "the workspace pool's DP scratch is smaller than the launch grid";
        return HT2GPU_ERR_ARG;
    }
    DevBatch db;
    db.seq = S.dSeq; db.qual = b->qual ? S.dQual : NULL; db.offs = S.dOffs; db.seeds = S.dSeeds;
    db.n_units = units; db.paired = b->paired; db.sw = h->P.bowtie2Dp ? wp->dSw : NULL; db.swPool = h->P.bowtie2Dp ? wp->dSwPool : NULL; db.minscTab = h->dMinsc;
    { static const int e = getenv("HT2GPU_ELECT") ? atoi(getenv("HT2GPU_ELECT")) : 8; db.elect = (uint32_t)(e < 1 ? 1 : (e > 32 ? 32 : e)); }
#ifdef HT2_ENABLE_SPLICED
    db.splT = (const Ht2SplTables*)h->dSplT; db.ssT = h->dSsT;
#endif
    DevOut o;
    o.reads = S.dReads; o.alns = S.dAlns; o.edits = S.dEdits; o.pairs = S.dPairs;
    o.capAlns = (uint32_t)S.capAlns; o.capEdits = (uint32_t)S.capEdits; o.capPairs = (uint32_t)S.capPairs;
    o.counters = S.dCounters;
    o.stats = h->dStats;
    CK(cudaMemsetAsync(S.dCounters, 0, 8 * sizeof(unsigned int), S.stream));
    if (evStart) CK(cudaEventRecord(evStart, S.stream));   // kernel time is counted from here: after the waits for the previous kernels
    Ht2Work* work = wp->dWork;
    const bool nospl = h->P.noSplicedAlignment != 0;   // the DNA-only instantiation has less code (DESIGN.md 4.1)
    if (h->graph) {
        if (nospl) ht2_align_pool_kernel<8, 4, true, true><<<grid, 256, 0, S.stream>>>(h->dBlob, h->P, db, o, work);
        else ht2_align_pool_kernel<8, 4, true, false><<<grid, 256, 0, S.stream>>>(h->dBlob, h->P, db, o, work);
    } else {
        switch (h->poolWarps * 100 + h->rgK) {
            case 802:
                if (nospl) ht2_align_pool_kernel<8, 2, false, true><<<grid, h->tpb, 0, S.stream>>>(h->dBlob, h->P, db, o, work);
                else ht2_align_pool_kernel<8, 2, false, false><<<grid, h->tpb, 0, S.stream>>>(h->dBlob, h->P, db, o, work);
                break;
            case 408:  ht2_align_pool_kernel<4, 8, false, false><<<grid, h->tpb, 0, S.stream>>>(h->dBlob, h->P, db, o, work); break;
            default:
                if (nospl) ht2_align_pool_kernel<8, 4, false, true><<<grid, h->tpb, 0, S.stream>>>(h->dBlob, h->P, db, o, work);
                else ht2_align_pool_kernel<8, 4, false, false><<<grid, h->tpb, 0, S.stream>>>(h->dBlob, h->P, db, o, work);
                break;
        }
    }
    CK(cudaGetLastError());
    return HT2GPU_OK;
}

// HT2GPU_STATS=1: per-state statistics of the pool kernel's rounds (investigation aid).
static void dumpStats(ht2gpu_handle* h)
{
    static const char* topN[] = {"START", "NEXTBWT", "PS", "ALIGN", "HYB_EXTEND", "HYB_PICK", "HYB_RET", "HYB_DP", "HYB_DP_RET", "POST_ALIGN", "AFTER_LOOP",
                                 "MATE_NEXT", "MATE_SEARCH", "MATE_ANCHOR", "MATE_RET", "MATE_DONE", "DONE"};
    static const char* frN[] = {"ENTER", "L_START", "L_WHILE", "L_COORD", "L_COORD_RET", "L_WHILE_TAIL", "L_STASH", "L_STASH_RET",
                                "L_AFTER_WHILE", "L_GCOORD", "L_GCOORD_RET", "L_TRIM", "L_TRIM_RET", "L_EXT", "R_START", "R_WHILE",
                                "R_COORD", "R_COORD_RET", "R_WHILE_TAIL", "R_STASH", "R_STASH_RET", "R_AFTER_WHILE", "R_GCOORD",
                                "R_GCOORD_RET", "R_TRIM", "R_TRIM_RET", "R_EXT", "FINAL_RET", "RETURN", "L_COMBINE", "L_GCOMBINE", "R_COMBINE", "R_GCOMBINE",
                                "SS_FULL", "L_SS", "L_SS_RET", "R_SS", "R_SS_RET"};
    std::vector<unsigned long long> st(1024 + 256 * 12);
    if (cudaMemcpy(st.data(), h->dStats, st.size() * 8, cudaMemcpyDeviceToHost) != cudaSuccess) return;
    cudaMemset(h->dStats, 0, st.size() * 8);
    unsigned long long totC = 0;
    for (int c = 0; c < 256; c++) totC += st[c * 4 + 2];
    fprintf(stderr, "%-16s %10s %7s %10s %9s %6s\n", "state", "rounds", "lanes", "cyc/round", "max cyc", "time%");
    for (int c = 0; c < 256; c++) {
        if (!st[c * 4]) continue;
        char nm[32];
        if (c == 0) snprintf(nm, sizeof nm, "NEED");
        else if (c == 1) snprintf(nm, sizeof nm, "FINISH");
        else if (c < 20) snprintf(nm, sizeof nm, "T_%s", c - 2 < 17 ? topN[c - 2] : "?");
        else snprintf(nm, sizeof nm, "F_%s", c - 20 < 38 ? frN[c - 20] : "?");
        fprintf(stderr, "%-16s %10llu %7.2f %10.0f %9llu %6.2f |", nm, st[c * 4], (double)st[c * 4 + 1] / st[c * 4],
                (double)st[c * 4 + 2] / st[c * 4], st[c * 4 + 3], 100.0 * st[c * 4 + 2] / (totC ? totC : 1));
        // cycles per round by group size: 1, 2-3, 4-7, 8-15, 16-31, 32 lanes
        for (int bk = 0; bk < 6; bk++) {
            unsigned long long n = st[1024 + (c * 6 + bk) * 2], cy = st[1024 + (c * 6 + bk) * 2 + 1];
            fprintf(stderr, " %6.0f(%llu)", n ? (double)cy / n / 1000.0 : 0.0, n);
        }
        fprintf(stderr, "\n");
    }
}

static int checkBatch(ht2gpu_handle* h, const ht2gpu_read_batch_t* b)
{
    if (b->paired && (b->n_reads & 1)) { h->err = "paired batch needs an even number of reads"; return HT2GPU_ERR_ARG; }
    if (h->graph && h->img->header()->altsUnsupported) {
        h->err = "this graph index holds splice-site / exon ALTs; alignment through them is not implemented in this build "
                 "(SNP / indel ALTs are; ht2gpu_seed_search works on any graph index)";
        return HT2GPU_ERR_UNSUPPORTED;
    }
    return HT2GPU_OK;
}

// Structured results (ht2gpu_align_batch / ht2gpu_align_resident): slot 0.
static int runBatch(ht2gpu_handle* h, const ht2gpu_read_batch_t* b, int iters, ht2gpu_result_batch_t* res)
{
    if (!h || !b || !res) return HT2GPU_ERR_ARG;
    memset(res, 0, sizeof(*res));
    int rc = checkBatch(h, b);
    if (rc) return rc;
    if (b->n_reads == 0) return HT2GPU_OK;
    CK(cudaSetDevice(h->device));
    SamSlot& S = h->slots[0];
    rc = slotInit(h, S);
    if (rc) return rc;
    const uint32_t units = b->paired ? b->n_reads / 2 : b->n_reads;
    uint64_t h2d = 0;
    CK(cudaEventRecord(S.ev[0], S.stream));
    rc = uploadBatch(h, S, b, NULL, NULL, 0, h2d);
    if (rc) return rc;
    size_t capA = (size_t)b->n_reads * 2 + 1024, capE = (size_t)b->n_reads * 4 + 4096, capP = (size_t)units * 2 + 1024;
    unsigned int counters[4] = {0, 0, 0, 0};
    float msKernel = 0;
    uint32_t nLaunch = 0;
    for (int attempt = 0; attempt < 4; attempt++) {
        rc = ensureOut(h, S, units, capA, capE, capP);
        if (rc) return rc;
        {
            std::lock_guard<std::mutex> lk(h->pool->mu);
            CK(cudaStreamWaitEvent(S.stream, h->pool->evDone, 0));
            for (int it = 0; it < iters; it++) { rc = launchAlign(h, S, b, units, it == 0 ? S.ev[1] : NULL); if (rc) return rc; nLaunch++; }
            CK(cudaEventRecord(S.ev[2], S.stream));
            CK(cudaEventRecord(h->pool->evDone, S.stream));
        }
        CK(cudaMemcpyAsync(counters, S.dCounters, sizeof(counters), cudaMemcpyDeviceToHost, S.stream));
        CK(cudaStreamSynchronize(S.stream));
        CK(cudaEventElapsedTime(&msKernel, S.ev[1], S.ev[2]));
        if (counters[0] <= S.capAlns && counters[1] <= S.capEdits && counters[2] <= S.capPairs) break;
        // result pools were too small: grow and re-run (results are deterministic)
        capA = counters[0] + 1024; capE = counters[1] + 4096; capP = counters[2] + 1024;
    }
    if (h->dStats) dumpStats(h);
    auto up = [](size_t v) { return (v + 63) & ~(size_t)63; };
    const size_t szR = up((size_t)units * sizeof(ht2gpu_read_result_t)), szA = up((size_t)counters[0] * sizeof(ht2gpu_aln_t)),
                 szE = up((size_t)counters[1] * sizeof(ht2gpu_edit_t)), szP = up((size_t)counters[2] * 4);
    ResPriv* pv = new ResPriv();
    if (!pinnedGet(szR + szA + szE + szP + 64, *pv)) { delete pv; h->err = "cudaHostAlloc failed for the result batch"; return HT2GPU_ERR_CUDA; }
    res->priv = pv;   // from here on ht2gpu_free_results returns the buffer, also on error paths
    uint8_t* hb = (uint8_t*)pv->buf;
    ht2gpu_read_result_t* hReads = (ht2gpu_read_result_t*)hb;
    ht2gpu_aln_t* hAlns = (ht2gpu_aln_t*)(hb + szR);
    ht2gpu_edit_t* hEdits = (ht2gpu_edit_t*)(hb + szR + szA);
    uint16_t* hPairs = (uint16_t*)(hb + szR + szA + szE);
    CK(cudaMemcpyAsync(hReads, S.dReads, (size_t)units * sizeof(ht2gpu_read_result_t), cudaMemcpyDeviceToHost, S.stream));
    if (counters[0]) CK(cudaMemcpyAsync(hAlns, S.dAlns, (size_t)counters[0] * sizeof(ht2gpu_aln_t), cudaMemcpyDeviceToHost, S.stream));
    if (counters[1]) CK(cudaMemcpyAsync(hEdits, S.dEdits, (size_t)counters[1] * sizeof(ht2gpu_edit_t), cudaMemcpyDeviceToHost, S.stream));
    if (counters[2]) CK(cudaMemcpyAsync(hPairs, S.dPairs, (size_t)counters[2] * 4, cudaMemcpyDeviceToHost, S.stream));
    CK(cudaEventRecord(S.ev[3], S.stream));
    CK(cudaStreamSynchronize(S.stream));
    float msH2d = 0, msD2h = 0;
    CK(cudaEventElapsedTime(&msH2d, S.ev[0], S.ev[1]));
    CK(cudaEventElapsedTime(&msD2h, S.ev[2], S.ev[3]));
    res->n_reads = units; res->reads = hReads;
    res->n_alns = counters[0]; res->alns = hAlns;
    res->n_edits = counters[1]; res->edits = hEdits;
    res->n_pairs = counters[2]; res->pairs = hPairs;
    res->ms_h2d = msH2d; res->ms_kernel = msKernel; res->ms_d2h = msD2h;
    res->h2d_bytes = h2d;
    res->d2h_bytes = (uint64_t)units * sizeof(ht2gpu_read_result_t) + (uint64_t)counters[0] * sizeof(ht2gpu_aln_t) +
                     (uint64_t)counters[1] * sizeof(ht2gpu_edit_t) + (uint64_t)counters[2] * 4 + sizeof(counters);
    res->n_launches = nLaunch;
    // Reads that exceeded a device-side capacity are flagged in reads[i].err and counted; the batch itself succeeds
    // (the reference has no such limits: a caller that needs byte parity must treat flagged reads as failed).
    uint32_t nErr = 0, anyErr = 0;
    for (uint32_t i = 0; i < units; i++) if (hReads[i].err) { nErr++; anyErr |= hReads[i].err; }
    res->n_err_reads = nErr;
    if (nErr) {
        char buf[160]; snprintf(buf, sizeof(buf), "device capacity exceeded for %u read(s) (err bits 0x%x); see reads[i].err", nErr, anyErr);
        h->err = buf;
    }
    return HT2GPU_OK;
}

extern "C" int ht2gpu_align_batch(ht2gpu_handle_t* h, const ht2gpu_read_batch_t* b, ht2gpu_result_batch_t* res)
{
    return runBatch(h, b, 1, res);
}
extern "C" int ht2gpu_align_resident(ht2gpu_handle_t* h, const ht2gpu_read_batch_t* b, int iters, ht2gpu_result_batch_t* res)
{
    return runBatch(h, b, iters < 1 ? 1 : iters, res);
}
extern "C" void ht2gpu_free_results(ht2gpu_result_batch_t* res)
{
    if (res && res->priv) { ResPriv* pv = (ResPriv*)res->priv; pinnedPut(*pv); delete pv; res->priv = NULL; }
}

// ---------------------------------------------------------------------------
// SAM on the device: align + finishRead for a batch, text back in pinned host memory
// ---------------------------------------------------------------------------
static Ht2SamIn samIn(const ht2gpu_handle* h, const SamSlot& S)
{
    Ht2SamIn in;
    in.blob = h->dBlob; in.minscTab = h->dMinsc;
    in.seq = S.dSeq; in.qual = S.batch.qual ? S.dQual : NULL; in.offs = S.dOffs; in.names = S.dNames; in.nameOffs = S.dNameOffs;
    in.n_reads = S.batch.n_reads; in.paired = S.batch.paired;
    in.reads = S.dReads; in.alns = S.dAlns; in.edits = S.dEdits; in.pairs = S.dPairs;
    in.khits = h->P.khits; in.secondary = h->P.secondary; in.mixed = h->P.mixed; in.discord = h->P.discord; in.ssT = h->dSsT;
    in.colCount = h->collectSs ? S.dCounters + 6 : NULL; in.colRecs = S.dColRecs; in.colCap = (uint32_t)S.capCol;
    in.noUnal = h->samOut.noUnal; in.omitSecSeq = h->samOut.omitSecSeq; in.rgTag = h->dRgTag;
    in.unitOut = h->recordOut ? S.dOut : NULL;
    return in;
}

// Enqueue [align, SAM count, block scan, SAM write] for the slot's uploaded batch.  withAlign = false re-runs
// only the SAM kernels (after the text buffer was grown).
static int enqueueKernels(ht2gpu_handle* h, SamSlot& S, bool withAlign)
{
    const uint32_t units = S.units;
    const uint32_t nBlk = (units + HT2_SAM_TPB - 1) / HT2_SAM_TPB;
    CK(growBuf(S.dSamLen, S.capSamLen, units));
    CK(growBuf(S.dBlk, S.capBlk, (size_t)nBlk + 2));
    if (h->collectSs) CK(growBuf(S.dColRecs, S.capCol, (size_t)S.batch.n_reads * 4 + 1024, 1, 1));
    if (h->recordOut) {
        CK(growBuf(S.dOut, S.capOut, units));
        if (units > S.capHOut) {
            if (S.hOut) CK(cudaFreeHost(S.hOut));
            S.hOut = NULL; S.capHOut = 0;
            CK(cudaHostAlloc(&S.hOut, (size_t)units + units / 8 + 4096, cudaHostAllocPortable));
            S.capHOut = (size_t)units + units / 8 + 4096;
        }
    }
    std::lock_guard<std::mutex> lk(h->pool->mu);
    CK(cudaStreamWaitEvent(S.stream, h->pool->evDone, 0));
    if (withAlign) { int rc = launchAlign(h, S, &S.batch, units, S.ev[2]); if (rc) return rc; S.nLaunch++; }
    else CK(cudaEventRecord(S.ev[2], S.stream));
    CK(cudaEventRecord(S.ev[3], S.stream));
    if (h->collectSs) CK(cudaMemsetAsync(S.dCounters + 6, 0, sizeof(unsigned int), S.stream));
    // the counting pass tallies the batch's ReportingMetrics; a re-run (ht2gpu_wait_sam) must not count it twice
    CK(cudaMemsetAsync(S.dTally, 0, HT2_T_N * sizeof(unsigned long long), S.stream));
    const Ht2SamIn in = samIn(h, S);
    if (S.evSplit[0]) CK(cudaEventRecord(S.evSplit[0], S.stream));
    ht2_sam_kernel<false><<<nBlk, HT2_SAM_TPB, 0, S.stream>>>(in, units, S.dSamLen, S.dBlk, NULL, 0, S.dCounters, S.dTally, 0);
    if (S.evSplit[1]) CK(cudaEventRecord(S.evSplit[1], S.stream));
    ht2_sam_scan_kernel<<<1, 1024, 0, S.stream>>>(S.dBlk, nBlk);
    if (S.evSplit[2]) CK(cudaEventRecord(S.evSplit[2], S.stream));
    ht2_sam_kernel<true><<<nBlk, HT2_SAM_TPB, h->samStage, S.stream>>>(in, units, S.dSamLen, S.dBlk, S.dSam, (unsigned long long)S.capSam, S.dCounters,
                                                                        S.dTally, h->samStage);
    CK(cudaGetLastError());
    S.nLaunch += 3;
    CK(cudaEventRecord(S.ev[4], S.stream));
    CK(cudaEventRecord(h->pool->evDone, S.stream));
    // meta: total SAM bytes, result counters, reads with errors
    CK(cudaMemcpyAsync(&S.hMeta[0], S.dBlk + nBlk, sizeof(unsigned long long), cudaMemcpyDeviceToHost, S.stream));
    CK(cudaMemcpyAsync(&S.hMeta[1], S.dCounters, 8 * sizeof(unsigned int), cudaMemcpyDeviceToHost, S.stream));
    CK(cudaMemcpyAsync(&S.hMeta[HT2_META_TALLY], S.dTally, HT2_T_N * sizeof(unsigned long long), cudaMemcpyDeviceToHost, S.stream));
    if (h->recordOut) CK(cudaMemcpyAsync(S.hOut, S.dOut, units, cudaMemcpyDeviceToHost, S.stream));
    return HT2GPU_OK;
}

extern "C" int ht2gpu_sam_slots(const ht2gpu_handle_t*) { return HT2GPU_N_SLOTS; }
extern "C" void* ht2gpu_host_alloc(size_t bytes) { void* p = NULL; return cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocPortable) == cudaSuccess ? p : NULL; }
extern "C" void ht2gpu_host_free(void* p) { if (p) cudaFreeHost(p); }
extern "C" void ht2gpu_set_error(ht2gpu_handle_t* h, const char* msg) { if (h) h->err = msg ? msg : ""; }
extern "C" void* ht2gpu_ctx_get(ht2gpu_handle_t* h) { return h ? h->pipeCtx : NULL; }
extern "C" void ht2gpu_ctx_set(ht2gpu_handle_t* h, void* ctx, void (*release)(void*)) { if (h) { h->pipeCtx = ctx; h->pipeCtxFree = release; } }

extern "C" int ht2gpu_submit_sam(ht2gpu_handle_t* h, int slot, const ht2gpu_read_batch_t* b, const char* names,
                                 const uint32_t* name_offs, size_t names_bytes)
{
    if (!h || !b || slot < 0 || slot >= HT2GPU_N_SLOTS || (b->n_reads && (!names || !name_offs))) return HT2GPU_ERR_ARG;
    int rc = checkBatch(h, b);
    if (rc) return rc;
    CK(cudaSetDevice(h->device));
    SamSlot& S = h->slots[slot];
    rc = slotInit(h, S);
    if (rc) return rc;
    if (S.pending) { h->err = "ht2gpu_submit_sam: the slot still holds a batch (call ht2gpu_wait_sam first)"; return HT2GPU_ERR_ARG; }
    S.batch = *b; S.units = b->paired ? b->n_reads / 2 : b->n_reads; S.namesBytes = names_bytes; S.nLaunch = 0; S.h2dBytes = 0;
    S.pending = true; S.outValid = false;
    if (b->n_reads == 0) return HT2GPU_OK;
    CK(cudaEventRecord(S.ev[0], S.stream));
    rc = uploadBatch(h, S, b, names, name_offs, names_bytes, S.h2dBytes);
    if (rc) return rc;
    CK(cudaEventRecord(S.ev[1], S.stream));
    rc = ensureOut(h, S, S.units, (size_t)b->n_reads * 2 + 1024, (size_t)b->n_reads * 4 + 4096, (size_t)S.units * 2 + 1024);
    if (rc) return rc;
    // SAM text: ~2.2 bytes per base + ~170 per record at one record per read; grown from the measured size if short
    // (+ "\tRG:Z:<id>" per record with a read group)
    const size_t rgBytes = h->samOut.rgId.empty() ? 0 : h->samOut.rgTag().size() + 1;
    const size_t est = (size_t)((double)b->offs[b->n_reads] * 2.6) + (size_t)b->n_reads * (260 + rgBytes) + names_bytes + 4096;
    if (est > S.capSam) CK(growBuf(S.dSam, S.capSam, est, 1, 1));
    return enqueueKernels(h, S, true);
}

extern "C" int ht2gpu_wait_sam(ht2gpu_handle_t* h, int slot, ht2gpu_sam_result_t* out)
{
    if (!h || !out || slot < 0 || slot >= HT2GPU_N_SLOTS) return HT2GPU_ERR_ARG;
    SamSlot& S = h->slots[slot];
    memset(out, 0, sizeof(*out));
    if (!S.init || !S.pending) { h->err = "ht2gpu_wait_sam: nothing was submitted on this slot"; return HT2GPU_ERR_ARG; }
    S.pending = false;
    out->n_units = S.units;
    if (S.batch.n_reads == 0) { out->sam = S.hSam ? S.hSam : (char*)""; S.outValid = h->recordOut; return HT2GPU_OK; }
    CK(cudaSetDevice(h->device));
    for (int attempt = 0; ; attempt++) {
        CK(cudaStreamSynchronize(S.stream));
        const unsigned int* c = (const unsigned int*)&S.hMeta[1];
        const bool poolsOk = c[0] <= S.capAlns && c[1] <= S.capEdits && c[2] <= S.capPairs;
        const bool textOk = S.hMeta[0] <= S.capSam;
        if (poolsOk && textOk) break;
        if (attempt >= 3) { h->err = "ht2gpu_wait_sam: result pools still too small after three re-runs"; return HT2GPU_ERR_CUDA; }
        // a pool was too small: grow it and re-run (results are deterministic); rare, sizes are kept afterwards
        if (!poolsOk) { int rc = ensureOut(h, S, S.units, (size_t)c[0] + 1024, (size_t)c[1] + 4096, (size_t)c[2] + 1024); if (rc) return rc; }
        if (!textOk) CK(growBuf(S.dSam, S.capSam, (size_t)S.hMeta[0] + 4096, 9, 8));
        int rc = enqueueKernels(h, S, !poolsOk);
        if (rc) return rc;
    }
    const size_t total = (size_t)S.hMeta[0];
    if (total + 1 > S.capHSam) {
        if (S.hSam) cudaFreeHost(S.hSam);
        S.hSam = NULL; S.capHSam = 0;
        const size_t cap = total + total / 8 + 4096;
        CK(cudaHostAlloc(&S.hSam, cap, cudaHostAllocPortable));
        S.capHSam = cap;
    }
    CK(cudaMemcpyAsync(S.hSam, S.dSam, total, cudaMemcpyDeviceToHost, S.stream));
    CK(cudaEventRecord(S.ev[5], S.stream));
    CK(cudaStreamSynchronize(S.stream));
    S.hSam[total] = 0;
    if (h->collectSs) {
        const unsigned int nrec = ((const unsigned int*)&S.hMeta[1])[6];
        if (nrec > S.capCol) { h->err = "ht2gpu_wait_sam: more junction records than the batch's buffer holds"; return HT2GPU_ERR_CAPACITY; }
        std::vector<Ht2SsRec> recs(nrec);
        if (nrec) CK(cudaMemcpy(recs.data(), S.dColRecs, (size_t)nrec * sizeof(Ht2SsRec), cudaMemcpyDeviceToHost));
        std::lock_guard<std::mutex> lk(h->novelMu);
        h->novel.add(recs.data(), recs.size());
    }
    {
        std::lock_guard<std::mutex> lk(h->countMu);
        uint64_t* tot = (uint64_t*)&h->counts;
        for (int k = 0; k < HT2_T_N; k++) tot[k] += S.hMeta[HT2_META_TALLY + k];
    }
    if (h->dStats) dumpStats(h);
    if (S.evSplit[0]) {   // HT2GPU_SAM_SPLIT=1: the three SAM kernels of the batch's last SAM pass (investigation aid)
        float ms[3];
        CK(cudaEventElapsedTime(&ms[0], S.evSplit[0], S.evSplit[1]));
        CK(cudaEventElapsedTime(&ms[1], S.evSplit[1], S.evSplit[2]));
        CK(cudaEventElapsedTime(&ms[2], S.evSplit[2], S.ev[4]));
        fprintf(stderr, "sam kernels: count %.3f ms  scan %.3f ms  write %.3f ms  total %.3f ms  |  %zu bytes of SAM, %u units  |  "
                "%.1f GB/s over the three, %.1f GB/s over the writing pass\n", ms[0], ms[1], ms[2], ms[0] + ms[1] + ms[2], total, S.units,
                total / ((ms[0] + ms[1] + ms[2]) * 1e6), total / (ms[2] * 1e6));
    }
    const unsigned int* c = (const unsigned int*)&S.hMeta[1];
    S.outValid = h->recordOut;
    out->sam = S.hSam; out->sam_len = total;
    out->n_alns = c[0]; out->n_err_reads = c[4];
    CK(cudaEventElapsedTime(&out->ms_h2d, S.ev[0], S.ev[1]));
    CK(cudaEventElapsedTime(&out->ms_align, S.ev[2], S.ev[3]));
    CK(cudaEventElapsedTime(&out->ms_sam, S.ev[3], S.ev[4]));
    CK(cudaEventElapsedTime(&out->ms_d2h, S.ev[4], S.ev[5]));
    out->h2d_bytes = S.h2dBytes; out->d2h_bytes = total + 9 * sizeof(unsigned long long) + (h->recordOut ? S.units : 0);
    out->n_launches = S.nLaunch;
    if (c[4]) {
        char buf[160]; snprintf(buf, sizeof(buf), "device capacity exceeded for %u read(s) of the batch; their SAM records are unreliable", c[4]);
        h->err = buf;
    }
    return HT2GPU_OK;
}

extern "C" int ht2gpu_align_sam(ht2gpu_handle_t* h, const ht2gpu_read_batch_t* b, const char* names, const uint32_t* name_offs,
                                size_t names_bytes, ht2gpu_sam_result_t* out)
{
    int rc = ht2gpu_submit_sam(h, 0, b, names, name_offs, names_bytes);
    if (rc) { if (h && h->slots[0].init) h->slots[0].pending = false; return rc; }
    return ht2gpu_wait_sam(h, 0, out);
}

// ---------------------------------------------------------------------------
// seed search (linear and graph indexes)
// ---------------------------------------------------------------------------
struct SeedPriv {
    std::vector<uint32_t> firstHit;
    std::vector<ht2gpu_seed_hit_t> hits;
    std::vector<uint16_t> iedges;
    std::vector<ht2gpu_seed_coord_t> coords;
};

extern "C" int ht2gpu_index_is_graph(const ht2gpu_handle_t* h) { return h && h->graph ? 1 : 0; }

// ---------------------------------------------------------------------------------------------------------------
// ht2gpu_sw_selftest: the warp-wide DP fill (swFillCoop) against the lane fill (swFill, itself pinned to a plain
// scalar statement of the recurrences by the host self-test, tests/hostsim --sw-selftest) on random problems:
// every H, E and F cell, every last-row score and the best score must be equal.  One warp per problem.
// ---------------------------------------------------------------------------------------------------------------
struct SwTestProblem {
    int32_t mmpMax, mmpMin, npen, mmcostConstant, rdGapConst, rdGapLinear, rfGapConst, rfGapLinear, gapbar;
    uint32_t nrow, ncol;
    int64_t minsc;
    uint8_t rd[HT2_SW_MAX_RDLEN], qu[HT2_SW_MAX_RDLEN], rf[HT2_SW_MAXCOLS + 8];
};
__global__ void __launch_bounds__(32)
ht2_sw_selftest_kernel(const SwTestProblem* probs, uint32_t n, Ht2SwScratch* scr, uint32_t* pools, unsigned long long* out)
{
    const uint32_t lane = threadIdx.x;
    Ht2SwScratch* S0 = scr + (size_t)blockIdx.x * 2; Ht2SwScratch* S1 = S0 + 1;
    uint32_t* p0 = pools + (size_t)blockIdx.x * 2 * HT2_SW_POOL_WORDS; uint32_t* p1 = p0 + HT2_SW_POOL_WORDS;
    __shared__ Ht2ParamsCore P;
    for (uint32_t it = blockIdx.x; it < n; it += gridDim.x) {
        const SwTestProblem& q = probs[it];
        __syncwarp();
        if (lane == 0) {
            memset(&P, 0, sizeof(P));
            P.mmpMax = q.mmpMax; P.mmpMin = q.mmpMin; P.npen = q.npen; P.mmcostConstant = q.mmcostConstant != 0;
            P.rdGapConst = q.rdGapConst; P.rdGapLinear = q.rdGapLinear; P.rfGapConst = q.rfGapConst; P.rfGapLinear = q.rfGapLinear;
            P.gapbar = q.gapbar;
        }
        __syncwarp();
        Ht2AlignerT<false> A0, A1;
        A0.blob = NULL; A0.H = NULL; A0.P = &P; A0.W = NULL; A0.sw = S0; A0.swPl = p0; A0.swStride = 1; A0.swStage = 0;
        A1 = A0; A1.sw = S1; A1.swPl = p1;
        long long best0 = 0;
        if (lane == 0) {
            best0 = A0.swFill(q.rd, q.qu, q.nrow, q.rf, q.ncol, q.minsc);
            S1->jrd = q.rd; S1->jqu = q.qu; S1->jrf = q.rf; S1->nrow = q.nrow; S1->jncol = q.ncol; S1->jmsc = q.minsc; S1->jbest = 0;
        }
        __syncwarp();
        A1.swFillCoop(S1, p1, lane);
        unsigned long long bad = 0;
        for (uint32_t c = lane; c < q.nrow * q.ncol; c += 32) {
            const uint32_t row = c % q.nrow, col = c / q.nrow;
            for (int pl = 0; pl < 3; pl++) if (A0.swRaw(pl, S0->seg, row, col) != A1.swRaw(pl, S1->seg, row, col)) bad++;
        }
        for (uint32_t j = lane; j < q.ncol; j += 32) if (S0->lastH[j] != S1->lastH[j]) bad++;
        if (lane == 0 && best0 != S1->jbest) bad++;
        if (bad) atomicAdd(&out[0], bad);
        if (lane == 0) { atomicAdd(&out[1], 1ull); atomicAdd(&out[2], (unsigned long long)q.nrow * q.ncol); if (best0 != HT2_MIN_I64) atomicAdd(&out[3], 1ull); }
    }
}
extern "C" int ht2gpu_sw_selftest(int device, uint32_t n, uint32_t seed, uint64_t out[4])
{
    if (cudaSetDevice(device) != cudaSuccess) return HT2GPU_ERR_CUDA;
    std::vector<SwTestProblem> probs(n);
    uint32_t rng = seed ? seed : 1;
    auto rnd = [&](uint32_t m) { rng = rng * 1664525u + 1013904223u; return (rng >> 8) % m; };
    for (uint32_t it = 0; it < n; it++) {
        SwTestProblem& q = probs[it];
        memset(&q, 0, sizeof(q));
        q.mmpMax = 2 + rnd(6); q.mmpMin = 1 + rnd(q.mmpMax); q.npen = 1 + rnd(2); q.mmcostConstant = rnd(4) == 0;
        q.rdGapConst = 1 + rnd(8); q.rdGapLinear = 1 + rnd(4); q.rfGapConst = 1 + rnd(8); q.rfGapLinear = 1 + rnd(4);
        q.gapbar = 1 + rnd(12);
        // rows 1..256: the first problems take 256 and every 32k +- 1 (the warp fill's row blocks), the rest any length;
        // a quarter of the rectangles are narrowed by up to 20 columns, as frameSeedExtensionRect trims at a contig end
        static const uint32_t edgeRows[] = {256, 1, 31, 33, 63, 65, 95, 97, 127, 129, 159, 161, 191, 193, 223, 225, 255};
        q.nrow = it < sizeof(edgeRows) / sizeof(edgeRows[0]) ? edgeRows[it] : 1 + rnd(HT2_SW_MAX_RDLEN);
        q.ncol = q.nrow + 40 - (rnd(4) == 0 ? rnd(21) : 0);
        for (uint32_t j = 0; j < q.ncol + 8; j++) q.rf[j] = rnd(50) == 0 ? 4 : rnd(4);
        uint32_t k = 0;
        for (uint32_t j = q.ncol - q.nrow > 20 ? 20 : q.ncol - q.nrow; k < q.nrow && j < q.ncol;) {   // the read: the window with substitutions and small indels
            const uint32_t r = rnd(100);
            if (r < 3) q.rd[k++] = (uint8_t)rnd(4);
            else if (r < 6) j++;
            else { q.rd[k++] = r < 12 ? (uint8_t)rnd(5) : q.rf[j]; j++; }
        }
        while (k < q.nrow) q.rd[k++] = (uint8_t)rnd(4);
        for (uint32_t i = 0; i < q.nrow; i++) q.qu[i] = (uint8_t)(33 + rnd(42));
        q.minsc = -(int64_t)(10 + rnd(3 * q.nrow));
    }
    const int grid = 64;
    SwTestProblem* dP = NULL; Ht2SwScratch* dS = NULL; uint32_t* dPool = NULL; unsigned long long* dOut = NULL;
    int rc = HT2GPU_OK;
    if (cudaMalloc(&dP, sizeof(SwTestProblem) * (size_t)(n ? n : 1)) != cudaSuccess || cudaMalloc(&dS, sizeof(Ht2SwScratch) * 2 * grid) != cudaSuccess ||
        cudaMalloc(&dPool, sizeof(uint32_t) * (size_t)HT2_SW_POOL_WORDS * 2 * grid) != cudaSuccess || cudaMalloc(&dOut, 4 * sizeof(unsigned long long)) != cudaSuccess) rc = HT2GPU_ERR_CUDA;
    if (rc == HT2GPU_OK) {
        cudaMemcpy(dP, probs.data(), sizeof(SwTestProblem) * (size_t)n, cudaMemcpyHostToDevice);
        cudaMemset(dOut, 0, 4 * sizeof(unsigned long long));
        cudaMemset(dS, 0, sizeof(Ht2SwScratch) * 2 * grid);
        size_t lim = 0; cudaDeviceGetLimit(&lim, cudaLimitStackSize);
        if (lim < 8192) cudaDeviceSetLimit(cudaLimitStackSize, 8192);
        ht2_sw_selftest_kernel<<<grid, 32>>>(dP, n, dS, dPool, dOut);
        unsigned long long o4[4] = {0, 0, 0, 0};
        if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpy(o4, dOut, sizeof(o4), cudaMemcpyDeviceToHost) != cudaSuccess) rc = HT2GPU_ERR_CUDA;
        for (int i = 0; i < 4; i++) out[i] = o4[i];
    }
    cudaFree(dP); cudaFree(dS); cudaFree(dPool); cudaFree(dOut);
    return rc;
}

namespace {
struct DevTmp {   // temporaries of one ht2gpu_seed_search / ht2gpu_sw_extend call: freed on every return path
    std::vector<void*> ptrs;
    template <typename T> cudaError_t alloc(T*& p, size_t bytes) { void* q = NULL; cudaError_t e = cudaMalloc(&q, bytes); if (e == cudaSuccess) ptrs.push_back(q); p = (T*)q; return e; }
    ~DevTmp() { for (void* q : ptrs) cudaFree(q); }
};
}

// ---------------------------------------------------------------------------------------------------------------
// ht2gpu_sw_extend: the --bowtie2-dp seed extension on its own, one job per lane, through the production code:
// warp fill = ht2_dp_round (the pool kernel's DP round) then swExtendAnchor -> swFinish; lane fill = swExtendAnchor
// (swPrepare + swFill + swFinish).  A warp holds whatever jobs it is given -- ones that fill, ones whose anchor
// already spans the read, ones refused -- as a round of the pool kernel does.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32)
ht2_sw_extend_kernel(const uint8_t* __restrict__ blob, Ht2ParamsCore P, const ht2gpu_sw_job_t* jobs, const uint8_t* seq,
                     const uint8_t* qual, uint32_t n, Ht2Work* work, Ht2SwScratch* scr, uint32_t* pools, int warpFill,
                     ht2gpu_sw_result_t* res, ht2gpu_edit_t* edits)
{
    const uint32_t lane = threadIdx.x, j = blockIdx.x * 32 + lane;
    Ht2AlignerT<false, true> A;
    A.bind(blob, &P, NULL);
    A.sw = scr + j; A.swPl = pools + (size_t)j * HT2_SW_POOL_WORDS; A.swStride = 1;
    Ht2Work* W = NULL;
    if (j < n) {
        const ht2gpu_sw_job_t& q = jobs[j];
        W = work + j;                                           // zeroed by the host
        Ht2Read& R = W->rd[0];
        const uint32_t len = q.read_len < HT2_MAX_RDLEN ? q.read_len : HT2_MAX_RDLEN;
        R.len = len;
        for (uint32_t i = 0; i < len; i++) {
            const uint8_t c = seq[q.read_off + i], rc = seq[q.read_off + len - 1 - i];
            R.seq[0][i] = c; R.qual[0][i] = qual[q.read_off + i];
            R.seq[1][i] = rc < 4 ? (uint8_t)(rc ^ 3) : (uint8_t)4; R.qual[1][i] = qual[q.read_off + len - 1 - i];
        }
        W->cfgMinsc[0] = q.minsc; W->cfgMinsc[1] = HT2_IDX_MAX32;
        W->curRdi = 0; W->hybHj = 0;
        W->rnd.init(q.seed);
        A.initHit(W->genomeHits[0], q.fw != 0, q.rdoff, q.len, 0, 0, q.tidx, q.toff, q.toff);
        A.sw->jbest = HT2_MIN_I64;                              // stays so unless swPrepare frames the problem
    }
    bool found = false;
    if (warpFill) {
        ht2_dp_round(A, work + (size_t)blockIdx.x * 32, j < n ? (int)lane : -1, lane);
        if (W) found = A.swExtendAnchor(0, W->genomeHits[0]);
    } else if (W) {
        A.attach(W);
        found = A.swExtendAnchor(0, W->genomeHits[0]);
    }
    if (!W) return;
    const Ht2Hit& gh = W->genomeHits[0];
    ht2gpu_sw_result_t& r = res[j];
    r.found = found ? 1u : 0u; r.err = W->err; r.toff = gh.toff; r.n_edits = gh.nedits;
    r.score = gh.score; r.best = A.sw->jbest;
    r.rnd_next = W->rnd.nextU32();
    // the edits are already in the reference's convention: it inverts a reverse-strand list twice (nextAlignment, hybridSearch)
    const uint32_t ne = gh.nedits < HT2GPU_SW_MAX_EDITS ? gh.nedits : HT2GPU_SW_MAX_EDITS;
    for (uint32_t k = 0; k < ne; k++) {
        const Ht2Edit& e = gh.edits[k];
        ht2gpu_edit_t& d = edits[(size_t)j * HT2GPU_SW_MAX_EDITS + k];
        d.pos = e.pos; d.chr = e.chr; d.qchr = e.qchr; d.type = e.type; d.pad = e.pad; d.snp_id = e.snpID;
    }
}

extern "C" int ht2gpu_sw_extend(ht2gpu_handle_t* h, uint32_t n, const ht2gpu_sw_job_t* jobs, const uint8_t* seq, const uint8_t* qual,
                                int warp_fill, ht2gpu_sw_result_t* res, ht2gpu_edit_t* edits)
{
    if (!h || (n && (!jobs || !seq || !qual || !res || !edits))) return HT2GPU_ERR_ARG;
    if (h->graph) { h->err = "ht2gpu_sw_extend: linear indexes only"; return HT2GPU_ERR_UNSUPPORTED; }
    if (n == 0) return HT2GPU_OK;
    size_t bases = 0;
    for (uint32_t i = 0; i < n; i++) { const size_t e = (size_t)jobs[i].read_off + jobs[i].read_len; if (e > bases) bases = e; }
    CK(cudaSetDevice(h->device));
    const uint32_t nt = (n + 31) / 32 * 32;                  // every lane of a launched warp indexes its own scratch
    DevTmp tmp;
    ht2gpu_sw_job_t* dJobs = NULL; uint8_t *dSeq = NULL, *dQual = NULL; Ht2Work* dWork = NULL; Ht2SwScratch* dScr = NULL;
    uint32_t* dPool = NULL; ht2gpu_sw_result_t* dRes = NULL; ht2gpu_edit_t* dEd = NULL;
    CK(tmp.alloc(dJobs, sizeof(ht2gpu_sw_job_t) * n));
    CK(tmp.alloc(dSeq, bases + 1));
    CK(tmp.alloc(dQual, bases + 1));
    CK(tmp.alloc(dWork, sizeof(Ht2Work) * n));
    CK(tmp.alloc(dScr, sizeof(Ht2SwScratch) * nt));
    CK(tmp.alloc(dPool, sizeof(uint32_t) * (size_t)HT2_SW_POOL_WORDS * nt));
    CK(tmp.alloc(dRes, sizeof(ht2gpu_sw_result_t) * n));
    CK(tmp.alloc(dEd, sizeof(ht2gpu_edit_t) * (size_t)HT2GPU_SW_MAX_EDITS * n));
    CK(cudaMemcpy(dJobs, jobs, sizeof(ht2gpu_sw_job_t) * n, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dSeq, seq, bases, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dQual, qual, bases, cudaMemcpyHostToDevice));
    CK(cudaMemset(dWork, 0, sizeof(Ht2Work) * n));
    CK(cudaMemset(dScr, 0, sizeof(Ht2SwScratch) * nt));
    CK(cudaMemset(dEd, 0, sizeof(ht2gpu_edit_t) * (size_t)HT2GPU_SW_MAX_EDITS * n));
    size_t lim = 0;
    CK(cudaDeviceGetLimit(&lim, cudaLimitStackSize));
    if (lim < 8192) CK(cudaDeviceSetLimit(cudaLimitStackSize, 8192));
    ht2_sw_extend_kernel<<<nt / 32, 32>>>(h->dBlob, h->P, dJobs, dSeq, dQual, n, dWork, dScr, dPool, warp_fill, dRes, dEd);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(res, dRes, sizeof(ht2gpu_sw_result_t) * n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(edits, dEd, sizeof(ht2gpu_edit_t) * (size_t)HT2GPU_SW_MAX_EDITS * n, cudaMemcpyDeviceToHost));
    return HT2GPU_OK;
}

extern "C" int ht2gpu_seed_search(ht2gpu_handle_t* h, const ht2gpu_read_batch_t* b, uint32_t maxRange, ht2gpu_seed_result_t* res)
{
    if (!h || !b || !res) return HT2GPU_ERR_ARG;
    memset(res, 0, sizeof(*res));
    SeedPriv* pv = new SeedPriv();
    res->priv = pv;
    const uint32_t n = b->n_reads;
    res->n_reads = n;
    pv->firstHit.assign((size_t)n + 1, 0);
    res->first_hit = pv->firstHit.data();
    if (n == 0) return HT2GPU_OK;
    CK(cudaSetDevice(h->device));
    SamSlot& S = h->slots[0];
    int rc = slotInit(h, S);
    if (rc) return rc;
    uint64_t h2d = 0;
    rc = uploadBatch(h, S, b, NULL, NULL, 0, h2d);
    if (rc) return rc;
    DevBatch db;
    db.seq = S.dSeq; db.qual = NULL; db.offs = S.dOffs; db.seeds = S.dSeeds; db.n_units = n; db.paired = 0; db.sw = NULL; db.swPool = NULL; db.minscTab = h->dMinsc; db.elect = 32;
#ifdef HT2_ENABLE_SPLICED
    db.splT = NULL; db.ssT = NULL;
#endif
    DevTmp tmp;
    uint32_t *dCounts = NULL, *dOffs3 = NULL;
    unsigned long long* dTot = NULL;
    SeedOut so; memset(&so, 0, sizeof(so));
    CK(tmp.alloc(dCounts, (size_t)n * 12));
    CK(tmp.alloc(dOffs3, (size_t)n * 12));
    CK(tmp.alloc(dTot, 3 * sizeof(unsigned long long)));
    CK(cudaMemsetAsync(dTot, 0, 3 * sizeof(unsigned long long), S.stream));
    so.counts = dCounts; so.offs = dOffs3; so.totals = dTot;
    const int tpb = 128;
    int grid = (int)((n + tpb - 1) / tpb);
    const int maxGrid = h->nSM * 16;
    if (grid > maxGrid) grid = maxGrid;
    CK(cudaEventRecord(S.ev[1], S.stream));
    if (h->graph) ht2_seed_kernel<true, false><<<grid, tpb, 0, S.stream>>>(h->dBlob, h->P, db, n, maxRange, so);
    else ht2_seed_kernel<false, false><<<grid, tpb, 0, S.stream>>>(h->dBlob, h->P, db, n, maxRange, so);
    CK(cudaGetLastError());
    CK(cudaEventRecord(S.ev[2], S.stream));
    std::vector<uint32_t> counts((size_t)n * 3), offs((size_t)n * 3);
    CK(cudaMemcpyAsync(counts.data(), dCounts, (size_t)n * 12, cudaMemcpyDeviceToHost, S.stream));
    CK(cudaStreamSynchronize(S.stream));
    float ms0 = 0, ms1 = 0;
    CK(cudaEventElapsedTime(&ms0, S.ev[1], S.ev[2]));
    uint64_t th = 0, te = 0, tc = 0;
    for (uint32_t i = 0; i < n; i++) {
        offs[3 * (size_t)i] = (uint32_t)th; offs[3 * (size_t)i + 1] = (uint32_t)te; offs[3 * (size_t)i + 2] = (uint32_t)tc;
        pv->firstHit[i] = (uint32_t)th;
        th += counts[3 * (size_t)i]; te += counts[3 * (size_t)i + 1]; tc += counts[3 * (size_t)i + 2];
    }
    pv->firstHit[n] = (uint32_t)th;
    if (th > 0xfffffff0ull || tc > 0xfffffff0ull) { h->err = "seed search result too large for one batch"; return HT2GPU_ERR_CAPACITY; }
    ht2gpu_seed_hit_t* dHits = NULL; uint16_t* dIe = NULL; ht2gpu_seed_coord_t* dCo = NULL;
    CK(tmp.alloc(dHits, (th + 1) * sizeof(ht2gpu_seed_hit_t)));
    CK(tmp.alloc(dIe, (te + 1) * 4));
    CK(tmp.alloc(dCo, (tc + 1) * sizeof(ht2gpu_seed_coord_t)));
    CK(cudaMemcpyAsync(dOffs3, offs.data(), (size_t)n * 12, cudaMemcpyHostToDevice, S.stream));
    so.hits = dHits; so.iedges = dIe; so.coords = dCo;
    CK(cudaEventRecord(S.ev[1], S.stream));
    if (h->graph) ht2_seed_kernel<true, true><<<grid, tpb, 0, S.stream>>>(h->dBlob, h->P, db, n, maxRange, so);
    else ht2_seed_kernel<false, true><<<grid, tpb, 0, S.stream>>>(h->dBlob, h->P, db, n, maxRange, so);
    CK(cudaGetLastError());
    CK(cudaEventRecord(S.ev[2], S.stream));
    pv->hits.resize(th); pv->iedges.resize(te * 2); pv->coords.resize(tc);
    unsigned long long tot[3] = {0, 0, 0};
    if (th) CK(cudaMemcpyAsync(pv->hits.data(), dHits, th * sizeof(ht2gpu_seed_hit_t), cudaMemcpyDeviceToHost, S.stream));
    if (te) CK(cudaMemcpyAsync(pv->iedges.data(), dIe, te * 4, cudaMemcpyDeviceToHost, S.stream));
    if (tc) CK(cudaMemcpyAsync(pv->coords.data(), dCo, tc * sizeof(ht2gpu_seed_coord_t), cudaMemcpyDeviceToHost, S.stream));
    CK(cudaMemcpyAsync(tot, dTot, sizeof(tot), cudaMemcpyDeviceToHost, S.stream));
    CK(cudaStreamSynchronize(S.stream));
    CK(cudaEventElapsedTime(&ms1, S.ev[1], S.ev[2]));
    res->n_hits = (uint32_t)th; res->hits = pv->hits.data();
    res->n_iedges = (uint32_t)te; res->iedges = pv->iedges.data();
    res->n_coords = (uint32_t)tc; res->coords = pv->coords.data();
    res->n_lf = tot[0]; res->alg_bytes = tot[1]; res->err = (uint32_t)tot[2];
    res->ms_kernel = ms0 + ms1;
    if (tot[2]) { h->err = "seed search: device capacity exceeded for some reads"; return HT2GPU_ERR_CAPACITY; }
    return HT2GPU_OK;
}

extern "C" void ht2gpu_free_seed_results(ht2gpu_seed_result_t* res)
{
    if (res && res->priv) { delete (SeedPriv*)res->priv; res->priv = NULL; }
}

// ---------------------------------------------------------------------------
// host back end (SAM)
// ---------------------------------------------------------------------------
extern "C" int ht2gpu_sam_header(ht2gpu_handle_t* h, char** out, size_t* out_len)
{
    if (!h || !out) return HT2GPU_ERR_ARG;
    std::string s;
    ht2_sam_header(s, *h->img, &h->samOut);
    char* p = (char*)malloc(s.size() + 1);
    memcpy(p, s.data(), s.size()); p[s.size()] = 0;
    *out = p; if (out_len) *out_len = s.size();
    return HT2GPU_OK;
}
extern "C" void ht2gpu_free_text(char* p) { free(p); }

// The run's read-only splice-site DB: --known-splicesite-infile / --novel-splicesite-infile (hisat2.cpp:4101-4116,
// SpliceSiteDB::read splice_site.cpp:727).  Replaces a DB loaded earlier.  Call between batches, not during one.
extern "C" int ht2gpu_load_splicesites(ht2gpu_handle_t* h, const char* known_path, const char* novel_path, uint32_t* n_sites)
{
    if (!h) return HT2GPU_ERR_ARG;
#ifdef HT2_ENABLE_SPLICED
    std::vector<Ht2SsFile> files;
    if (known_path && *known_path) files.push_back({known_path, true});
    if (novel_path && *novel_path) files.push_back({novel_path, false});
    if (h->collectSs && files.size()) { h->err = "ht2gpu: a splice-site DB cannot be loaded while novel splice sites are collected"; return HT2GPU_ERR_UNSUPPORTED; }
    if (h->dSsT) { cudaFree(h->dSsT); h->dSsT = NULL; }
    h->ssBlob.clear();
    if (n_sites) *n_sites = 0;
    if (files.empty()) return HT2GPU_OK;
    for (const Ht2SsFile& f : files) { FILE* t = fopen(f.path.c_str(), "rb"); if (!t) { h->err = "ht2gpu: cannot open " + f.path; return HT2GPU_ERR_INDEX; } fclose(t); }
    std::string err; uint32_t ns = 0;
    if (!ht2_ssdb_build(*h->img, files, h->ssBlob, ns, err)) { h->err = err; h->ssBlob.clear(); return HT2GPU_ERR_INDEX; }
    CK(cudaSetDevice(h->device));
    CK(cudaMalloc(&h->dSsT, h->ssBlob.size()));
    CK(cudaMemcpy(h->dSsT, h->ssBlob.data(), h->ssBlob.size(), cudaMemcpyHostToDevice));
    if (n_sites) *n_sites = ns;
    return HT2GPU_OK;
#else
    (void)known_path; (void)novel_path; (void)n_sites;
    h->err = "ht2gpu: built without spliced alignment"; return HT2GPU_ERR_UNSUPPORTED;
#endif
}

// --novel-splicesite-outfile (hisat2.cpp:4092, aln_sink.h:1571-1580, splice_site.cpp:190-350, 565-651): collect the
// junctions of every printed alignment while batches run through ht2gpu_*_sam / ht2gpu_run_reads, then write the
// filtered site list.  Deterministic only with an empty DB (a site learned from one read would otherwise steer later
// reads in the reference), so collecting is refused while a DB is loaded.
extern "C" int ht2gpu_collect_splicesites(ht2gpu_handle_t* h, int enable)
{
    if (!h) return HT2GPU_ERR_ARG;
    if (enable && h->dSsT) { h->err = "ht2gpu: --novel-splicesite-outfile together with a loaded splice-site DB is order dependent in the reference; not supported"; return HT2GPU_ERR_UNSUPPORTED; }
    if (enable && h->P.noSplicedAlignment) { h->err = "ht2gpu: novel splice sites need spliced alignment"; return HT2GPU_ERR_UNSUPPORTED; }
    std::lock_guard<std::mutex> lk(h->novelMu);
    if (enable && !h->collectSs) h->novel.sites.clear();
    h->collectSs = enable != 0;
    return HT2GPU_OK;
}
extern "C" int ht2gpu_write_novel_splicesites(ht2gpu_handle_t** hs, int n, const char* path, uint64_t* n_written)
{
    if (!hs || n < 1 || !hs[0] || !path) return HT2GPU_ERR_ARG;
    Ht2NovelSites all;
    for (int i = 0; i < n; i++) { if (!hs[i]) return HT2GPU_ERR_ARG; std::lock_guard<std::mutex> lk(hs[i]->novelMu); all.merge(hs[i]->novel); }
    std::string err;
    if (!all.write(*hs[0]->img, path, n_written, err)) { hs[0]->err = err; return HT2GPU_ERR_INDEX; }
    return HT2GPU_OK;
}

extern "C" int ht2gpu_format_sam(ht2gpu_handle_t* h, const ht2gpu_read_batch_t* b, const char* names,
                                 const ht2gpu_result_batch_t* res, char** out, size_t* out_len)
{
    if (!h || !b || !res || !names || !out) return HT2GPU_ERR_ARG;
    unsigned nth = std::thread::hardware_concurrency();
    if (const char* e = getenv("HT2GPU_THREADS")) nth = (unsigned)atoi(e);
    return ht2_format_batch(*h->img, h->P, b, names, res, out, out_len, nth, h->ssBlob.empty() ? NULL : h->ssBlob.data(),
                            NULL, NULL, 0, &h->samOut) ? HT2GPU_OK : HT2GPU_ERR_ARG;
}

// Read outcomes for --un / --al / --un-conc / --al-conc / --al-conc-disc (ht2gpu.h): the counting pass stores them
// only while enabled, so a handle that never asks runs exactly the kernels and copies it ran without them.
extern "C" int ht2gpu_record_outcomes(ht2gpu_handle_t* h, int enable)
{
    if (!h) return HT2GPU_ERR_ARG;
    for (int k = 0; k < HT2GPU_N_SLOTS; k++)
        if (h->slots[k].pending) { h->err = "ht2gpu_record_outcomes: a batch is in flight (call ht2gpu_wait_sam first)"; return HT2GPU_ERR_ARG; }
    h->recordOut = enable != 0;
    return HT2GPU_OK;
}

extern "C" int ht2gpu_unit_outcomes(ht2gpu_handle_t* h, int slot, const uint8_t** bytes, uint32_t* n_units)
{
    if (!h || !bytes || !n_units || slot < 0 || slot >= HT2GPU_N_SLOTS) return HT2GPU_ERR_ARG;
    const SamSlot& S = h->slots[slot];
    *bytes = NULL; *n_units = 0;
    if (!S.init || !S.outValid) {
        h->err = "ht2gpu_unit_outcomes: the slot holds no outcomes (ht2gpu_record_outcomes, then ht2gpu_wait_sam)";
        return HT2GPU_ERR_ARG;
    }
    *bytes = S.hOut; *n_units = S.units;
    return HT2GPU_OK;
}

// SAM output settings (--no-unal, --omit-sec-seq, --no-sq, --rg-id / --rg).  The read group's "RG:Z:<id>" is uploaded
// once here; the SAM kernels print it from device memory.
extern "C" int ht2gpu_set_sam_output(ht2gpu_handle_t* h, const ht2gpu_sam_output_t* cfg)
{
    if (!h || !cfg || cfg->n_rg < 0 || (cfg->n_rg > 0 && !cfg->rg)) return HT2GPU_ERR_ARG;
    for (int k = 0; k < HT2GPU_N_SLOTS; k++)
        if (h->slots[k].pending) { h->err = "ht2gpu_set_sam_output: a batch is in flight (call ht2gpu_wait_sam first)"; return HT2GPU_ERR_ARG; }
    Ht2SamOutput so;
    so.noUnal = cfg->no_unal != 0; so.omitSecSeq = cfg->omit_sec_seq != 0; so.noSq = cfg->no_sq != 0;
    if (cfg->rg_id) so.rgId = cfg->rg_id;
    for (int i = 0; i < cfg->n_rg; i++) { if (!cfg->rg[i]) return HT2GPU_ERR_ARG; so.rg.push_back(cfg->rg[i]); }
    CK(cudaSetDevice(h->device));
    for (int k = 0; k < HT2GPU_N_SLOTS; k++) if (h->slots[k].init) CK(cudaStreamSynchronize(h->slots[k].stream));
    if (h->dRgTag) { CK(cudaFree(h->dRgTag)); h->dRgTag = NULL; }
    const std::string tag = so.rgTag();
    if (!tag.empty()) {
        CK(cudaMalloc(&h->dRgTag, tag.size() + 1));
        CK(cudaMemcpy(h->dRgTag, tag.c_str(), tag.size() + 1, cudaMemcpyHostToDevice));
    }
    h->samOut = so;
    return HT2GPU_OK;
}

// The output settings of two handles are the same (ht2gpu_run_reads_multi: one run prints one kind of record)
bool ht2_same_sam_output(const ht2gpu_handle_t* a, const ht2gpu_handle_t* b) { return a->samOut == b->samOut; }

extern "C" int ht2gpu_align_counts(ht2gpu_handle_t** hs, int n, int reset, ht2gpu_align_counts_t* out)
{
    if (!hs || n < 1 || !out) return HT2GPU_ERR_ARG;
    for (int i = 0; i < n; i++) if (!hs[i]) return HT2GPU_ERR_ARG;
    memset(out, 0, sizeof(*out));
    uint64_t* o = (uint64_t*)out;
    for (int i = 0; i < n; i++) {
        std::lock_guard<std::mutex> lk(hs[i]->countMu);
        const uint64_t* c = (const uint64_t*)&hs[i]->counts;
        for (int k = 0; k < HT2_T_N; k++) o[k] += c[k];
        if (reset) memset(&hs[i]->counts, 0, sizeof(hs[i]->counts));
    }
    return HT2GPU_OK;
}
