// ht2_hostsim.cpp -- TEST-ONLY host build of the per-read state machine.
//
// Compiles ht2_core.h for the CPU so parity against oracle/_ref can be
// debugged on machines without a GPU.  Not part of the product: the shipped
// library (libht2gpu.so) has no CPU path and fails loudly without CUDA.
// usage: ht2_hostsim <index_base> <reads.fa> <out.sam> [--spliced]
//        ht2_hostsim --sw-extend <index_base> <jobs.txt> [<golden>]   (tools/swjobs.py jobs; see swExtend below)
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <string>
#include <vector>
#include <chrono>
#include "../../hisat2_b200/csrc/ht2_host.h"
#include "../../hisat2_b200/csrc/ht2_seed.h"

// Runs the explicit-stack state machine the kernels use (ht2_machine.h) to completion.
template <typename ALIGNER>
static void runRead(ALIGNER& A) {
    A.machineStart();
    while (!A.machineDone()) A.machineStep();
}

// `ht2_hostsim --seed-dump <index> <reads.fa> <no_spliced>`: host build of ht2_seed.h / ht2_graph.h,
// printing the record format of oracle/ref_dump.cpp (H / G / C lines).
template <bool GRAPH>
static void seedDump(const Ht2Image& img, const Ht2Params& P, const std::vector<Ht2HostRead>& reads) {
    const Ht2ImageHeader* H = (const Ht2ImageHeader*)img.blob.data();
    Ht2Fm<uint32_t> fm; fm.init(img.blob.data(), &H->global);
    for (size_t ri = 0; ri < reads.size(); ri++) {
        const std::vector<uint8_t>& fwv = reads[ri].seq;
        const uint32_t len = (uint32_t)fwv.size();
        if (len == 0) continue;
        std::vector<uint8_t> rc(len);
        for (uint32_t i = 0; i < len; i++) { uint8_t c = fwv[len - 1 - i]; rc[i] = c < 4 ? (uint8_t)(c ^ 3) : 4; }
        for (int fwi = 0; fwi < 2; fwi++) {
            const uint8_t* seq = fwi == 0 ? fwv.data() : rc.data();
            Ht2SeedState st; memset(&st, 0, sizeof(st)); st.len = len;
            unsigned nh = 0;
            while (!st.done) {
                Ht2SeedHit ph;
                bool ps = !GRAPH && !P.noSplicedAlignment, as = true;
                ht2_seed_partial<GRAPH>(fm, P, seq, st, ph, ps, as);
                printf("H %zu %d %u %u %u %u %u %u %u\n", ri, fwi == 0, ph.bwoff, ph.len, ph.top, ph.bot, ph.hit_type, ps, as);
                const bool blank = ph.top == HT2_IDX_MAX32;
                if (GRAPH && !blank) {
                    printf("G %zu %d %u %u %u %u", ri, fwi == 0, nh, ph.node_top, ph.node_bot, ph.niedges);
                    for (uint32_t e = 0; e < ph.niedges; e++) printf(" %u:%u", ph.iedges[e][0], ph.iedges[e][1]);
                    printf("\n");
                }
                if (!blank && ph.node_bot - ph.node_top <= 4) {
                    for (uint32_t i = 0; i < ph.node_bot - ph.node_top; i++) {
                        uint32_t row; uint32_t joff = ht2_seed_elt_offset<GRAPH>(fm, ph, i, row, st);
                        uint32_t tidx = HT2_IDX_MAX32, toff = 0, lo = 0, hi = H->global.nFrag, elt = HT2_IDX_MAX32;
                        while (true) {
                            uint32_t old = elt; elt = lo + ((hi - lo) >> 1);
                            if (old == elt) break;
                            uint32_t lower = fm.rstarts[elt * 3], upper = (elt == H->global.nFrag - 1) ? fm.g->len : fm.rstarts[(elt + 1) * 3];
                            if (lower <= joff) { if (upper > joff) { tidx = fm.rstarts[elt * 3 + 1]; toff = joff - lower + fm.rstarts[elt * 3 + 2]; break; } lo = elt; }
                            else hi = elt;
                        }
                        printf("C %zu %d %u %u %u %u %u\n", ri, fwi == 0, nh, row, joff, tidx, toff);
                    }
                }
                nh++;
                if (st.done) break;
                if (!ps) { if (st.cur + 1 < st.len) st.cur++; }
            }
        }
    }
}

#ifdef HT2_ENABLE_SPLICED
static std::vector<uint8_t> g_ssBlob;      // HT2_SS=<known-splicesite file>[,<novel-splicesite file>]: the run's splice-site DB (ht2_ssdb.h)
#define HT2_SS_BLOB (g_ssBlob.empty() ? (const uint8_t*)NULL : g_ssBlob.data())
#define HT2_SET_SPLT(A) do { (A).splT = &ht2_spl_tables(); (A).ssT = HT2_SS_BLOB; } while (0)
#else
#define HT2_SS_BLOB ((const uint8_t*)NULL)
#define HT2_SET_SPLT(A) (void)0
#endif

template <bool GRAPH>
static int alignAll(Ht2Image* img, Ht2Params& P, std::vector<Ht2HostRead>& reads, std::vector<Ht2HostRead>& reads2, bool pairedMode,
                    const char* outPath) {
    std::string sam;
    ht2_sam_header(sam, *img);
    // The results are handed over in the C ABI's batch structures (what the kernels' finish step writes,
    // ht2_gpu.cu ht2_finish_unit) and ht2_format_batch -- the body of ht2gpu_format_sam, i.e. the formatter of
    // ht2_sam.h that the device SAM kernel also runs -- prints them, on HT2_THREADS host threads
    const bool viaBatch = true;
    std::vector<ht2gpu_read_result_t> bReads; std::vector<ht2gpu_aln_t> bAlns; std::vector<ht2gpu_edit_t> bEdits; std::vector<uint16_t> bPairs;
    auto collect = [&](const Ht2Work* Wk) {
        ht2gpu_read_result_t rr; memset(&rr, 0, sizeof(rr));
        rr.aln_off = (uint32_t)bAlns.size(); rr.pair_off = (uint32_t)(bPairs.size() / 2);
        rr.n_aln[0] = (uint16_t)Wk->nRes[0]; rr.n_aln[1] = (uint16_t)Wk->nRes[1]; rr.n_pairs = Wk->nPairs;
        rr.rng_state = Wk->rnd.last; rr.err = Wk->err;
        for (uint32_t m = 0; m < 2; m++) for (uint32_t i = 0; i < Wk->nRes[m]; i++) {
            const Ht2Res& r = Wk->res[m][i];
            ht2gpu_aln_t d; memset(&d, 0, sizeof(d));
            d.tidx = r.tidx; d.toff = r.toff; d.score = (int32_t)r.score; d.fw = (uint8_t)r.fw; d.mate = (uint8_t)m;
            d.n_edits = (uint16_t)r.nedits; d.trim5 = (uint16_t)r.trim5p; d.trim3 = (uint16_t)r.trim3p; d.ref_extent = r.rfextent;
            d.edit_off = (uint32_t)bEdits.size();
            const Ht2Edit* red = Wk->resEdits + r.editOff;
            for (uint32_t k = 0; k < r.nedits; k++) {
                ht2gpu_edit_t e; e.pos = red[k].pos; e.chr = red[k].chr; e.qchr = red[k].qchr; e.type = red[k].type; e.pad = red[k].pad; e.snp_id = red[k].snpID;
                bEdits.push_back(e);
            }
            bAlns.push_back(d);
        }
        for (uint32_t k = 0; k < Wk->nPairs; k++) { bPairs.push_back(Wk->pairs[k][0]); bPairs.push_back(Wk->pairs[k][1]); }
        bReads.push_back(rr);
    };
    Ht2Work* W = new Ht2Work();
    Ht2SwScratch* swScratch = P.bowtie2Dp ? new Ht2SwScratch() : NULL;
    uint32_t* swPool = P.bowtie2Dp ? new uint32_t[HT2_SW_POOL_WORDS] : NULL;
    Ht2AlignerT<GRAPH> A;
    size_t nerr = 0;
    uint64_t nLF = 0;
    long long finishNs = 0;
    uint32_t mx[8] = {0,0,0,0,0,0,0,0};
    for (size_t i = 0; pairedMode && i < reads.size(); i++) {
        Ht2HostRead& r1 = reads[i]; Ht2HostRead& r2 = reads2[i];
        r1.seed = ht2_gen_rand_seed(r1, 0); r2.seed = ht2_gen_rand_seed(r2, 0);
        int64_t ms1 = ht2_minsc(P, (uint32_t)r1.seq.size()), ms2 = ht2_minsc(P, (uint32_t)r2.seq.size());
        Ht2ReadFilters f1 = ht2_filters(r1, ms1), f2 = ht2_filters(r2, ms2);
        A.bind(img->blob.data(), &P, W); A.sw = swScratch; A.swPl = swPool; A.swStride = 1; HT2_SET_SPLT(A);
        W->err = 0; W->localindexatts = 0; W->maxLocalindexatts = 0; W->nLF = 0; W->nSides = 0; W->algBytes = 0; W->maxPool = W->maxDepth = W->maxEdits = 0;
        bool p1 = f1.pass(), p2 = f2.pass();
        W->rnd.init((p1 && p2) ? (r1.seed ^ r2.seed) : r1.seed);
        A.nofw[0] = P.gMate1fw ? P.nofw : P.norc; A.norc[0] = P.gMate1fw ? P.norc : P.nofw;
        A.nofw[1] = P.gMate2fw ? P.nofw : P.norc; A.norc[1] = P.gMate2fw ? P.norc : P.nofw;
        A.sinkReset(true);
        if (r1.seq.size() > HT2_MAX_RDLEN || r2.seq.size() > HT2_MAX_RDLEN) W->err |= HT2_ERR_RDLEN;
        if (!W->err) {
            if (p1 && p2) {
                A.paired = true; A.rightendonly = false; A.minsc[0] = ms1; A.minsc[1] = ms2;
                ht2_fill_read(W->rd[0], r1); ht2_fill_read(W->rd[1], r2);
                runRead(A);
            } else if (p1 || p2) {
                A.paired = false; A.rightendonly = !p1;
                bool nf = A.nofw[p1 ? 0 : 1], nr = A.norc[p1 ? 0 : 1];
                A.nofw[0] = nf; A.norc[0] = nr; A.nofw[1] = true; A.norc[1] = true;
                A.minsc[0] = p1 ? ms1 : ms2; A.minsc[1] = HT2_IDX_MAX32;
                ht2_fill_read(W->rd[0], p1 ? r1 : r2);
                runRead(A);
            }
        }
        nLF += W->nLF;
        if (W->err) { nerr++; fprintf(stderr, "pair %zu (%s): err=0x%x\n", i, r1.name.c_str(), W->err); }
        { uint32_t v[8] = {W->maxPool, W->maxDepth, W->maxEdits, W->nSearched[0] > W->nSearched[1] ? W->nSearched[0] : W->nSearched[1], W->nRes[0] > W->nRes[1] ? W->nRes[0] : W->nRes[1], W->nGenomeHits, W->nPairs, 0};
          for (int k = 0; k < 8; k++) if (v[k] > mx[k]) mx[k] = v[k]; }
        if (!(p1 || p2) || (W->err & HT2_ERR_RDLEN)) { W->nRes[0] = W->nRes[1] = 0; W->nPairs = 0; }
        collect(W);
    }
    for (size_t i = 0; !pairedMode && i < reads.size(); i++) {
        Ht2HostRead& rd = reads[i];
        rd.seed = ht2_gen_rand_seed(rd, 0);
        int64_t minsc = ht2_minsc(P, (uint32_t)rd.seq.size());
        Ht2ReadFilters f = ht2_filters(rd, minsc);
        A.bind(img->blob.data(), &P, W); A.sw = swScratch; A.swPl = swPool; A.swStride = 1; HT2_SET_SPLT(A);
        W->err = 0; W->localindexatts = 0; W->maxLocalindexatts = 0; W->nLF = 0; W->nSides = 0; W->algBytes = 0; W->maxPool = W->maxDepth = W->maxEdits = 0;
        W->rnd.init(rd.seed);
        A.paired = false; A.rightendonly = false;
        A.nofw[0] = P.nofw; A.norc[0] = P.norc; A.nofw[1] = true; A.norc[1] = true;
        A.minsc[0] = minsc; A.minsc[1] = HT2_IDX_MAX32;
        A.sinkReset(false);
        if (rd.seq.size() > HT2_MAX_RDLEN) W->err |= HT2_ERR_RDLEN;
        if (f.pass() && !W->err) {
            ht2_fill_read(W->rd[0], rd);
            runRead(A);
        }
        nLF += W->nLF;
        { uint32_t v[8] = {W->maxPool, W->maxDepth, W->maxEdits, W->nSearched[0], W->nRes[0], W->nGenomeHits, W->hits[0][0].nhits, W->hits[0][1].nhits};
          for (int k = 0; k < 8; k++) if (v[k] > mx[k]) mx[k] = v[k]; }
        if (W->err) { nerr++; fprintf(stderr, "read %zu (%s): err=0x%x\n", i, rd.name.c_str(), W->err); }
        if (!f.pass() || (W->err & HT2_ERR_RDLEN)) { W->nRes[0] = W->nRes[1] = 0; W->nPairs = 0; }
        collect(W);
    }
    if (viaBatch) {
        std::vector<uint8_t> seq, qual; std::vector<uint64_t> offs(1, 0); std::string names;
        auto add = [&](const Ht2HostRead& r) { seq.insert(seq.end(), r.seq.begin(), r.seq.end()); qual.insert(qual.end(), r.qual.begin(), r.qual.end());
                                               offs.push_back(seq.size()); names += r.name; names.push_back('\0'); };
        for (size_t i = 0; i < reads.size(); i++) { add(reads[i]); if (pairedMode) add(reads2[i]); }
        ht2gpu_read_batch_t rb; memset(&rb, 0, sizeof(rb));
        rb.n_reads = (uint32_t)(offs.size() - 1); rb.paired = pairedMode ? 1 : 0; rb.seq = seq.data(); rb.qual = qual.data(); rb.offs = offs.data();
        ht2gpu_result_batch_t res; memset(&res, 0, sizeof(res));
        res.n_reads = (uint32_t)bReads.size(); res.reads = bReads.data(); res.n_alns = (uint32_t)bAlns.size(); res.alns = bAlns.data();
        res.n_edits = (uint32_t)bEdits.size(); res.edits = bEdits.data(); res.n_pairs = (uint32_t)(bPairs.size() / 2); res.pairs = bPairs.data();
        char* txt = NULL; size_t len = 0;
        const unsigned nth = getenv("HT2_THREADS") ? (unsigned)atoi(getenv("HT2_THREADS")) : 1;
        auto t0 = std::chrono::steady_clock::now();
        // HT2_SS_OUT=<file>: --novel-splicesite-outfile through the formatter's junction collection
        const char* ssOut = getenv("HT2_SS_OUT");
        uint32_t colCount = 0; std::vector<Ht2SsRec> colRecs(ssOut ? rb.n_reads * 4 + 16 : 0);
        if (!ht2_format_batch(*img, P, &rb, names.c_str(), &res, &txt, &len, nth, HT2_SS_BLOB, ssOut ? &colCount : NULL, colRecs.data(), (uint32_t)colRecs.size())) { fprintf(stderr, "ht2_format_batch failed\n"); return 1; }
        if (ssOut) {
            Ht2NovelSites ns; ns.add(colRecs.data(), colCount < colRecs.size() ? colCount : colRecs.size());
            uint64_t nw = 0; std::string e2;
            if (!ns.write(*img, ssOut, &nw, e2)) { fprintf(stderr, "%s\n", e2.c_str()); return 1; }
            fprintf(stderr, "novel splice sites: %u junction records, %zu sites, %llu written\n", colCount, ns.sites.size(), (unsigned long long)nw);
        }
        finishNs += (std::chrono::steady_clock::now() - t0).count();
        sam.append(txt, len); free(txt);
    }
    FILE* fo = fopen(outPath, "wb");
    fwrite(sam.data(), 1, sam.size(), fo);
    fclose(fo);
    fprintf(stderr, "SAM back end: %.1f ms total, %.2f us per read\n", finishNs / 1e6, finishNs / 1e3 / (double)reads.size());
    fprintf(stderr, "reads=%zu errors=%zu LF=%llu maxPool=%u maxDepth=%u maxEdits=%u maxSearched=%u maxRes=%u maxGH=%u maxPH=%u/%u sizeof(Work)=%zu\n", reads.size(), nerr, (unsigned long long)nLF, mx[0], mx[1], mx[2], mx[3], mx[4], mx[5], mx[6], mx[7], sizeof(Ht2Work));
    return 0;
}

// --sw-selftest N SEED: pins the striped s16x2 fill (ht2_sw.h swFill) and the plane-derived backtrace against
// an independent, plain scalar statement of the same saturating Gotoh recurrences: every last-row score must
// be equal, and the edits returned for the best candidate must turn the read into the reference window
// they claim, at exactly that score.
static int swSelfTest(int n, unsigned seed) {
    Ht2Params P; memset(&P, 0, sizeof(P));
    Ht2Work* W = new Ht2Work(); Ht2SwScratch* S = new Ht2SwScratch();
    Ht2AlignerT<false> A; A.blob = NULL; A.H = NULL; A.P = &P; A.W = W; A.sw = S; A.swPl = new uint32_t[HT2_SW_POOL_WORDS]; A.swStride = 1; A.swStage = 0;
    uint32_t rng = seed ? seed : 1;
    auto rnd = [&](uint32_t m) { rng = rng * 1664525u + 1013904223u; return (rng >> 8) % m; };
    int bad = 0; long cells = 0, traced = 0;
    for (int it = 0; it < n; it++) {
        P.mmpMax = 2 + rnd(6); P.mmpMin = 1 + rnd(P.mmpMax); P.npen = 1 + rnd(2); P.mmcostConstant = rnd(4) == 0;
        P.rdGapConst = 1 + rnd(8); P.rdGapLinear = 1 + rnd(4); P.rfGapConst = 1 + rnd(8); P.rfGapLinear = 1 + rnd(4);
        P.gapbar = 1 + rnd(12);
        // rows 1..256: the first problems take 256 and every 32k +- 1 (the warp fill's row blocks), the rest any length;
        // a quarter of the rectangles are narrowed by up to 20 columns, as frameSeedExtensionRect trims at a contig end
        static const uint32_t edgeRows[] = {256, 1, 31, 33, 63, 65, 95, 97, 127, 129, 159, 161, 191, 193, 223, 225, 255};
        const uint32_t nrow = it < (int)(sizeof(edgeRows) / sizeof(edgeRows[0])) ? edgeRows[it] : 1 + rnd(HT2_SW_MAX_RDLEN);
        const uint32_t ncol = nrow + 40 - (rnd(4) == 0 ? rnd(21) : 0);
        std::vector<uint8_t> ref(ncol + 8), rd, qu;
        for (auto& c : ref) c = rnd(50) == 0 ? 4 : rnd(4);
        for (uint32_t j = ncol - nrow > 20 ? 20 : ncol - nrow; rd.size() < nrow && j < ncol;) {   // the read: the window with substitutions and small indels
            uint32_t r = rnd(100);
            if (r < 3) { rd.push_back((uint8_t)rnd(4)); }                        // insertion in the read
            else if (r < 6) { j++; }                                               // deletion
            else { rd.push_back(r < 12 ? (uint8_t)rnd(5) : ref[j]); j++; }
        }
        while (rd.size() < nrow) rd.push_back((uint8_t)rnd(4));
        for (uint32_t i = 0; i < nrow; i++) qu.push_back((uint8_t)(33 + rnd(42)));
        const int64_t minsc = -(int64_t)(10 + rnd(3 * nrow));
        W->err = 0;
        int64_t best = A.swFill(rd.data(), qu.data(), nrow, ref.data(), ncol, minsc);
        // scalar statement (score space: 0 = perfect, no floor needed in 64-bit; barrier = -inf)
        const int64_t NEG = -(1ll << 40);
        std::vector<int64_t> Hp(nrow, NEG), Ep(nrow, NEG), Hc(nrow), Ec(nrow), last(ncol);
        const int rdo = P.rdGapConst + P.rdGapLinear, rde = P.rdGapLinear, rfo = P.rfGapConst + P.rfGapLinear, rfe = P.rfGapLinear;
        for (uint32_t j = 0; j < ncol; j++) {
            int64_t f = NEG, hup = NEG;
            for (uint32_t i = 0; i < nrow; i++) {
                const bool gb = i < (uint32_t)P.gapbar || nrow - 1 - i < (uint32_t)P.gapbar;
                const int rdc = rd[i], rfc = ref[j];
                const int pen = (rdc > 3 || rfc > 3) ? P.npen : (rdc == rfc ? 0 : ht2_mmpen(P, (int)qu[i] - 33));
                int64_t e = NEG; if (!gb && j > 0) e = std::max(Ep[i] - rde, Hp[i] - rdo); else if (j > 0) e = Ep[i] - rde;
                int64_t ff = NEG; if (!gb && i > 0) ff = std::max(f - rfe, hup - rfo);
                const int64_t hd = (i == 0) ? 0 : (j == 0 ? NEG : Hp[i - 1]);
                int64_t h = std::max(std::max(hd - pen, e), ff);
                if (h < NEG) h = NEG; if (e < NEG) e = NEG;
                Hc[i] = h; Ec[i] = e; f = ff; hup = h;
            }
            last[j] = Hc[nrow - 1]; Hp = Hc; Ep = Ec;
        }
        int64_t sbest = NEG; for (uint32_t j = 0; j < ncol; j++) sbest = std::max(sbest, last[j]);
        cells += (long)nrow * ncol;
        const bool reach = sbest >= minsc && sbest > -16000;
        if ((best != HT2_MIN_I64) != reach || (reach && best != sbest)) { fprintf(stderr, "selftest %d: best %lld vs scalar %lld (minsc %lld)\n", it, (long long)best, (long long)sbest, (long long)minsc); bad++; continue; }
        if (!reach) continue;
        for (uint32_t j = 0; j < ncol; j++) if (last[j] > -16000 && S->lastH[j] != last[j]) { fprintf(stderr, "selftest %d: column %u %d vs %lld\n", it, j, S->lastH[j], (long long)last[j]); bad++; break; }
        // backtrace from the best, right-most candidate; check the edits against read and window
        uint32_t cc = 0; for (uint32_t j = 0; j < ncol; j++) if (last[j] == sbest) cc = j;
        typename Ht2AlignerT<false>::SwRect rect; rect.refl = 0; rect.refr = ncol - 1; rect.triml = 0; rect.trimr = 0; rect.corel = 0; rect.corer = ncol + nrow;
        uint32_t ned = 0, off = 0; int64_t score = 0;
        if (!A.swBacktrace(rd.data(), qu.data(), nrow, ref.data(), rect, (int)nrow, nrow - 1, cc, ned, off, score)) { fprintf(stderr, "selftest %d: backtrace failed\n", it); bad++; continue; }
        traced++;
        int64_t sc2 = 0; uint32_t rp = off, k = 0; bool ok = score == sbest; int prevGap = 0; uint32_t prevPos = 0;
        for (uint32_t i = 0; i < nrow && ok; i++) {
            while (k < ned && S->ned[k].type == HT2_EDIT_READ_GAP && S->ned[k].pos == i) {   // reference bases skipped before row i
                ok = ok && S->ned[k].chr == "ACGTN"[ref[rp]]; sc2 -= (prevGap == 1 && prevPos == i) ? rde : rdo; prevGap = 1; prevPos = i; rp++; k++;
            }
            if (k < ned && S->ned[k].pos == i && S->ned[k].type == HT2_EDIT_REF_GAP) { sc2 -= (prevGap == 2 && prevPos + 1 == i) ? rfe : rfo; prevGap = 2; prevPos = i; k++; continue; }
            const int rdc = rd[i], rfc = ref[rp];
            if (k < ned && S->ned[k].pos == i && S->ned[k].type == HT2_EDIT_MM) {
                ok = ok && (rdc != rfc || rdc > 3) && S->ned[k].chr == "ACGTN"[rfc] && S->ned[k].qchr == "ACGTN"[rdc];
                sc2 -= (rdc > 3 || rfc > 3) ? P.npen : ht2_mmpen(P, (int)qu[i] - 33); k++;
            } else ok = ok && rdc == rfc && rdc <= 3;
            prevGap = 0; rp++;
        }
        ok = ok && k == ned && rp == cc + 1 && sc2 == sbest;
        if (!ok) { fprintf(stderr, "selftest %d: edits do not reproduce the alignment (score %lld, recomputed %lld, optimum %lld)\n", it, (long long)score, (long long)sc2, (long long)sbest); bad++; }
    }
    printf("sw selftest: %d problems, %ld cells, %ld backtraces, %d failures\n", n, cells, traced, bad);
    return bad ? 1 : 0;
}

// --sw-extend INDEX JOBS [GOLDEN]: the --bowtie2-dp seed extension (swExtendAnchor = swPrepare + swFill + swFinish)
// on the jobs of tools/swjobs.py, one result line per job in the format of oracle/ref_sw plus the error bits:
//   <id> <found> <off|-> <score|-> <best|-> <rnd.nextU32() after> <edits|-> <err>
// With GOLDEN (tests/golden/sw_extend_ref.txt), every job's first seven fields must equal the reference's (its best
// only where it reaches minsc), except for the jobs the device refuses by design: reads over 256 bases and minsc
// below -15000 (HT2_ERR_SW), alignments of more than HT2_MAX_EDITS edits, and jobs the reference finds nothing for
// whose rejected candidates ran past the backtrace's HT2_SW_MAX_EDITS edits (HT2_ERR_EDITS).  Prints a summary line; exit 1 on a mismatch.
static int swExtend(const char* index, const char* jobsPath, const char* goldenPath) {
    std::string err;
    Ht2Image* img = ht2_image_load(index, err);
    if (!img) { fprintf(stderr, "%s\n", err.c_str()); return 1; }
    FILE* fj = fopen(jobsPath, "r");
    if (!fj) { fprintf(stderr, "cannot open %s\n", jobsPath); return 1; }
    std::vector<std::string> golden;
    if (goldenPath) {
        FILE* fg = fopen(goldenPath, "r");
        if (!fg) { fprintf(stderr, "cannot open %s\n", goldenPath); return 1; }
        char* gl = NULL; size_t gcap = 0;
        while (getline(&gl, &gcap, fg) > 0) { std::string s(gl); while (!s.empty() && (s.back() == '\n' || s.back() == '\r')) s.pop_back(); golden.push_back(s); }
        free(gl); fclose(fg);
        if (!golden.empty()) golden.erase(golden.begin());   // the job stream's sha1
    }
    Ht2Params P;
    ht2_default_params(P, *img, true);
    P.bowtie2Dp = 2;
    Ht2Work* W = new Ht2Work();
    Ht2SwScratch* S = new Ht2SwScratch();
    uint32_t* pool = new uint32_t[HT2_SW_POOL_WORDS];
    Ht2AlignerT<false> A;
    char* line = NULL; size_t cap = 0;
    size_t n = 0, bad = 0, flagged = 0;
    std::vector<char> rd(4096), qu(4096);
    while (getline(&line, &cap, fj) > 0) {
        long long id, mpMax, mpMin, ignq, np, rdc, rdl, rfc, rfl, gbar, fw, tidx, toff, rdoff, len, minsc; unsigned long long seed;
        if (sscanf(line, "%lld %lld %lld %lld %lld %lld %lld %lld %lld %lld %lld %lld %lld %lld %lld %lld %llu %4095s %4095s", &id, &mpMax, &mpMin,
                   &ignq, &np, &rdc, &rdl, &rfc, &rfl, &gbar, &fw, &tidx, &toff, &rdoff, &len, &minsc, &seed, rd.data(), qu.data()) != 19) {
            fprintf(stderr, "malformed job line: %s", line); return 1;
        }
        P.mmpMax = (int)mpMax; P.mmpMin = (int)mpMin; P.mmcostConstant = ignq != 0; P.npen = (int)np;
        P.rdGapConst = (int)rdc; P.rdGapLinear = (int)rdl; P.rfGapConst = (int)rfc; P.rfGapLinear = (int)rfl; P.gapbar = (int)gbar;
        Ht2HostRead hr;
        for (const char* c = rd.data(); *c; c++) hr.seq.push_back((uint8_t)ht2_asc2code((uint8_t)*c));
        for (const char* c = qu.data(); *c; c++) hr.qual.push_back((uint8_t)*c);
        memset(W, 0, sizeof(Ht2Work));
        A.bind(img->blob.data(), &P, W); A.sw = S; A.swPl = pool; A.swStride = 1;
        A.minsc[0] = minsc; A.minsc[1] = HT2_IDX_MAX32;
        ht2_fill_read(W->rd[0], hr);
        W->rnd.init((uint32_t)seed);
        Ht2Hit gh; memset(&gh, 0, sizeof(gh));
        Ht2AlignerT<false>::initHit(gh, fw != 0, (uint32_t)rdoff, (uint32_t)len, 0, 0, (uint32_t)tidx, (uint32_t)toff, (uint32_t)toff);
        const bool found = A.swExtendAnchor(0, gh);
        const bool dp = (uint32_t)len < W->rd[0].len;
        char out[8192]; int o = 0;
        o += snprintf(out + o, sizeof(out) - o, "%lld %d ", id, found ? 1 : 0);
        if (found && dp) o += snprintf(out + o, sizeof(out) - o, "%u %lld ", gh.toff, (long long)gh.score);
        else o += snprintf(out + o, sizeof(out) - o, "- - ");
        if (dp && S->jbest != HT2_MIN_I64 && !W->err) o += snprintf(out + o, sizeof(out) - o, "%lld ", (long long)S->jbest);
        else o += snprintf(out + o, sizeof(out) - o, "- ");
        o += snprintf(out + o, sizeof(out) - o, "%u ", W->rnd.nextU32());
        if (found && dp) {   // the reference inverts a reverse-strand edit list twice (nextAlignment, hybridSearch)
            for (uint32_t k = 0; k < gh.nedits; k++)
                o += snprintf(out + o, sizeof(out) - o, "%s%u:%u:%c:%c", k ? "," : "", gh.edits[k].pos, gh.edits[k].type, gh.edits[k].chr, gh.edits[k].qchr);
        }
        if (!found || !dp || gh.nedits == 0) o += snprintf(out + o, sizeof(out) - o, "-");
        snprintf(out + o, sizeof(out) - o, " %u", W->err);
        printf("%s\n", out);
        if (W->err) flagged++;
        if (goldenPath) {
            if (n >= golden.size()) { fprintf(stderr, "job %lld: no golden line\n", id); bad++; n++; continue; }
            std::string g = golden[n];
            {   // the reference's best is the best last-row score even below minsc; the device keeps only a best >= minsc
                std::vector<std::string> f; size_t a = 0;
                for (size_t b; (b = g.find(' ', a)) != std::string::npos; a = b + 1) f.push_back(g.substr(a, b - a));
                f.push_back(g.substr(a));
                if (f.size() == 7 && f[4] != "-" && atoll(f[4].c_str()) < minsc) { f[4] = "-"; g = f[0]; for (size_t k = 1; k < 7; k++) g += " " + f[k]; }
            }
            // expected refusals: reads over the planes' 256 rows, minsc below -15000, more edits than a hit holds
            size_t gedits = 0; { size_t p = g.rfind(' '); std::string e = g.substr(p + 1); if (e != "-") { gedits = 1; for (char c : e) if (c == ',') gedits++; } }
            uint32_t want = 0;
            if (dp && (W->rd[0].len > HT2_SW_MAX_RDLEN || minsc < -15000)) want = HT2_ERR_SW;
            else if (dp && gedits > HT2_MAX_EDITS) want = HT2_ERR_EDITS;
            std::string mine(out); mine = mine.substr(0, mine.rfind(' '));
            // a rejected candidate whose path runs past the backtrace's HT2_SW_MAX_EDITS edits is flagged as well
            const bool overran = W->err == HT2_ERR_EDITS && !want && g.compare(0, g.find(' ') + 2, std::to_string(id) + " 0") == 0;
            if (!overran && (W->err != want || (!want && mine != g))) {
                fprintf(stderr, "job %lld differs (err %u, expected %u)\n  host:      %s\n  reference: %s\n", id, W->err, want, mine.c_str(), g.c_str());
                bad++;
            }
        }
        n++;
    }
    free(line); fclose(fj);
    if (goldenPath && n != golden.size()) { fprintf(stderr, "%zu jobs, %zu golden lines\n", n, golden.size()); bad++; }
    fprintf(stderr, "sw extend: %zu jobs, %zu flagged, %zu mismatches\n", n, flagged, bad);
    return bad ? 1 : 0;
}

int main(int argc, char** argv) {
    if (argc >= 3 && !strcmp(argv[1], "--sw-selftest")) return swSelfTest(atoi(argv[2]), argc > 3 ? (unsigned)atoi(argv[3]) : 1u);
    if (argc >= 4 && !strcmp(argv[1], "--sw-extend")) return swExtend(argv[2], argv[3], argc > 4 ? argv[4] : NULL);
    if (argc >= 5 && !strcmp(argv[1], "--seed-dump")) {
        std::string err;
        Ht2Image* img = ht2_image_load(argv[2], err);
        if (!img) { fprintf(stderr, "%s\n", err.c_str()); return 1; }
        std::vector<Ht2HostRead> reads;
        if (!ht2_read_fasta(argv[3], reads, 0, err)) { fprintf(stderr, "%s\n", err.c_str()); return 1; }
        Ht2Params P;
        ht2_default_params(P, *img, atoi(argv[4]) != 0);
        const Ht2ImageHeader* H = (const Ht2ImageHeader*)img->blob.data();
        if (H->global.linearFM) seedDump<false>(*img, P, reads); else seedDump<true>(*img, P, reads);
        return 0;
    }
    if (argc < 4) { fprintf(stderr, "usage: %s index reads.fa out.sam\n", argv[0]); return 2; }
    std::string err;
    Ht2Image* img = ht2_image_load(argv[1], err);
    if (!img) { fprintf(stderr, "%s\n", err.c_str()); return 1; }
    std::vector<Ht2HostRead> reads;
    // usage: ht2_hostsim index reads.fa out.sam            (unpaired)
    //        ht2_hostsim index reads_1.fa out.sam reads_2.fa (paired, --fr)
    const bool pairedMode = argc > 4;
    if (!ht2_read_reads(argv[2], reads, pairedMode ? 1 : 0, err)) { fprintf(stderr, "%s\n", err.c_str()); return 1; }
    std::vector<Ht2HostRead> reads2;
    if (pairedMode && !ht2_read_reads(argv[4], reads2, 2, err)) { fprintf(stderr, "%s\n", err.c_str()); return 1; }
    Ht2Params P;
    ht2_default_params(P, *img, true);
#ifdef HT2_ENABLE_SPLICED
    if (const char* ssf = getenv("HT2_SS")) {
        std::vector<Ht2SsFile> files;
        std::string a(ssf); size_t c = a.find(',');
        files.push_back({a.substr(0, c), true});
        if (c != std::string::npos) files.push_back({a.substr(c + 1), false});
        uint32_t ns = 0;
        if (!ht2_ssdb_build(*img, files, g_ssBlob, ns, err)) { fprintf(stderr, "%s\n", err.c_str()); return 1; }
        fprintf(stderr, "splice-site DB: %u sites\n", ns);
    }
#endif
    // HT2_OPTS="khits=1,mp_max=4,...": the ht2gpu_options_t fields, mapped like applyOptions (ht2_gpu.cu)
    if (const char* os = getenv("HT2_OPTS")) {
        std::string o(os); size_t p0 = 0;
        bool kseedsGiven = false;
        char smT = 0; double smC = (double)0.0f, smL = (double)-0.2f;
        while (p0 < o.size()) {
            size_t c = o.find(',', p0); if (c == std::string::npos) c = o.size();
            std::string kv = o.substr(p0, c - p0); p0 = c + 1;
            size_t e = kv.find('='); if (e == std::string::npos) continue;
            std::string k = kv.substr(0, e); int v = atoi(kv.c_str() + e + 1);
            if (k == "khits") P.khits = (uint32_t)v; else if (k == "max_seeds") { P.kseeds = (uint32_t)v; kseedsGiven = true; }
            else if (k == "secondary") P.secondary = v; else if (k == "mp_max") P.mmpMax = v; else if (k == "mp_min") P.mmpMin = v;
            else if (k == "sp_max") P.scpMax = v; else if (k == "sp_min") P.scpMin = v; else if (k == "np") P.npen = v;
            else if (k == "rdg_const") P.rdGapConst = v; else if (k == "rdg_linear") P.rdGapLinear = v;
            else if (k == "rfg_const") P.rfGapConst = v; else if (k == "rfg_linear") P.rfGapLinear = v;
            else if (k == "ignore_quals") P.mmcostConstant = v; else if (k == "nofw") P.nofw = v; else if (k == "norc") P.norc = v;
            else if (k == "min_frag") P.minFrag = (uint32_t)v; else if (k == "max_frag") P.maxFrag = (uint32_t)v;
            else if (k == "no_mixed") P.mixed = v ? 0 : 1; else if (k == "no_discordant") P.discord = v ? 0 : 1;
            else if (k == "spliced") P.noSplicedAlignment = v ? 0 : 1;   // experiment only: spliced joins are flagged (HT2_ERR_SPLICE), not built
            else if (k == "min_intronlen") P.minIntronLen = (uint32_t)v; else if (k == "max_intronlen") P.maxIntronLen = (uint32_t)v;
            else if (k == "pen_cansplice") P.canSplPen = v;
#ifdef HT2_ENABLE_SPLICED
            else if (k == "pen_noncansplice") P.noncanSplPen = v;
#endif
            else if (k == "bowtie2_dp") P.bowtie2Dp = (uint32_t)v; else if (k == "gbar") P.gapbar = v;
            else if (k == "score_min_type") smT = (char)v; else if (k == "score_min_const") { smC = atof(kv.c_str() + e + 1); if (!smT) smT = 'L'; }
            else if (k == "score_min_coeff") { smL = atof(kv.c_str() + e + 1); if (!smT) smT = 'L'; }
            else if (k == "score_min") {   // score_min=L:0:-0.5
                const char* t = kv.c_str() + e + 1; char ty = t[0]; double C = 0, L = 0;
                if (sscanf(t + 1, ":%lf:%lf", &C, &L) < 1 || !ht2_set_score_min(P, ty, C, L)) { fprintf(stderr, "bad score_min %s\n", t); return 2; }
            }
            else { fprintf(stderr, "unknown option %s\n", k.c_str()); return 2; }
        }
        if (!kseedsGiven) P.kseeds = P.khits * 2 > 5 ? P.khits * 2 : 5;
        if (smT && !ht2_set_score_min(P, smT, smC, smL)) { fprintf(stderr, "bad score_min_type\n"); return 2; }
    }
    const Ht2ImageHeader* Hh = (const Ht2ImageHeader*)img->blob.data();
    return Hh->global.linearFM ? alignAll<false>(img, P, reads, reads2, pairedMode, argv[3])
                               : alignAll<true>(img, P, reads, reads2, pairedMode, argv[3]);
}

