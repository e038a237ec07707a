// ht2_sam.h -- the SAM back end of one read (pair): AlnSinkWrap::finishRead, allocation-free, host + device.
//
// One source serves the device kernel (ht2_sam_kernel in ht2_gpu.cu: one thread per unit, a counting pass
// and a writing pass) and the host entry points (ht2gpu_format_sam, tests/hostsim).  It turns the flat result
// records of the alignment kernel (ht2gpu_read_result_t / ht2gpu_aln_t / ht2gpu_edit_t) plus the read batch
// into the reference's SAM records, byte for byte:
//   AlnSinkWrap::finishRead            aln_sink.h:1939-2560   (concordant > discordant > unpaired > unaligned)
//   AlnSinkWrap::selectByScore         aln_sink.h:2680-2755   (HISAT2 score key, Fisher-Yates over equal keys)
//   AlnSetSumm                         aligner_result.cpp:1167-1260
//   BowtieMapq2::mapq                  unique.h:170-420
//   AlnSinkSam::appendMate             aln_sink.h:3024-3250
//   StackedAln (CIGAR / MD:Z)          aligner_result.h:723-895, aligner_result.cpp:660-1000
//   SamConfig::printAlignedOptFlags    sam.h:525-1032
//   AlnRes::setFragmentLength          aligner_result.h:1631-1697
#ifndef HT2_SAM_H_
#define HT2_SAM_H_

#include "ht2_core.h"
#include "../../include/ht2gpu.h"

#ifndef HT2_SAM_MAXSEL
#define HT2_SAM_MAXSEL (HT2_MAX_RES > HT2_MAX_PAIRS ? HT2_MAX_RES : HT2_MAX_PAIRS)
#endif
#define HT2_SAM_MAXCOLS (HT2_MAX_RDLEN + HT2_SW_MAX_EDITS + 8)

// Everything one batch's formatter reads; all pointers live in the memory space the caller runs in.
struct Ht2SamIn {
    const uint8_t*  blob;        // index image (reference names, ALT table + names)
    const int32_t*  minscTab;    // --score-min per read length (Ht2Params::minscTab)
    const uint8_t*  seq;         // read batch (ht2gpu_read_batch_t)
    const uint8_t*  qual;        // NULL = all 'I'
    const uint64_t* offs;
    const char*     names;       // read i's name = names + nameOffs[i], '\0'-terminated
    const uint32_t* nameOffs;
    uint32_t        n_reads;
    int32_t         paired;
    const ht2gpu_read_result_t* reads;
    const ht2gpu_aln_t*         alns;
    const ht2gpu_edit_t*        edits;
    const uint16_t*             pairs;
    uint32_t khits, secondary, mixed, discord;
    const uint8_t*  ssT;         // the run's splice-site DB (ht2_ssdb.h) or NULL: template-length adjustment of concordant pairs
    uint32_t*       colCount;    // --novel-splicesite-outfile: junctions of the printed alignments (write pass only), or NULL
    Ht2SsRec*       colRecs;
    uint32_t        colCap;
    // SAM output settings (ht2gpu_set_sam_output)
    uint32_t        noUnal;      // --no-unal: appendMate prints nothing for rs == NULL (aln_sink.h:3040)
    uint32_t        omitSecSeq;  // --omit-sec-seq: SEQ / QUAL '*' in non-primary records (aln_sink.h:3190-3215)
    const char*     rgTag;       // "RG:Z:<id>" or NULL (sam.h:780, 1102)
    uint8_t*        unitOut;     // ht2gpu_record_outcomes: the counting pass stores each unit's HT2GPU_OUTCOME_* bits here, or NULL
};

// ReportingMetrics (aln_sink.h:2007-2346) of the units a formatter pass went through, in the field order of
// ht2gpu_align_counts_t.  The *_rep counters need -M: hisat2.cpp:1882-1884 sets mhits to 0 whatever the options
// (line 1883), so pairMax / unpair1Max / unpair2Max are never set and nconcord_rep, nunp_0_rep and nunp_rep stay 0;
// they are not kept.
enum { HT2_T_NREAD, HT2_T_NPAIRED, HT2_T_NUNPAIRED, HT2_T_NCONCORD_0, HT2_T_NCONCORD_UNI1, HT2_T_NCONCORD_UNI2, HT2_T_NDISCORD,
       HT2_T_NUNP_0_0, HT2_T_NUNP_0_UNI1, HT2_T_NUNP_0_UNI2, HT2_T_NUNP_0, HT2_T_NUNP_UNI1, HT2_T_NUNP_UNI2, HT2_T_N };
struct Ht2SamTally { uint32_t c[HT2_T_N]; uint32_t outcome; };   // outcome: the last unit's HT2GPU_OUTCOME_* bits
static_assert(sizeof(ht2gpu_align_counts_t) == HT2_T_N * sizeof(uint64_t), "ht2gpu_align_counts_t follows the tally's order");

// Where a pass's text goes: p + n (WRITE) or only the byte count n (the counting pass).  Ht2SamFmt::unit formats
// one unit through an Ht2SamCur and adds its length to n.
template <bool WRITE>
struct Ht2SamOut {
    char*    p;
    uint64_t n;
};

HT2_HD bool ht2_sam_isspace(char ch) { return ch == ' ' || (ch >= 9 && ch <= 13); }

// The emission helpers below are called from dozens of fields.  Each is one out-of-line leaf that takes the
// destination by value and returns the bytes it wrote (or would write, WRITE = false), so a caller's cursor stays
// in registers and no helper is copied into every call site.

// v in decimal: the digits are counted first and then stored from the last one backwards, in place.
template <bool WRITE> HT2_NI uint32_t ht2_sam_i64(char* d, int64_t v) {
    uint64_t u = v < 0 ? (uint64_t)0 - (uint64_t)v : (uint64_t)v;
    uint32_t k = 1;
    if (u >> 32) { for (uint64_t q = u; q >= 10; q /= 10) k++; }
    else { for (uint32_t q = (uint32_t)u; q >= 10; q /= 10) k++; }
    const uint32_t len = k + (v < 0);
    if (WRITE) {
        char* e = d + len;
        for (; u >> 32; u /= 10) *--e = (char)('0' + u % 10);
        uint32_t w = (uint32_t)u;
        do { *--e = (char)('0' + w % 10); w /= 10; } while (w);
        if (v < 0) *d = '-';
    }
    return len;
}

#ifdef __CUDA_ARCH__
// the 4 bytes at p, from the two aligned words that hold them (p need not be aligned; neither word is read past
// the one that holds p[3])
__device__ __forceinline__ uint32_t ht2_sam_ld4(const char* p) {
    const uintptr_t a = (uintptr_t)p;
    const uint32_t sh = (uint32_t)(a & 3) * 8;
    const uint32_t* w = (const uint32_t*)(a & ~(uintptr_t)3);
    return sh ? __funnelshift_r(w[0], w[1], sh) : w[0];
}
#endif

// Length of s up to its first '\0' or white space; atEnd = it stopped at the '\0'.  The device reads aligned words
// (no word past the one holding the stop byte, so nothing outside the string's allocation granule).
HT2_HD uint32_t ht2_sam_token(const char* s, bool& atEnd) {
#ifdef __CUDA_ARCH__
    const uintptr_t a = (uintptr_t)s;
    const uint32_t* w = (const uint32_t*)(a & ~(uintptr_t)3);
    const uint32_t head = (uint32_t)(a & 3);
    const uint32_t before = (1u << (8 * head)) - 1u;        // bytes ahead of s read as 'A'
    uint32_t x = (w[0] & ~before) | (0x41414141u & before);
    for (uint32_t k = 0;; k += 4) {
        const uint32_t z = __vcmpeq4(x, 0u);
        const uint32_t st = z | __vcmpeq4(x, 0x20202020u) | (__vcmpgeu4(x, 0x09090909u) & __vcmpleu4(x, 0x0d0d0d0du));
        if (st) {
            const uint32_t b = (uint32_t)(__ffs(st) - 1) >> 3;
            atEnd = (z >> (8 * b)) & 1u;
            return k + b - head;
        }
        x = w[(k >> 2) + 1];
    }
#else
    uint32_t i = 0;
    while (s[i] && !ht2_sam_isspace(s[i])) i++;
    atEnd = !s[i];
    return i;
#endif
}

// len bytes of s (all of them before its terminator); 4 to a store once the destination is aligned on the device
HT2_HD void ht2_sam_copy(char* d, const char* s, uint32_t len) {
    uint32_t i = 0;
#ifdef __CUDA_ARCH__
    for (; i < len && ((uintptr_t)(d + i) & 3); i++) d[i] = s[i];
    for (; i + 4 <= len; i += 4) *(uint32_t*)(d + i) = ht2_sam_ld4(s + i);
#endif
    for (; i < len; i++) d[i] = s[i];
}

// A read or reference name up to its first white space, at most cap bytes; with omitSlashMate a trailing /1, /2
// or /3 of the whole name is dropped.  White space cannot come after the '/'
// of such a suffix, so the suffix only matters when the name ends at its terminator.
template <bool WRITE> HT2_NI uint32_t ht2_sam_name(char* d, const char* name, bool omitSlashMate, uint32_t cap) {
    bool atEnd;
    uint32_t len = ht2_sam_token(name, atEnd);
    if (atEnd && omitSlashMate && len >= 2 && name[len - 2] == '/' &&
        (name[len - 1] == '1' || name[len - 1] == '2' || name[len - 1] == '3')) len -= 2;
    if (len > cap) len = cap;
    if (WRITE) ht2_sam_copy(d, name, len);
    return len;
}

// a '\0'-terminated string of the run (read group, ALT names)
template <bool WRITE> HT2_NI uint32_t ht2_sam_str(char* d, const char* z) {
    uint32_t i = 0;
    for (; z[i]; i++) if (WRITE) d[i] = z[i];
    return i;
}

// One unit's text: d + [0, n), a 32-bit offset from the unit's first byte.
template <bool WRITE>
struct Ht2SamCur {
    char*    d;
    uint32_t n;
    HT2_HD char* at() const { return WRITE ? d + n : NULL; }
    HT2_HD void c(char ch) { if (WRITE) d[n] = ch; n++; }
    // a literal: its length is known at compile time, its bytes are immediates at fixed offsets from one address
    template <uint32_t N> HT2_HD void s(const char (&lit)[N]) {
        if (WRITE) {
            char* q = d + n;
#pragma unroll
            for (uint32_t i = 0; i + 1 < N; i++) q[i] = lit[i];
        }
        n += N - 1;
    }
    HT2_HD void str(const char* z) { n += ht2_sam_str<WRITE>(at(), z); }
    HT2_HD void i64(int64_t v) { n += ht2_sam_i64<WRITE>(at(), v); }
    HT2_HD void name(const char* z, bool omitSlashMate, uint32_t cap) { n += ht2_sam_name<WRITE>(at(), z, omitSlashMate, cap); }
    // cnt bytes, byte i = byteAt(i); once the destination is 4-byte aligned, bytes i..i+3 = word4(i), one store (SEQ / QUAL)
    template <typename F, typename G> HT2_HD void run(uint32_t cnt, F byteAt, G word4) {
        if (WRITE) {
            char* q = d + n;
            uint32_t i = 0;
            for (; i < cnt && ((uintptr_t)(q + i) & 3); i++) q[i] = byteAt(i);
            for (; i + 4 <= cnt; i += 4) *(uint32_t*)(q + i) = word4(i);
            for (; i < cnt; i++) q[i] = byteAt(i);
        }
        n += cnt;
    }
};

struct Ht2SamKey { int64_t score; int64_t h2; bool valid; };
HT2_HD bool ht2_sam_key_gt(const Ht2SamKey& a, const Ht2SamKey& b) {   // AlnScore::operator> (aligner_result.h:143-157)
    if (!b.valid) return a.valid;
    if (!a.valid) return false;
    return a.score > b.score || (a.score == b.score && a.h2 > b.h2);
}
HT2_HD bool ht2_sam_key_eq(const Ht2SamKey& a, const Ht2SamKey& b) { return a.valid && b.valid && a.score == b.score && a.h2 == b.h2; }

struct Ht2SamSumm {   // AlnSetSumm (aligner_result.cpp:1167-1260)
    Ht2SamKey best[2], secbest[2], bestPaired, secbestPaired;
    bool paired;
    uint32_t numAlns[2], numAlnsPaired;
    int64_t orefid, orefoff;
    HT2_HD void reset() {
        best[0].valid = best[1].valid = secbest[0].valid = secbest[1].valid = false;
        bestPaired.valid = secbestPaired.valid = false;
        paired = false; numAlns[0] = numAlns[1] = numAlnsPaired = 0; orefid = -1; orefoff = -1;
    }
};

// AlnFlags::pairing (aligner_result.h:383-398)
enum { HT2_PAIR_CONCORD_MATE1 = 1, HT2_PAIR_CONCORD_MATE2, HT2_PAIR_DISCORD_MATE1, HT2_PAIR_DISCORD_MATE2,
       HT2_PAIR_UNPAIRED_MATE1, HT2_PAIR_UNPAIRED_MATE2, HT2_PAIR_UNPAIRED };
struct Ht2SamFlags {
    int pairing; bool primary; bool oppAligned;
    HT2_HD bool partOfPair() const { return pairing < HT2_PAIR_UNPAIRED; }
    HT2_HD bool readMate1() const { return pairing == HT2_PAIR_CONCORD_MATE1 || pairing == HT2_PAIR_DISCORD_MATE1 || pairing == HT2_PAIR_UNPAIRED_MATE1; }
    HT2_HD bool concordant() const { return pairing == HT2_PAIR_CONCORD_MATE1 || pairing == HT2_PAIR_CONCORD_MATE2; }
    HT2_HD bool discordant() const { return pairing == HT2_PAIR_DISCORD_MATE1 || pairing == HT2_PAIR_DISCORD_MATE2; }
    HT2_HD bool unpairedMate() const { return pairing == HT2_PAIR_UNPAIRED_MATE1 || pairing == HT2_PAIR_UNPAIRED_MATE2; }
};

// One read of the batch as the formatter sees it.
struct Ht2SamRead {
    const uint8_t* seq; const uint8_t* qual; const char* name;
    uint32_t len; int mate;            // 0 unpaired, 1, 2
    uint8_t lenfilt, nfilt, scfilt;    // 1 = passes (hisat2.cpp:3417-3440)
};

struct Ht2SamFmt {
    const Ht2SamIn* in;
    const Ht2ImageHeader* IH;
    const Ht2Alt* altTab;
    uint32_t nAlts;

    HT2_HD void bind(const Ht2SamIn* i) {
        in = i; IH = (const Ht2ImageHeader*)i->blob; nAlts = IH->nAlts; altTab = (const Ht2Alt*)(i->blob + IH->o_alts);
    }
    HT2_HD const char* refName(uint32_t tidx) const {
        const uint32_t* no = (const uint32_t*)(in->blob + IH->o_nameOffs);
        return (const char*)in->blob + IH->o_names + no[tidx];
    }
    HT2_HD const char* altName(uint32_t si) const {
        const uint32_t* no = (const uint32_t*)(in->blob + IH->o_altNameOffs);
        return (const char*)in->blob + IH->o_altNames + no[si];
    }
    HT2_HD int64_t minscOf(uint32_t len) const { return in->minscTab[len <= HT2_PARAMS_MAX_RDLEN ? len : HT2_PARAMS_MAX_RDLEN]; }

    HT2_HD void mkRead(uint32_t i, int mate, Ht2SamRead& rd) const {
        const uint64_t o0 = in->offs[i];
        rd.seq = in->seq + o0; rd.qual = in->qual ? in->qual + o0 : NULL;
        rd.len = (uint32_t)(in->offs[i + 1] - o0);
        rd.name = in->names + in->nameOffs[i];
        rd.mate = mate;
        // ht2_filters (hisat2.cpp:3417-3440; Scoring::nFilter with nCeil = L,0,0.15)
        int64_t m = minscOf(rd.len); if (m > 0) m = 0;
        const uint32_t maxns = (uint32_t)((double)0.0f + (double)0.15f * (double)rd.len);
        uint32_t ns = 0;
#ifdef __CUDA_ARCH__
        {   // base codes are 0..4, so bit 2 marks an N; aligned words, bytes outside the read masked off
            const uintptr_t a = (uintptr_t)rd.seq;
            const uint32_t* w = (const uint32_t*)(a & ~(uintptr_t)3);
            const uint32_t head = (uint32_t)(a & 3), end = head + rd.len;
            for (uint32_t k = 0; k < end; k += 4) {
                uint32_t m = 0x04040404u;
                if (k == 0) m &= ~((1u << (8 * head)) - 1u);
                if (k + 4 > end) m &= (1u << (8 * (end - k))) - 1u;
                ns += (uint32_t)__popc(w[k >> 2] & m);
            }
        }
#else
        for (uint32_t k = 0; k < rd.len; k++) ns += (rd.seq[k] == 4);
#endif
        rd.nfilt = ns <= maxns; rd.scfilt = (0 >= m); rd.lenfilt = rd.len >= 2;
    }

    // AlnScore::calculate_hisat2_score (aligner_result.h:322-348), repeat = 0.  The splice part of the key
    // follows from the edits alone: GenomeHit::spliced() and the splicescore rule of calculateScore
    // (hi_aligner.h:3745-3817) in the hit's (reference-forward) orientation.
    HT2_HD int64_t h2score(const ht2gpu_aln_t& al, uint32_t rdlen) const {
        int64_t score = al.score;
        int64_t splicescore = 255, transcript_score = 0;
#ifdef HT2_ENABLE_SPLICED
        {
            const ht2gpu_edit_t* ed = in->edits + al.edit_off;
            const uint32_t n = al.n_edits;
            bool spl = false, known = true; double ss = 0; uint32_t nss = 0;
            for (uint32_t e = 0; e < n; e++) {
                if (ed[e].type != HT2_EDIT_SPL) continue;
                const Ht2Edit& se = *(const Ht2Edit*)&ed[e];
                spl = true; known = known && ht2_spl_known(se);
                if (ht2_spl_known(se)) continue;
                uint32_t before = 0, after = 0;   // in hit order: plain mismatches before, mismatches + gaps after
                for (uint32_t k = 0; k < n; k++) {
                    if (k == e) continue;
                    const ht2gpu_edit_t& o2 = ed[k];
                    const bool isBefore = al.fw ? (k < e) : (k > e);
                    if (isBefore) { if (o2.type == HT2_EDIT_MM && o2.snp_id == HT2_IDX_MAX32) before++; }
                    else if (o2.type == HT2_EDIT_MM || o2.type == HT2_EDIT_READ_GAP || o2.type == HT2_EDIT_REF_GAP) after++;
                }
                const uint32_t q = ed[e].pos + al.trim5;              // 5'->3' offset of the splice in the read
                int left_anchor = (int)(al.fw ? q : rdlen - q), right_anchor = (int)rdlen - left_anchor;
                left_anchor -= (int)(before * 2); right_anchor -= (int)(after * 2);
                int shorter = left_anchor < right_anchor ? left_anchor : right_anchor;
                if (shorter <= 0) shorter = 1;
                if (shorter <= 15) { nss++; ss += (double)ht2_spl_len(se); }
            }
            if (nss > 1) ss /= (double)nss;
            splicescore = (int64_t)(ss / 100);     // TAlScore splicescore = splicescore_ / 100 (aligner_result.h:339)
            if (splicescore > 255) splicescore = 0; else splicescore = 255 - splicescore;
            transcript_score = (spl && known) ? 2 : (spl ? 1 : 0);
        }
#else
        (void)rdlen;
#endif
        int64_t trim = (int64_t)al.trim5 + (int64_t)al.trim3;
        if (trim > 65535) trim = 0; else trim = 65535 - trim;
        return (int64_t)((uint64_t)score << 32) | (transcript_score << 24) | (splicescore << 16) | trim;
    }

    HT2_HD void addUnp(Ht2SamSumm& s, int j, const ht2gpu_aln_t* rs, uint32_t n, uint32_t rdlen) const {
        for (uint32_t i = 0; i < n; i++) {
            Ht2SamKey sc = {rs[i].score, h2score(rs[i], rdlen), true};
            if (ht2_sam_key_gt(sc, s.best[j])) { s.secbest[j] = s.best[j]; s.best[j] = sc; }
            else if (ht2_sam_key_gt(sc, s.secbest[j])) s.secbest[j] = sc;
        }
        s.numAlns[j] = n;
    }

    // AlnSinkWrap::selectByScore (aln_sink.h:2680-2755).  rs1 (+ rs2 and pairs for concordant pairs); writes the
    // selected element indexes to sel[] and returns their number.  The sort key is (score key, index), both
    // descending -- std::sort + reverse of pair<key, index> in the reference's restatement -- so the order is total.
    // One candidate (nearly every read) is selected as it is, without the sort arrays; no shuffle draws from rnd
    // either way, as a run of equal keys needs two candidates.
    HT2_HD uint32_t selectByScore(const ht2gpu_aln_t* rs1, uint32_t n1, uint32_t len1, const ht2gpu_aln_t* rs2, uint32_t len2,
                                  const uint16_t* pairs, uint32_t npairs, bool usePairs, uint64_t num, uint16_t* sel, Ht2Rng& rnd) const {
        if ((usePairs ? npairs : n1) == 1 && num > 0) { sel[0] = 0; return 1; }
        return selectMany(rs1, n1, len1, rs2, len2, pairs, npairs, usePairs, num, sel, rnd);
    }
    HT2_NI uint32_t selectMany(const ht2gpu_aln_t* rs1, uint32_t n1, uint32_t len1, const ht2gpu_aln_t* rs2, uint32_t len2,
                               const uint16_t* pairs, uint32_t npairs, bool usePairs, uint64_t num, uint16_t* sel, Ht2Rng& rnd) const {
        uint32_t sz = usePairs ? npairs : n1;
        if (sz > HT2_SAM_MAXSEL) sz = HT2_SAM_MAXSEL;   // cannot happen: the kernel's per-read capacities are smaller
        if (sz < num) num = sz;
        if (sz < 1) return 0;
        int64_t key[HT2_SAM_MAXSEL];
        uint16_t idx[HT2_SAM_MAXSEL];
        for (uint32_t i = 0; i < sz; i++) {
            const int64_t k = usePairs ? h2score(rs1[pairs[2 * i]], len1) + h2score(rs2[pairs[2 * i + 1]], len2) : h2score(rs1[i], len1);
            // insertion into descending (key, index) order
            uint32_t j = i;
            while (j > 0 && key[j - 1] <= k) { key[j] = key[j - 1]; idx[j] = idx[j - 1]; j--; }   // equal keys: the later index sorts first
            key[j] = k; idx[j] = (uint16_t)i;
        }
        // equal-key runs are shuffled (ds.h:836-847)
        uint32_t streak = 0;
        for (uint32_t i = 1; i <= sz; i++) {
            if (i < sz && key[i] == key[i - 1]) { if (streak == 0) streak = 1; streak++; }
            else {
                if (streak > 1) {
                    const uint32_t begin = i - streak;
                    uint32_t left = streak;
                    for (uint32_t q = begin; q < begin + streak - 1; q++) {
                        const uint32_t rndi = rnd.nextU32() % left;
                        if (rndi > 0) { const uint16_t t = idx[q]; idx[q] = idx[q + rndi]; idx[q + rndi] = t; }
                        left--;
                    }
                }
                streak = 0;
            }
        }
        uint32_t nsel = 0;
        for (uint32_t i = 0; i < sz && i < num; i++) sel[nsel++] = idx[i];
        if (!in->secondary) {
            for (uint32_t i = 0; i + 1 < nsel; i++) if (key[i] != key[i + 1]) { nsel = i + 1; break; }
        }
        return nsel;
    }

    // BowtieMapq2::mapq (unique.h:170-400) for monotone scoring, canMax=false, exhausted=false.
    HT2_HD int mapqV2(const Ht2SamSumm& s, bool mate1, uint32_t rdlen, uint32_t ordlen) const {
        const Ht2SamKey& bst = s.paired ? s.bestPaired : s.best[mate1 ? 0 : 1];
        const Ht2SamKey& sec = s.paired ? s.secbestPaired : s.secbest[mate1 ? 0 : 1];
        const bool hasSecbest = sec.valid;
        const bool equalSecbest = hasSecbest && ht2_sam_key_eq(bst, sec);
        if (!hasSecbest || !equalSecbest) return 60;
        int64_t scMin = minscOf(rdlen);
        if (s.paired) scMin += minscOf(ordlen);
        const int64_t diff = 0 - scMin;
        const int64_t best = bst.score;
        const int64_t bestOver = best - scMin;
        const int64_t secbest = sec.score;
        const int64_t a = best < 0 ? -best : best, b = secbest < 0 ? -secbest : secbest;
        const int64_t bestdiff = a - b < 0 ? b - a : a - b;
        int ret;
        if (bestdiff >= diff * (double)0.9f) ret = (bestOver == diff) ? 39 : 33;
        else if (bestdiff >= diff * (double)0.8f) ret = (bestOver == diff) ? 38 : 27;
        else if (bestdiff >= diff * (double)0.7f) ret = (bestOver == diff) ? 37 : 26;
        else if (bestdiff >= diff * (double)0.6f) ret = (bestOver == diff) ? 36 : 22;
        else if (bestdiff >= diff * (double)0.5f) {
            if (bestOver == diff) ret = 35;
            else if (bestOver >= diff * (double)0.84f) ret = 25;
            else if (bestOver >= diff * (double)0.68f) ret = 16;
            else ret = 5;
        } else if (bestdiff >= diff * (double)0.4f) {
            if (bestOver == diff) ret = 34;
            else if (bestOver >= diff * (double)0.84f) ret = 21;
            else if (bestOver >= diff * (double)0.68f) ret = 14;
            else ret = 4;
        } else if (bestdiff >= diff * (double)0.3f) {
            if (bestOver == diff) ret = 32;
            else if (bestOver >= diff * (double)0.88f) ret = 18;
            else if (bestOver >= diff * (double)0.67f) ret = 15;
            else ret = 3;
        } else if (bestdiff >= diff * (double)0.2f) {
            if (bestOver == diff) ret = 31;
            else if (bestOver >= diff * (double)0.88f) ret = 17;
            else if (bestOver >= diff * (double)0.67f) ret = 11;
            else ret = 0;
        } else if (bestdiff >= diff * (double)0.1f) {
            if (bestOver == diff) ret = 30;
            else if (bestOver >= diff * (double)0.88f) ret = 12;
            else if (bestOver >= diff * (double)0.67f) ret = 7;
            else ret = 0;
        } else if (bestdiff > 0) {
            ret = (bestOver >= diff * (double)0.67f) ? 6 : 2;
        } else {
            ret = (bestOver >= diff * (double)0.67f) ? 1 : 0;
        }
        return ret;
    }

    // AlnRes::setFragmentLength (aligner_result.h:1631-1697) with an empty splice-site DB; st2/en2 are the
    // extents shifted right by the alignment's own introns (getCoords, :1132-1147)
    HT2_HD void extents(const ht2gpu_aln_t& r, int64_t& st, int64_t& en, int64_t& st2, int64_t& en2) const {
        const int64_t trim_st = r.fw ? r.trim5 : r.trim3, trim_en = r.fw ? r.trim3 : r.trim5;
        int64_t introns = 0;
#ifdef HT2_ENABLE_SPLICED
        for (uint32_t e = 0; e < r.n_edits; e++) { const ht2gpu_edit_t& ed = in->edits[r.edit_off + e]; if (ed.type == HT2_EDIT_SPL) introns += ht2_spl_len(*(const Ht2Edit*)&ed); }
#endif
        st = (int64_t)r.toff - trim_st;
        en = (int64_t)r.toff + r.ref_extent - 1 + trim_en;
        st2 = st + introns; en2 = en + introns;
    }
    HT2_HD int64_t fragmentLength(const ht2gpu_aln_t& me, const ht2gpu_aln_t& o, bool meMate1, bool useSs = false) const {
        int64_t st, en, st2, en2, ost, oen, ost2, oen2;
        extents(me, st, en, st2, en2); extents(o, ost, oen, ost2, oen2);
        bool imUpstream;
        if (st < ost) imUpstream = true;
        else if (st == ost) {
            if (me.fw && o.fw && meMate1) imUpstream = true;
            else if (me.fw && !o.fw) imUpstream = true;
            else imUpstream = false;
        } else imUpstream = false;
        int64_t up, dn, up_right, dn_left;
        if (imUpstream) { up = st2 < ost ? st2 : ost; up_right = en2 < oen ? en2 : oen; dn_left = st2 > ost ? st2 : ost; dn = en2 > oen ? en2 : oen; }
        else { up = st < ost2 ? st : ost2; up_right = en < oen2 ? en : oen2; dn_left = st > ost2 ? st : ost2; dn = en > oen2 ? en : oen2; }
        // concordant pairs, templateLenAdjustment (the default): the longest known intron that lies strictly between the
        // mates does not count (AlnRes::setFragmentLength, aligner_result.h:1666-1683)
        int64_t intron_len = 0;
        if (useSs && in->ssT != NULL && up_right + 100 < dn_left) {
            Ht2SsView ssv; ssv.init(in->ssT);
            uint32_t lo, hi;
            ssv.rightSites(me.tidx, (uint32_t)up_right, (uint32_t)(dn_left - up_right), lo, hi);
            for (uint32_t si = lo; si < hi; si++) {
                const Ht2SsSite& ss = ssv.fw[si];
                if ((int64_t)ss.left <= up || (int64_t)ss.right >= dn) continue;
                const int64_t l = (int64_t)(ss.right - ss.left - 1);
                if (intron_len < l) intron_len = l;
            }
        }
        int64_t fraglen = 1 + dn - up - intron_len;
        if (!imUpstream) fraglen = -fraglen;
        return fraglen;
    }

    template <bool W> HT2_HD void putRefName(Ht2SamCur<W>& o, uint32_t tidx) const { o.name(refName(tidx), false, 0xffffffffu); }
    template <bool W> HT2_HD void putSeqQual(Ht2SamCur<W>& o, const Ht2SamRead& rd, bool fw) const {
        const uint32_t n = rd.len;
        if (n == 0) { o.s("*\t*"); return; }   // aln_sink.h:3194, 3210
        const uint8_t* sq = rd.seq; const uint8_t* ql = rd.qual;
        auto fwBase = [&](uint32_t i) { return "ACGTN"[sq[i]]; };
        auto rcBase = [&](uint32_t i) { const uint8_t c = sq[n - i - 1]; return "TGCAN"[c < 4 ? c : 4]; };
        auto fwQual = [&](uint32_t i) { return (char)ql[i]; };
        auto rcQual = [&](uint32_t i) { return (char)ql[n - i - 1]; };
#ifdef __CUDA_ARCH__
        // four bytes per step: aligned word loads of the read, base codes (0..4) to letters with one byte permute
        // (selector nibble = code; byte 4 of the pair is 'N'), the reverse strand's order by one more permute
        auto letters = [](uint32_t codes, uint32_t table) {
            const uint32_t y = codes | (codes >> 4);
            return __byte_perm(table, 0x4Eu, __byte_perm(y, 0, 0x0020));
        };
        const char* sc = (const char*)sq; const char* qc = (const char*)ql;
        auto fwBase4 = [&](uint32_t i) { return letters(ht2_sam_ld4(sc + i), 0x54474341u); };                          // "ACGT"
        auto rcBase4 = [&](uint32_t i) { return letters(__byte_perm(ht2_sam_ld4(sc + n - i - 4), 0, 0x0123), 0x41434754u); };   // "TGCA"
        auto fwQual4 = [&](uint32_t i) { return ht2_sam_ld4(qc + i); };
        auto rcQual4 = [&](uint32_t i) { return __byte_perm(ht2_sam_ld4(qc + n - i - 4), 0, 0x0123); };
#else
        auto word = [](auto byteAt, uint32_t i) {
            return (uint32_t)(uint8_t)byteAt(i) | ((uint32_t)(uint8_t)byteAt(i + 1) << 8) |
                   ((uint32_t)(uint8_t)byteAt(i + 2) << 16) | ((uint32_t)(uint8_t)byteAt(i + 3) << 24);
        };
        auto fwBase4 = [&](uint32_t i) { return word(fwBase, i); };
        auto rcBase4 = [&](uint32_t i) { return word(rcBase, i); };
        auto fwQual4 = [&](uint32_t i) { return word(fwQual, i); };
        auto rcQual4 = [&](uint32_t i) { return word(rcQual, i); };
#endif
        if (fw) o.run(n, fwBase, fwBase4);
        else o.run(n, rcBase, rcBase4);
        o.c('\t');
        if (!ql) o.run(n, [&](uint32_t) { return 'I'; }, [&](uint32_t) { return 0x49494949u; });
        else if (fw) o.run(n, fwQual, fwQual4);
        else o.run(n, rcQual, rcQual4);
    }
    template <bool W> HT2_HD void putYF(Ht2SamCur<W>& o, const Ht2SamRead& rd) const {
        if (!rd.lenfilt) o.s("\tYF:Z:LN");
        else if (!rd.nfilt) o.s("\tYF:Z:NS");
        else if (!rd.scfilt) o.s("\tYF:Z:SC");
    }
    // the read group follows YT:Z / YF:Z and precedes XS:A / NH:i (sam.h:780, 1102)
    template <bool W> HT2_HD void putRG(Ht2SamCur<W>& o) const {
        if (in->rgTag) { o.c('\t'); o.str(in->rgTag); }
    }
    template <bool W> HT2_HD void putYT(Ht2SamCur<W>& o, const Ht2SamFlags& fl) const {
        o.s("\tYT:Z:");
        if (fl.concordant()) o.s("CP"); else if (fl.discordant()) o.s("DP"); else if (fl.unpairedMate()) o.s("UP"); else o.s("UU");
    }

    // SpliceSiteDB::addSpliceSite (splice_site.cpp:190-350) for one printed alignment: every junction whose anchors
    // are long enough (15 bases + 2 per mismatch / gap on its side, + 6 without a canonical motif) is recorded with the
    // alignment's edit distance.  Alignments with soft-trimmed ends are skipped.  (The threshold of a junction that is
    // followed by another one uses the NEXT junction's direction and the mismatches seen so far -- as the reference.)
    HT2_NI void collectSites(const ht2gpu_aln_t* rs, uint32_t rdlen) const {
        if (rs->trim5 + rs->trim3 > 0) return;
        const ht2gpu_edit_t* ed = in->edits + rs->edit_off;
        const uint32_t ned = rs->n_edits;
        uint32_t editdist = 0; bool spliced = false;
        for (uint32_t k = 0; k < ned; k++) {
            if (ed[k].type == HT2_EDIT_SPL) spliced = true;
            else if (ed[k].type == HT2_EDIT_MM || ed[k].type == HT2_EDIT_READ_GAP || ed[k].type == HT2_EDIT_REF_GAP) editdist++;
        }
        if (!spliced) return;
        const bool fw = rs->fw != 0;
        // edit k in left-to-right order and its position there (Edit::invertPoss for the reverse strand)
        auto at = [&](uint32_t k) -> const ht2gpu_edit_t& { return fw ? ed[k] : ed[ned - 1 - k]; };
        auto posOf = [&](uint32_t k) -> uint32_t {
            const ht2gpu_edit_t& e = at(k);
            if (fw) return e.pos;
            return (e.type == HT2_EDIT_READ_GAP || e.type == HT2_EDIT_SPL) ? rdlen - e.pos : rdlen - e.pos - 1;
        };
        auto isEd = [&](const ht2gpu_edit_t& e) { return e.type == HT2_EDIT_MM || e.type == HT2_EDIT_READ_GAP || e.type == HT2_EDIT_REF_GAP; };
        auto splLen = [&](const ht2gpu_edit_t& e) { return (uint32_t)e.chr | ((uint32_t)e.qchr << 8) | ((uint32_t)(e.pad & 15) << 16); };
        auto splDir = [&](const ht2gpu_edit_t& e) { return (uint32_t)(e.pad >> 4) & 7u; };
        auto push = [&](uint32_t l, uint32_t r, uint32_t d) {
#ifdef __CUDA_ARCH__
            const uint32_t idx = atomicAdd(in->colCount, 1u);
#else
            const uint32_t idx = __sync_fetch_and_add(in->colCount, 1u);
#endif
            if (idx < in->colCap) { Ht2SsRec rec; rec.ref = rs->tidx; rec.left = l; rec.right = r; rec.dirEd = d | (editdist << 8); in->colRecs[idx] = rec; }
        };
        const uint32_t minAnchorLen = 15;
        uint32_t refoff = rs->toff, leftAnchor = 0, rightAnchor = 0, eidx = 0, last = 0, mm = 0;
        uint32_t sl = 0, sr = 0, sd = 0; bool inited = false;
        for (uint32_t i = 0; i < rdlen; i++, refoff++) {
            while (eidx < ned && posOf(eidx) == i) {
                const ht2gpu_edit_t& e = at(eidx);
                if (e.type == HT2_EDIT_READ_GAP) refoff++;
                else if (e.type == HT2_EDIT_REF_GAP) refoff--;
                if (isEd(e)) mm++;
                if (e.type == HT2_EDIT_SPL) {
                    if (inited) {
                        rightAnchor = posOf(eidx) - posOf(last);
                        const uint32_t unk = splDir(e) == HT2_SPL_UNKNOWN ? 6u : 0u;
                        uint32_t mm2 = 0;
                        for (uint32_t j = eidx + 1; j < ned; j++) if (isEd(at(j))) mm2++;
                        if (leftAnchor >= minAnchorLen + mm * 2 + unk && rightAnchor >= minAnchorLen + mm2 * 2 + unk) push(sl, sr, sd);
                        leftAnchor = rightAnchor; rightAnchor = 0;
                    } else leftAnchor = posOf(eidx);
                    sl = refoff - 1; sr = refoff + splLen(e); sd = splDir(e); inited = true;
                    refoff += splLen(e);
                    last = eidx;
                }
                eidx++;
            }
        }
        if (inited) {
            rightAnchor = rdlen - posOf(last);
            const uint32_t unk = splDir(at(last)) == HT2_SPL_UNKNOWN ? 6u : 0u;
            uint32_t mm2 = 0;
            for (uint32_t j = last + 1; j < ned; j++) if (isEd(at(j))) mm2++;
            if (leftAnchor >= minAnchorLen + mm * 2 + unk && rightAnchor >= minAnchorLen + mm2 * 2 + unk) push(sl, sr, sd);
        }
    }

    // StackedAln of a gapped alignment (StackedAln::init / leftAlign, aligner_result.cpp:660-790), built in this
    // frame, then its CIGAR (mdz = false: StackedAln::buildCigar, aligner_result.cpp:793-850) or its MD:Z string
    // (mdz = true: StackedAln::buildMdz, aligner_result.cpp:852-1000).  Out of line so that the column arrays are no
    // part of the gapless path's frame; a gapped record builds its stack twice.
    template <bool W>
    HT2_NI uint32_t putStacked(char* d, const uint8_t* seq, uint32_t rdlen, const ht2gpu_aln_t* rs, bool mdz) const {
        Ht2SamCur<W> o = {d, 0};
        const ht2gpu_edit_t* ed = in->edits + rs->edit_off;
        const uint32_t ned = rs->n_edits;
        uint32_t trimLS = rs->trim5, trimRS = rs->trim3;
        const uint32_t len_trimmed = rdlen - trimLS - trimRS;
        if (!rs->fw) { const uint32_t t = trimLS; trimLS = trimRS; trimRS = t; }
        // columns of (ref, rel, read, snp)
        char stRef[HT2_SAM_MAXCOLS], stRel[HT2_SAM_MAXCOLS], stRead[HT2_SAM_MAXCOLS];
        uint8_t stSnp[HT2_SAM_MAXCOLS];
        uint32_t ln = 0;
        {
            // AlnRes::initStacked (aligner_result.h:1856-1873): edits and read in reference-forward orientation
            uint32_t rdoff = trimLS;
            auto rdc = [&](uint32_t i) -> int { if (rs->fw) return seq[i]; const uint8_t c = seq[rdlen - i - 1]; return c < 4 ? (c ^ 3) : 4; };
            for (uint32_t k = 0; k < ned && ln + 2 < HT2_SAM_MAXCOLS; k++) {
                const ht2gpu_edit_t& e = rs->fw ? ed[k] : ed[ned - 1 - k];
                uint32_t epos = e.pos;
                if (!rs->fw) epos = (e.type == HT2_EDIT_READ_GAP || e.type == HT2_EDIT_SPL) ? len_trimmed - e.pos : len_trimmed - e.pos - 1;   // Edit::invertPoss
                const uint32_t pos = epos + trimLS;
                while (rdoff < pos && ln + 2 < HT2_SAM_MAXCOLS) { const int c = rdc(rdoff++); stRef[ln] = "ACGTN"[c]; stRel[ln] = '='; stSnp[ln] = 0; stRead[ln] = "ACGTN"[c]; ln++; }
                const uint8_t isSnp = e.snp_id != HT2_IDX_MAX32;
                if (e.type == HT2_EDIT_MM) { const int c = rdc(rdoff++); stRef[ln] = (char)e.chr; stRel[ln] = 'X'; stSnp[ln] = isSnp; stRead[ln] = "ACGTN"[c]; ln++; }
                else if (e.type == HT2_EDIT_REF_GAP) { const int c = rdc(rdoff++); stRef[ln] = '-'; stRel[ln] = 'I'; stSnp[ln] = isSnp; stRead[ln] = "ACGTN"[c]; ln++; }
                else if (e.type == HT2_EDIT_READ_GAP) { stRef[ln] = (char)e.chr; stRel[ln] = 'D'; stSnp[ln] = isSnp; stRead[ln] = '-'; ln++; }
                else if (e.type == HT2_EDIT_SPL) { stRef[ln] = 'N'; stRel[ln] = 'N'; stSnp[ln] = 0; stRead[ln] = 'N'; ln++; }   // aligner_result.cpp:711-718
            }
            while (rdoff < rdlen - trimRS && ln + 1 < HT2_SAM_MAXCOLS) { const int c = rdc(rdoff++); stRef[ln] = "ACGTN"[c]; stRel[ln] = '='; stSnp[ln] = 0; stRead[ln] = "ACGTN"[c]; ln++; }
            // StackedAln::leftAlign(false) (aligner_result.cpp:727-790)
            for (uint32_t i = 0; i < ln; i++) {
                const char r = stRel[i];
                if (r != '=' && r != 'X' && r != 'N') {
                    if (stSnp[i]) continue;
                    uint32_t glen = 1;
                    for (uint32_t j = i + 1; j < ln; j++) { if (r != stRel[j]) break; glen++; }
                    uint32_t l = i - 1;                 // wraps for i == 0 exactly like the reference's size_t
                    uint32_t rr = l + glen;
                    char* gp = (r == 'I') ? stRef : stRead;
                    const char* ngp = (r == 'I') ? stRead : stRef;
                    while (l > 0 && l < ln && ngp[l] == ngp[rr]) {
                        if (stRel[l] == 'I' || stRel[l] == 'D') break;
                        if (stRel[l] == 'X' || stRel[l] == 'N') break;   // pastMms == false
                        { const char t = gp[l]; gp[l] = gp[rr]; gp[rr] = t; }
                        { const char t = stRel[l]; stRel[l] = stRel[rr]; stRel[rr] = t; }
                        l--; rr--;
                    }
                    i += (glen - 1);
                }
            }
        }
        if (!mdz) {
            if (trimLS > 0) { o.i64(trimLS); o.c('S'); }
            uint32_t numSkips = 0;
            for (uint32_t i = 0; i < ln; i++) {
                char op = stRel[i];
                if (op == 'X' || op == '=') op = 'M';
                uint64_t run = 1;
                if (op != 'N') {
                    for (; i + run < ln; run++) {
                        char op2 = stRel[i + run];
                        if (op2 == 'X' || op2 == '=') op2 = 'M';
                        if (op2 != op) break;
                    }
                    i += (uint32_t)(run - 1);
                } else {   // the numSkips-th splice edit in reference-forward order (aligner_result.cpp:815-833)
                    uint32_t seen = 0; run = 0;
                    for (uint32_t k = 0; k < ned; k++) {
                        const ht2gpu_edit_t& e = rs->fw ? ed[k] : ed[ned - 1 - k];
                        if (e.type != HT2_EDIT_SPL) continue;
                        if (seen == numSkips) { run = ht2_spl_len(*(const Ht2Edit*)&e); break; }
                        seen++;
                    }
                    numSkips++;
                }
                o.i64((int64_t)run); o.c(op);
            }
            if (trimRS > 0) { o.i64(trimRS); o.c('S'); }
        } else {
            bool mm_last = false, rdgap_last = false, first_print = true;
            for (uint32_t i = 0; i < ln; i++) {
                const char op = stRel[i];
                if (op == '=') {
                    uint32_t run = 1, ninserts = 0;
                    for (; i + run < ln; run++) {
                        if (stRel[i + run] == '=') {}
                        else if (stRel[i + run] == 'I' || stRel[i + run] == 'N') ninserts++;   // insertions and introns do not count
                        else break;
                    }
                    i += (run - 1);
                    const uint32_t r = run - ninserts;
                    if (r > 0) { o.i64(r); first_print = false; mm_last = false; rdgap_last = false; }
                } else if (op == 'X') {
                    if (rdgap_last || mm_last || first_print) o.c('0');
                    o.c(stRef[i]);
                    first_print = false; mm_last = true; rdgap_last = false;
                } else if (op == 'D') {
                    if (mm_last || first_print) o.c('0');
                    if (!rdgap_last) o.c('^');
                    o.c(stRef[i]);
                    first_print = false; mm_last = false; rdgap_last = true;
                }
            }
            if (mm_last || rdgap_last) o.c('0');
        }
        return o.n;
    }

    // the fields of an unaligned record after FLAG
    template <bool W>
    HT2_NI uint32_t putUnaligned(char* d, const Ht2SamRead& rd, const Ht2SamSumm& summ, const Ht2SamFlags& fl) const {
        Ht2SamCur<W> o = {d, 0};
        if (summ.orefid != -1) { putRefName(o, (uint32_t)summ.orefid); o.c('\t'); o.i64(summ.orefoff + 1); o.s("\t0\t*\t=\t"); o.i64(summ.orefoff + 1); o.s("\t0\t"); }
        else o.s("*\t0\t0\t*\t*\t0\t0\t");
        putSeqQual(o, rd, true);
        putYT(o, fl);
        putYF(o, rd);
        putRG(o);
        o.c('\n');
        return o.n;
    }

#ifdef HT2_ENABLE_SPLICED
    // XS:A of a spliced alignment: AlnRes::spliced_whichsense_transcript (aligner_result.h:1288-1318, sam.h:925-937);
    // '+', '-' or 0 for none
    HT2_NI char xsSense(const ht2gpu_edit_t* ed, uint32_t ned) const {
        uint32_t whichsense = HT2_SPL_UNKNOWN;
        for (uint32_t i = 0; i < ned; i++) {
            if (ed[i].type != HT2_EDIT_SPL) continue;
            const uint32_t d = ht2_spl_dir(*(const Ht2Edit*)&ed[i]);
            if (whichsense == HT2_SPL_UNKNOWN) whichsense = d;
            else if (d != HT2_SPL_UNKNOWN) {
                if ((whichsense == HT2_SPL_FW || whichsense == HT2_SPL_SEMI_FW) && d != HT2_SPL_FW && d != HT2_SPL_SEMI_FW) return 0;
                if ((whichsense == HT2_SPL_RC || whichsense == HT2_SPL_SEMI_RC) && d != HT2_SPL_RC && d != HT2_SPL_SEMI_RC) return 0;
            }
        }
        if (whichsense == HT2_SPL_UNKNOWN) return 0;
        return (whichsense == HT2_SPL_FW || whichsense == HT2_SPL_SEMI_FW) ? '+' : '-';
    }
#endif

    // Zs:Z: the known ALTs the alignment went through (sam.h:983-1032); edits in reference-forward order
    template <bool W>
    HT2_NI uint32_t putZs(char* d, const ht2gpu_aln_t* rs, uint32_t len_trimmed) const {
        Ht2SamCur<W> o = {d, 0};
        const ht2gpu_edit_t* ed = in->edits + rs->edit_off;
        const uint32_t ned = rs->n_edits;
        auto nedAt = [&](uint32_t i, uint32_t& pos) -> const ht2gpu_edit_t& {   // Edit::invertPoss (edit.cpp:70-111), sort = false
            const ht2gpu_edit_t& e = rs->fw ? ed[i] : ed[ned - 1 - i];
            pos = e.pos;
            if (!rs->fw) pos = (e.type == HT2_EDIT_READ_GAP || e.type == HT2_EDIT_SPL) ? len_trimmed - e.pos : len_trimmed - e.pos - 1;
            return e;
        };
        bool first = true;
        uint32_t prev = 0xffffffffu;
        for (uint32_t i = 0; i < ned; i++) {
            uint32_t epos;
            const ht2gpu_edit_t& e = nedAt(i, epos);
            if (e.type == HT2_EDIT_SPL || e.snp_id >= nAlts) continue;   // a splice edit keeps its site probability in the snpID word
            const uint32_t si = e.snp_id;
            const Ht2Alt& snp = altTab[si];
            if (si == prev) continue;
            if (first) o.s("\tZs:Z:"); else o.c(',');
            uint64_t pos = epos;
            uint32_t j = i;
            while (j > 0) {
                uint32_t ppos;
                const ht2gpu_edit_t& pe = nedAt(j - 1, ppos);
                if (pe.snp_id < nAlts) {
                    const Ht2Alt& snp2 = altTab[pe.snp_id];
                    if (snp2.type == HT2_ALT_SNP_SGL) pos -= (ppos + 1);
                    else if (snp2.type == HT2_ALT_SNP_DEL) pos -= ppos;
                    else if (snp2.type == HT2_ALT_SNP_INS) pos -= (ppos + snp.len);
                    break;
                }
                j--;
            }
            o.i64((int64_t)pos);
            if (snp.type == HT2_ALT_SNP_SGL) o.s("|S|"); else if (snp.type == HT2_ALT_SNP_DEL) o.s("|D|"); else o.s("|I|");
            o.str(altName(si));
            first = false;
            prev = si;
        }
        return o.n;
    }

    // AlnSinkSam::appendMate (aln_sink.h:3024-3250): one record at d; returns its length.  The common record (aligned,
    // gapless, no ALTs) runs in this frame; gapped CIGAR / MD:Z, unaligned records, XS:A, Zs:Z and the junction
    // collection are out of line.
    template <bool W>
    HT2_NI uint32_t appendMate(char* d, const Ht2SamRead& rd, uint32_t ordlen, const ht2gpu_aln_t* rs, const ht2gpu_aln_t* rso,
                               const Ht2SamSumm& summ, const Ht2SamFlags& fl, bool fraglenSet, int64_t fraglen, bool haveOscore) const {
        if (rs == NULL && in->noUnal) return 0;
        Ht2SamCur<W> o = {d, 0};
        o.name(rd.name, fl.partOfPair(), 255);
        o.c('\t');
        int flag = 0;
        if (fl.partOfPair()) {
            flag |= 1;
            if (fl.concordant()) flag |= 2;
            if (!fl.oppAligned) flag |= 8;
            flag |= fl.readMate1() ? 64 : 128;
            if (fl.oppAligned && rso != NULL && !rso->fw) flag |= 32;
        }
        if (!fl.primary) flag |= 256;
        if (rs != NULL && !rs->fw) flag |= 16;
        if (rs == NULL) flag |= 4;
        o.i64(flag);
        o.c('\t');
        if (rs == NULL) return o.n + putUnaligned<W>(o.at(), rd, summ, fl);
        if (W && in->colCount != NULL) collectSites(rs, rd.len);   // AlnSinkSam::append (aln_sink.h:1571, 1579)
        const ht2gpu_edit_t* ed = in->edits + rs->edit_off;
        const uint32_t ned = rs->n_edits;
        // Gapless alignments (mismatches only; the vast majority): CIGAR and MD:Z follow from the edit positions
        // directly -- what StackedAln::buildCigar / buildMdz print for a stack without I/D columns, with nothing for
        // leftAlign to move.  Everything else goes through the stacked form (putStacked).
        bool gapless = true;
        for (uint32_t i = 0; i < ned; i++) if (ed[i].type != HT2_EDIT_MM) { gapless = false; break; }
        uint32_t trimLS = rs->trim5, trimRS = rs->trim3;
        const uint32_t len_trimmed = rd.len - trimLS - trimRS;
        if (!rs->fw) { const uint32_t t = trimLS; trimLS = trimRS; trimRS = t; }
        putRefName(o, rs->tidx);
        o.c('\t');
        o.i64((int64_t)rs->toff + 1);
        o.c('\t');
        o.i64(mapqV2(summ, rd.mate < 2, rd.len, ordlen));
        o.c('\t');
        if (gapless) {
            if (trimLS > 0) { o.i64(trimLS); o.c('S'); }
            if (len_trimmed > 0) { o.i64(len_trimmed); o.c('M'); }
            if (trimRS > 0) { o.i64(trimRS); o.c('S'); }
        } else o.n += putStacked<W>(o.at(), rd.seq, rd.len, rs, false);
        o.c('\t');
        if (fl.partOfPair()) {
            if (rso != NULL && rs->tidx != rso->tidx) { putRefName(o, rso->tidx); o.c('\t'); }
            else o.s("=\t");
            o.i64((int64_t)(rso ? rso->toff : rs->toff) + 1);
            o.c('\t');
        } else o.s("*\t0\t");
        o.i64(fraglenSet ? fraglen : 0);
        o.c('\t');
        if (!fl.primary && in->omitSecSeq) o.s("*\t*");
        else putSeqQual(o, rd, rs->fw != 0);
        // optional flags (sam.h:525-1010)
        o.s("\tAS:i:"); o.i64(rs->score);
        const Ht2SamKey& sb = summ.secbest[rd.mate < 2 ? 0 : 1];
        if (sb.valid) { o.s("\tZS:i:"); o.i64(sb.score); }
        o.s("\tXN:i:0");
        // counts exclude edits that are known ALTs (snpID < #alts, sam.h:574-647)
        uint32_t num_mm = 0, num_go = 0, num_gx = 0, NM = 0;
        bool spliced = false;
        for (uint32_t i = 0; i < ned; i++) {
            if (ed[i].type == HT2_EDIT_SPL) spliced = true;
            else if (ed[i].snp_id >= nAlts) NM++;
        }
        for (uint32_t i = 0; i < ned; i++) {
            const ht2gpu_edit_t& e = ed[i];
            if (e.type == HT2_EDIT_MM) { if (e.snp_id >= nAlts) num_mm++; }
            else if (e.type == HT2_EDIT_READ_GAP) {
                if (e.snp_id >= nAlts) { num_go++; num_gx++; }
                while (i + 1 < ned && ed[i + 1].pos == ed[i].pos && ed[i + 1].type == HT2_EDIT_READ_GAP) { i++; if (ed[i].snp_id >= nAlts) num_gx++; }
            } else if (e.type == HT2_EDIT_REF_GAP) {
                if (e.snp_id >= nAlts) { num_go++; num_gx++; }
                while (i + 1 < ned && ed[i + 1].pos == ed[i].pos + 1 && ed[i + 1].type == HT2_EDIT_REF_GAP) { i++; if (ed[i].snp_id >= nAlts) num_gx++; }
            }
        }
        o.s("\tXM:i:"); o.i64(num_mm);
        o.s("\tXO:i:"); o.i64(num_go);
        o.s("\tXG:i:"); o.i64(num_gx);
        o.s("\tNM:i:"); o.i64(NM);
        o.s("\tMD:Z:");
        if (gapless) {   // <matches>[<ref char><matches>]..., a 0 between adjacent mismatches and at either end
            uint32_t prevEnd = 0;
            for (uint32_t k = 0; k < ned; k++) {
                const ht2gpu_edit_t& e = rs->fw ? ed[k] : ed[ned - 1 - k];
                const uint32_t p = rs->fw ? e.pos : len_trimmed - e.pos - 1;
                o.i64((int64_t)(p - prevEnd));
                o.c((char)e.chr);
                prevEnd = p + 1;
            }
            o.i64((int64_t)(len_trimmed - prevEnd));
        } else o.n += putStacked<W>(o.at(), rd.seq, rd.len, rs, true);
        if (summ.paired && haveOscore && rso) { o.s("\tYS:i:"); o.i64(rso->score); }
        putYT(o, fl);
        putYF(o, rd);
        putRG(o);
#ifdef HT2_ENABLE_SPLICED
        if (spliced) { const char xs = xsSense(ed, ned); if (xs) { o.s("\tXS:A:"); o.c(xs); } }
#else
        (void)spliced;
#endif
        o.s("\tNH:i:");
        if (fl.concordant() || fl.discordant()) o.i64(summ.numAlnsPaired);
        else o.i64((fl.pairing == HT2_PAIR_UNPAIRED || fl.readMate1()) ? summ.numAlns[0] : summ.numAlns[1]);
        if (nAlts > 0) o.n += putZs<W>(o.at(), rs, len_trimmed);
        o.c('\n');
        return o.n;
    }

    // finishRead for an unpaired read (aln_sink.h:2213-2557, unpaired branches)
    template <bool W> HT2_HD void finishUnpaired(Ht2SamCur<W>& o, uint32_t u, Ht2SamTally* t) const {
        const ht2gpu_read_result_t& rr = in->reads[u];
        Ht2SamRead rd; mkRead(u, 0, rd);
        Ht2Rng rnd; rnd.last = rr.rng_state;
        const ht2gpu_aln_t* rs = in->alns + rr.aln_off;
        const uint32_t n = rr.n_aln[0];
        const uint64_t nunpair1 = n < in->khits ? n : in->khits;   // ReportingState::getReport
        Ht2SamSumm summ; summ.reset();
        Ht2SamFlags fl = {HT2_PAIR_UNPAIRED, true, false};
        if (t) { t->c[HT2_T_NREAD]++; t->c[HT2_T_NUNPAIRED]++; t->outcome = nunpair1 > 0 ? HT2GPU_OUTCOME_AL1 : 0; }
        if (nunpair1 > 0) {
            addUnp(summ, 0, rs, n, rd.len);
            uint16_t sel[HT2_SAM_MAXSEL];
            const uint32_t nsel = selectByScore(rs, n, rd.len, NULL, 0, NULL, 0, false, nunpair1, sel, rnd);
            summ.numAlns[0] = nsel;
            if (t) { t->c[HT2_T_NUNP_UNI1] += (uint32_t)(nsel == 1); t->c[HT2_T_NUNP_UNI2] += (uint32_t)(nsel != 1); }   // aln_sink.h:2290-2299
            for (uint32_t i = 0; i < nsel; i++) {
                fl.primary = (i == 0);
                o.n += appendMate<W>(o.at(), rd, 0, &rs[sel[i]], NULL, summ, fl, false, 0, false);
            }
        } else {
            if (t) t->c[HT2_T_NUNP_0]++;
            o.n += appendMate<W>(o.at(), rd, 0, NULL, NULL, summ, fl, false, 0, false);
        }
    }

    // AlnSinkWrap::finishRead for a pair (aln_sink.h:1939-2557)
    template <bool W> HT2_HD void finishPaired(Ht2SamCur<W>& o, uint32_t u, Ht2SamTally* t) const {
        const ht2gpu_read_result_t& rr = in->reads[u];
        if (t) { t->c[HT2_T_NREAD]++; t->c[HT2_T_NPAIRED]++; }
        Ht2SamRead rd1, rd2; mkRead(2 * u, 1, rd1); mkRead(2 * u + 1, 2, rd2);
        Ht2Rng rnd; rnd.last = rr.rng_state;
        const ht2gpu_aln_t* rs1u = in->alns + rr.aln_off;
        const ht2gpu_aln_t* rs2u = rs1u + rr.n_aln[0];
        const uint32_t n1 = rr.n_aln[0], n2 = rr.n_aln[1], np = rr.n_pairs;
        const uint16_t* pairs = in->pairs + 2 * (size_t)rr.pair_off;
        // ReportingState replay (aln_sink.cpp:72-131, 139-170)
        uint64_t nconcord_ = 0;
        {
            int64_t best = HT2_MIN_SCORE;
            for (uint32_t i = 0; i < np; i++) {
                const int64_t sc = (int64_t)rs1u[pairs[2 * i]].score + rs2u[pairs[2 * i + 1]].score;
                if (sc > best) { best = sc; nconcord_ = 0; }
                nconcord_++;
            }
        }
        const bool discordant = in->discord && np == 0 && n1 == 1 && n2 == 1;
        uint16_t sel[HT2_SAM_MAXSEL];
        if (nconcord_ > 0) {
            const uint64_t nconcord = in->khits < nconcord_ ? in->khits : nconcord_;
            Ht2SamSumm summ; summ.reset();
            summ.paired = true;
            for (uint32_t i = 0; i < np; i++) {
                const ht2gpu_aln_t& a = rs1u[pairs[2 * i]]; const ht2gpu_aln_t& b = rs2u[pairs[2 * i + 1]];
                Ht2SamKey sc = {(int64_t)a.score + b.score, h2score(a, rd1.len) + h2score(b, rd2.len), true};
                if (ht2_sam_key_gt(sc, summ.bestPaired)) { summ.secbestPaired = summ.bestPaired; summ.bestPaired = sc; }
                else if (ht2_sam_key_gt(sc, summ.secbestPaired)) summ.secbestPaired = sc;
            }
            addUnp(summ, 0, rs1u, n1, rd1.len); addUnp(summ, 1, rs2u, n2, rd2.len);
            const uint32_t nsel = selectByScore(rs1u, n1, rd1.len, rs2u, rd2.len, pairs, np, true, nconcord, sel, rnd);
            summ.numAlnsPaired = nsel;
            if (t) {   // select1_.size(), aln_sink.h:2100-2110
                t->c[HT2_T_NCONCORD_UNI1] += (uint32_t)(nsel == 1); t->c[HT2_T_NCONCORD_UNI2] += (uint32_t)(nsel != 1);
                t->outcome = HT2GPU_OUTCOME_AL1 | HT2GPU_OUTCOME_AL2 | HT2GPU_OUTCOME_CONC;
            }
            Ht2SamFlags fl1 = {HT2_PAIR_CONCORD_MATE1, true, true}, fl2 = {HT2_PAIR_CONCORD_MATE2, true, true};
            for (uint32_t i = 0; i < nsel; i++) {
                const ht2gpu_aln_t& a = rs1u[pairs[2 * sel[i]]]; const ht2gpu_aln_t& b = rs2u[pairs[2 * sel[i] + 1]];
                fl1.primary = fl2.primary = (i == 0);
                o.n += appendMate<W>(o.at(), rd1, rd2.len, &a, &b, summ, fl1, true, fragmentLength(a, b, true, true), true);
                o.n += appendMate<W>(o.at(), rd2, rd1.len, &b, &a, summ, fl2, true, fragmentLength(b, a, false, true), true);
            }
            return;
        } else if (discordant) {
            if (t) { t->c[HT2_T_NCONCORD_0]++; t->c[HT2_T_NDISCORD]++; t->outcome = HT2GPU_OUTCOME_AL1 | HT2GPU_OUTCOME_AL2; }   // aln_sink.h:2191-2192
            Ht2SamSumm summ; summ.reset();
            summ.paired = true;
            const ht2gpu_aln_t& a = rs1u[0]; const ht2gpu_aln_t& b = rs2u[0];
            { Ht2SamKey sc = {(int64_t)a.score + b.score, h2score(a, rd1.len) + h2score(b, rd2.len), true}; summ.bestPaired = sc; }
            addUnp(summ, 0, rs1u, n1, rd1.len); addUnp(summ, 1, rs2u, n2, rd2.len);
            summ.numAlnsPaired = 1; // AlnSetSumm::init counts rs1->size()
            const uint16_t dp[2] = {0, 0};
            (void)selectByScore(rs1u, n1, rd1.len, rs2u, rd2.len, dp, 1, true, 1, sel, rnd);
            Ht2SamFlags fl1 = {HT2_PAIR_DISCORD_MATE1, true, true}, fl2 = {HT2_PAIR_DISCORD_MATE2, true, true};
            const bool sameRef = a.tidx == b.tidx; // setMateParams (aligner_result.h:1594-1618)
            o.n += appendMate<W>(o.at(), rd1, rd2.len, &a, &b, summ, fl1, sameRef, sameRef ? fragmentLength(a, b, true) : 0, true);
            o.n += appendMate<W>(o.at(), rd2, rd1.len, &b, &a, summ, fl2, sameRef, sameRef ? fragmentLength(b, a, false) : 0, true);
            return;
        }
        uint64_t nunpair1 = 0, nunpair2 = 0;
        if (in->mixed && n1 + n2 > 0) {
            nunpair1 = n1 < in->khits ? n1 : in->khits;
            nunpair2 = n2 < in->khits ? n2 : in->khits;
        }
        const bool rep1 = nunpair1 > 0, rep2 = nunpair2 > 0;
        Ht2SamSumm summ1, summ2; summ1.reset(); summ2.reset();
        uint16_t sel2[HT2_SAM_MAXSEL];
        uint32_t nsel1 = 0, nsel2 = 0;
        const ht2gpu_aln_t *repRs1 = NULL, *repRs2 = NULL;
        if (rep1) {
            addUnp(summ1, 0, rs1u, n1, rd1.len);
            if (rep2) addUnp(summ1, 1, rs2u, n2, rd2.len);
            nsel1 = selectByScore(rs1u, n1, rd1.len, NULL, 0, NULL, 0, false, nunpair1, sel, rnd);
            repRs1 = &rs1u[sel[0]];
        }
        if (rep2) {
            addUnp(summ2, 1, rs2u, n2, rd2.len);
            if (rep1) addUnp(summ2, 0, rs1u, n1, rd1.len);
            nsel2 = selectByScore(rs2u, n2, rd2.len, NULL, 0, NULL, 0, false, nunpair2, sel2, rnd);
            repRs2 = &rs2u[sel2[0]];
        }
        // numAlns1/2 setters are applied to both summaries (aln_sink.h:2238-2239, 2263-2264)
        if (rep1) { summ1.numAlns[0] = nsel1; summ2.numAlns[0] = nsel1; }
        if (rep2) { summ1.numAlns[1] = nsel2; summ2.numAlns[1] = nsel2; }
        if (t) {   // aln_sink.h:2271-2346 (constant indexes: the device tally stays in registers)
            t->c[HT2_T_NCONCORD_0]++;
            t->c[HT2_T_NUNP_0_0] += (uint32_t)!rep1 + (uint32_t)!rep2;
            t->c[HT2_T_NUNP_0_UNI1] += (uint32_t)(rep1 && nsel1 == 1) + (uint32_t)(rep2 && nsel2 == 1);
            t->c[HT2_T_NUNP_0_UNI2] += (uint32_t)(rep1 && nsel1 != 1) + (uint32_t)(rep2 && nsel2 != 1);
            t->outcome = (rep1 ? HT2GPU_OUTCOME_AL1 : 0) | (rep2 ? HT2GPU_OUTCOME_AL2 : 0);
        }
        Ht2SamFlags fl1 = {HT2_PAIR_UNPAIRED_MATE1, true, repRs2 != NULL}, fl2 = {HT2_PAIR_UNPAIRED_MATE2, true, repRs1 != NULL};
        int64_t refid = -1, refoff = -1;
        if (rep1) {
            // AlnSink::reportHits (aln_sink.h:730-790)
            if (repRs2 != NULL) {
                const ht2gpu_aln_t* r1pri = &rs1u[sel[0]]; const ht2gpu_aln_t* r2pri = &rs2u[sel2[0]];
                o.n += appendMate<W>(o.at(), rd1, rd2.len, r1pri, r2pri, summ1, fl1, false, 0, false);
                o.n += appendMate<W>(o.at(), rd2, rd1.len, r2pri, r1pri, summ1, fl2, false, 0, false);
                fl1.primary = fl2.primary = false;
                for (uint32_t i = 1; i < nsel1; i++) o.n += appendMate<W>(o.at(), rd1, rd2.len, &rs1u[sel[i]], r2pri, summ1, fl1, false, 0, false);
                for (uint32_t i = 1; i < nsel2; i++) o.n += appendMate<W>(o.at(), rd2, rd1.len, &rs2u[sel2[i]], r1pri, summ1, fl2, false, 0, false);
                fl1.primary = fl2.primary = true;
            } else {
                for (uint32_t i = 0; i < nsel1; i++) {
                    fl1.primary = (i == 0);
                    o.n += appendMate<W>(o.at(), rd1, 0, &rs1u[sel[i]], NULL, summ1, fl1, false, 0, false);
                }
                fl1.primary = true;
            }
            refid = rs1u[sel[0]].tidx; refoff = rs1u[sel[0]].toff;
        }
        if (rep2 && !rep1) {
            for (uint32_t i = 0; i < nsel2; i++) {
                fl2.primary = (i == 0);
                o.n += appendMate<W>(o.at(), rd2, 0, &rs2u[sel2[i]], NULL, summ2, fl2, false, 0, false);
            }
            fl2.primary = true;
            refid = rs2u[sel2[0]].tidx; refoff = rs2u[sel2[0]].toff;
        }
        if (nunpair1 == 0) {
            Ht2SamSumm s; s.reset();
            if (nunpair2 > 0) { s.orefid = refid; s.orefoff = refoff; }
            Ht2SamFlags fl = {HT2_PAIR_UNPAIRED_MATE1, true, repRs2 != NULL};
            o.n += appendMate<W>(o.at(), rd1, 0, NULL, NULL, s, fl, false, 0, false);
        }
        if (nunpair2 == 0) {
            Ht2SamSumm s; s.reset();
            if (nunpair1 > 0) { s.orefid = refid; s.orefoff = refoff; }
            Ht2SamFlags fl = {HT2_PAIR_UNPAIRED_MATE2, true, repRs1 != NULL};
            o.n += appendMate<W>(o.at(), rd2, 0, NULL, NULL, s, fl, false, 0, false);
        }
    }

    // t != NULL: also tally the unit's outcome (the counting pass)
    template <bool W> HT2_HD void unit(Ht2SamOut<W>& o, uint32_t u, Ht2SamTally* t = NULL) const {
        Ht2SamCur<W> c = {W ? o.p + o.n : NULL, 0};
        if (in->paired) finishPaired(c, u, t); else finishUnpaired(c, u, t);
        if (t && in->unitOut) in->unitOut[u] = (uint8_t)t->outcome;
        o.n += c.n;
    }
};

#endif // HT2_SAM_H_
