// ht2_pair.h -- paired-end policy, pairReads and the anchor search of alignMate.
// Included from ht2_core.h.
#ifndef HT2_PAIR_H_
#define HT2_PAIR_H_

// PairedEndPolicy::peClassifyPair (pe.cpp:38-132) with the hisat2 defaults
// olapOk = containOk = expandToFit = true, dovetailOk = false (hisat2.cpp:348-352).
// Returns true iff the pair is NOT discordant.
template <bool GRAPH, bool NOSPL, bool DP> HT2_NI bool Ht2AlignerT<GRAPH, NOSPL, DP>::peConcordant(int64_t off1, uint32_t len1, bool fw1, int64_t off2, uint32_t len2, bool fw2) const
{
    uint32_t maxfrag = P->maxFrag;
    if (len1 > maxfrag) maxfrag = len1;
    if (len2 > maxfrag) maxfrag = len2;
    uint32_t minfrag = P->minFrag;
    if (minfrag < 1) minfrag = 1;
    bool oneLeft = false;
    switch (P->pePolicy) {
        case 0: if (fw1 != fw2) return false; oneLeft = fw1; break;   // FF
        case 1: if (fw1 != fw2) return false; oneLeft = !fw1; break;  // RR
        case 2: if (fw1 == fw2) return false; oneLeft = fw1; break;   // FR
        default: if (fw1 == fw2) return false; oneLeft = !fw1; break; // RF
    }
    int64_t fraglo = off1 < off2 ? off1 : off2;
    int64_t h1 = off1 + len1, h2 = off2 + len2;
    int64_t fraghi = h1 > h2 ? h1 : h2;
    uint64_t frag = (uint64_t)(fraghi - fraglo);
    if (frag > maxfrag || frag < minfrag) return false;
    int64_t lo1 = off1, hi1 = off1 + len1 - 1, lo2 = off2, hi2 = off2 + len2 - 1;
    bool containment = (lo1 >= lo2 && hi1 <= hi2) || (lo2 >= lo1 && hi2 <= hi1);
    bool olap = (lo1 <= lo2 && hi1 >= lo2) || (lo1 <= hi2 && hi1 >= hi2) || containment;
    if (!olap) {
        if ((oneLeft && lo2 < lo1) || (!oneLeft && lo1 < lo2)) return false;
    }
    if ((oneLeft && (hi1 > hi2 || lo2 < lo1)) || (!oneLeft && (hi2 > hi1 || lo1 < lo2))) return false; // dovetail
    return true;
}

// HI_Aligner::pairReads (hi_aligner.h:5948-6057) + AlnSinkWrap::report for a
// pair (aln_sink.h:2565-2611) + ReportingState::foundConcordant (aln_sink.cpp:72-92).
template <bool GRAPH, bool NOSPL, bool DP> HT2_NI void Ht2AlignerT<GRAPH, NOSPL, DP>::pairReads()
{
    const uint32_t n1 = W->nRes[0], n2 = W->nRes[1];
    uint32_t start_i = W->concordInspected[0], start_j = W->concordInspected[1];
    W->concordInspected[0] = n1;
    W->concordInspected[1] = n2;
    for (uint32_t i = 0; i < n1; i++) {
        for (uint32_t j = (i >= start_i ? 0 : start_j); j < n2; j++) {
            const Ht2Res& r1 = W->res[0][i];
            const Ht2Res& r2 = W->res[1][j];
            if (r1.tidx != r2.tidx) continue;
            // Coord left/right of each mate; orient() == fw
            int64_t left = r1.toff, right = (int64_t)r1.toff + r1.rfextent - 1;
            int64_t left2 = r2.toff, right2 = (int64_t)r2.toff + r2.rfextent - 1;
#ifdef HT2_ENABLE_SPLICED   // AlnRes::refcoord_right adds the introns (aligner_result.h:1255-1268)
            for (uint32_t e = 0; e < r1.nedits; e++) if (isSpl(W->resEdits[r1.editOff + e])) right += ht2_spl_len(W->resEdits[r1.editOff + e]);
            for (uint32_t e = 0; e < r2.nedits; e++) if (isSpl(W->resEdits[r2.editOff + e])) right2 += ht2_spl_len(W->resEdits[r2.editOff + e]);
#endif
            if ((r1.fw != 0) == (P->gMate1fw != 0)) {
                if ((r2.fw != 0) != (P->gMate2fw != 0)) continue;
            } else {
                if ((r2.fw != 0) == (P->gMate2fw != 0)) continue;
                int64_t t = left; left = left2; left2 = t;
                t = right; right = right2; right2 = t;
            }
            if (left > left2) continue;
            if (right > right2) continue;
            if (right + (int64_t)(int)P->maxIntronLen < left2) continue;
            bool dna_frag_pass = true;
            if (noSpl()) {
                if (r1.toff < r2.toff) dna_frag_pass = peConcordant(r1.toff, r1.rfextent, r1.fw != 0, r2.toff, r2.rfextent, r2.fw != 0);
                else dna_frag_pass = peConcordant(r2.toff, r2.rfextent, r2.fw != 0, r1.toff, r1.rfextent, r1.fw != 0);
            }
            if (!noSpl() || dna_frag_pass) {
                int64_t threshold = W->bestPair;
                if (W->bestUnp[0] >= minsc[0] && W->bestUnp[1] >= minsc[1]) {
                    double t = (double)(W->bestUnp[0] + W->bestUnp[1]) -
                               (double)(uint64_t)((uint64_t)r1.rdlen + (uint64_t)r2.rdlen) * 0.03 * (double)ht2_mmpen(*P, 255);
                    int64_t tmp = (int64_t)t;
                    if (tmp > threshold) threshold = tmp;
                }
                int64_t score = r1.score + r2.score;
                if (score >= threshold || P->secondary) {
                    // sink.report(0, &r1, &r2)
                    if (score > W->concordBest) { W->concordBest = score; W->nconcord = 0; }
                    W->nconcord++;
                    if (W->nPairs >= HT2_MAX_PAIRS) { W->err |= HT2_ERR_PAIRS; return; }
                    W->pairs[W->nPairs][0] = (uint16_t)i;
                    W->pairs[W->nPairs][1] = (uint16_t)j;
                    W->nPairs++;
                    if (score > W->bestPair) { W->best2Pair = W->bestPair; W->bestPair = score; }
                    else if (score > W->best2Pair) W->best2Pair = score;
                }
            }
        }
    }
}

// anchor search part of alignMate (hi_aligner.h:5600-5717): fills W->genomeHits
template <bool GRAPH, bool NOSPL, bool DP> HT2_NI void Ht2AlignerT<GRAPH, NOSPL, DP>::alignMateAnchors(uint32_t rdi, bool fw, uint32_t tidx, uint32_t toff)
{
    const uint32_t ordi = 1 - rdi;
    const bool ofw = (fw == (P->gMate2fw != 0)) ? (P->gMate1fw != 0) : (P->gMate2fw != 0);
    const uint32_t rdlen = W->rd[ordi].len;
    const uint32_t minKL = P->minKLocal;
    W->nGenomeHits = 0;
    Ht2Coord coords[HT2_MAX_COORDS];
    int lid = localIndexId(tidx, toff);
    bool first = true;
    uint32_t count = 0;
    uint32_t max_hitlen = 0;
    while (count++ < 2) {
        if (first) first = false;
        else {
            if (W->nGenomeHits > 0) break;
            lid = lid >= 0 ? (fw ? nextLocal(lid) : prevLocal(lid)) : -1;
            if (lid < 0 || localGeom(lid)->len == 0) break;
        }
        if (lid < 0 || localGeom(lid)->len == 0) break;
        Ht2Fm<uint16_t> lfm; lfm.init(blob, localGeom(lid));
        uint32_t hitoff = rdlen - 1;
        while (hitoff >= minKL - 1) {
            uint32_t hitlen = 0;
            uint32_t top = 0xffff, bot = 0xffff, node_top = 0xffff, node_bot = 0xffff;
            bool uniqueStop = false;
            uint32_t nelt = gfmSearch(lfm, ordi, ofw, hitoff, hitlen, top, bot, node_top, node_bot,
                                      uniqueStop, minKL, 0xffffu, P->kseeds, true);
            if (nelt > 0 && nelt <= P->kseeds && hitlen > max_hitlen) {
                uint32_t ncoords = 0;
                getGenomeCoordsLocal(lfm, top, bot, node_top, node_bot, ofw, hitoff - hitlen + 1, hitlen, coords, ncoords, HT2_MAX_COORDS);
                W->nGenomeHits = 0;
                for (uint32_t ri = 0; ri < ncoords; ri++) {
                    const Ht2Coord& coord = coords[ri];
                    if (noSpl()) {
                        if (coord.off + P->maxFrag * 2 < toff || toff + P->maxFrag * 2 < coord.off) continue;
                    }
                    if (W->nGenomeHits >= HT2_MAX_GHITS) { W->err |= HT2_ERR_GHITS; break; }
                    adjustWithALTCoord(hitoff - hitlen + 1, hitlen, coord, ordi);   // plain init on linear indexes (hi_aligner.h:5692)
                }
                max_hitlen = hitlen;
            }
            if (hitlen > 0) hitoff -= (hitlen - 1);
            if (hitoff > 0) hitoff -= 1;
        }
    }
    const uint32_t maxsize = P->kseeds;
    if (W->nGenomeHits > maxsize) {
        uint32_t left = W->nGenomeHits;
        for (uint32_t i = 0; i + 1 < W->nGenomeHits; i++) {
            uint32_t rndi = W->rnd.nextU32() % left;
            if (rndi > 0) {
                Ht2Hit* t = poolAlloc();
                copyHit(*t, W->genomeHits[i]); uint32_t hc = W->genomeHits[i].hitcount;
                copyHit(W->genomeHits[i], W->genomeHits[i + rndi]); W->genomeHits[i].hitcount = W->genomeHits[i + rndi].hitcount;
                copyHit(W->genomeHits[i + rndi], *t); W->genomeHits[i + rndi].hitcount = hc;
                W->poolTop--;
            }
            left--;
        }
        W->nGenomeHits = maxsize;
    }
}

#endif // HT2_PAIR_H_
