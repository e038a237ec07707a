// ht2_alt.h -- ALT-aware extension for graph (SNP) indexes.  Textually included INSIDE
// struct Ht2AlignerT (ht2_core.h); everything here is a member.
//
// Restates GenomeHit::alignWithALTs / alignWithALTs_recur (hi_aligner.h:683-783, 2763-3550) for
// SNP ALTs (single-base, deletion, insertion) and splice-site ALTs: a mismatch-bounded scan, then for
// every ALT in reach of the scanned stretch a recursive continuation that consumes the ALT with a
// zero-penalty edit carrying its id, or with a known splice edit across the site's intron.  Exon ALTs
// are skipped there (they only feed the splice-site DB).  Haplotype filtering (off by default,
// hisat2.cpp:522) and CODIS are not built.
//
// Under --no-spliced-alignment the reference drops the splice-site ALTs when it loads the index
// (gfm.h:760-771).  The image keeps them, so that its ALT ids do not depend on options; every walk here
// skips them instead (altSs), which visits the same ALTs in the same order.
//
// Scratch state of one alignWithALTs call lives in W->alt (Ht2AltScratch).
#if !defined(__CUDA_ARCH__) && defined(HT2_TRACE)
#define HT2_GERR(k) (fprintf(stderr, "graph capacity site %d\n", k), W->err |= HT2_ERR_GRAPH)
#else
#define HT2_GERR(k) (W->err |= HT2_ERR_GRAPH)
#endif

    HT2_HD const Ht2Alt* altTable() const { return (const Ht2Alt*)(blob + H->o_alts); }
    HT2_HD uint32_t numAlts() const { return H->nAlts; }
    // EList::bsearchLoBound with a key that only has 'pos' set (alt.h:89-103): first ALT with pos >= p
    HT2_HD uint32_t altLoBound(uint32_t p) const {
        const Ht2Alt* a = altTable();
        uint32_t lo = 0, hi = numAlts();
        while (lo < hi) { uint32_t mid = lo + ((hi - lo) >> 1); if (a[mid].pos < p) lo = mid + 1; else hi = mid; }
        return lo;
    }
    HT2_HD static bool altIsSnp(const Ht2Alt& a) { return a.type == HT2_ALT_SNP_SGL || a.type == HT2_ALT_SNP_DEL || a.type == HT2_ALT_SNP_INS; }
    // a splice-site ALT the run loaded (see above); altSsFw: the site as read (left < right), else its reversed copy
    HT2_HD bool altSs(const Ht2Alt& a) const { return a.type == HT2_ALT_SPLICESITE && !noSpl(); }
    HT2_HD bool altSsFw(const Ht2Alt& a) const { return altSs(a) && a.pos < a.len; }
    // the known splice edit of a splice-site ALT [left, right] (hi_aligner.h:3030-3040, 3430-3440)
    HT2_HD bool pushSsEdit(uint32_t pos, const Ht2Alt& a, uint32_t left, uint32_t right, bool front) {
        const uint32_t intronLen = right - left + 1;
        if (intronLen > HT2_MAX_SPL_LEN) { HT2_GERR(12); return false; }
        Ht2Edit e = mkAltEdit(pos, 'A', 'A', HT2_EDIT_SPL, 0);
        ht2_spl_set(e, intronLen, (a.seq & 0xff) ? HT2_SPL_FW : HT2_SPL_RC, true, 0.0f);
        return front ? tmpInsertFront(e) : tmpPush(e);
    }
    // a splice site as read among ALTs [a, b)
    HT2_HD bool ssInRange(uint32_t a, uint32_t b) const {
        const Ht2Alt* alts = altTable();
        for (uint32_t s = a; s < b; s++) if (altSsFw(alts[s])) return true;
        return false;
    }

    // tmp_edits helpers
    HT2_HD bool tmpPush(const Ht2Edit& e) {
        Ht2AltScratch& S = W->alt;
        if (S.ntmp >= HT2_ALT_TMP_EDITS) { W->err |= HT2_ERR_EDITS; return false; }
        S.tmp[S.ntmp++] = e; return true;
    }
    HT2_HD bool tmpInsertFront(const Ht2Edit& e) {
        Ht2AltScratch& S = W->alt;
        if (S.ntmp >= HT2_ALT_TMP_EDITS) { W->err |= HT2_ERR_EDITS; return false; }
        for (uint32_t i = S.ntmp; i > 0; i--) S.tmp[i] = S.tmp[i - 1];
        S.tmp[0] = e; S.ntmp++; return true;
    }
    HT2_HD void tmpEraseFront(uint32_t n) {
        Ht2AltScratch& S = W->alt;
        for (uint32_t i = 0; i + n < S.ntmp; i++) S.tmp[i] = S.tmp[i + n];
        S.ntmp -= n;
    }
    HT2_HD void editsFromTmp(Ht2Hit& h) {
        uint32_t n = W->alt.ntmp;
        if (n > HT2_MAX_EDITS) { W->err |= HT2_ERR_EDITS; n = HT2_MAX_EDITS; }   // the alignment itself needs more edits than a hit holds
        for (uint32_t i = 0; i < n; i++) h.edits[i] = W->alt.tmp[i];
        h.nedits = n;
    }
    HT2_HD void candClear() { W->alt.ncand = 0; }
    HT2_HD void candPushTmp() {
        Ht2AltScratch& S = W->alt;
        if (!S.wantCands) return;
        if (S.ncand >= HT2_ALT_CANDS) { HT2_GERR(1); return; }
        if (S.ntmp > HT2_MAX_EDITS) { W->err |= HT2_ERR_EDITS; return; }
        for (uint32_t i = 0; i < S.ntmp; i++) S.cand[S.ncand][i] = S.tmp[i];
        S.candN[S.ncand] = (uint8_t)S.ntmp;
        S.ncand++;
    }
    HT2_HD static Ht2Edit mkAltEdit(uint32_t pos, char chr, char qchr, uint8_t type, uint32_t snpID) {
        Ht2Edit e; e.pos = pos; e.chr = (uint8_t)chr; e.qchr = (uint8_t)qchr; e.type = type; e.pad = 0; e.snpID = snpID; return e;
    }

    // reference window [rfoff, rfoff+rflen) of tidx into one of the per-depth buffers; positions < 0 read as 4.
    // Returns NULL on capacity problems (flagged).
    HT2_NI const uint8_t* altFetch(uint32_t tidx, int rfoff, uint32_t rflen) {
        Ht2AltScratch& S = W->alt;
        if (S.nbuf >= HT2_ALT_BUFS || rflen > HT2_REFBUF) { HT2_GERR(2); return NULL; }
        uint8_t* buf = S.ref[S.nbuf++];
        const uint32_t lead = rfoff < 0 ? (uint32_t)(-rfoff) : 0;
        if (lead == 0) return getStretch(buf, tidx, (uint32_t)rfoff, rflen);
        for (uint32_t i = 0; i < lead && i < rflen; i++) buf[i] = 4;
        if (rflen > lead) getStretch(buf + lead, tidx, 0, rflen - lead, false);
        return buf;
    }

    // alignWithALTs_recur, left == true (hi_aligner.h:2822-3167)
    HT2_NI uint32_t altLeft(Ht2Hit& h, const uint8_t* seq, uint32_t joinedOff, uint32_t rdoff, uint32_t rdlen,
                            const uint8_t* rfseq, uint32_t tidx, int rfoff, uint32_t rflen, uint32_t mm,
                            uint32_t tmp_numNs, uint32_t* numNs, uint32_t dep, bool prevSs) {
        Ht2AltScratch& S = W->alt;
        if (S.numALTsTried > P->maxAltsTried + dep) return 0;
        if (dep >= HT2_ALT_MAXDEP) { HT2_GERR(3); return 0; }
        if (rfoff < -16) return 0;
        const uint32_t contig_len = refLen(tidx);
        if (rfoff >= 0 && (uint32_t)rfoff >= contig_len) return 0;
        if (rfoff >= 0 && (uint32_t)rfoff + rflen > contig_len) rflen = contig_len - (uint32_t)rfoff;
        else if (rfoff < 0 && rflen > contig_len) rflen = contig_len;
        if (rflen == 0) return 0;
        const uint32_t bufMark = S.nbuf;
        if (rfseq == NULL) { rfseq = altFetch(tidx, rfoff, rflen); if (rfseq == NULL) { S.nbuf = bufMark; return 0; } }
        uint32_t ret = 0;
        {
            uint32_t tmp_mm = 0;
            int min_rd_i = (int)rdoff, mm_min_rd_i = (int)rdoff;
            uint32_t mm_tmp_numNs = 0;
            for (int rf_i = (int)rflen - 1; rf_i >= 0 && mm_min_rd_i >= 0; rf_i--, mm_min_rd_i--) {
                const int rf_bp = rfseq[rf_i], rd_bp = seq[mm_min_rd_i];
                if (rf_bp != rd_bp || rd_bp == 4) {
                    if (tmp_mm == 0) min_rd_i = mm_min_rd_i;
                    if (tmp_mm >= mm) break;
                    tmp_mm++;
                    tmpInsertFront(mkAltEdit((uint32_t)mm_min_rd_i, ht2_code2asc(rf_bp), ht2_code2asc(rd_bp), HT2_EDIT_MM, HT2_IDX_MAX32));
                }
                if (rf_bp == 4) { if (tmp_mm == 0) tmp_numNs++; mm_tmp_numNs++; }
            }
            if (tmp_mm == 0) min_rd_i = mm_min_rd_i;
            if (mm_min_rd_i < S.best_rdoff) {
                S.best_rdoff = mm_min_rd_i;
                editsFromTmp(h);
                if (numNs) *numNs = mm_tmp_numNs;
            }
            if (mm_min_rd_i < 0) { S.nbuf = bufMark; return rdlen; }
            if (tmp_mm > 0) { tmpEraseFront(tmp_mm); tmp_mm = 0; }

            // ALTs in reach of this stretch (hi_aligner.h:2871-2903)
            const Ht2Alt* alts = altTable();
            const uint32_t nalts = numAlts();
            int first = 0, second = 0;
            if (nalts > 0) {
                const uint32_t minK = 16;
                uint32_t rd_diff = rdoff - (uint32_t)mm_min_rd_i;
                rd_diff = (rd_diff > minK ? rd_diff - minK : 0);
                const uint32_t key = (rd_diff >= joinedOff) ? joinedOff : joinedOff - rd_diff;
                first = second = (int)altLoBound(key);
                if ((uint32_t)first >= nalts) first = second = second - 1;
                for (; first >= 0; first--) {
                    const Ht2Alt& alt = alts[first];
                    if (altIsSnp(alt)) {
                        if (alt.type == HT2_ALT_SNP_DEL && !alt.reversed) continue;
                        if (alt.pos + rdlen < joinedOff) break;
                    } else if (altSs(alt)) {
                        if (alt.pos < alt.len) continue;
                        if (alt.pos + rdlen - 1 < joinedOff) break;
                    } else continue;
                }
            }
            const uint32_t orig_nedits = S.ntmp;
            for (; second > first; second--) {
                Ht2Alt alt = alts[second];
                if (alt.pos >= joinedOff) continue;
                const bool ss = altSs(alt);
                if (ss) {   // the reversed copy, turned back into [left, right] = [pos, len]
                    if (alt.pos < alt.len) continue;
                    const uint32_t t = alt.pos; alt.pos = alt.len; alt.len = t;
                }
                if (alt.type == HT2_ALT_SNP_DEL) {
                    if (!alt.reversed) continue;
                    alt.pos = alt.pos - alt.len + 1;
                }
                if (!altIsSnp(alt) && !ss) continue;
                bool alt_compatible = false;
                int rf_i = (int)rflen - 1, rd_i = (int)rdoff;
                int diff = 0;
                if (alt.type == HT2_ALT_SNP_SGL) diff = (int)(joinedOff - alt.pos - 1);
                else if (alt.type == HT2_ALT_SNP_DEL) {
                    if (alt.pos + alt.len >= joinedOff) continue;
                    diff = (int)(joinedOff - (alt.pos + alt.len));
                } else if (ss) diff = (int)(joinedOff - (alt.len + 1));
                else diff = (int)(joinedOff - alt.pos);
                if (rf_i < diff || rd_i < diff) continue;
                rf_i -= diff; rd_i -= diff;
                int rd_bp = seq[rd_i];
                if (rd_i < min_rd_i) {
                    if (alt.type == HT2_ALT_SNP_INS) { if (rd_i + 1 >= min_rd_i) continue; }
                    break;
                }
                if (alt.type == HT2_ALT_SNP_SGL) {
                    if (rd_bp == (int)alt.seq) {
                        const int rf_bp = rfseq[rf_i];
                        tmpInsertFront(mkAltEdit((uint32_t)rd_i, ht2_code2asc(rf_bp), ht2_code2asc(rd_bp), HT2_EDIT_MM, (uint32_t)second));
                        rd_i--; rf_i--;
                        alt_compatible = true;
                    }
                } else if (alt.type == HT2_ALT_SNP_DEL) {
                    if (rfoff + rf_i > (int)alt.len) {
                        if (rf_i > (int)alt.len) {
                            for (uint32_t i = 0; i < alt.len; i++) {
                                const int rf_bp = rfseq[rf_i - (int)i];
                                tmpInsertFront(mkAltEdit((uint32_t)(rd_i + 1), ht2_code2asc(rf_bp), '-', HT2_EDIT_READ_GAP, (uint32_t)second));
                            }
                        } else {
                            // long deletion: the window does not reach far enough to the left
                            const int new_rfoff = rfoff - (int)alt.len;
                            const uint32_t new_rflen = (uint32_t)rf_i + alt.len + 10;
                            const uint32_t m = S.nbuf;
                            const uint8_t* new_rfseq = altFetch(tidx, new_rfoff, new_rflen);
                            if (new_rfseq == NULL) break;
                            for (int i = 0; i < (int)alt.len; i++) {
                                const int rf_bp = new_rfseq[rf_i - i + (int)alt.len];
                                tmpInsertFront(mkAltEdit((uint32_t)(rd_i + 1), ht2_code2asc(rf_bp), '-', HT2_EDIT_READ_GAP, (uint32_t)second));
                            }
                            S.nbuf = m;
                        }
                        rf_i -= (int)alt.len;
                        alt_compatible = true;
                    }
                } else if (ss) {
                    // no splice right after a splice (hi_aligner.h:3021-3024)
                    if (!(rd_i == (int)rdoff && prevSs)) {
                        if (!pushSsEdit((uint32_t)(rd_i + 1), alt, alt.pos, alt.len, true)) break;
                        alt_compatible = true;
                    }
                } else { // insertion
                    if (rd_i > (int)alt.len) {
                        bool same_seq = true;
                        for (uint32_t i = 0; i < alt.len; i++) {
                            rd_bp = seq[rd_i - (int)i];
                            const int snp_bp = (int)((alt.seq >> (i << 1)) & 0x3);
                            if (rd_bp != snp_bp) { same_seq = false; break; }
                            tmpInsertFront(mkAltEdit((uint32_t)(rd_i - (int)i), '-', ht2_code2asc(rd_bp), HT2_EDIT_REF_GAP, (uint32_t)second));
                        }
                        if (same_seq) { rd_i -= (int)alt.len; alt_compatible = true; }
                    }
                }
                if (alt_compatible) {
                    S.numALTsTried++;
                    if (rd_i < 0) {
                        S.best_rdoff = rd_i;
                        editsFromTmp(h);
                        S.nbuf = bufMark;
                        return rdlen;
                    }
                    const uint32_t next_joinedOff = alt.pos;
                    int next_rfoff = rfoff;
                    const int next_rdoff = rd_i;
                    const uint8_t* next_rfseq = rfseq;
                    int next_rflen = rf_i + 1;
                    const int next_rdlen = rd_i + 1;
                    if (ss) {   // continue left of the intron
                        next_rfoff -= (int)(alt.len - alt.pos + 1);
                        next_rfseq = NULL;
                    }
                    if (next_rflen < next_rdlen) {
                        int add_len = next_rdlen + 10 - next_rflen;
                        if (next_rfoff < add_len) add_len = next_rfoff;
                        next_rfoff -= add_len;
                        next_rflen += add_len;
                        next_rfseq = NULL;
                    }
                    const uint32_t alignedLen = altLeft(h, seq, next_joinedOff, (uint32_t)next_rdoff, (uint32_t)next_rdlen, next_rfseq,
                                                        tidx, next_rfoff, (uint32_t)next_rflen, mm, tmp_numNs, numNs, dep + 1, ss);
                    if (alignedLen == (uint32_t)next_rdlen) { S.nbuf = bufMark; return rdlen; }
                }
                // restore
                if (orig_nedits < S.ntmp) tmpEraseFront(S.ntmp - orig_nedits);
            }
            ret = 0;
        }
        S.nbuf = bufMark;
        return ret;
    }

    // alignWithALTs_recur, left == false (hi_aligner.h:3168-3548)
    HT2_NI uint32_t altRight(Ht2Hit& h, const uint8_t* seq, uint32_t joinedOff, uint32_t rdoff_add, uint32_t rdoff, uint32_t rdlen,
                             const uint8_t* rfseq, uint32_t tidx, int rfoff, uint32_t rflen, uint32_t mm,
                             uint32_t tmp_numNs, uint32_t* numNs, uint32_t dep) {
        Ht2AltScratch& S = W->alt;
        if (S.numALTsTried > P->maxAltsTried + dep) return 0;
        if (dep >= HT2_ALT_MAXDEP) { HT2_GERR(4); return 0; }
        if (rfoff < -16) return 0;
        const uint32_t contig_len = refLen(tidx);
        if (rfoff >= 0 && (uint32_t)rfoff >= contig_len) return 0;
        if (rfoff >= 0 && (uint32_t)rfoff + rflen > contig_len) rflen = contig_len - (uint32_t)rfoff;
        else if (rfoff < 0 && rflen > contig_len) rflen = contig_len;
        if (rflen == 0) return 0;
        const uint32_t bufMark = S.nbuf;
        if (rfseq == NULL) { rfseq = altFetch(tidx, rfoff, rflen); if (rfseq == NULL) { S.nbuf = bufMark; return 0; } }
        uint32_t tmp_mm = 0, max_rd_i = 0, mm_max_rd_i = 0, mm_tmp_numNs = 0;
        for (uint32_t rf_i = 0; rf_i < rflen && mm_max_rd_i < rdlen; rf_i++, mm_max_rd_i++) {
            const int rf_bp = rfseq[rf_i], rd_bp = seq[rdoff + mm_max_rd_i];
            if (rf_bp != rd_bp || rd_bp == 4) {
                if (tmp_mm == 0) max_rd_i = mm_max_rd_i;
                if (tmp_mm >= mm) break;
                tmp_mm++;
                tmpPush(mkAltEdit(mm_max_rd_i + rdoff_add, ht2_code2asc(rf_bp), ht2_code2asc(rd_bp), HT2_EDIT_MM, HT2_IDX_MAX32));
            }
            if (rf_bp == 4) { if (tmp_mm == 0) tmp_numNs++; mm_tmp_numNs++; }
        }
        if (tmp_mm == 0) max_rd_i = mm_max_rd_i;
        if ((int)(mm_max_rd_i + rdoff) > S.best_rdoff) {
            S.best_rdoff = (int)(mm_max_rd_i + rdoff);
            editsFromTmp(h);
            if (numNs) *numNs = mm_tmp_numNs;
            candClear();
        } else if ((int)(mm_max_rd_i + rdoff) == S.best_rdoff) {
            candPushTmp();
        }
        if (mm_max_rd_i == rflen) { S.nbuf = bufMark; return mm_max_rd_i; }

        // ALTs in reach (hi_aligner.h:3211-3234)
        const Ht2Alt* alts = altTable();
        const uint32_t nalts = numAlts();
        uint32_t first, second;
        {
            const uint32_t minK = 16;
            const uint32_t rd_diff = (max_rd_i > minK ? max_rd_i - minK : 0);
            first = second = altLoBound(joinedOff + rd_diff);
            if (first >= nalts) { S.nbuf = bufMark; return 0; }
            for (; second < nalts; second++) {
                const Ht2Alt& alt = alts[second];
                if (alt.type == HT2_ALT_SPLICESITE && !altSsFw(alt)) continue;
                if (alt.type == HT2_ALT_SNP_DEL && alt.reversed) continue;
                if (alt.pos > joinedOff + max_rd_i) break;
            }
        }
        if (mm_max_rd_i == rdlen && !ssInRange(first, second)) { S.nbuf = bufMark; return mm_max_rd_i; }   // a splice site in reach is still tried
        if (tmp_mm > 0) { S.ntmp -= tmp_mm; tmp_mm = 0; }
        const uint32_t orig_nedits = S.ntmp;
        for (; first < second; first++) {
            const Ht2Alt& alt = alts[first];
            const bool ss = altSsFw(alt);
            if (!altIsSnp(alt) && !ss) continue;
            if (alt.type == HT2_ALT_SNP_DEL && alt.reversed) continue;
            bool alt_compatible = false;
            uint32_t rf_i, rd_i;
            rf_i = rd_i = alt.pos - joinedOff;
            if (rd_i >= rdlen) continue;
            int rf_bp = rfseq[rf_i];
            int rd_bp = seq[rdoff + rd_i];
            if (alt.type == HT2_ALT_SNP_SGL) {
                if (rd_bp == (int)alt.seq) {
                    tmpPush(mkAltEdit(rd_i + rdoff_add, ht2_code2asc(rf_bp), ht2_code2asc(rd_bp), HT2_EDIT_MM, first));
                    rd_i++; rf_i++;
                    alt_compatible = true;
                }
            } else if (alt.type == HT2_ALT_SNP_DEL) {
                bool try_del = rd_i > 0;
                if (rd_i == 0 && dep > 0) {
                    // avoid consecutive deletions
                    if (S.ntmp > 0 && S.tmp[S.ntmp - 1].type != HT2_EDIT_READ_GAP) try_del = true;
                }
                if (try_del) {
                    if (rf_i + alt.len <= rflen) {
                        for (uint32_t i = 0; i < alt.len; i++) {
                            rf_bp = rfseq[rf_i + i];
                            tmpPush(mkAltEdit(rd_i + rdoff_add, ht2_code2asc(rf_bp), '-', HT2_EDIT_READ_GAP, first));
                        }
                        rf_i += alt.len;
                        alt_compatible = true;
                    } else {
                        // long deletion: fetch a longer window from the same start
                        const uint32_t new_rflen = rf_i + alt.len + 10;
                        const uint32_t m = S.nbuf;
                        const uint8_t* new_rfseq = altFetch(tidx, rfoff, new_rflen);
                        if (new_rfseq == NULL) break;
                        for (uint32_t i = 0; i < alt.len; i++) {
                            rf_bp = new_rfseq[rf_i + i];
                            tmpPush(mkAltEdit(rd_i + rdoff_add, ht2_code2asc(rf_bp), '-', HT2_EDIT_READ_GAP, first));
                        }
                        S.nbuf = m;
                        rf_i += alt.len;
                        alt_compatible = true;
                    }
                }
            } else if (ss) {
                // no two introns in a row (hi_aligner.h:3413-3421)
                bool try_splice = rd_i > 0;
                if (rd_i == 0 && dep > 0) {
                    if (S.ntmp > 0 && S.tmp[S.ntmp - 1].type != HT2_EDIT_SPL) try_splice = true;
                }
                if (try_splice) {
                    if (!pushSsEdit(rd_i + rdoff_add, alt, alt.pos, alt.len, false)) break;
                    alt_compatible = true;
                }
            } else { // insertion
                if (rd_i + alt.len <= rdlen && rf_i > 0) {
                    bool same_seq = true;
                    for (uint32_t i = 0; i < alt.len; i++) {
                        rd_bp = seq[rdoff + rd_i + i];
                        const int snp_bp = (int)((alt.seq >> ((alt.len - i - 1) << 1)) & 0x3);
                        if (rd_bp != snp_bp) { same_seq = false; break; }
                        tmpPush(mkAltEdit(rd_i + i + rdoff_add, '-', ht2_code2asc(rd_bp), HT2_EDIT_REF_GAP, first));
                    }
                    if (same_seq) { rd_i += alt.len; alt_compatible = true; }
                }
            }
            if (alt_compatible) {
                S.numALTsTried++;
                if (rd_i == rdlen) {
                    if (S.best_rdoff < (int)(rdoff + rd_i)) candClear();
                    candPushTmp();
                    S.best_rdoff = (int)(rdoff + rd_i);
                    editsFromTmp(h);
                    S.nbuf = bufMark;
                    return rd_i;
                }
                uint32_t next_joinedOff = 0;
                int next_rfoff = rfoff + (int)rf_i;
                const uint32_t next_rdoff = rdoff + rd_i;
                const uint8_t* next_rfseq = rfseq + rf_i;
                uint32_t next_rflen = rflen - rf_i;     // wraps like the reference's index_t when rf_i > rflen (long deletion)
                const uint32_t next_rdlen = rdlen - rd_i;
                if (alt.type == HT2_ALT_SNP_SGL) next_joinedOff = alt.pos + 1;
                else if (alt.type == HT2_ALT_SNP_DEL) { next_joinedOff = alt.pos + alt.len; if (rflen <= rf_i) next_rflen = 0; }
                else if (ss) {   // continue right of the intron
                    next_joinedOff = alt.len + 1;
                    next_rfoff += (int)(alt.len - alt.pos + 1);
                    next_rfseq = NULL;
                }
                else next_joinedOff = alt.pos;
                if (next_rflen < next_rdlen) { next_rflen = next_rdlen + 10; next_rfseq = NULL; }
                const uint32_t alignedLen = altRight(h, seq, next_joinedOff, rdoff_add + rd_i, next_rdoff, next_rdlen, next_rfseq, tidx,
                                                     next_rfoff, next_rflen, mm, tmp_numNs, numNs, dep + 1);
                if (alignedLen > 0) {
                    // after a splice, a later splice site in reach is still tried (hi_aligner.h:3517-3530)
                    if (!(ss && ssInRange(first + 1, second)) && rd_i + alignedLen == rdlen) { S.nbuf = bufMark; return rd_i + alignedLen; }
                }
            }
            if (orig_nedits < S.ntmp) S.ntmp = orig_nedits;
        }
        S.nbuf = bufMark;
        return 0;
    }

    // GenomeHit::alignWithALTs (hi_aligner.h:683-783).  h.edits is both input and result ("edits").
    HT2_NI uint32_t alignWithALTs(Ht2Hit& h, const uint8_t* seq, uint32_t joinedOff, uint32_t base_rdoff, uint32_t rdoff, uint32_t rdlen,
                                  uint32_t tidx, int rfoff, uint32_t rflen, bool left, bool wantCands, uint32_t mm, uint32_t* numNs) {
        Ht2AltScratch& S = W->alt;
        S.best_rdoff = (int)rdoff;
        if (numNs) *numNs = 0;
        S.numALTsTried = 0;
        S.nbuf = 0;
        S.wantCands = wantCands ? 1 : 0;
        S.ncand = 0;
        for (uint32_t i = 0; i < h.nedits; i++) S.tmp[i] = h.edits[i];
        S.ntmp = h.nedits;
        const uint32_t nedits = h.nedits;
        if (left) altLeft(h, seq, joinedOff, rdoff, rdlen, NULL, tidx, rfoff, rflen, mm, 0, numNs, 0, false);
        else altRight(h, seq, joinedOff, rdoff - base_rdoff, rdoff, rdlen, NULL, tidx, rfoff, rflen, mm, 0, numNs, 0);
        uint32_t extlen = left ? (rdoff - (uint32_t)S.best_rdoff) : ((uint32_t)S.best_rdoff - rdoff);
        if (left && S.best_rdoff < 0) extlen = rdoff + 1;
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
            if (extlen == 0 && h.nedits > nedits) {
                if (left) {
                    const uint32_t added = h.nedits - nedits;
                    for (uint32_t i = 0; i + added < h.nedits; i++) h.edits[i] = h.edits[i + added];
                    h.nedits = nedits;
                } else h.nedits = nedits;
            }
        }
        return extlen;
    }

    // =====================================================================================
    // graph search inside the aligner (partial search, global / local GFM search, coordinates)
    // =====================================================================================

    // HI_Aligner::partialSearch on a graph index: the generic chain step of ht2_seed.h, stored as a BWTHit
    // with its in-edge list (hi_aligner.h:6361-6601).
    // Returns false when the search was parked after a slice of steps (W->psG): call again to continue.
#ifndef HT2_PSG_SLICE
#define HT2_PSG_SLICE 8
#endif
    HT2_NI bool partialSearchGraph(uint32_t rdi, bool fw, bool& pseudogeneStop, bool& anchorStop) {
        Ht2ReadHits& hit = W->hits[rdi][fw ? 0 : 1];
        if (!W->psG.active && hit.nhits >= HT2_MAX_PHITS) { W->err |= HT2_ERR_PHITS; hit.cur = W->rd[rdi].len; hit.done = 1; return true; }
        Ht2SeedState st;
        st.len = W->rd[rdi].len; st.cur = hit.cur; st.done = hit.done;
        st.numPartialSearch = hit.numPartialSearch; st.numUniqueSearch = hit.numUniqueSearch;
        st.err = 0; st.nLF = 0; st.algBytes = 0;
        Ht2SeedHit sh;
        const bool finished = ht2_seed_partial<true>(gfm, *P, W->rd[rdi].seq[fw ? 0 : 1], st, sh, pseudogeneStop, anchorStop, &W->psG, HT2_PSG_SLICE);
        hit.numPartialSearch = st.numPartialSearch;
        W->nLF += st.nLF; W->algBytes += st.algBytes;
        if (st.err) HT2_GERR(5);
        if (!finished) return false;
        hit.cur = st.cur; hit.done = st.done; hit.numUniqueSearch = st.numUniqueSearch;
        Ht2BwtHit& ph = hit.hits[hit.nhits++];
        ph.top = sh.top; ph.bot = sh.bot; ph.node_top = sh.node_top; ph.node_bot = sh.node_bot;
        ph.bwoff = sh.bwoff; ph.len = sh.len; ph.hit_type = sh.hit_type; ph.hasCoords = 0;
        ph.ieOff = (uint8_t)hit.nie; ph.ieN = 0;
        if (sh.niedges > 0) {
            if (hit.nie + sh.niedges > HT2_IE_POOL) { HT2_GERR(6); }
            else {
                for (uint32_t e = 0; e < sh.niedges; e++) { hit.ie[hit.nie + e][0] = sh.iedges[e][0]; hit.ie[hit.nie + e][1] = sh.iedges[e][1]; }
                ph.ieN = sh.niedges; hit.nie += sh.niedges;
            }
        }
        return true;
    }

    // globalGFMSearch / localGFMSearch on a graph index (hi_aligner.h:6606-6744, 6751-6892); the in-edge list
    // of the result is left in W->curIe (the reference's _node_iedge_count / _local_node_iedge_count).
    template <typename IT>
    HT2_NI uint32_t gfmSearchGraph(const Ht2Fm<IT>& fm, uint32_t rdi, bool fw, uint32_t rdoff, uint32_t& hitlen,
                                   uint32_t& top, uint32_t& bot, uint32_t& node_top, uint32_t& node_bot,
                                   bool& uniqueStop, uint32_t minUniqueLen, uint32_t maxHitLen, uint32_t maxHits, bool local) {
        const bool uniqueStop_ = uniqueStop;
        uniqueStop = false;
        W->nCurIe = 0;
        const uint32_t ftabLen = fm.g->ftabChars;
        const uint32_t len = W->rd[rdi].len;
        const uint8_t* seq = W->rd[rdi].seq[fw ? 0 : 1];
        const uint32_t offset = len - rdoff - 1;
        uint32_t dep = offset;
        if (local) top = bot = node_top = node_bot = 0;
        const uint32_t left = len - dep;
        if (left < ftabLen + 1) { hitlen = left; return 0; }
        for (uint32_t i = 0; i < ftabLen; i++) {
            if (seq[len - dep - 1 - i] > 3) { hitlen = i + 1; return 0; }
        }
        uint32_t rtop = 0, rbot = 0, ntop = 0, nbot = 0;
        ht2_ftab_lohi(fm, seq, len - dep - ftabLen, rtop, rbot);
        W->algBytes += 2 * (uint32_t)sizeof(IT);
        dep += ftabLen;
        if (rtop >= rbot) { hitlen = ftabLen; return 0; }
        Ht2SeedState st; st.err = 0; st.nLF = 0; st.algBytes = 0;
        uint16_t tie[HT2G_MAX_IEDGES][2];
        uint32_t ntie = 0;
        while (dep < len) {
            const int c = seq[len - dep - 1];
            uint32_t ttop = 0, tbot = 0, tntop = 0, tnbot = 0;
            ntie = 0;
            if (c <= 3) ht2_seed_step<true, IT>(fm, rtop, rbot, c, P->kseeds, ttop, tbot, tntop, tnbot, tie, ntie, st);
            if (ttop >= tbot) break;
            rtop = ttop; rbot = tbot; ntop = tntop; nbot = tnbot;
            W->nCurIe = ntie;
            for (uint32_t e = 0; e < ntie; e++) { W->curIe[e][0] = tie[e][0]; W->curIe[e][1] = tie[e][1]; }
            dep++;
            if (uniqueStop_) {
                if (rbot - rtop == 1 && dep - offset >= minUniqueLen) { uniqueStop = true; break; }
            }
            if (local && dep - offset >= maxHitLen) break;
        }
        W->nLF += st.nLF; W->algBytes += st.algBytes;
        if (st.err) HT2_GERR(7);
        uint32_t nelt = 0;
        if (ntop < nbot && nbot - ntop <= maxHits) {
            top = rtop; bot = rbot; node_top = ntop; node_bot = nbot;
            nelt = nbot - ntop;
            hitlen = dep - offset;
        }
        return nelt;
    }

    // first BW row of element i of a node range (group_walk.h:545-560)
    HT2_HD static uint32_t elementRow(uint32_t top, const uint16_t (*ie)[2], uint32_t nie, uint32_t i) {
        uint32_t num_iedges = 0;
        for (uint32_t e = 0; e < nie; e++) { if (i <= ie[e][0]) break; num_iedges += ie[e][1]; }
        return top + i + num_iedges;
    }

    // HI_Aligner::getGenomeCoords on a graph index (hi_aligner.h:5774-5855); appends to W->coords.  The
    // offsets come from the group walk (ht2_gwalk.h), not from independent per-node walks.
    HT2_NI bool getGenomeCoordsGraph(uint32_t top, uint32_t bot, uint32_t node_top, uint32_t node_bot, const uint16_t (*ie)[2], uint32_t nie,
                                     bool fw, uint32_t maxelt, uint32_t rdlen, bool rejectStraddle, bool& straddled) {
        straddled = false;
        uint32_t nelt = node_bot - node_top;
        if (nelt > maxelt) nelt = maxelt;
        Ht2GroupWalk<uint32_t> gw(gfm, W->gw);
        gw.init(top, bot, node_top, nelt, ie, nie);
        bool ok = true;
        for (uint32_t i = 0; i < nelt && i < HT2_GW_MAXELT; i++) {
            const uint32_t joff = gw.resolve(i);
            if (W->gw.err) break;
            uint32_t tidx = 0, toff = 0;
            bool straddled2 = false;
            joinedToTextOff(gfm, rdlen, joff, tidx, toff, rejectStraddle, straddled2);
            straddled |= straddled2;
            if (tidx == HT2_IDX_MAX32) { ok = false; break; }
            if (W->nCoords >= HT2_MAX_COORDS) { W->err |= HT2_ERR_COORDS; ok = false; break; }
            Ht2Coord& c = W->coords[W->nCoords++];
            c.ref = straddled2 ? HT2_IDX_MAX32 : tidx;
            c.off = toff; c.fw = fw ? 1 : 0; c.joinedOff = joff;
        }
        W->nLF += W->gw.nLF; W->algBytes += W->gw.nLF * 3u * HT2_GSIDE_BYTES + 4u * nelt;
        if (W->gw.err) { HT2_GERR(10); return false; }
        return ok;
    }

    // HI_Aligner::getGenomeCoords_local on a graph local index (hi_aligner.h:5861-5941); uses W->curIe.
    HT2_NI bool getGenomeCoordsLocalGraph(const Ht2Fm<uint16_t>& lfm, uint32_t top, uint32_t bot, uint32_t node_top, uint32_t node_bot, bool fw,
                                          uint32_t rdoff, uint32_t rdlen, Ht2Coord* out, uint32_t& nout, uint32_t cap) {
        const uint32_t nelt = node_bot - node_top;
        Ht2GroupWalk<uint16_t> gw(lfm, W->gw);
        gw.init(top, bot, node_top, nelt, W->curIe, W->nCurIe);
        bool ok = true;
        for (uint32_t i = 0; i < nelt && i < HT2_GW_MAXELT; i++) {
            const uint32_t joff = gw.resolve(i);
            if (W->gw.err) break;
            uint32_t tidx = 0, toff = 0;
            bool straddled2 = false;
            const bool found = joinedToTextOff(lfm, rdlen, joff, tidx, toff, true, straddled2);
            if (!found) continue;
            const uint32_t global_toff = toff + lfm.g->localOffset;
            const uint32_t joinedOff = joff + lfm.g->joinedOffset;
            if (global_toff < rdoff) continue;
            if (nout >= cap) { W->err |= HT2_ERR_COORDS; ok = false; break; }
            Ht2Coord& c = out[nout++];
            c.ref = lfm.g->tidx; c.off = global_toff; c.fw = fw ? 1 : 0; c.joinedOff = joinedOff;
        }
        W->nLF += W->gw.nLF; W->algBytes += W->gw.nLF * 3u * HT2_GSIDE_BYTES + 2u * nelt;
        if (W->gw.err) { HT2_GERR(11); return false; }
        return ok;
    }

    // GenomeHit::findOffDiffs (hi_aligner.h:2545-2650), SNP indels only (splice sites are skipped).  Entries are (|diff|, sign) with
    // sign stored as 0 / 1 / 2 for -1 / 0 / +1 so that the pair ordering of the reference's sort is the
    // ordering of the two unsigned values.  Returns single_offDiffs_size.
    HT2_NI uint32_t findOffDiffs(uint32_t start, uint32_t end) {
        uint32_t (*od)[2] = W->offDiffs;
        uint32_t n = 0;
        od[n][0] = 0; od[n][1] = 1; n++;
        const Ht2Alt* alts = altTable();
        const uint32_t nalts = numAlts();
        uint32_t first = altLoBound(start), second;
        for (second = first; second < nalts; second++) {
            const Ht2Alt& alt = alts[second];
            if (alt.type == HT2_ALT_SPLICESITE && !altSsFw(alt)) continue;
            if (alt.type == HT2_ALT_SNP_DEL && alt.reversed) continue;
            if (alt.pos >= end) break;
        }
        if (first >= second) { W->nOffDiffs = n; return n; }
        auto isIndel = [](const Ht2Alt& a) { return (a.type == HT2_ALT_SNP_DEL && !a.reversed) || a.type == HT2_ALT_SNP_INS; };
        for (uint32_t s = second; s > first; s--) {
            const Ht2Alt& alt = alts[s - 1];
            if (!isIndel(alt)) continue;
            if (n >= 40) { HT2_GERR(8); break; }
            od[n][0] = alt.len; od[n][1] = (alt.type == HT2_ALT_SNP_DEL) ? 2u : 0u; n++;
        }
        if (n > 1) {
            // sort + unique on (first, second)
            for (uint32_t i = 1; i < n; i++) {
                uint32_t a0 = od[i][0], a1 = od[i][1]; uint32_t j = i;
                while (j > 0 && (od[j - 1][0] > a0 || (od[j - 1][0] == a0 && od[j - 1][1] > a1))) { od[j][0] = od[j - 1][0]; od[j][1] = od[j - 1][1]; j--; }
                od[j][0] = a0; od[j][1] = a1;
            }
            uint32_t m = 1;
            for (uint32_t i = 1; i < n; i++) if (od[i][0] != od[m - 1][0] || od[i][1] != od[m - 1][1]) { od[m][0] = od[i][0]; od[m][1] = od[i][1]; m++; }
            n = m;
        }
        const uint32_t single = n;
        for (uint32_t s = second; s > first; s--) {
            const Ht2Alt& alt = alts[s - 1];
            if (!isIndel(alt)) continue;
            int off = (alt.type == HT2_ALT_SNP_DEL) ? (int)alt.len : -(int)alt.len;
            for (uint32_t s2 = s - 1; s2 > first; s2--) {
                const Ht2Alt& alt2 = alts[s2 - 1];
                if (!isIndel(alt2)) continue;
                if (alt2.type == HT2_ALT_SNP_DEL) { if (alt2.pos + alt2.len >= alt.pos) continue; off += (int)alt2.len; }
                else { if (alt2.pos >= alt.pos) continue; off -= (int)alt2.len; }
                bool found = false;
                for (uint32_t i = 0; i < n; i++) {
                    const int cmp = (int)od[i][0] * ((int)od[i][1] - 1);
                    if (off == cmp) { found = true; break; }
                }
                if (!found) {
                    if (n >= 40) { HT2_GERR(9); break; }
                    od[n][0] = (uint32_t)(off < 0 ? -off : off); od[n][1] = off > 0 ? 2u : 0u; n++;
                }
            }
        }
        W->nOffDiffs = n;
        return single;
    }

    // shared body of the two adjustWithALT versions: try the offset differences until the seed aligns over
    // its whole length through the ALTs (hi_aligner.h:2296-2350, 2407-2470).  asGenomeHit: the static version --
    // h is the last element of W->genomeHits, a result equal to an earlier genome hit does not count, and the
    // equally long alternatives (candidate_edits) are appended as further genome hits.
    HT2_NI bool adjustTry(Ht2Hit& h, uint32_t rdi, bool asGenomeHit) {
#if !defined(__CUDA_ARCH__) && defined(HT2_TRACE)
        if (h.tidx >= H->nRefs) fprintf(stderr, "adjustTry: bad tidx %u toff %u joined %u rdoff %u len %u asGH %d st %u nframes %u pc %d\n", h.tidx, h.toff, h.joinedOff, h.rdoff, h.len, (int)asGenomeHit, W->st, W->nFrames, W->nFrames ? (int)W->frames[W->nFrames-1].pc : -1);
#endif
        const uint32_t width = 1u << (gfm.g->offRate + 2);
        const uint32_t single = findOffDiffs(h.joinedOff >= width ? h.joinedOff - width : 0, h.joinedOff + width);
        const uint8_t* seq = W->rd[rdi].seq[h.fw ? 0 : 1];
        const uint32_t orig_joinedOff = h.joinedOff, orig_toff = h.toff;
        bool found = false;
        const uint32_t max_extra = (P->maxAltsTried / 4) > 4 ? (P->maxAltsTried / 4) : 4;
        uint32_t n = W->nOffDiffs;
        if (n - single > max_extra) n = single + max_extra;
        for (uint32_t o = 0; o < n && !found; o++) {
            const uint32_t d = W->offDiffs[o][0]; const uint32_t sgn = W->offDiffs[o][1];
            if (sgn >= 1) { h.joinedOff = orig_joinedOff + d; h.toff = orig_toff + d; }
            else {
                if (orig_toff < d) continue;
                h.joinedOff = orig_joinedOff - d; h.toff = orig_toff - d;
            }
            if (asGenomeHit) h.nedits = 0;
            const uint32_t reflen = h.len + 10;
            const uint32_t alignedLen = alignWithALTs(h, seq, h.joinedOff, h.rdoff, h.rdoff, h.len, h.tidx, (int)h.toff, reflen,
                                                      false, asGenomeHit, 0, NULL);
            if (alignedLen == h.len) {
                found = true;
                if (asGenomeHit) {
                    for (uint32_t i = 0; i + 1 < W->nGenomeHits; i++) if (hitEq(W->genomeHits[i], h)) found = false;
                    if (found) {
                        const uint32_t ncand = W->alt.ncand;
                        for (uint32_t e = 0; e < ncand; e++) {
                            if (W->nGenomeHits >= HT2_MAX_GHITS) { W->err |= HT2_ERR_GHITS; break; }
                            Ht2Hit& nh = W->genomeHits[W->nGenomeHits];
                            copyHit(nh, W->genomeHits[W->nGenomeHits - 1]);
                            nh.nedits = W->alt.candN[e];
                            for (uint32_t k = 0; k < nh.nedits; k++) nh.edits[k] = W->alt.cand[e][k];
                            W->nGenomeHits++;
                            for (uint32_t i = 0; i + 1 < W->nGenomeHits; i++) {
                                if (hitEq(W->genomeHits[i], W->genomeHits[W->nGenomeHits - 1])) { W->nGenomeHits--; break; }
                            }
                        }
                    }
                }
            } else h.nedits = 0;
        }
        return found;
    }

    // GenomeHit::adjustWithALT, member version (hi_aligner.h:2395-2478)
    HT2_NI bool adjustWithALT(Ht2Hit& h, uint32_t rdi) {
        if (!GRAPH) return true;
        return adjustTry(h, rdi, false);
    }

    // GenomeHit::findSSOffs (hi_aligner.h:2485-2540): the joined-offset shifts a BWT hit whose path crossed splice
    // edges of the graph may need -- every intron of a site in [start, end), and the distances from a site's left
    // end to the right ends of other sites near its right end -- as sorted, unique (|shift|, sign) pairs with sign
    // 0 / 1 / 2 for -1 / 0 / +1, the first being (0, 0).  Returns the number of pairs.
    HT2_NI uint32_t findSSOffs(uint32_t start, uint32_t end, uint32_t (*so)[2]) {
        uint32_t n = 0;
        so[n][0] = 0; so[n][1] = 1; n++;
        if (H->nSpliceSites == 0 || noSpl()) return n;
        const Ht2Alt* alts = altTable();
        const uint32_t nalts = numAlts();
        for (uint32_t i = altLoBound(start); i < nalts; i++) {
            const Ht2Alt& alt = alts[i];
            if (alt.pos >= end) break;
            if (alt.type != HT2_ALT_SPLICESITE) continue;
            if (n >= HT2_SS_OFFS) { HT2_GERR(13); return n; }
            if (alt.pos < alt.len) {
                so[n][0] = alt.len - alt.pos + 1; so[n][1] = 2; n++;
                const uint32_t relax = 5;
                for (uint32_t j = altLoBound(alt.len > relax ? alt.len - relax : 0); j < nalts; j++) {
                    const Ht2Alt& alt2 = alts[j];
                    if (alt2.type != HT2_ALT_SPLICESITE) continue;
                    if (alt2.pos < alt2.len) continue;
                    if (alt2.pos + alt2.len == alt.pos + alt.len) continue;
                    if (alt2.pos > alt.len + relax) break;
                    if (n >= HT2_SS_OFFS) { HT2_GERR(13); return n; }
                    if (alt2.len < alt.pos) { so[n][0] = alt.pos - alt2.len; so[n][1] = 0; }
                    else { so[n][0] = alt2.len - alt.pos; so[n][1] = 2; }
                    n++;
                }
            } else {
                so[n][0] = alt.pos - alt.len + 1; so[n][1] = 0; n++;
            }
        }
        if (n > 1) {   // sort + unique on (first, second)
            for (uint32_t i = 1; i < n; i++) {
                const uint32_t a0 = so[i][0], a1 = so[i][1]; uint32_t j = i;
                while (j > 0 && (so[j - 1][0] > a0 || (so[j - 1][0] == a0 && so[j - 1][1] > a1))) { so[j][0] = so[j - 1][0]; so[j][1] = so[j - 1][1]; j--; }
                so[j][0] = a0; so[j][1] = a1;
            }
            uint32_t m = 1;
            for (uint32_t i = 1; i < n; i++) if (so[i][0] != so[m - 1][0] || so[i][1] != so[m - 1][1]) { so[m][0] = so[i][0]; so[m][1] = so[i][1]; m++; }
            n = m;
        }
        return n;
    }

    // GenomeHit::adjustWithALT, static version used by getAnchorHits (hi_aligner.h:2239-2388): for each splice shift
    // of findSSOffs, appends the adjusted hit (and its equally good alternatives) to W->genomeHits.  The result is
    // the last shift's, as in the reference.
    HT2_NI bool adjustWithALTCoord(uint32_t rdoff, uint32_t len, const Ht2Coord& coord, uint32_t rdi) {
        if (!GRAPH) {
            if (W->nGenomeHits >= HT2_MAX_GHITS) { W->err |= HT2_ERR_GHITS; return false; }
            initHit(W->genomeHits[W->nGenomeHits++], coord.fw != 0, rdoff, len, 0, 0, coord.ref, coord.off, coord.joinedOff);
            return true;
        }
        const uint32_t width = 1u << (gfm.g->offRate + 2);
        uint32_t ssOffs[HT2_SS_OFFS][2];
        const uint32_t nss = findSSOffs(coord.joinedOff >= width ? coord.joinedOff - width : 0, coord.joinedOff + width, ssOffs);
        bool found = false;
        for (uint32_t s = 0; s < nss; s++) {
            uint32_t off = coord.off, joinedOff = coord.joinedOff;
            if (ssOffs[s][0] > 0) {
                if (ssOffs[s][1] > 1) { off += ssOffs[s][0]; joinedOff += ssOffs[s][0]; }
                else { off -= ssOffs[s][0]; joinedOff -= ssOffs[s][0]; }
            }
            const uint32_t before = W->nGenomeHits;
            if (W->nGenomeHits >= HT2_MAX_GHITS) { W->err |= HT2_ERR_GHITS; return false; }
            Ht2Hit& gh = W->genomeHits[W->nGenomeHits++];
            initHit(gh, coord.fw != 0, rdoff, len, 0, 0, coord.ref, off, joinedOff);
            if (!adjustTry(gh, rdi, true)) W->nGenomeHits = before;
            found = W->nGenomeHits > before;
        }
        return found;
    }
