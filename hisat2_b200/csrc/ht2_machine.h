// ht2_machine.h -- the per-read alignment policy as an explicit state machine.
//
// Same behaviour as the recursive formulation in ht2_core_impl.h (which mirrors
// HI_Aligner::go / nextBWT / align, SplicedAligner::hybridSearch /
// hybridSearch_recur and alignMate line by line), but with every loop that
// contains a recursive call turned into resumable states and the recursion
// turned into an explicit frame stack in the workspace.  One call of step()
// executes ONE segment.  On the GPU each lane owns a read and all lanes of a
// warp sit in the same dispatcher loop, so lanes that are in the same state
// execute the same segment together (convergent instruction fetch) instead of
// each lane wandering through a deep call tree on its own.
//
// Included at the end of ht2_core.h (inside no namespace); defines members of
// Ht2Aligner declared there.
#ifndef HT2_MACHINE_H_
#define HT2_MACHINE_H_

enum {
    // top-level states (HI_Aligner::go, hi_aligner.h:4048-4149)
    TS_START = 0, TS_NEXTBWT, TS_PS, TS_ALIGN, TS_HYB_EXTEND, TS_HYB_PICK, TS_HYB_RET, TS_HYB_DP, TS_HYB_DP_RET, TS_POST_ALIGN,
    TS_AFTER_LOOP, TS_MATE_NEXT, TS_MATE_SEARCH, TS_MATE_ANCHOR, TS_MATE_RET, TS_MATE_DONE, TS_DONE
};
enum {
    // frame states (SplicedAligner::hybridSearch_recur, spliced_aligner.h:331-2052)
    F_ENTER = 0,
    F_L_START, F_L_WHILE, F_L_COORD, F_L_COORD_RET, F_L_WHILE_TAIL, F_L_STASH, F_L_STASH_RET, F_L_AFTER_WHILE,
    F_L_GCOORD, F_L_GCOORD_RET, F_L_TRIM, F_L_TRIM_RET, F_L_EXT,
    F_R_START, F_R_WHILE, F_R_COORD, F_R_COORD_RET, F_R_WHILE_TAIL, F_R_STASH, F_R_STASH_RET, F_R_AFTER_WHILE,
    F_R_GCOORD, F_R_GCOORD_RET, F_R_TRIM, F_R_TRIM_RET, F_R_EXT,
    F_FINAL_RET, F_RETURN,
    // the expensive half of the four *COORD states (extend + combineWith): its own states, so that a round gathers only
    // slots that really have a pair of hits to join (the cheap half -- build the hit, compatibleWith -- is glue)
    F_L_COMBINE, F_L_GCOMBINE, F_R_COMBINE, F_R_GCOMBINE,
    // the three uses of a populated splice-site DB (spliced_aligner.h:409-668, 685-811, 1365-1494)
    F_SS_FULL, F_L_SS, F_L_SS_RET, F_R_SS, F_R_SS_RET
};

// push a child frame (== a recursive call of hybridSearch_recur)
template <bool GRAPH, bool NOSPL, bool DP> HT2_NI void Ht2AlignerT<GRAPH, NOSPL, DP>::pushFrame(uint32_t rdi, const Ht2Hit* hit, uint32_t hitoff, uint32_t hitlen, bool alignMate, uint32_t dep)
{
    if (W->nFrames >= HT2_DEPTH_CAP) { W->err |= HT2_ERR_DEPTH; W->childRet = HT2_MIN_I64; return; }
    Ht2Frame& f = W->frames[W->nFrames++];
    f.pc = F_ENTER; f.rdi = (uint8_t)rdi; f.alignMate = alignMate ? 1 : 0; f.hit = hit; f.hitoff = hitoff; f.hitlen = hitlen; f.dep = dep;
}

// One segment of one hybridSearch_recur activation.
template <bool GRAPH, bool NOSPL, bool DP> HT2_NI void Ht2AlignerT<GRAPH, NOSPL, DP>::runFrame()
{
    Ht2Frame& f = W->frames[W->nFrames - 1];
    const uint32_t rdi = f.rdi;
    const Ht2Hit& hit = *f.hit;
    const uint32_t hitoff = f.hitoff, hitlen = f.hitlen;
    const bool alignMate = f.alignMate != 0;
    const uint32_t rdlen = W->rd[rdi].len;
    const uint32_t minK = P->minK, minKL = P->minKLocal;
    const int64_t mmpMax = P->mmpMax;
    const uint32_t max_count = 2;
    switch (f.pc) {
    case F_ENTER: {
        f.maxsc = HT2_MIN_I64;
        f.cushion = 0;
        if (noSpl())
            f.cushion = alignMate ? (int64_t)((double)rdlen * 0.03 * (double)ht2_mmpen(*P, 255)) : 0;
        f.poolMark = W->poolTop;
        if (hit.score + f.cushion < minsc[rdi]) { f.pc = F_RETURN; break; }
        if (f.dep >= HT2_MAX_DEPTH) { f.pc = F_RETURN; break; }
        HT2_HIWATER(maxDepth, f.dep);
        if (hitoff == hit.rdoff - hit.trim5 && hitlen == hit.len + hit.trim5 + hit.trim3) {
            if (isSearched(hit, rdi)) { f.pc = F_RETURN; break; }
            addSearched(hit, rdi);
        }
        if (W->err) { f.pc = F_RETURN; break; }
        f.nLocalHits = 0;
        const bool ss = !ssdbEmpty() && !noSpl();   // with --no-spliced-alignment the DB branches reduce to the plain ones
        f.ssi = HT2_IDX_MAX32; f.ssHi = 0;
        if (hitoff == 0 && hitlen == rdlen) {
            if (!redundant(rdi, hit)) {
                if (ss) { f.pc = F_SS_FULL; break; }
                reportHit(rdi, hit);
                if (hit.score > f.maxsc) f.maxsc = hit.score;
            }
            f.pc = F_RETURN;
        } else if (hitoff > 0 && (hitoff + hitlen == rdlen || hitoff + hitoff < rdlen - hitlen)) f.pc = ss ? F_L_SS : F_L_START;
        else f.pc = ss ? F_R_SS : F_R_START;
        break;
    }
#ifdef HT2_ENABLE_SPLICED
    // ------------------------------------------------ splice-site DB: a full-length hit (spliced_aligner.h:409-664) --
    // Known / novel sites next to the hit's first and last exon-like fragment are tried as alternative ends of the
    // alignment: a read that runs a few bases into the next exon aligns those bases as mismatches or soft clips
    // otherwise.  No recursion in here: one heavy segment.
    case F_SS_FULL: {
        Ht2SsView ssv; ssv.init(ssT);
        enum { MAXL = 24 };
        Ht2Hit* list[MAXL]; uint32_t n = 0;
        int64_t best_score = hit.score;
        list[n] = poolAlloc(); copyHit(*list[n], hit); list[n]->hitcount = hit.hitcount; n++;
        uint32_t fragoff = 0, fraglen = 0, left = 0, right = 0;
        getLeft(hit, fragoff, fraglen, left, NULL, rdi);
        const uint32_t minMatchLen = minK;
        if (fraglen >= minMatchLen && left >= minMatchLen && hit.trim5 == 0) {
            uint32_t lo, hi;
            ssv.leftSites(hit.tidx, left + minMatchLen, minMatchLen, lo, hi);
            for (uint32_t si = lo; si < hi && !W->err; si++) {
                const Ht2SsSite ss1 = ssv.bw[si];
                if (left + fraglen - 1 < ss1.right) continue;
                const uint32_t frag2off = ss1.left - (ss1.right - left);
                if (frag2off + 1 < hitoff) continue;
                if (fragoff + ss1.right < left + 1) continue;
                const uint32_t readoff = fragoff + ss1.right - left - 1;
                uint32_t joinedOff = 0;
                if (!textOffToJoined(hit.tidx, ss1.left, joinedOff)) continue;
                Ht2Hit* tp = poolAlloc();
                Ht2Hit& tempHit = *tp;
                initHit(tempHit, hit.fw != 0, readoff + 1, 0, 0, 0, hit.tidx, ss1.left + 1, joinedOff + 1);
                uint32_t leftext = readoff + 1, rightext = 0;
                extend(tempHit, rdi, leftext, rightext, 0);
                bool keep = false;
                if (tempHit.len > 0 && compatibleWith(tempHit, hit, rdi)) {
                    int64_t msc = minsc[rdi] > best_score ? minsc[rdi] : best_score;
                    const bool combined = combineWith(tempHit, hit, rdi, msc, &ss1);
                    if (W->bestUnp[rdi] > msc) msc = W->bestUnp[rdi];
                    uint32_t anchor = 0, ned = 0;
                    getLeftAnchor(tempHit, anchor, ned);
                    if (combined && tempHit.score >= msc && ned <= anchor / 4) {   // no short anchors with many mismatches
                        if (!isSearched(tempHit, rdi) && !redundant(rdi, tempHit)) {
                            if (tempHit.score > best_score) best_score = tempHit.score;
                            if (n < MAXL) { list[n++] = tp; keep = true; } else W->err |= HT2_ERR_POOL;
                        }
                    }
                }
                if (!keep) W->poolTop--;
            }
        }
        const uint32_t num = n;
        for (uint32_t i = 0; i < num && !W->err; i++) {
            const Ht2Hit& canHit = *list[i];
            getRight(canHit, fragoff, fraglen, right, NULL, rdi);
            if (canHit.score < best_score) continue;
            if (!(fraglen >= minMatchLen && canHit.trim3 == 0)) continue;
            uint32_t lo, hi;
            ssv.rightSites(canHit.tidx, right + fraglen - minMatchLen, minMatchLen, lo, hi);
            for (uint32_t si = lo; si < hi && !W->err; si++) {
                const Ht2SsSite ss1 = ssv.fw[si];
                if (right > ss1.left) continue;
                const uint32_t readoff = fragoff + ss1.left - right + 1;
                if (readoff >= rdlen) continue;
                uint32_t joinedOff = 0;
                if (!textOffToJoined(canHit.tidx, ss1.right, joinedOff)) continue;
                Ht2Hit* cp = poolAlloc();        // the combined hit, kept when it survives ...
                Ht2Hit* tp = poolAlloc();        // ... the fragment beyond the site, always released
                Ht2Hit& tempHit = *tp;
                initHit(tempHit, canHit.fw != 0, readoff, 0, 0, 0, canHit.tidx, ss1.right, joinedOff);
                uint32_t leftext = 0, rightext = rdlen - readoff;
                extend(tempHit, rdi, leftext, rightext, 0);
                bool keep = false;
                if (tempHit.len > 0 && compatibleWith(canHit, tempHit, rdi)) {
                    Ht2Hit& combinedHit = *cp;
                    copyHit(combinedHit, canHit); combinedHit.hitcount = canHit.hitcount;
                    int64_t msc = minsc[rdi] > best_score ? minsc[rdi] : best_score;
                    const bool combined = combineWith(combinedHit, tempHit, rdi, msc, &ss1);
                    if (W->bestUnp[rdi] > msc) msc = W->bestUnp[rdi];
                    uint32_t anchor = 0, ned = 0;
                    getRightAnchor(combinedHit, anchor, ned);
                    if (combined && combinedHit.score >= msc && ned <= anchor / 4) {
                        if (!isSearched(combinedHit, rdi) && !redundant(rdi, combinedHit)) {
                            if (combinedHit.score > best_score) best_score = tempHit.score;   // sic: the fragment's score (spliced_aligner.h:632)
                            if (n < MAXL) { list[n++] = cp; keep = true; } else W->err |= HT2_ERR_POOL;
                        }
                    }
                }
                W->poolTop--;                    // tempHit
                if (!keep) W->poolTop--;         // combinedHit
            }
        }
        for (uint32_t i = 0; i < n && !W->err; i++) {
            const Ht2Hit& canHit = *list[i];
            if (!P->secondary && canHit.score < best_score) continue;
            if (i > 0 && !isSearched(canHit, rdi)) addSearched(canHit, rdi);
            if (!redundant(rdi, canHit)) {
                reportHit(rdi, canHit);
                if (canHit.score > f.maxsc) f.maxsc = canHit.score;
            }
        }
        f.pc = F_RETURN;
        break;
    }
    // ------------------------- splice-site DB: a partial hit to be extended to the left (spliced_aligner.h:685-811) --
    case F_L_SS: {
        Ht2SsView ssv; ssv.init(ssT);
        uint32_t fragoff = 0, fraglen = 0, left = 0;
        getLeft(hit, fragoff, fraglen, left, NULL, rdi);
        const uint32_t minMatchLen = minKL;
        if (f.ssi == HT2_IDX_MAX32) {
            f.ssi = 0; f.ssHi = 0;
            if (fraglen >= minMatchLen && left >= minMatchLen)
                ssv.leftSites(hit.tidx, left + minMatchLen, minMatchLen + (minMatchLen < fragoff ? minMatchLen : fragoff), f.ssi, f.ssHi);
        }
        f.pc = F_L_START;
        while (f.ssi < f.ssHi && !W->err) {
            const Ht2SsSite ss1 = ssv.bw[f.ssi++];
            if (left + fraglen - 1 < ss1.right) continue;
            if (fragoff + ss1.right < left + 1) continue;
            const uint32_t readoff = fragoff + ss1.right - left - 1;
            uint32_t joinedOff = 0;
            if (!textOffToJoined(hit.tidx, ss1.left, joinedOff)) continue;
            Ht2Hit* tp = poolAlloc();
            Ht2Hit& tempHit = *tp;
            initHit(tempHit, hit.fw != 0, readoff + 1, 0, 0, 0, hit.tidx, ss1.left + 1, joinedOff + 1);
            uint32_t leftext = readoff + 1, rightext = 0;
            extend(tempHit, rdi, leftext, rightext, 0);
            if (tempHit.len > 0 && compatibleWith(tempHit, hit, rdi)) {
                const bool combined = combineWith(tempHit, hit, rdi, minsc[rdi], &ss1);
                const int64_t msc = sinkFloor(rdi, f.cushion);
                if (combined && tempHit.score >= msc &&
                    tempHit.score + (int64_t)((uint32_t)ht2_scpen(*P, 0) * hit.rdoff) >= hit.score) {   // soft-clipping might be better
                    f.pc = F_L_SS_RET;
                    pushFrame(rdi, tp, tempHit.rdoff, tempHit.len + tempHit.trim3, alignMate, f.dep + 1);
                    break;
                }
            }
            W->poolTop--;
        }
        break;
    }
    case F_L_SS_RET: {
        if (W->childRet > f.maxsc) f.maxsc = W->childRet;
        W->poolTop--;   // tempHit
        f.pc = F_L_SS;
        break;
    }
    // ----------------------- splice-site DB: a partial hit to be extended to the right (spliced_aligner.h:1365-1494) --
    case F_R_SS: {
        Ht2SsView ssv; ssv.init(ssT);
        uint32_t fragoff = 0, fraglen = 0, right = 0;
        getRight(hit, fragoff, fraglen, right, NULL, rdi);
        const uint32_t minMatchLen = minKL;
        if (f.ssi == HT2_IDX_MAX32) {
            f.ssi = 0; f.ssHi = 0;
            if (fraglen >= minMatchLen) {
                const uint32_t right_unmapped_len = rdlen - fragoff - fraglen;
                ssv.rightSites(hit.tidx, right + fraglen - minMatchLen, minMatchLen + (minMatchLen < right_unmapped_len ? minMatchLen : right_unmapped_len), f.ssi, f.ssHi);
            }
        }
        f.pc = F_R_START;
        while (f.ssi < f.ssHi && !W->err) {
            const Ht2SsSite ss1 = ssv.fw[f.ssi++];
            if (right > ss1.left) continue;
            const uint32_t readoff = fragoff + ss1.left - right + 1;
            if (readoff >= rdlen) continue;
            uint32_t joinedOff = 0;
            if (!textOffToJoined(hit.tidx, ss1.right, joinedOff)) continue;
            Ht2Hit* cp = poolAlloc();
            Ht2Hit* tp = poolAlloc();
            Ht2Hit& tempHit = *tp;
            initHit(tempHit, hit.fw != 0, readoff, 0, 0, 0, hit.tidx, ss1.right, joinedOff);
            uint32_t leftext = 0, rightext = rdlen - readoff;
            extend(tempHit, rdi, leftext, rightext, 0);
            bool go = false;
            if (tempHit.len > 0 && compatibleWith(hit, tempHit, rdi)) {
                Ht2Hit& combinedHit = *cp;
                copyHit(combinedHit, hit); combinedHit.hitcount = hit.hitcount;
                const bool combined = combineWith(combinedHit, tempHit, rdi, minsc[rdi], &ss1);
                const int64_t msc = sinkFloor(rdi, f.cushion);
                if (combined && combinedHit.score >= msc &&
                    combinedHit.score + (int64_t)((uint32_t)ht2_scpen(*P, 0) * (rdlen - hit.rdoff - hit.len - hit.trim5)) >= hit.score) go = true;
            }
            W->poolTop--;       // tempHit
            if (go) {
                f.pc = F_R_SS_RET;
                pushFrame(rdi, cp, cp->rdoff - cp->trim5, cp->len + cp->trim5, alignMate, f.dep + 1);
                break;
            }
            W->poolTop--;       // combinedHit
        }
        break;
    }
    case F_R_SS_RET: {
        if (W->childRet > f.maxsc) f.maxsc = W->childRet;
        W->poolTop--;   // combinedHit
        f.pc = F_R_SS;
        break;
    }
#endif
    // ------------------------------------------------------------ left --
    case F_L_START: {
        f.use_localindex = 1;
        if (hitoff == hit.rdoff && hitoff <= minK) {
            uint32_t leftext = HT2_IDX_MAX32, rightext = 0;
            Ht2Hit* t = poolAlloc();
            copyHit(*t, hit);
            extend(*t, rdi, leftext, rightext, 1);
            if (t->rdoff == 0) f.use_localindex = 0;
            W->poolTop--;
        }
        f.lid = localIndexId(hit.tidx, hit.toff);
        f.success = 0; f.first = 1; f.count = 0;
        f.prev_score = hit.score;
        f.pc = F_L_WHILE;
        break;
    }
    case F_L_WHILE: {
        if (!(!f.success && f.count++ < max_count && f.use_localindex)) { f.pc = F_L_AFTER_WHILE; break; }
        if (W->localindexatts >= W->maxLocalindexatts) { f.pc = F_L_AFTER_WHILE; break; }
        if (f.first) f.first = 0;
        else {
            f.lid = f.lid >= 0 ? prevLocal(f.lid) : -1;
            if (f.lid < 0 || localGeom(f.lid)->len == 0) { f.pc = F_L_AFTER_WHILE; break; }
        }
        if (f.lid < 0) { f.pc = F_L_AFTER_WHILE; break; }
        Ht2Fm<uint16_t> lfm; lfm.init(blob, localGeom(f.lid));
        uint32_t extlen = 0;
        uint32_t top = 0xffff, bot = 0xffff, node_top = 0xffff, node_bot = 0xffff;
        uint32_t extoff = hitoff - 1;
        if (extoff > 0) extoff -= 1;
        if (extoff < P->minAnchorLen) extoff = P->minAnchorLen;
        uint32_t nelt = HT2_IDX_MAX32;
        const uint32_t max_nelt = 5;
        bool no_extension = false;
        bool uniqueStop = false;
        for (; extoff < rdlen; extoff++) {
            extlen = 0;
            uniqueStop = true;
            W->localindexatts++;
            if (lfm.g->len == 0) { nelt = 0; top = bot = node_top = node_bot = 0; }
            else nelt = gfmSearch(lfm, rdi, hit.fw != 0, extoff, extlen, top, bot, node_top, node_bot,
                                  uniqueStop, minKL, 0xffffu, P->kseeds, true);
            if (extoff + 1 - extlen >= hitoff) { no_extension = true; break; }
            if (nelt <= max_nelt) break;
        }
        f.uniqueStop = uniqueStop ? 1 : 0; f.extoff = extoff; f.extlen = extlen;
        f.ncoords = 0; f.ri = -1;
        if (nelt > 0 && nelt <= max_nelt && extlen >= P->minAnchorLen && !no_extension) {
            uint32_t nc = 0;
            getGenomeCoordsLocal(lfm, top, bot, node_top, node_bot, hit.fw != 0, extoff + 1 - extlen, extlen, f.coords, nc, 8);
            sortCoords(f.coords, nc);
            f.ncoords = nc; f.ri = (int)nc - 1;
        }
        f.pc = F_L_COORD;
        break;
    }
    case F_L_COORD: {
        if (f.ri < 0) { f.pc = F_L_WHILE_TAIL; break; }
        const Ht2Coord& coord = f.coords[f.ri];
        Ht2Hit* tp = poolAlloc();
        Ht2Hit& tempHit = *tp;
        initHit(tempHit, coord.fw != 0, f.extoff + 1 - f.extlen, f.extlen, 0, 0, coord.ref, coord.off, coord.joinedOff);
        if (GRAPH && !adjustWithALT(tempHit, rdi)) { W->poolTop--; f.ri--; break; }   // spliced_aligner.h:946, 1139, 1635, 1826
        if (!compatibleWith(tempHit, hit, rdi)) {
            W->poolTop--;
            if (f.count == 1) { f.ri--; break; }
            f.pc = F_L_WHILE_TAIL; break;
        }
        f.tempHit = tp; f.pc = F_L_COMBINE;
        break;
    }
    case F_L_COMBINE: {
        Ht2Hit* tp = f.tempHit;
        Ht2Hit& tempHit = *tp;
        if (f.uniqueStop) {
            uint32_t leftext = HT2_IDX_MAX32, rightext = 0;
            extend(tempHit, rdi, leftext, rightext, 0);
        }
        bool combined = combineWith(tempHit, hit, rdi, minsc[rdi]);
        int64_t msc = sinkFloor(rdi, f.cushion);
        f.pc = F_L_COORD;
        if (combined && tempHit.score >= msc) {
            if (tempHit.score >= f.prev_score - mmpMax) {
                f.pc = F_L_COORD_RET;
                pushFrame(rdi, tp, tempHit.rdoff, tempHit.len + tempHit.trim3, alignMate, f.dep + 1);
                break;
            } else if (f.nLocalHits < 16) {
                f.localHits[f.nLocalHits++] = (uint16_t)(tp - W->pool);
                f.ri--;
                break; // keep tempHit on the pool
            } else W->err |= HT2_ERR_POOL;
        }
        W->poolTop--;
        f.ri--;
        break;
    }
    case F_L_COORD_RET: {
        if (W->childRet > f.maxsc) f.maxsc = W->childRet;
        W->poolTop--; // tempHit
        f.ri--;
        f.pc = F_L_COORD;
        break;
    }
    case F_L_WHILE_TAIL: {
        if (f.maxsc >= f.prev_score - mmpMax) f.success = 1;
        if (!f.success && (W->localindexatts >= W->maxLocalindexatts || f.count == max_count || prevLocal(f.lid) < 0)) {
            f.ti = 0; f.pc = F_L_STASH;
        } else f.pc = F_L_WHILE;
        break;
    }
    case F_L_STASH: {
        if (f.ti >= f.nLocalHits) { f.pc = F_L_WHILE; break; }
        Ht2Hit& tempHit = W->pool[f.localHits[f.ti]];
        int64_t msc = sinkFloor(rdi, f.cushion);
        if (tempHit.score >= msc) {
            f.pc = F_L_STASH_RET;
            pushFrame(rdi, &tempHit, tempHit.rdoff, tempHit.len + tempHit.trim3, alignMate, f.dep + 1);
        } else f.ti++;
        break;
    }
    case F_L_STASH_RET: {
        if (W->childRet > f.maxsc) f.maxsc = W->childRet;
        f.ti++; f.pc = F_L_STASH;
        break;
    }
    case F_L_AFTER_WHILE: {
        if (f.success) { f.pc = F_RETURN; break; }
        f.ncoords = 0; f.ri = -1;
        if (hitoff > minK && W->localindexatts < W->maxLocalindexatts) {
            uint32_t extlen = 0;
            uint32_t top = HT2_IDX_MAX32, bot = HT2_IDX_MAX32, node_top = HT2_IDX_MAX32, node_bot = HT2_IDX_MAX32;
            uint32_t extoff = hitoff - 1;
            bool uniqueStop = true;
            uint32_t nelt = gfmSearch(gfm, rdi, hit.fw != 0, extoff, extlen, top, bot, node_top, node_bot,
                                      uniqueStop, minK, HT2_IDX_MAX32, P->kseeds, false);
            f.uniqueStop = uniqueStop ? 1 : 0; f.extoff = extoff; f.extlen = extlen;
            if (nelt > 0 && nelt <= 5 && extlen >= minK) {
                W->nCoords = 0;
                bool straddled = false;
                getGenomeCoords(top, bot, node_top, node_bot, hit.fw != 0, bot - top, extlen, true, straddled);
                uint32_t nc = W->nCoords < 8 ? W->nCoords : 8;
                for (uint32_t i = 0; i < nc; i++) f.coords[i] = W->coords[i];
                if (nc > 1) sortCoords(f.coords, nc);
                f.ncoords = nc; f.ri = (int)nc - 1;
            }
        }
        f.pc = F_L_GCOORD;
        break;
    }
    case F_L_GCOORD: {
        if (f.ri < 0) { f.pc = F_L_TRIM; break; }
        const Ht2Coord& coord = f.coords[f.ri];
        Ht2Hit* tp = poolAlloc();
        Ht2Hit& tempHit = *tp;
        initHit(tempHit, coord.fw != 0, f.extoff + 1 - f.extlen, f.extlen, 0, 0, coord.ref, coord.off, coord.joinedOff);
        if (GRAPH && !adjustWithALT(tempHit, rdi)) { W->poolTop--; f.ri--; break; }   // spliced_aligner.h:946, 1139, 1635, 1826
        if (!compatibleWith(tempHit, hit, rdi)) { W->poolTop--; f.ri--; break; }
        f.tempHit = tp; f.pc = F_L_GCOMBINE;
        break;
    }
    case F_L_GCOMBINE: {
        Ht2Hit* tp = f.tempHit;
        Ht2Hit& tempHit = *tp;
        if (f.uniqueStop) {
            uint32_t leftext = HT2_IDX_MAX32, rightext = 0;
            extend(tempHit, rdi, leftext, rightext, 0);
        }
        bool combined = combineWith(tempHit, hit, rdi, minsc[rdi]);
        int64_t msc = sinkFloor(rdi, f.cushion);
        f.pc = F_L_GCOORD;
        if (combined && tempHit.score >= msc) {
            f.pc = F_L_GCOORD_RET;
            pushFrame(rdi, tp, tempHit.rdoff, tempHit.len + tempHit.trim3, alignMate, f.dep + 1);
            break;
        }
        W->poolTop--; f.ri--;
        break;
    }
    case F_L_GCOORD_RET: {
        if (W->childRet > f.maxsc) f.maxsc = W->childRet;
        W->poolTop--; f.ri--;
        f.pc = F_L_GCOORD;
        break;
    }
    case F_L_TRIM: {
        Ht2Hit* tp = poolAlloc();
        f.tempHit = tp;
        copyHit(*tp, hit);
        int64_t floor_ = f.maxsc > minsc[rdi] ? f.maxsc : minsc[rdi];
        uint32_t trimMax = (uint32_t)((tp->score - floor_) / ht2_scpen(*P, 0));
        if (tp->rdoff < trimMax) {
            Ht2Hit* trp = poolAlloc();
            copyHit(*trp, *tp);
            trp->trim5 = tp->rdoff; // GenomeHit::trim5 (hi_aligner.h:831-854)
            calculateScore(*trp, rdi);
            int64_t tmp_score = trp->score;
            if (tmp_score > f.maxsc && tmp_score >= minsc[rdi]) {
                f.pc = F_L_TRIM_RET;
                pushFrame(rdi, trp, 0, trp->len + trp->trim5 + trp->trim3, alignMate, f.dep + 1);
                break;
            }
            W->poolTop--;
        }
        f.pc = F_L_EXT;
        break;
    }
    case F_L_TRIM_RET: {
        if (W->childRet > f.maxsc) f.maxsc = W->childRet;
        W->poolTop--; // trimedHit
        f.pc = F_L_EXT;
        break;
    }
    case F_L_EXT: {
        Ht2Hit& tempHit = *f.tempHit;
        int64_t msc = minsc[rdi];
        uint32_t mm = (uint32_t)((tempHit.score - msc) / mmpMax);
        uint32_t leftext = HT2_IDX_MAX32, rightext = 0;
        uint32_t num_mismatch_allowed = 1;
        if (hitoff <= minKL) num_mismatch_allowed = tempHit.rdoff < mm ? tempHit.rdoff : mm;
        extend(tempHit, rdi, leftext, rightext, num_mismatch_allowed);
        msc = sinkFloor(rdi, f.cushion);
        uint32_t need = minKL < hit.rdoff ? minKL : hit.rdoff;
        f.pc = F_RETURN;
        if (tempHit.score >= msc && leftext >= need) {
            f.pc = F_FINAL_RET;
            pushFrame(rdi, &tempHit, tempHit.rdoff, tempHit.len + tempHit.trim3, alignMate, f.dep + 1);
        } else if (hitoff > minKL) {
            uint32_t jumplen = hitoff > minK ? minK : minKL;
            int64_t expected_score = hit.score - (int64_t)((hit.rdoff - hitoff) / jumplen) * mmpMax - mmpMax;
            if (expected_score >= msc) {
                f.pc = F_FINAL_RET;
                pushFrame(rdi, f.hit, hitoff - jumplen, hitlen + jumplen, alignMate, f.dep + 1);
            }
        }
        break;
    }
    // ----------------------------------------------------------- right --
    case F_R_START: {
        f.use_localindex = 1;
        if (hit.len == hitlen && hitoff + hitlen + minK > rdlen) {
            uint32_t leftext = 0, rightext = HT2_IDX_MAX32;
            Ht2Hit* t = poolAlloc();
            copyHit(*t, hit);
            extend(*t, rdi, leftext, rightext, 1);
            if (t->rdoff + t->len == rdlen) f.use_localindex = 0;
            W->poolTop--;
        }
        f.lid = localIndexId(hit.tidx, hit.toff);
        f.success = 0; f.first = 1; f.count = 0;
        f.prev_score = hit.score;
        f.pc = F_R_WHILE;
        break;
    }
    case F_R_WHILE: {
        if (!(!f.success && f.count++ < max_count && f.use_localindex)) { f.pc = F_R_AFTER_WHILE; break; }
        if (W->localindexatts >= W->maxLocalindexatts) { f.pc = F_R_AFTER_WHILE; break; }
        if (f.first) f.first = 0;
        else {
            f.lid = f.lid >= 0 ? nextLocal(f.lid) : -1;
            if (f.lid < 0 || localGeom(f.lid)->len == 0) { f.pc = F_R_AFTER_WHILE; break; }
        }
        if (f.lid < 0) { f.pc = F_R_AFTER_WHILE; break; }
        Ht2Fm<uint16_t> lfm; lfm.init(blob, localGeom(f.lid));
        uint32_t extlen = 0;
        uint32_t top = 0xffff, bot = 0xffff, node_top = 0xffff, node_bot = 0xffff;
        uint32_t extoff = hitoff + hitlen + minKL;
        if (extoff + 1 < rdlen) extoff += 1;
        if (extoff >= rdlen) extoff = rdlen - 1;
        uint32_t nelt = HT2_IDX_MAX32;
        const uint32_t max_nelt = 5;
        bool no_extension = false;
        bool uniqueStop = false;
        uint32_t maxHitLen = extoff - hitoff - hitlen;
        if (maxHitLen < minKL) maxHitLen = minKL;
        for (; maxHitLen < extoff + 1 && extoff < rdlen;) {
            extlen = 0;
            uniqueStop = false;
            W->localindexatts++;
            if (lfm.g->len == 0) { nelt = 0; top = bot = node_top = node_bot = 0; }
            else nelt = gfmSearch(lfm, rdi, hit.fw != 0, extoff, extlen, top, bot, node_top, node_bot,
                                  uniqueStop, minKL, maxHitLen & 0xffffu, P->kseeds, true);
            if (extoff < hitoff + hitlen) { no_extension = true; break; }
            if (nelt <= max_nelt) break;
            if (extoff + 1 < rdlen) extoff++;
            else {
                if (extlen < maxHitLen) break;
                else maxHitLen++;
            }
        }
        f.extoff = extoff; f.extlen = extlen;
        f.ncoords = 0; f.ri = 0;
        if (nelt > 0 && nelt <= max_nelt && extlen >= P->minAnchorLen && !no_extension) {
            uint32_t nc = 0;
            getGenomeCoordsLocal(lfm, top, bot, node_top, node_bot, hit.fw != 0, extoff + 1 - extlen, extlen, f.coords, nc, 8);
            if (nc > 1) sortCoords(f.coords, nc);
            f.ncoords = nc;
        }
        f.pc = F_R_COORD;
        break;
    }
    case F_R_COORD: {
        if (f.ri >= (int)f.ncoords) { f.pc = F_R_WHILE_TAIL; break; }
        const Ht2Coord& coord = f.coords[f.ri];
        Ht2Hit* tp = poolAlloc();
        Ht2Hit& tempHit = *tp;
        initHit(tempHit, coord.fw != 0, f.extoff + 1 - f.extlen, f.extlen, 0, 0, coord.ref, coord.off, coord.joinedOff);
        if (GRAPH && !adjustWithALT(tempHit, rdi)) { W->poolTop--; f.ri++; break; }   // spliced_aligner.h:946, 1139, 1635, 1826
        if (!compatibleWith(hit, tempHit, rdi)) {
            W->poolTop--;
            if (f.count == 1) { f.ri++; break; }
            f.pc = F_R_WHILE_TAIL; break;
        }
        f.tempHit = tp; f.pc = F_R_COMBINE;
        break;
    }
    case F_R_COMBINE: {
        Ht2Hit* tp = f.tempHit;
        Ht2Hit& tempHit = *tp;
        uint32_t leftext = 0, rightext = HT2_IDX_MAX32;
        extend(tempHit, rdi, leftext, rightext, 0);
        Ht2Hit* cp = poolAlloc();
        Ht2Hit& combinedHit = *cp;
        copyHit(combinedHit, hit);
        bool combined = combineWith(combinedHit, tempHit, rdi, minsc[rdi]);
        int64_t msc = sinkFloor(rdi, f.cushion);
        // keep the combined hit in tempHit's slot so the pool stays a stack
        copyHit(tempHit, combinedHit);
        W->poolTop--; // combinedHit slot
        f.pc = F_R_COORD;
        if (combined && tempHit.score >= msc) {
            if (tempHit.score >= f.prev_score - mmpMax) {
                f.pc = F_R_COORD_RET;
                pushFrame(rdi, tp, tempHit.rdoff - tempHit.trim5, tempHit.len + tempHit.trim5, alignMate, f.dep + 1);
                break;
            } else if (f.nLocalHits < 16) {
                f.localHits[f.nLocalHits++] = (uint16_t)(tp - W->pool);
                f.ri++;
                break;
            } else W->err |= HT2_ERR_POOL;
        }
        W->poolTop--;
        f.ri++;
        break;
    }
    case F_R_COORD_RET: {
        if (W->childRet > f.maxsc) f.maxsc = W->childRet;
        W->poolTop--;
        f.ri++;
        f.pc = F_R_COORD;
        break;
    }
    case F_R_WHILE_TAIL: {
        if (f.maxsc >= f.prev_score - mmpMax) f.success = 1;
        if (!f.success && (W->localindexatts >= W->maxLocalindexatts || f.count == max_count || nextLocal(f.lid) < 0)) {
            f.ti = 0; f.pc = F_R_STASH;
        } else f.pc = F_R_WHILE;
        break;
    }
    case F_R_STASH: {
        if (f.ti >= f.nLocalHits) { f.pc = F_R_WHILE; break; }
        Ht2Hit& tempHit = W->pool[f.localHits[f.ti]];
        int64_t msc = sinkFloor(rdi, f.cushion);
        if (tempHit.score >= msc) {
            f.pc = F_R_STASH_RET;
            pushFrame(rdi, &tempHit, tempHit.rdoff - tempHit.trim5, tempHit.len + tempHit.trim5, alignMate, f.dep + 1);
        } else f.ti++;
        break;
    }
    case F_R_STASH_RET: {
        if (W->childRet > f.maxsc) f.maxsc = W->childRet;
        f.ti++; f.pc = F_R_STASH;
        break;
    }
    case F_R_AFTER_WHILE: {
        if (f.success) { f.pc = F_RETURN; break; }
        f.ncoords = 0; f.ri = 0;
        if (hitoff + hitlen + minK + 1 < rdlen && W->localindexatts < W->maxLocalindexatts) {
            uint32_t extlen = 0;
            uint32_t top = HT2_IDX_MAX32, bot = HT2_IDX_MAX32, node_top = HT2_IDX_MAX32, node_bot = HT2_IDX_MAX32;
            uint32_t extoff = hitoff + hitlen + minK + 1;
            bool uniqueStop = true;
            uint32_t nelt = gfmSearch(gfm, rdi, hit.fw != 0, extoff, extlen, top, bot, node_top, node_bot,
                                      uniqueStop, minK, HT2_IDX_MAX32, P->kseeds, false);
            f.extoff = extoff; f.extlen = extlen;
            if (nelt > 0 && nelt <= 5 && extlen >= minK) {
                W->nCoords = 0;
                bool straddled = false;
                getGenomeCoords(top, bot, node_top, node_bot, hit.fw != 0, bot - top, extlen, true, straddled);
                uint32_t nc = W->nCoords < 8 ? W->nCoords : 8;
                for (uint32_t i = 0; i < nc; i++) f.coords[i] = W->coords[i];
                sortCoords(f.coords, nc);
                f.ncoords = nc;
            }
        }
        f.pc = F_R_GCOORD;
        break;
    }
    case F_R_GCOORD: {
        if (f.ri >= (int)f.ncoords) { f.pc = F_R_TRIM; break; }
        const Ht2Coord& coord = f.coords[f.ri];
        Ht2Hit* tp = poolAlloc();
        Ht2Hit& tempHit = *tp;
        initHit(tempHit, coord.fw != 0, f.extoff + 1 - f.extlen, f.extlen, 0, 0, coord.ref, coord.off, coord.joinedOff);
        if (GRAPH && !adjustWithALT(tempHit, rdi)) { W->poolTop--; f.ri++; break; }   // spliced_aligner.h:946, 1139, 1635, 1826
        if (!compatibleWith(hit, tempHit, rdi)) { W->poolTop--; f.ri++; break; }
        f.tempHit = tp; f.pc = F_R_GCOMBINE;
        break;
    }
    case F_R_GCOMBINE: {
        Ht2Hit* tp = f.tempHit;
        Ht2Hit& tempHit = *tp;
        uint32_t leftext = 0, rightext = HT2_IDX_MAX32;
        extend(tempHit, rdi, leftext, rightext, 0);
        Ht2Hit* cp = poolAlloc();
        Ht2Hit& combinedHit = *cp;
        copyHit(combinedHit, hit);
        bool combined = combineWith(combinedHit, tempHit, rdi, minsc[rdi]);
        int64_t msc = sinkFloor(rdi, f.cushion);
        copyHit(tempHit, combinedHit);
        W->poolTop--;
        f.pc = F_R_GCOORD;
        if (combined && tempHit.score >= msc) {
            f.pc = F_R_GCOORD_RET;
            pushFrame(rdi, tp, tempHit.rdoff - tempHit.trim5, tempHit.len + tempHit.trim5, alignMate, f.dep + 1);
            break;
        }
        W->poolTop--; f.ri++;
        break;
    }
    case F_R_GCOORD_RET: {
        if (W->childRet > f.maxsc) f.maxsc = W->childRet;
        W->poolTop--; f.ri++;
        f.pc = F_R_GCOORD;
        break;
    }
    case F_R_TRIM: {
        Ht2Hit* tp = poolAlloc();
        f.tempHit = tp;
        copyHit(*tp, hit);
        uint32_t trimLen = rdlen - hitoff - tp->len - tp->trim5;
        int64_t floor_ = f.maxsc > minsc[rdi] ? f.maxsc : minsc[rdi];
        uint32_t trimMax = (uint32_t)((tp->score - floor_) / ht2_scpen(*P, 0));
        if (trimLen < trimMax) {
            Ht2Hit* trp = poolAlloc();
            copyHit(*trp, *tp);
            trp->trim3 = trimLen; // GenomeHit::trim3 (hi_aligner.h:855-876)
            calculateScore(*trp, rdi);
            int64_t tmp_score = trp->score;
            if (tmp_score > f.maxsc && tmp_score >= minsc[rdi]) {
                f.pc = F_R_TRIM_RET;
                pushFrame(rdi, trp, trp->rdoff - trp->trim5, trp->len + trp->trim5 + trp->trim3, alignMate, f.dep + 1);
                break;
            }
            W->poolTop--;
        }
        f.pc = F_R_EXT;
        break;
    }
    case F_R_TRIM_RET: {
        if (W->childRet > f.maxsc) f.maxsc = W->childRet;
        W->poolTop--;
        f.pc = F_R_EXT;
        break;
    }
    case F_R_EXT: {
        Ht2Hit& tempHit = *f.tempHit;
        int64_t msc = minsc[rdi];
        uint32_t leftext = 0, rightext = HT2_IDX_MAX32;
        uint32_t mm = (uint32_t)((tempHit.score - msc) / mmpMax);
        uint32_t num_mismatch_allowed = 1;
        if (rdlen - hitoff - hitlen <= minKL) {
            uint32_t r = rdlen - tempHit.rdoff - tempHit.len;
            num_mismatch_allowed = r < mm ? r : mm;
        }
        extend(tempHit, rdi, leftext, rightext, num_mismatch_allowed);
        msc = sinkFloor(rdi, f.cushion);
        uint32_t need = rdlen - hit.len - hit.rdoff;
        if (minKL < need) need = minKL;
        f.pc = F_RETURN;
        if (tempHit.score >= msc && rightext >= need) {
            f.pc = F_FINAL_RET;
            pushFrame(rdi, &tempHit, tempHit.rdoff - tempHit.trim5, tempHit.len + tempHit.trim5, alignMate, f.dep + 1);
        } else if (hitoff + hitlen + minKL < rdlen) {
            uint32_t jumplen = hitoff + hitlen + minK < rdlen ? minK : minKL;
            int64_t expected_score = hit.score - (int64_t)((hitlen - hit.len) / jumplen) * mmpMax - mmpMax;
            if (expected_score >= msc) {
                f.pc = F_FINAL_RET;
                pushFrame(rdi, f.hit, hitoff, hitlen + jumplen, alignMate, f.dep + 1);
            }
        }
        break;
    }
    case F_FINAL_RET: {
        if (W->childRet > f.maxsc) f.maxsc = W->childRet;
        f.pc = F_RETURN;
        break;
    }
    default: // F_RETURN
        W->poolTop = f.poolMark;
        W->childRet = f.maxsc;
        W->nFrames--;
        break;
    }
}

// One segment of the top-level control (go / nextBWT / align / hybridSearch / alignMate).
template <bool GRAPH, bool NOSPL, bool DP> HT2_NI void Ht2AlignerT<GRAPH, NOSPL, DP>::runTop()
{
    switch (W->st) {
    case TS_START: {
        for (uint32_t rdi = 0; rdi < 2; rdi++) {
            for (uint32_t fwi = 0; fwi < 2; fwi++) {
                Ht2ReadHits& h = W->hits[rdi][fwi];
                h.len = W->rd[rdi].len; h.cur = 0; h.done = 0; h.numPartialSearch = 0; h.numUniqueSearch = 0; h.nhits = 0; h.nie = 0;
            }
            W->nSearched[rdi] = 0;
        }
        W->searchedTop = 0;
        W->nGenomeHits = 0; W->poolTop = 0; W->nFrames = 0;
        W->concordInspected[0] = W->concordInspected[1] = 0;
        W->found[0][0] = W->found[0][1] = 1; W->found[1][0] = W->found[1][1] = paired ? 1 : 0;
        W->st = TS_NEXTBWT;
        break;
    }
    case TS_NEXTBWT: { // HI_Aligner::nextBWT up to the point where a partial search is needed
        uint32_t rdi; bool fw;
        if (!pickNextReadToSearch(rdi, fw)) { W->st = TS_AFTER_LOOP; break; }
        uint32_t fwi = fw ? 0 : 1;
        Ht2ReadHits& hit = W->hits[rdi][fwi];
        bool anchorStop = P->anchorStop != 0;
        if (!P->secondary) {
            uint32_t numSearched = hit.numPartialSearch - hit.numUniqueSearch;
            int64_t bestScore = W->bestUnp[rdi];
            if (bestScore >= minsc[rdi]) {
                uint32_t maxmm = (uint32_t)((-bestScore + P->mmpMax - 1) / P->mmpMax);
                if (numSearched > maxmm + bestSpliced(rdi) + 1) {
                    hit.done = 1;
                    if (paired) {
                        if (W->bestUnp[1 - rdi] >= minsc[1 - rdi] && W->nPairs > 0) W->st = TS_AFTER_LOOP;
                        // else: continue the while loop == stay in TS_NEXTBWT
                    } else W->st = TS_AFTER_LOOP;
                    break;
                }
            }
            Ht2ReadHits& rchit = W->hits[rdi][1 - fwi];
            if (rchit.done && bestScore < minsc[rdi]) {
                if (numSearched > (rchit.numPartialSearch - rchit.numUniqueSearch) + (anchorStop ? 1u : 0u)) {
                    hit.done = 1;
                    W->st = TS_AFTER_LOOP;
                    break;
                }
            }
        }
        W->curRdi = (uint8_t)rdi; W->curFw = fw ? 1 : 0;
        W->st = TS_PS;
        break;
    }
    case TS_PS: {
        const uint32_t rdi = W->curRdi; const bool fw = W->curFw != 0;
        Ht2ReadHits& hit = W->hits[rdi][fw ? 0 : 1];
        bool pseudogeneStop = gfm.g->linearFM && !noSpl();
        bool anchorStop = P->anchorStop != 0;
        if (!partialSearch(rdi, fw, pseudogeneStop, anchorStop)) break;   // parked after a slice of LF steps: stay in TS_PS
        if (hit.done) { W->st = TS_ALIGN; break; }
        if (!pseudogeneStop) { if (hit.cur + 1 < hit.len) hit.cur++; }
        if (anchorStop) { hit.done = 1; W->st = TS_ALIGN; break; }
        W->st = TS_NEXTBWT;
        break;
    }
    case TS_ALIGN: { // HI_Aligner::align up to hybridSearch
        const uint32_t rdi = W->curRdi; const bool fw = W->curFw != 0;
        Ht2ReadHits& hit = W->hits[rdi][fw ? 0 : 1];
        bool any = false;
        for (uint32_t i = 0; i < hit.nhits; i++) if (hit.hits[i].bot > hit.hits[i].top) { any = true; break; }
        if (!any) { W->alignRet = 0; W->st = TS_POST_ALIGN; break; }
        int64_t bestScore = W->bestUnp[rdi];
        if (bestScore < minsc[rdi]) bestScore = minsc[rdi];
        uint32_t maxmm = (uint32_t)((-bestScore + P->mmpMax - 1) / P->mmpMax);
        uint32_t numActualPartialSearch = hit.numPartialSearch - hit.numUniqueSearch;
        if (!P->secondary && numActualPartialSearch > maxmm + bestSpliced(rdi) + 1) { W->alignRet = 1; W->st = TS_POST_ALIGN; break; }
        const uint32_t maxsize = P->khits > P->kseeds ? P->khits : P->kseeds;
        W->nGenomeHits = 0;
        uint32_t numHits = getAnchorHits(rdi, fw, maxsize);
        if (numHits <= 0) { W->alignRet = 0; W->st = TS_POST_ALIGN; break; }
        uint64_t add = (uint64_t)(-minsc[rdi] / P->mmpMax) * numHits * (P->secondary ? 2 : 1);
        W->maxLocalindexatts = W->localindexatts + (uint32_t)(add > 10 ? add : 10);
        W->alignRet = 1;
        W->st = TS_HYB_EXTEND;
        break;
    }
    case TS_HYB_EXTEND: { // SplicedAligner::hybridSearch, first loop
        const uint32_t rdi = W->curRdi;
        for (uint32_t hi = 0; hi < W->nGenomeHits; hi++) {
            uint32_t leftext = HT2_IDX_MAX32, rightext = HT2_IDX_MAX32;
            extend(W->genomeHits[hi], rdi, leftext, rightext, 0);
        }
#if !defined(__CUDA_ARCH__) && defined(HT2_TRACE)
        for (uint32_t gi = 0; gi < W->nGenomeHits; gi++) { Ht2Hit& g = W->genomeHits[gi]; fprintf(stderr, "ext %u rdoff %u len %u toff %u joined %u hitcount %u ned %u score %lld\n", gi, g.rdoff, g.len, g.toff, g.joinedOff, g.hitcount, g.nedits, (long long)g.score); }
#endif
        for (uint32_t i = 0; i < W->nGenomeHits; i++) W->genomeHitsDone[i] = 0;
        W->hybIter = 0;
        W->st = TS_HYB_PICK;
        break;
    }
    case TS_HYB_PICK: {
        const uint32_t rdi = W->curRdi;
        if (W->hybIter >= W->nGenomeHits) { W->st = TS_POST_ALIGN; break; }
        uint32_t hj = 0;
        for (; hj < W->nGenomeHits; hj++) if (!W->genomeHitsDone[hj]) break;
        if (hj >= W->nGenomeHits) { W->st = TS_POST_ALIGN; break; }
        for (uint32_t hk = hj + 1; hk < W->nGenomeHits; hk++) {
            if (W->genomeHitsDone[hk]) continue;
            Ht2Hit& gj = W->genomeHits[hj]; Ht2Hit& gk = W->genomeHits[hk];
            if (gk.hitcount > gj.hitcount || (gk.hitcount == gj.hitcount && gk.len > gj.len)) hj = hk;
        }
        W->hybHj = hj;
        Ht2Hit& gh = W->genomeHits[hj];
        W->st = TS_HYB_RET;
        pushFrame(rdi, &gh, gh.rdoff, gh.len, false, 0);
        break;
    }
    case TS_HYB_RET: {
        // --bowtie2-dp: dynamic programming around the anchor, then one more recursion on the
        // full-length hit (spliced_aligner.h:209-320)
        if (DP && (P->bowtie2Dp == 2 || (P->bowtie2Dp == 1 && W->childRet < minsc[W->curRdi]))) {
            Ht2Hit& gh = W->genomeHits[W->hybHj];
            if (!W->err) {
                if (gh.len < W->rd[W->curRdi].len) { W->st = TS_HYB_DP; break; }   // a DP problem: its own heavy state, so that
                                                                                   // the lanes of a round all run the fill
                W->st = TS_HYB_DP_RET;                                             // already full length (swExtendAnchor's first line)
                pushFrame(W->curRdi, &gh, gh.rdoff, gh.len, false, 0);
                break;
            }
        }
        W->genomeHitsDone[W->hybHj] = 1;
        W->hybIter++;
        W->st = TS_HYB_PICK;
        break;
    }
    case TS_HYB_DP: {
        Ht2Hit& gh = W->genomeHits[W->hybHj];
        if (DP && swExtendAnchor(W->curRdi, gh)) {
            W->st = TS_HYB_DP_RET;
            pushFrame(W->curRdi, &gh, gh.rdoff, gh.len, false, 0);
            break;
        }
        W->genomeHitsDone[W->hybHj] = 1;
        W->hybIter++;
        W->st = TS_HYB_PICK;
        break;
    }
    case TS_HYB_DP_RET: {
        W->genomeHitsDone[W->hybHj] = 1;
        W->hybIter++;
        W->st = TS_HYB_PICK;
        break;
    }
    case TS_POST_ALIGN: { // back in go()'s while body
        W->found[W->curRdi][W->curFw ? 0 : 1] = W->alignRet;
        if (!W->found[0][0] && !W->found[0][1] && !W->found[1][0] && !W->found[1][1]) { W->st = TS_AFTER_LOOP; break; }
        if (paired) pairReads();
        W->st = W->err ? TS_DONE : TS_NEXTBWT;
        break;
    }
    case TS_AFTER_LOOP: {
        W->st = TS_DONE;
        if (paired && !W->err) {
            if (W->nPairs == 0 && (W->bestUnp[0] >= minsc[0] || W->bestUnp[1] >= minsc[1])) {
                W->mateSize[0] = W->nRes[0]; W->mateSize[1] = W->nRes[1];
                W->mateI = 0; W->mateJ = 0;
                W->st = TS_MATE_NEXT;
            }
        }
        break;
    }
    case TS_MATE_NEXT: { // for i in 0..1, j < rs_size[i]: alignMate(i, ...)
        while (W->mateI < 2 && W->mateJ >= W->mateSize[W->mateI]) { W->mateI++; W->mateJ = 0; }
        if (W->mateI >= 2) { W->st = TS_MATE_DONE; break; }
        W->st = TS_MATE_SEARCH;
        break;
    }
    case TS_MATE_SEARCH: { // HI_Aligner::alignMate, anchor search part (hi_aligner.h:5600-5717)
        const Ht2Res& res = W->res[W->mateI][W->mateJ];
        alignMateAnchors(W->mateI, res.fw != 0, res.tidx, res.toff);
        W->hybIter = 0;
        W->st = TS_MATE_ANCHOR;
        break;
    }
    case TS_MATE_ANCHOR: {
        const uint32_t ordi = 1 - W->mateI;
        if (W->hybIter >= W->nGenomeHits) { W->mateJ++; W->st = TS_MATE_NEXT; break; }
        Ht2Hit& gh = W->genomeHits[W->hybIter];
        uint32_t leftext = HT2_IDX_MAX32, rightext = HT2_IDX_MAX32;
        extend(gh, ordi, leftext, rightext, 0);
        W->st = TS_MATE_RET;
        pushFrame(ordi, &gh, gh.rdoff, gh.len, true, 0);
        break;
    }
    case TS_MATE_RET: {
        W->hybIter++;
        W->st = TS_MATE_ANCHOR;
        break;
    }
    case TS_MATE_DONE: {
        pairReads(); // mate_found is always true once alignMate ran (hi_aligner.h:5766)
        W->st = TS_DONE;
        break;
    }
    default:
        W->st = TS_DONE;
        break;
    }
}

// Run one read (pair) to completion (host build and the one-lane-per-read kernel loop).
template <bool GRAPH, bool NOSPL, bool DP> HT2_HD void Ht2AlignerT<GRAPH, NOSPL, DP>::machineStart() { W->st = TS_START; W->nFrames = 0; W->psCont = 0; W->psG.active = 0; }
template <bool GRAPH, bool NOSPL, bool DP> HT2_HD bool Ht2AlignerT<GRAPH, NOSPL, DP>::machineDone() const { return W->st == TS_DONE && W->nFrames == 0; }
template <bool GRAPH, bool NOSPL, bool DP> HT2_HD void Ht2AlignerT<GRAPH, NOSPL, DP>::machineStep()
{
    if (W->nFrames > 0) runFrame();
    else runTop();
}
// "Heavy" states are the ones worth regrouping lanes for (index searches,
// reference extension, combine); everything else is short glue that is chained
// onto the end of the previous segment.
template <bool GRAPH, bool NOSPL, bool DP> HT2_HD bool Ht2AlignerT<GRAPH, NOSPL, DP>::machineAtHeavyState() const
{
    if (W->nFrames > 0) {
        switch (W->frames[W->nFrames - 1].pc) {
            case F_ENTER: case F_L_START: case F_L_WHILE: case F_L_COMBINE: case F_L_AFTER_WHILE: case F_L_GCOMBINE: case F_L_TRIM: case F_L_EXT:
            case F_R_START: case F_R_WHILE: case F_R_COMBINE: case F_R_AFTER_WHILE: case F_R_GCOMBINE: case F_R_TRIM: case F_R_EXT:
            case F_SS_FULL: case F_L_SS: case F_R_SS:
                return true;
            default: return false;
        }
    }
    switch (W->st) {
        case TS_PS: case TS_ALIGN: case TS_HYB_EXTEND: case TS_MATE_SEARCH: case TS_MATE_ANCHOR: case TS_DONE: return true;
        case TS_HYB_DP: return true;                 // the dynamic-programming extension runs here
        default: return false;
    }
}
// run one heavy segment plus the glue that follows it
template <bool GRAPH, bool NOSPL, bool DP> HT2_HD void Ht2AlignerT<GRAPH, NOSPL, DP>::machineRun()
{
    do { machineStep(); } while (!machineAtHeavyState());
}

#endif // HT2_MACHINE_H_
