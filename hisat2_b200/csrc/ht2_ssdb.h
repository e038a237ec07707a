// ht2_ssdb.h -- the populated splice-site DB of a run, read-only: the splice-site and exon ALTs of the index
// (SpliceSiteDB::read(gfm, alts), splice_site.cpp:653-720), then the sites of --known-splicesite-infile /
// --novel-splicesite-infile (SpliceSiteDB::read(ifstream&, known), splice_site.cpp:727-775).  One position-independent
// blob, built on the host once per handle and kept in HBM:
//
//   Ht2SsHeader | refOff[nRefs + 1] | fw[nSites] | bw[nSites] | exons[nExons]
//
// The reference keeps two red-black trees per reference sequence, keyed (left, right, dir) and (right, left, dir)
// (SpliceSitePos::operator<, splice_site.h:137-148), and answers range queries by in-order traversal
// (getSpliceSites_recur, splice_site.cpp:401-433): the result list is the keys in [lo, hi] in key order.  Here the
// two trees are two sorted arrays of the same sites and a query is a lower bound plus a scan.  The exon list is the
// reference's sorted _exons (Exon::operator<, splice_site.h:426-435).
// Temporary sites (sites added while reads are aligned, splice_site.cpp:190-350) are not represented: their effect
// depends on the order in which the reference's threads finish reads.
#ifndef HT2_SSDB_H_
#define HT2_SSDB_H_
#include <stdint.h>
#include "ht2_image.h"

#define HT2_SS_MAGIC 0x53533248u   /* "H2SS" */
enum { HT2_SPL_UNKNOWN = 1, HT2_SPL_FW, HT2_SPL_RC, HT2_SPL_SEMI_FW, HT2_SPL_SEMI_RC };   // splice_site.h SPL_* (the codes Ht2Edit keeps)

struct Ht2SsSite { uint32_t left, right; uint32_t dir; uint32_t known; };   // left = last base of the upstream exon, right = first base of the downstream exon (0-based)
struct Ht2SsHeader { uint32_t magic, nRefs, nSites, nExons; };
// An exon ALT of the index, widened by 10 bases at each end and clamped to its sequence (0-based, inclusive)
struct Ht2SsExon { uint32_t ref, left, right, pad; };
// One junction of one printed alignment, as SpliceSiteDB::addSpliceSite would record it (--novel-splicesite-outfile):
// appended by the SAM write pass, aggregated on the host (ht2_index.h Ht2NovelSites)
struct Ht2SsRec { uint32_t ref, left, right; uint32_t dirEd; };   // dirEd = direction | edit distance of the alignment << 8

struct Ht2SsView {
    const Ht2SsHeader* h;
    const uint32_t* refOff;
    const Ht2SsSite* fw;   // sorted by (left, right, dir)  -- _fwIndex
    const Ht2SsSite* bw;   // sorted by (right, left, dir)  -- _bwIndex
    const Ht2SsExon* ex;   // sorted by (ref, left, right)  -- _exons
    HT2_HD void init(const uint8_t* blob) {
        h = (const Ht2SsHeader*)blob;
        refOff = (const uint32_t*)(blob + sizeof(Ht2SsHeader));
        fw = (const Ht2SsSite*)(blob + sizeof(Ht2SsHeader) + (((size_t)h->nRefs + 1 + 3) & ~(size_t)3) * 4);
        bw = fw + h->nSites;
        ex = (const Ht2SsExon*)(bw + h->nSites);
    }
    // SpliceSiteDB::insideExon(ref, left, right) (splice_site.cpp:508-526): from the last exon that starts at or
    // before 'left', walk back while exons still reach 'left'; true when one covers [left, right].  As in the
    // reference, the walk does not stop at the reference sequence's first exon.
    HT2_HD bool insideExon(uint32_t ref, uint32_t left, uint32_t right) const {
        uint32_t l = 0, r = h->nExons;
        while (l < r) {   // lower bound of (ref, left + 1, 0)
            const uint32_t m = l + ((r - l) >> 1);
            const Ht2SsExon& e = ex[m];
            if (e.ref < ref || (e.ref == ref && e.left < left + 1)) l = m + 1; else r = m;
        }
        for (; l > 0; l--) {
            const Ht2SsExon& e = ex[l - 1];
            if (e.right < left) break;
            if (e.left <= left && right <= e.right) return true;
        }
        return false;
    }
    // SpliceSiteDB::getLeftSpliceSites(ref, left, range): sites whose RIGHT end lies in [left + 1 - range, left], in
    // (right, left, dir) order (splice_site.cpp:370-383) -> index range [lo, hi) of bw
    HT2_HD void leftSites(uint32_t ref, uint32_t left, uint32_t range, uint32_t& lo, uint32_t& hi) const {
        const uint32_t a = refOff[ref], b = refOff[ref + 1];
        const uint32_t kmin = left + 1 - range, kmax = left;
        uint32_t l = a, r = b;
        while (l < r) { const uint32_t m = l + ((r - l) >> 1); if (bw[m].right < kmin) l = m + 1; else r = m; }
        lo = l;
        while (l < b && bw[l].right <= kmax) l++;
        hi = l;
    }
    // SpliceSiteDB::getRightSpliceSites(ref, right, range): sites whose LEFT end lies in [right, right + range - 1], in
    // (left, right, dir) order (splice_site.cpp:385-399) -> index range [lo, hi) of fw
    HT2_HD void rightSites(uint32_t ref, uint32_t right, uint32_t range, uint32_t& lo, uint32_t& hi) const {
        const uint32_t a = refOff[ref], b = refOff[ref + 1];
        const uint32_t kmin = right, kmax = right + range - 1;
        uint32_t l = a, r = b;
        while (l < r) { const uint32_t m = l + ((r - l) >> 1); if (fw[m].left < kmin) l = m + 1; else r = m; }
        lo = l;
        while (l < b && fw[l].left <= kmax) l++;
        hi = l;
    }
};
#endif
