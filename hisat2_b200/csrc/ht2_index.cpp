// ht2_index.cpp -- host parser: HISAT2 .ht2 files -> packed index image.
//
// Reads <base>.1.ht2 .. <base>.8.ht2 exactly as laid out by the reference's
// loaders and re-packs the arrays into the single position-independent blob
// described in ht2_image.h.  Formats follow (not copied from):
//   gfm.h:5917-6458  GFM::readIntoMemory     (.1 header/body, .2 SA sample)
//   hgfm.h:2453-2651 HGFM::readIntoMemory    (.5 header)
//   hgfm.h:1106-1530 LocalGFM::readIntoMemory (.5 body, .6 SA sample)
//   reference.cpp:30-390 BitPairReference    (.3 records, .4 packed bases)
//   gfm.h:714-778, alt.h:197-204             (.7 ALTs)
// Little-endian files only (the reference refuses byte-swapped mmap too).
#include "ht2_index.h"
#include "ht2_fm.h"

#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

namespace {

struct FileBuf {
    std::vector<uint8_t> d;
    size_t pos = 0;
    explicit FileBuf(const std::string& path, bool optional = false) {
        FILE* f = fopen(path.c_str(), "rb");
        if (!f) {
            if (optional) return;
            throw std::runtime_error("ht2: could not open index file " + path);
        }
        fseek(f, 0, SEEK_END);
        long sz = ftell(f);
        fseek(f, 0, SEEK_SET);
        d.resize((size_t)sz);
        if (sz > 0 && fread(d.data(), 1, (size_t)sz, f) != (size_t)sz) {
            fclose(f);
            throw std::runtime_error("ht2: short read on " + path);
        }
        fclose(f);
    }
    void need(size_t n) const {
        if (pos + n > d.size()) throw std::runtime_error("ht2: truncated index file");
    }
    uint32_t u32() { need(4); uint32_t v; memcpy(&v, &d[pos], 4); pos += 4; return v; }
    int32_t  i32() { return (int32_t)u32(); }
    uint16_t u16() { need(2); uint16_t v; memcpy(&v, &d[pos], 2); pos += 2; return v; }
    uint64_t u64() { need(8); uint64_t v; memcpy(&v, &d[pos], 8); pos += 8; return v; }
    const uint8_t* take(size_t n) { need(n); const uint8_t* p = &d[pos]; pos += n; return p; }
    bool eof() const { return pos >= d.size(); }
};

struct Blob {
    std::vector<uint8_t> d;
    uint64_t alloc(size_t n, size_t align) {
        size_t off = (d.size() + align - 1) / align * align;
        d.resize(off + n, 0);
        return off;
    }
    uint64_t put(const void* src, size_t n, size_t align) {
        uint64_t off = alloc(n, align);
        if (n) memcpy(&d[off], src, n);
        return off;
    }
};

// GFMParams::init (gfm.h:134-176), for entry width 'eb' bytes.
void initGeom(Ht2Gfm& g, uint32_t len, uint32_t gbwtLen, uint32_t numNodes,
              int32_t lineRate, int32_t offRate, int32_t ftabChars,
              uint32_t eftabLen, uint32_t eb)
{
    memset(&g, 0, sizeof(g));
    g.entryBytes = eb;
    const uint32_t entryMax = (eb == 4) ? 0xffffffffu : 0xffffu;
    // all arithmetic in the reference happens in index_t (wraps for uint16)
    auto wrap = [&](uint32_t v) { return v & entryMax; };
    g.linearFM = (wrap(len + 1) == gbwtLen || gbwtLen == 0) ? 1 : 0;
    g.len = len;
    g.gbwtLen = (gbwtLen == 0 ? wrap(len + 1) : gbwtLen);
    g.numNodes = (numNodes == 0 ? wrap(len + 1) : numNodes);
    uint32_t gbwtSz = g.linearFM ? wrap(g.gbwtLen / 4 + 1) : wrap(g.gbwtLen / 2 + 1);
    g.offRate = (uint32_t)offRate;
    g.offMask = wrap(entryMax << offRate);
    g.ftabChars = (uint32_t)ftabChars;
    g.eftabLen = eftabLen;
    g.ftabLen = wrap((1u << (ftabChars * 2)) + 1);
    g.offsLen = wrap((g.numNodes + (1u << offRate) - 1) >> offRate);
    g.sideSz = 1u << lineRate;
    if (g.linearFM) {
        g.sideGbwtSz = g.sideSz - eb * 4;
        g.sideGbwtLen = g.sideGbwtSz << 2;
    } else {
        g.sideGbwtSz = g.sideSz - eb * 6;
        g.sideGbwtLen = g.sideGbwtSz << 1;
    }
    g.numSides = (gbwtSz + g.sideGbwtSz - 1) / g.sideGbwtSz;
    g.ftabCmp = g.linearFM ? g.len : g.gbwtLen;
}

// Re-lay a linear BWT (.ht2 sides: sideGbwtSz bytes of 2-bit chars + 4 occ
// entries, gfm.h:2952-2991) as 32-byte rank sides (ht2_image.h).  The occ
// entries of the file are cross-checked against the recount on the way.
void relayLinear(Blob& b, Ht2Gfm& g, const uint8_t* old, uint32_t z)
{
    const uint32_t eb = g.entryBytes;
    const uint32_t oldSz = g.sideSz, oldBwtSz = g.sideGbwtSz, oldLen = g.sideGbwtLen;
    const uint32_t nSides = (g.gbwtLen >> HT2_SIDE_SHIFT) + 1;   // a range end may equal gbwtLen
    // one zeroed side of slack so 16-byte side loads of row gbwtLen+small stay inside the blob
    g.o_gfm = b.alloc((size_t)(nSides + 1) * HT2_SIDE_BYTES, 128);
    uint32_t cnt[4] = {0, 0, 0, 0};
    for (uint32_t row = 0; row <= g.gbwtLen; row++) {
        if (row % oldLen == 0 && row < g.gbwtLen) {
            const uint8_t* tr = old + (size_t)(row / oldLen) * oldSz + oldBwtSz;
            for (int c = 0; c < 4; c++) {
                uint32_t v;
                if (eb == 4) memcpy(&v, tr + 4 * c, 4); else { uint16_t v16; memcpy(&v16, tr + 2 * c, 2); v = v16; }
                if (v != cnt[c]) throw std::runtime_error("ht2: occ table of the index disagrees with its BWT");
            }
        }
        if ((row & (HT2_SIDE_CHARS - 1)) == 0) {
            uint32_t occ[4];
            for (int c = 0; c < 4; c++) occ[c] = g.fchr[c] + cnt[c];
            memcpy(&b.d[g.o_gfm + (size_t)(row >> HT2_SIDE_SHIFT) * HT2_SIDE_BYTES + 16], occ, 16);
        }
        if (row == g.gbwtLen) break;
        const uint32_t co = row % oldLen;
        const int c = (old[(size_t)(row / oldLen) * oldSz + (co >> 2)] >> ((co & 3) << 1)) & 3;
        const uint32_t nco = row & (HT2_SIDE_CHARS - 1);
        b.d[g.o_gfm + (size_t)(row >> HT2_SIDE_SHIFT) * HT2_SIDE_BYTES + (nco >> 2)] |= (uint8_t)(c << ((nco & 3) << 1));
        if (row != z) cnt[c]++;
    }
    g.sideSz = HT2_SIDE_BYTES;
    g.sideGbwtSz = 16;
    g.sideGbwtLen = HT2_SIDE_CHARS;
    g.numSides = nSides;
}

// Re-lay a graph BWT (.ht2 sides: 2-bit chars, F bits, M bits, F_loc/M_occ/occ trailer,
// gfm.h:3394-3398, 3146-3154, 3790-3795) as 64-byte graph rank sides (ht2_image.h).
void relayGraph(Blob& b, Ht2Gfm& g, const uint8_t* old, const std::vector<uint32_t>& zs)
{
    const uint32_t eb = g.entryBytes;
    const uint32_t oldSz = g.sideSz, oldBwtSz = g.sideGbwtSz, oldLen = g.sideGbwtLen;
    const uint32_t nSides = (g.gbwtLen >> HT2_SIDE_SHIFT) + 2;   // rank queries reach row gbwtLen + 1
    g.o_gfm = b.alloc((size_t)(nSides + 1) * HT2_GSIDE_BYTES, 128);
    auto bitAt = [&](uint32_t row, uint32_t byteOff) -> int {
        const uint8_t* side = old + (size_t)(row / oldLen) * oldSz;
        const uint32_t k = row % oldLen;
        return (side[byteOff + (k >> 3)] >> (k & 7)) & 1;
    };
    std::vector<uint32_t> fpos;                 // fpos[n-1] = row of the n-th set F bit
    fpos.reserve(g.numNodes + 1);
    for (uint32_t row = 0; row < g.gbwtLen; row++) if (bitAt(row, oldBwtSz >> 1)) fpos.push_back(row);
    uint32_t cnt[4] = {0, 0, 0, 0}, mcnt = 0;
    for (uint32_t row = 0; row <= g.gbwtLen + HT2_SIDE_CHARS; row++) {
        uint8_t* side = &b.d[g.o_gfm + (size_t)(row >> HT2_SIDE_SHIFT) * HT2_GSIDE_BYTES];
        if ((row >> HT2_SIDE_SHIFT) >= nSides) break;
        if (row < g.gbwtLen && row % oldLen == 0) {
            // cross-check the file's own trailer: M_occ and the char occ entries
            const uint8_t* tr = old + (size_t)(row / oldLen) * oldSz + oldBwtSz;
            for (int k = 0; k < 6; k++) {
                uint32_t v;
                if (eb == 4) memcpy(&v, tr + 4 * k, 4); else { uint16_t v16; memcpy(&v16, tr + 2 * k, 2); v = v16; }
                if (k == 0 && (mcnt == 0 || mcnt > fpos.size())) continue;
                const uint32_t want = (k == 0) ? fpos[mcnt - 1] : (k == 1) ? mcnt : cnt[k - 2];
                if (v != (eb == 4 ? want : (want & 0xffffu))) throw std::runtime_error("ht2: rank tables of the graph index disagree with its BWT");
            }
        }
        if ((row & (HT2_SIDE_CHARS - 1)) == 0) {
            uint32_t tr[6];
            for (int c = 0; c < 4; c++) tr[c] = g.fchr[c] + cnt[c];
            tr[4] = mcnt;
            tr[5] = (mcnt > 0 && mcnt <= fpos.size()) ? fpos[mcnt - 1] : (mcnt == 0 ? 0u : g.gbwtLen);
            memcpy(side + 32, tr, 24);
        }
        if (row >= g.gbwtLen) continue;
        const uint32_t co = row % oldLen;
        const uint8_t* os = old + (size_t)(row / oldLen) * oldSz;
        const int c = (os[co >> 2] >> ((co & 3) << 1)) & 3;
        const uint32_t nco = row & (HT2_SIDE_CHARS - 1);
        side[nco >> 2] |= (uint8_t)(c << ((nco & 3) << 1));
        if (bitAt(row, oldBwtSz >> 1)) side[16 + (nco >> 3)] |= (uint8_t)(1u << (nco & 7));
        if (bitAt(row, oldBwtSz - (oldBwtSz >> 2))) { side[24 + (nco >> 3)] |= (uint8_t)(1u << (nco & 7)); mcnt++; }
        bool isZ = false;
        for (uint32_t z : zs) if (z == row) isZ = true;
        if (!isZ) cnt[c]++;
    }
    g.sideSz = HT2_GSIDE_BYTES;
    g.sideGbwtSz = 32;
    g.sideGbwtLen = HT2_SIDE_CHARS;
    g.numSides = nSides;
}

// Body shared by the global (.1) and local (.5) formats, after the header
// ints: nPat plen[] nFrag rstarts[] gfm[] nzOffs zOffs[] fchr[5] ftab[] eftab[]
void readBody(FileBuf& f, Blob& b, Ht2Gfm& g)
{
    const uint32_t eb = g.entryBytes;
    auto rdIdx = [&]() -> uint32_t { return eb == 4 ? f.u32() : f.u16(); };
    g.nPat = rdIdx();
    g.o_plen = b.put(f.take((size_t)g.nPat * eb), (size_t)g.nPat * eb, 16);
    g.nFrag = rdIdx();
    g.o_rstarts = b.put(f.take((size_t)g.nFrag * 3 * eb), (size_t)g.nFrag * 3 * eb, 16);
    size_t tot = (size_t)g.numSides * g.sideSz;
    const uint8_t* sides = f.take(tot);
    g.nzOffs = rdIdx();
    const uint8_t* zp = f.take((size_t)g.nzOffs * eb);
    g.o_zoffs = b.put(zp, (size_t)g.nzOffs * eb, 16);
    g.zOff0 = 0xffffffffu;
    if (g.nzOffs) { if (eb == 4) memcpy(&g.zOff0, zp, 4); else { uint16_t v; memcpy(&v, zp, 2); g.zOff0 = v; } }
    for (int i = 0; i < 5; i++) g.fchr[i] = rdIdx();
    if (g.linearFM) {
        if (g.nzOffs != 1) throw std::runtime_error("ht2: linear index with other than one '$' row");
        relayLinear(b, g, sides, g.zOff0);
    } else {
        std::vector<uint32_t> zs(g.nzOffs);
        for (uint32_t i = 0; i < g.nzOffs; i++) { if (eb == 4) memcpy(&zs[i], zp + 4 * i, 4); else { uint16_t v; memcpy(&v, zp + 2 * i, 2); zs[i] = v; } }
        relayGraph(b, g, sides, zs);
    }
    g.o_ftab = b.put(f.take((size_t)g.ftabLen * eb), (size_t)g.ftabLen * eb, 16);
    g.o_eftab = b.put(f.take((size_t)g.eftabLen * eb), (size_t)g.eftabLen * eb, 16);
}


// Densify the suffix-array sample of a LINEAR index.  The .ht2 files sample every 2^offRate-th row (offRate 4 by
// default: gfm.h:5682 getOffset walks ~7.5 LF steps per resolved row, a third of all LF steps of a read); the
// image spends HBM instead -- 80 GB per H100 -- and keeps every 2^HT2_DENSE_OFFRATE-th row, so that
// tryOffset succeeds after ~1.5 steps.  The value of a row is a property of the index, not of the sampling:
// new[r] = old[row'] + steps for the first sampled row' on r's LF walk, exactly what getOffset returns.
#ifndef HT2_DENSE_OFFRATE
#define HT2_DENSE_OFFRATE 2
#endif
template <typename IT>
void densifySample(Blob& b, Ht2Gfm& g)
{
    if (!g.linearFM || g.len == 0 || g.offRate <= HT2_DENSE_OFFRATE) return;
    const uint32_t newRate = HT2_DENSE_OFFRATE;
    const uint32_t entryMax = (sizeof(IT) == 4) ? 0xffffffffu : 0xffffu;
    const uint32_t nNew = (g.numNodes + (1u << newRate) - 1) >> newRate;
    const uint64_t oNew = b.alloc((size_t)nNew * sizeof(IT), 128);   // may move the blob: take pointers afterwards
    Ht2Fm<IT> fm;
    fm.init(b.d.data(), &g);
    IT* out = (IT*)(b.d.data() + oNew);
    const uint32_t oldMask = g.offMask, oldRate = g.offRate, z0 = g.zOff0;
    unsigned nth = std::thread::hardware_concurrency();
    if (nth < 1) nth = 1;
    if (nth > 32) nth = 32;
    if (nNew < (1u << 16)) nth = 1;
    auto work = [&](unsigned t) {
        const uint32_t k0 = (uint32_t)((uint64_t)nNew * t / nth), k1 = (uint32_t)((uint64_t)nNew * (t + 1) / nth);
        for (uint32_t k = k0; k < k1; k++) {
            uint32_t row = k << newRate, steps = 0;
            uint32_t v;
            for (;;) {
                if (row == z0) { v = steps; break; }
                if ((row & oldMask) == row) { v = (uint32_t)fm.offs[row >> oldRate] + steps; break; }
                int c;
                row = ht2_lf_own(fm, row, c);
                steps++;
            }
            out[k] = (IT)v;
        }
    };
    if (nth == 1) work(0);
    else {
        std::vector<std::thread> th;
        for (unsigned t = 0; t < nth; t++) th.emplace_back(work, t);
        for (auto& x : th) x.join();
    }
    g.o_offs = oNew;
    g.offRate = newRate;
    g.offMask = (entryMax << newRate) & entryMax;
    g.offsLen = nNew;
}

} // namespace

Ht2Image* ht2_image_load(const char* base_c, std::string& err)
{
    try {
        const std::string base(base_c);
        Blob b;
        b.alloc(sizeof(Ht2ImageHeader), 128);
        Ht2ImageHeader h;
        memset(&h, 0, sizeof(h));
        h.magic = HT2_MAGIC;
        h.version = HT2_IMAGE_VERSION;

        // ---- .1.ht2 : global index ------------------------------------
        FileBuf f1(base + ".1.ht2");
        if (f1.u32() != 1) throw std::runtime_error("ht2: index has opposite endianness");
        f1.u32(); // version word
        uint32_t len = f1.u32(), gbwtLen = f1.u32(), numNodes = f1.u32();
        int32_t lineRate = f1.i32();
        f1.i32(); // linesPerSide
        int32_t offRate = f1.i32();
        int32_t ftabChars = f1.i32();
        uint32_t eftabLen = f1.u32();
        f1.i32(); // flags
        initGeom(h.global, len, gbwtLen, numNodes, lineRate, offRate, ftabChars, eftabLen, 4);
        readBody(f1, b, h.global);
        // reference names: '\n'-separated, '\0'-terminated (gfm.h:6270-6300)
        std::vector<std::string> names;
        {
            std::string cur;
            while (!f1.eof()) {
                char c = (char)*f1.take(1);
                if (c == '\0') break;
                if (c == '\n') { names.push_back(cur); cur.clear(); }
                else cur.push_back(c);
            }
            if (!cur.empty()) names.push_back(cur);
        }
        h.nRefs = h.global.nPat;
        while (names.size() < h.nRefs) names.push_back(std::to_string(names.size()));
        {
            std::string packed;
            std::vector<uint32_t> noffs;
            for (uint32_t i = 0; i < h.nRefs; i++) { noffs.push_back((uint32_t)packed.size()); packed += names[i]; packed.push_back('\0'); }
            noffs.push_back((uint32_t)packed.size());
            h.o_names = b.put(packed.data(), packed.size(), 16);
            h.namesBytes = packed.size();
            h.o_nameOffs = b.put(noffs.data(), noffs.size() * 4, 16);
        }

        // ---- .2.ht2 : SA sample ---------------------------------------
        {
            FileBuf f2(base + ".2.ht2");
            f2.u32(); // endian hint
            size_t n = (size_t)h.global.offsLen * 4;
            h.global.o_offs = b.put(f2.take(n), n, 128);
            densifySample<uint32_t>(b, h.global);
        }

        // ---- .5/.6.ht2 : local indexes --------------------------------
        std::vector<Ht2Gfm> locals;
        std::vector<uint32_t> localFirst(h.nRefs + 1, 0);
        {
            FileBuf f5(base + ".5.ht2", true), f6(base + ".6.ht2", true);
            if (!f5.d.empty()) {
                if (f5.u32() != 1) throw std::runtime_error("ht2: local index has opposite endianness");
                if (!f6.d.empty()) f6.u32();
                uint32_t nlocal = f5.u32();
                int32_t llineRate = f5.i32();
                f5.i32();
                int32_t loffRate = f5.i32();
                int32_t lftabChars = f5.i32();
                f5.i32(); // flags
                locals.resize(nlocal);
                std::vector<uint32_t> counts(h.nRefs, 0);
                for (uint32_t i = 0; i < nlocal; i++) {
                    Ht2Gfm& g = locals[i];
                    uint32_t tidx = f5.u32(), localOffset = f5.u32(), joinedOffset = f5.u32();
                    uint32_t llen = f5.u16(), lgbwtLen = f5.u16(), lnumNodes = f5.u16(), leftabLen = f5.u16();
                    initGeom(g, llen, lgbwtLen, lnumNodes, llineRate, loffRate, lftabChars, leftabLen, 2);
                    g.tidx = tidx; g.localOffset = localOffset; g.joinedOffset = joinedOffset;
                    if (tidx >= h.nRefs) throw std::runtime_error("ht2: local index tidx out of range");
                    counts[tidx]++;
                    if (llen == 0) continue; // empty local index (hgfm.h:1147-1150)
                    readBody(f5, b, g);
                    size_t n = (size_t)g.offsLen * 2;
                    g.o_offs = b.put(f6.take(n), n, 16);
                    densifySample<uint16_t>(b, g);
                }
                // the reference appends local indexes to the list of their
                // reference in file order (hgfm.h:2637-2641)
                for (uint32_t t = 0; t < h.nRefs; t++) localFirst[t + 1] = localFirst[t] + counts[t];
                uint32_t prev = 0;
                for (uint32_t i = 0; i < nlocal; i++) {
                    if (locals[i].tidx < prev) throw std::runtime_error("ht2: local indexes not grouped by reference");
                    prev = locals[i].tidx;
                }
            }
        }
        h.nLocal = (uint32_t)locals.size();
        h.o_localGfm = b.put(locals.data(), locals.size() * sizeof(Ht2Gfm), 128);
        h.o_localFirst = b.put(localFirst.data(), localFirst.size() * 4, 16);

        // ---- .3/.4.ht2 : 2-bit reference ------------------------------
        {
            FileBuf f3(base + ".3.ht2");
            if (f3.i32() != 1) throw std::runtime_error("ht2: reference has opposite endianness");
            uint32_t nrec = f3.u32();
            std::vector<Ht2RefRecord> recs(nrec);
            std::vector<uint32_t> refRecOffs;
            std::vector<uint64_t> refOffs;
            std::vector<uint32_t> refLens;
            uint64_t cumsz = 0;
            uint32_t cumlen = 0;
            for (uint32_t i = 0; i < nrec; i++) {
                recs[i].off = f3.u32();
                recs[i].len = f3.u32();
                recs[i].first = *f3.take(1) ? 1 : 0;
                recs[i].pad = 0;
                if (recs[i].first) {
                    refRecOffs.push_back(i);
                    refOffs.push_back(cumsz);
                    if (refRecOffs.size() > 1) refLens.push_back(cumlen);
                    cumlen = 0;
                } else if (i == 0) {
                    throw std::runtime_error("ht2: first reference record is not marked 'first'");
                }
                cumsz += recs[i].len;
                cumlen += recs[i].off + recs[i].len;
            }
            refRecOffs.push_back(nrec);
            refOffs.push_back(cumsz);
            refLens.push_back(cumlen);
            if (refLens.size() != h.nRefs)
                throw std::runtime_error("ht2: .3.ht2 reference count differs from .1.ht2");
            h.nRecs = nrec;
            h.o_recs = b.put(recs.data(), recs.size() * sizeof(Ht2RefRecord), 16);
            h.o_refRecOffs = b.put(refRecOffs.data(), refRecOffs.size() * 4, 16);
            h.o_refOffs = b.put(refOffs.data(), refOffs.size() * 8, 16);
            h.o_refLens = b.put(refLens.data(), refLens.size() * 4, 16);
            FileBuf f4(base + ".4.ht2");
            size_t need = (size_t)((cumsz + 3) >> 2);
            if (f4.d.size() < need) throw std::runtime_error("ht2: .4.ht2 shorter than .3.ht2 implies");
            h.refBufBytes = need;
            h.o_refBuf = b.put(f4.d.data(), need, 128);
            b.alloc(16, 16);
        }

        // ---- .7/.8.ht2 : ALTs and their names (gfm.h:714-903) ------------
        {
            FileBuf f7(base + ".7.ht2", true), f8(base + ".8.ht2", true);
            std::vector<Ht2Alt> alts;
            std::vector<std::string> names;
            if (f7.d.size() >= 8) {
                f7.u32(); // endian hint
                uint32_t nalt = f7.u32();
                for (uint32_t i = 0; i < nalt && !f7.eof(); i++) {
                    Ht2Alt a;
                    a.pos = f7.u32(); a.type = f7.u32(); a.len = f7.u32(); a.reversed = 0;
                    a.seq = f7.u64();
                    alts.push_back(a);
                }
                // names: whitespace-separated tokens after two 32-bit words
                size_t p8 = 8;
                while (names.size() < alts.size()) {
                    while (p8 < f8.d.size() && isspace((unsigned char)f8.d[p8])) p8++;
                    std::string nm;
                    while (p8 < f8.d.size() && !isspace((unsigned char)f8.d[p8])) nm.push_back((char)f8.d[p8++]);
                    names.push_back(nm);
                }
            }
            const size_t nalts = alts.size();
            for (size_t s2 = 0; s2 < nalts; s2++) {
                const Ht2Alt a = alts[s2];
                if (a.type == HT2_ALT_SNP_ALT) h.altsUnsupported = 1;
                if (a.type == HT2_ALT_EXON) h.nExons++;
                if (a.type == HT2_ALT_SPLICESITE) {    // reversed copy: left and right swapped, named "ssr" (gfm.h:873-879)
                    h.nSpliceSites++;
                    Ht2Alt r = a;
                    r.pos = a.len; r.len = a.pos;
                    alts.push_back(r);
                    names.push_back("ssr");
                } else if (a.type == HT2_ALT_SNP_DEL) {       // reversed copy at the deletion's last base (gfm.h:880-885)
                    Ht2Alt r = a;
                    r.pos = a.pos + a.len - 1;
                    r.reversed = 1;
                    r.seq = (a.seq & ~(uint64_t)0xff) | 1u;
                    alts.push_back(r);
                    names.push_back(names[s2]);
                }
            }
            if (alts.size() > 1 && alts.size() > nalts) {
                // EList<pair<ALT, index>>::sort with ALT::operator< (alt.h:89-103)
                auto altLess = [](const Ht2Alt& x, const Ht2Alt& y) {
                    if (x.pos != y.pos) return x.pos < y.pos;
                    if (x.type != y.type) {
                        if (x.type == HT2_ALT_NONE || y.type == HT2_ALT_NONE) return x.type == HT2_ALT_NONE;
                        if (x.type == HT2_ALT_SNP_INS) return true;
                        else if (y.type == HT2_ALT_SNP_INS) return false;
                        return x.type < y.type;
                    }
                    if (x.len != y.len) return x.len < y.len;
                    if (x.seq != y.seq) return x.seq < y.seq;
                    return false;
                };
                std::vector<uint32_t> order(alts.size());
                for (size_t i = 0; i < order.size(); i++) order[i] = (uint32_t)i;
                std::sort(order.begin(), order.end(), [&](uint32_t i, uint32_t j) {
                    if (altLess(alts[i], alts[j])) return true;
                    if (altLess(alts[j], alts[i])) return false;
                    return i < j;
                });
                std::vector<Ht2Alt> a2(alts.size());
                std::vector<std::string> n2(alts.size());
                for (size_t i = 0; i < order.size(); i++) { a2[i] = alts[order[i]]; n2[i] = names[order[i]]; }
                alts.swap(a2); names.swap(n2);
            }
            h.nAlts = (uint32_t)alts.size();
            h.o_alts = b.put(alts.data(), alts.size() * sizeof(Ht2Alt), 16);
            std::string packed;
            std::vector<uint32_t> noffs;
            for (size_t i = 0; i < names.size(); i++) { noffs.push_back((uint32_t)packed.size()); packed += names[i]; packed.push_back('\0'); }
            noffs.push_back((uint32_t)packed.size());
            h.o_altNames = b.put(packed.data(), packed.size(), 16);
            h.altNamesBytes = packed.size();
            h.o_altNameOffs = b.put(noffs.data(), noffs.size() * 4, 16);
        }

        b.alloc(0, 128);
        h.totalBytes = b.d.size();
        memcpy(b.d.data(), &h, sizeof(h));

        Ht2Image* img = new Ht2Image();
        img->blob.swap(b.d);
        return img;
    } catch (const std::exception& e) {
        err = e.what();
        return nullptr;
    }
}


// ---------------------------------------------------------------------------------------------------------------
// Splice-site DB blob (ht2_ssdb.h)
// ---------------------------------------------------------------------------------------------------------------
#include "ht2_ssdb.h"
#include <fstream>
#include <sstream>
#include <algorithm>
#include <set>
#include <tuple>
// the reference-name table of a handle (ht2_index.h): the splice-site DB matches and prints its names
void Ht2RefNames::build(const Ht2Image& img, int chrNames)
{
    const uint32_t nRefs = img.header()->nRefs;
    blob.assign((size_t)nRefs * 4, 0);
    for (uint32_t r = 0; r < nRefs; r++) {
        std::string n = img.refName(r);
        const bool chr = n.compare(0, 3, "chr") == 0;
        if (chrNames == HT2GPU_CHR_NAMES_REMOVE && chr) n = n.substr(3);
        else if (chrNames == HT2GPU_CHR_NAMES_ADD && !chr) n = "chr" + n;
        const uint32_t at = (uint32_t)blob.size();
        memcpy(blob.data() + (size_t)r * 4, &at, 4);
        blob.insert(blob.end(), n.c_str(), n.c_str() + n.size() + 1);
    }
}

std::string Ht2RefNames::token(uint32_t i) const
{
    const char* n = (*this)[i];
    size_t k = 0;
    while (n[k] && !isspace((unsigned char)n[k])) k++;
    return std::string(n, k);
}

bool ht2_ssdb_build(const Ht2Image& img, const std::vector<Ht2SsFile>& files, std::vector<uint8_t>& blob, uint32_t& nSites, std::string& err,
                    const Ht2RefNames* refNames, bool indexSites)
{
    const uint32_t nRefs = img.header()->nRefs;
    Ht2RefNames own;
    if (!refNames) { own.build(img, HT2GPU_CHR_NAMES_INDEX); refNames = &own; }
    std::vector<std::string> names(nRefs);
    for (uint32_t r = 0; r < nRefs; r++) names[r] = refNames->token(r);
    std::vector<std::vector<Ht2SsSite>> per(nRefs);
    std::vector<std::set<std::tuple<uint32_t, uint32_t, uint32_t>>> seen(nRefs);
    std::vector<Ht2SsExon> exons;
    {   // the index's splice sites and exons first (SpliceSiteDB::read(gfm, alts), splice_site.cpp:653-720)
        const Ht2ImageHeader* H = img.header();
        const uint8_t* blob0 = img.blob.data();
        const Ht2Alt* alts = (const Ht2Alt*)(blob0 + H->o_alts);
        const uint32_t* rstarts = (const uint32_t*)(blob0 + H->global.o_rstarts);
        const uint32_t* plen = (const uint32_t*)(blob0 + H->global.o_plen);
        const uint32_t nFrag = H->global.nFrag;
        for (uint32_t i = 0; i < H->nAlts; i++) {
            const Ht2Alt& a = alts[i];
            if (a.type != HT2_ALT_EXON && (a.type != HT2_ALT_SPLICESITE || !indexSites)) continue;
            if (a.pos > a.len) continue;   // the reversed copy of a splice site
            // joinedToTextOff(1, left, ...) with straddlers rejected (gfm.h:5527-5600)
            uint32_t lo = 0, hi = nFrag;
            while (lo < hi) { const uint32_t m = lo + ((hi - lo) >> 1); if (rstarts[m * 3] <= a.pos) lo = m + 1; else hi = m; }
            const uint32_t elt = lo - 1;
            const uint32_t upper = elt + 1 == nFrag ? H->global.len : rstarts[(elt + 1) * 3];
            if (lo == 0 || a.pos >= upper) { err = "ht2: a splice-site / exon ALT of the index lies outside the reference"; return false; }
            const uint32_t ref = rstarts[elt * 3 + 1], tlen = plen[ref];
            uint32_t left = a.pos - rstarts[elt * 3] + rstarts[elt * 3 + 2];
            uint32_t right = left + (a.len - a.pos);
            const uint32_t fw = (uint32_t)(a.seq & 0xff);
            if (a.type == HT2_ALT_SPLICESITE) {
                left -= 1; right += 1;
                Ht2SsSite st; st.left = left; st.right = right; st.dir = fw ? HT2_SPL_FW : HT2_SPL_RC; st.known = 1;
                if (seen[ref].insert(std::make_tuple(st.left, st.right, st.dir)).second) per[ref].push_back(st);
            } else {
                left = left >= 10 ? left - 10 : 0;
                right = right + 10 < tlen ? right + 10 : tlen - 1;
                Ht2SsExon e; e.ref = ref; e.left = left; e.right = right; e.pad = 0;
                exons.push_back(e);
            }
        }
        std::stable_sort(exons.begin(), exons.end(), [](const Ht2SsExon& x, const Ht2SsExon& y) {
            return x.ref != y.ref ? x.ref < y.ref : (x.left != y.left ? x.left < y.left : x.right < y.right); });
    }
    for (const Ht2SsFile& f : files) {
        std::ifstream in(f.path.c_str(), std::ios::in);
        if (!in.is_open()) continue;
        std::string refname, sl, sr, sd;
        while (in >> refname) {
            if (!(in >> sl >> sr >> sd)) { err = "ht2: truncated splice-site record in " + f.path; return false; }
            char* e1 = NULL; char* e2 = NULL;
            const unsigned long long l = strtoull(sl.c_str(), &e1, 10), r = strtoull(sr.c_str(), &e2, 10);
            if (*e1 || *e2 || l > 0xfffffffeull || r > 0xfffffffeull) { err = "ht2: malformed splice-site record in " + f.path + ": " + refname + " " + sl + " " + sr; return false; }
            uint32_t ref = 0;
            for (; ref < nRefs; ref++) if (names[ref] == refname) break;
            if (ref >= nRefs) continue;
            Ht2SsSite s; s.left = (uint32_t)l; s.right = (uint32_t)r; s.dir = sd[0] == '+' ? HT2_SPL_FW : HT2_SPL_RC; s.known = f.known ? 1u : 0u;
            if (seen[ref].insert(std::make_tuple(s.left, s.right, s.dir)).second) per[ref].push_back(s);   // a site already present is dropped (_fwIndex->add fails)
        }
    }
    nSites = 0;
    for (auto& v : per) nSites += (uint32_t)v.size();
    const size_t offWords = ((size_t)nRefs + 1 + 3) & ~(size_t)3;
    blob.assign(sizeof(Ht2SsHeader) + offWords * 4 + (size_t)nSites * 2 * sizeof(Ht2SsSite) + exons.size() * sizeof(Ht2SsExon), 0);
    Ht2SsHeader* h = (Ht2SsHeader*)blob.data();
    h->magic = HT2_SS_MAGIC; h->nRefs = nRefs; h->nSites = nSites; h->nExons = (uint32_t)exons.size();
    if (!exons.empty()) memcpy(blob.data() + sizeof(Ht2SsHeader) + offWords * 4 + (size_t)nSites * 2 * sizeof(Ht2SsSite), exons.data(), exons.size() * sizeof(Ht2SsExon));
    uint32_t* refOff = (uint32_t*)(blob.data() + sizeof(Ht2SsHeader));
    Ht2SsSite* fw = (Ht2SsSite*)(blob.data() + sizeof(Ht2SsHeader) + offWords * 4);
    Ht2SsSite* bw = fw + nSites;
    uint32_t at = 0;
    for (uint32_t r = 0; r < nRefs; r++) {
        refOff[r] = at;
        std::vector<Ht2SsSite> a = per[r], b = per[r];
        std::sort(a.begin(), a.end(), [](const Ht2SsSite& x, const Ht2SsSite& y) { return x.left != y.left ? x.left < y.left : (x.right != y.right ? x.right < y.right : x.dir < y.dir); });
        std::sort(b.begin(), b.end(), [](const Ht2SsSite& x, const Ht2SsSite& y) { return x.right != y.right ? x.right < y.right : (x.left != y.left ? x.left < y.left : x.dir < y.dir); });
        for (size_t i = 0; i < a.size(); i++) { fw[at + i] = a[i]; bw[at + i] = b[i]; }
        at += (uint32_t)a.size();
    }
    refOff[nRefs] = at;
    return true;
}


void Ht2NovelSites::add(const Ht2SsRec* recs, size_t n)
{
    for (size_t i = 0; i < n; i++) {
        const Ht2SsRec& r = recs[i];
        const uint32_t dir = r.dirEd & 0xffu, ed = r.dirEd >> 8;
        auto it = sites.find(std::make_tuple(r.ref, r.left, r.right, dir));
        if (it == sites.end()) sites[std::make_tuple(r.ref, r.left, r.right, dir)] = std::make_pair(1u, ed);
        else { it->second.first += 1; if (ed < it->second.second) it->second.second = ed; }
    }
}
void Ht2NovelSites::merge(const Ht2NovelSites& o)
{
    for (const auto& kv : o.sites) {
        auto it = sites.find(kv.first);
        if (it == sites.end()) sites[kv.first] = kv.second;
        else { it->second.first += kv.second.first; if (kv.second.second < it->second.second) it->second.second = kv.second.second; }
    }
}
bool Ht2NovelSites::write(const Ht2Image& img, const char* path, uint64_t* nWritten, std::string& err, const Ht2RefNames* names) const
{
    Ht2RefNames own;
    if (!names) { own.build(img, HT2GPU_CHR_NAMES_INDEX); names = &own; }
    FILE* f = fopen(path, "wb");
    if (!f) { err = std::string("ht2: cannot write ") + path; return false; }
    // calculate_splicesite_read_dist (splice_site.cpp:528-563): smallest read count whose cumulative share of the sites exceeds 0.7
    int64_t dist[100]; for (int i = 0; i < 100; i++) dist[i] = 0;
    for (const auto& kv : sites) { const uint32_t n = kv.second.first; if (n < 100) dist[n] += 1; else dist[99] += 1; }
    for (int i = 1; i < 100; i++) dist[i] += dist[i - 1];
    uint32_t cutoff = 0;
    for (int i = 0; i < 100; i++) { const float cmf = float(dist[i]) / dist[99]; if (cmf > 0.7) { cutoff = (uint32_t)i; break; } }
    const uint32_t cutoff2 = (uint32_t)(sites.size() / 100000);
    struct S { uint32_t ref, left, right, dir, numreads; };
    std::vector<S> list;
    uint64_t nw = 0;
    auto impl = [&](const S* ss) {   // print_impl (splice_site.cpp:605-651)
        size_t i = 0;
        while (i < list.size()) {
            const S tmp = list[i];
            bool do_print = true;
            if (ss != NULL && tmp.ref == ss->ref && ss->left < tmp.left + 10) {
                do_print = false;
                const int d = ((int)ss->left - (int)tmp.left) - ((int)ss->right - (int)tmp.right);
                if ((d < 0 ? -d : d) <= 10) {
                    if (tmp.numreads < ss->numreads) { list.erase(list.begin() + i); list.push_back(*ss); }
                    return;
                }
            }
            if (!do_print) { i++; continue; }
            const char c = (tmp.dir == HT2_SPL_FW || tmp.dir == HT2_SPL_SEMI_FW) ? '+' : ((tmp.dir == HT2_SPL_RC || tmp.dir == HT2_SPL_SEMI_RC) ? '-' : '.');
            fprintf(f, "%s\t%u\t%u\t%c\n", names->token(tmp.ref).c_str(), tmp.left, tmp.right, c);
            nw++;
            list.erase(list.begin() + i);
        }
        if (ss != NULL) list.push_back(*ss);
    };
    for (const auto& kv : sites) {   // std::map order = (ref, left, right, dir): the in-order walk of every _fwIndex in turn
        const S ss = {std::get<0>(kv.first), std::get<1>(kv.first), std::get<2>(kv.first), std::get<3>(kv.first), kv.second.first};
        if (ss.numreads >= cutoff || (kv.second.second == 0 && ss.numreads >= cutoff2)) impl(&ss);
    }
    impl(NULL);
    fclose(f);
    if (nWritten) *nWritten = nw;
    return true;
}
