// ht2_inflate.h -- gzip (RFC 1952 members of RFC 1951 DEFLATE) inflated in parallel chunks.
//
// A single-member gzip stream cannot be split without decoding it, so the compressed input is cut into chunks of a
// fixed compressed size and every chunk after the first is decoded speculatively (the pugz / rapidgzip approach):
//
//   1. find: in each chunk, the first bit offset where a block can begin -- a dynamic-Huffman header whose code-length,
//      literal/length and distance codes are complete, a byte-aligned stored header (LEN == ~NLEN after zero pad bits)
//      or a gzip member header (1f 8b 08, reserved flags clear);
//   2. decode: from that candidate, without the 32 KiB window before it, into 16-bit symbols: 0..255 are bytes, 256 + i
//      is byte i of the 32 KiB before the chunk (a marker); markers copied by later back-references stay markers.  A
//      chunk stops at the first block or member boundary at or past the next chunk's candidate;
//   3. confirm: a candidate counts only when the previous chunk stopped exactly on it.  A chunk without a candidate,
//      or one whose candidate was false, is merged into its predecessor, which continues through it (a cost in time,
//      never in output).  A stream with no findable boundaries (Z_FIXED) thus decodes sequentially;
//   4. window: in chunk order, each chunk's last 32 KiB are resolved from the previous chunk's window;
//   5. replace: every marker becomes its byte, in parallel;
//   6. verify: the CRC-32 of each chunk's part of each member, combined per member with crc32_combine arithmetic and
//      checked with ISIZE against the member's trailer.
//
// The input goes through in windows of compressed bytes (the 32 KiB window and the decoder state carry over), so the
// memory used is fixed whatever the size of the file.  Everything a chunk reads or writes is bounds-checked: corrupt
// input ends in an error status, never in an access outside the buffers.  A chunk stops only at a symbol boundary, and
// its state (bit position, phase, code lengths of the current block) is enough to resume it, in the same window
// (merging) or the next.
//
// The decoder (ht2z_candidate, ht2z_run, ht2z_next_win / ht2z_sym) is HT2_HD code: ht2_inflate.cu runs it as kernels, and the host
// backend below runs the same source in loops (tests/hostsim/ht2_gunzipsim.cpp).  ht2z_gunzip is the driver of both.
#ifndef HT2_INFLATE_H_
#define HT2_INFLATE_H_

#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../include/ht2gpu.h"
#include "ht2_image.h"

#define HT2Z_WSIZE 32768u
#define HT2Z_EV 64                  // member trailers recorded per chunk; a chunk stops (resumably) when its list is full
#define HT2Z_LFAST 10               // bits of the literal/length lookup table
#define HT2Z_DFAST 8                // bits of the distance lookup table
#define HT2Z_NONE (~(uint64_t)0)
#define HT2Z_PIECE 4096u            // bytes per CRC-32 piece

enum { HT2Z_PH_MEMBER = 0, HT2Z_PH_BLOCK, HT2Z_PH_HUFF, HT2Z_PH_STORED, HT2Z_PH_TRAILER };
// chunk status: STOP..EV_FULL end at a resumable state, the rest are errors of the input
enum { HT2Z_STOP = 0, HT2Z_END, HT2Z_PAD, HT2Z_NEED_INPUT, HT2Z_OUT_FULL, HT2Z_EV_FULL,
       HT2Z_E_HEADER, HT2Z_E_BTYPE, HT2Z_E_STORED, HT2Z_E_CODES, HT2Z_E_SYMBOL, HT2Z_E_DIST, HT2Z_E_GARBAGE };
enum { HT2Z_K_NONE = 0, HT2Z_K_BLOCK, HT2Z_K_STORED, HT2Z_K_MEMBER, HT2Z_K_RESUME };

struct Ht2zState {                  // a resumable decoder position (always at a symbol boundary)
    uint64_t bit;                   // absolute bit position in the compressed input
    uint32_t phase, last;           // HT2Z_PH_*, BFINAL of the current block
    uint32_t stored, pad;           // bytes left in the current stored block
    uint8_t  lens[320];             // PH_HUFF: code lengths of the current block (288 literal/length, 32 distance)
};
struct Ht2zEvent { uint32_t pos, crc, isize, pad; };   // a member trailer; pos = the member's end in the chunk output
struct Ht2zChunk {
    Ht2zState st;                   // in: where to start or continue; out: where the chunk stopped
    uint64_t  cand;                 // the candidate: its bit (stored blocks: the bit of LEN)
    uint64_t  stopBit;              // stop at the first block or member boundary at or past this bit
    uint32_t  kind, status, nout, nev, nblk;
    int32_t   base;                 // output position of the current member's start (negative: before the chunk)
    int32_t   lastStart;            // output position of the last member start inside the chunk, -1 = none
    uint32_t  cap;                  // symbols the chunk may hold: its slice and those of the chunks it absorbed
    Ht2zEvent ev[HT2Z_EV];
};

// ---------------------------------------------------------------------------------------------------------------------
// tables
// ---------------------------------------------------------------------------------------------------------------------
#define HT2Z_TABLES                                                                                                   \
    {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15},                                                \
    {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258}, \
    {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0},                           \
    {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,     \
     6145, 8193, 12289, 16385, 24577},                                                                                 \
    {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13}
struct Ht2zConst { uint8_t clOrder[19]; uint16_t lbase[29]; uint8_t lext[29]; uint16_t dbase[30]; uint8_t dext[30]; };
static const Ht2zConst ht2z_const_h = {HT2Z_TABLES};
#if defined(__CUDACC__)
__constant__ Ht2zConst ht2z_const_d = {HT2Z_TABLES};
#endif
HT2_HD const Ht2zConst& ht2z_k()
{
#if defined(__CUDA_ARCH__)
    return ht2z_const_d;
#else
    return ht2z_const_h;
#endif
}

// ---------------------------------------------------------------------------------------------------------------------
// bits: LSB first from bytes [base, end) of the input held at p (p[0] = input byte base)
// ---------------------------------------------------------------------------------------------------------------------
struct Ht2zBits {
    const uint8_t* p;
    uint64_t base, end, next;       // next: the next input byte to load into buf
    uint64_t buf;
    uint32_t cnt;                   // valid bits in buf
    HT2_HD void init(const uint8_t* src, uint64_t b, uint64_t e, uint64_t bit)
    {
        p = src; base = b; end = e; next = bit >> 3; buf = 0; cnt = 0;
        if (next < base) next = end;                 // before the buffer: reads as the end of the input
        refill();
        const uint32_t s = (uint32_t)(bit & 7);
        if (cnt >= s) drop(s); else cnt = 0;
    }
    HT2_HD void refill() { while (cnt <= 56 && next < end) { buf |= (uint64_t)p[next - base] << cnt; next++; cnt += 8; } }
    HT2_HD uint64_t pos() const { return next * 8 - cnt; }
    HT2_HD bool have(uint32_t n) { if (cnt < n) refill(); return cnt >= n; }
    HT2_HD uint32_t peek(uint32_t n) const { return (uint32_t)(buf & ((1ull << n) - 1)); }
    HT2_HD void drop(uint32_t n) { buf >>= n; cnt -= n; }
    HT2_HD uint32_t get(uint32_t n) { const uint32_t v = peek(n); drop(n); return v; }   // after have(n)
    HT2_HD void align() { drop(cnt & 7); }
};

// ---------------------------------------------------------------------------------------------------------------------
// canonical Huffman codes: a lookup table of the first FB bits, counts / symbols for the longer codes
// ---------------------------------------------------------------------------------------------------------------------
template <int NS, int FB>
struct Ht2zHuff { uint16_t count[16]; uint16_t sym[NS]; uint16_t fast[FB ? (1 << FB) : 1]; };

// zlib's rules: over-subscribed is an error; incomplete only for a single code of length 1 (allowIncomplete)
template <int NS, int FB>
HT2_HD bool ht2z_build(Ht2zHuff<NS, FB>& h, const uint8_t* len, int n, bool allowIncomplete)
{
    for (int i = 0; i < 16; i++) h.count[i] = 0;
    for (int i = 0; i < n; i++) h.count[len[i]]++;
    int left = 1, maxLen = 0;
    for (int l = 1; l < 16; l++) { left <<= 1; left -= h.count[l]; if (left < 0) return false; if (h.count[l]) maxLen = l; }
    if (left > 0 && maxLen > 0 && !(allowIncomplete && maxLen == 1)) return false;
    uint16_t offs[16], next[16];
    offs[1] = 0;
    for (int l = 1; l < 15; l++) offs[l + 1] = (uint16_t)(offs[l] + h.count[l]);
    uint32_t code = 0;
    for (int l = 1; l < 16; l++) { code = (code + h.count[l - 1] * (l > 1)) << 1; next[l] = (uint16_t)code; }
    if (FB) for (int i = 0; i < (1 << FB); i++) h.fast[i] = 0;
    for (int i = 0; i < n; i++) {
        const int l = len[i];
        if (!l) continue;
        h.sym[offs[l]++] = (uint16_t)i;
        const uint32_t c = next[l]++;
        if (FB && l <= FB) {
            uint32_t r = 0;
            for (int b = 0; b < l; b++) r |= ((c >> b) & 1) << (l - 1 - b);
            for (uint32_t j = r; j < (1u << FB); j += 1u << l) h.fast[j] = (uint16_t)((l << 9) | i);
        }
    }
    return true;
}

// >= 0 symbol, -1 invalid code, -2 input ends inside the code
template <int NS, int FB>
HT2_HD int ht2z_decode(Ht2zBits& br, const Ht2zHuff<NS, FB>& h)
{
    br.refill();
    if (FB) {
        const uint32_t e = h.fast[br.peek(FB)];
        if (e) { const uint32_t l = e >> 9; if (l > br.cnt) return -2; br.drop(l); return (int)(e & 511); }
    }
    int code = 0, first = 0, index = 0;
    uint64_t b = br.buf;
    for (int l = 1; l < 16; l++) {
        if ((uint32_t)l > br.cnt) return -2;
        code |= (int)(b & 1); b >>= 1;
        const int count = h.count[l];
        if (code - count < first) { br.drop((uint32_t)l); return h.sym[index + (code - first)]; }
        index += count; first += count; first <<= 1; code <<= 1;
    }
    return -1;
}

HT2_HD bool ht2z_complete(const uint16_t* count)
{
    int left = 1;
    for (int l = 1; l < 16; l++) { left <<= 1; left -= count[l]; if (left < 0) return false; }
    return left == 0;
}

// The header of a dynamic block, after BTYPE.  With lens, the code lengths go to lens[0..288) / lens[288..320) under
// zlib's rules; without (the block finder), only their counts are kept and every code must be complete (the distance
// code may also have one code or none), which is what zlib writes.  0 ok, -1 invalid, -2 input ends inside the header.
HT2_HD int ht2z_dynamic(Ht2zBits& br, uint8_t* lens)
{
    const Ht2zConst& K = ht2z_k();
    if (!br.have(14)) return -2;
    const int nlen = (int)br.get(5) + 257, ndist = (int)br.get(5) + 1, ncode = (int)br.get(4) + 4;
    if (nlen > 286 || ndist > 30) return -1;
    uint8_t cl[19];
    for (int i = 0; i < 19; i++) cl[i] = 0;
    if (!br.have((uint32_t)ncode * 3)) return -2;
    for (int i = 0; i < ncode; i++) cl[K.clOrder[i]] = (uint8_t)br.get(3);
    Ht2zHuff<19, 0> ch;
    if (!ht2z_build(ch, cl, 19, false)) return -1;
    uint16_t lc[16], dc[16];
    for (int i = 0; i < 16; i++) { lc[i] = 0; dc[i] = 0; }
    int n = 0, prev = -1, eob = 0;
    while (n < nlen + ndist) {
        const int s = ht2z_decode(br, ch);
        if (s < 0) return s;
        int rep = 1, v = s;
        if (s == 16) { if (prev < 0 || !br.have(2)) return prev < 0 ? -1 : -2; v = prev; rep = 3 + (int)br.get(2); }
        else if (s == 17) { if (!br.have(3)) return -2; v = 0; rep = 3 + (int)br.get(3); }
        else if (s == 18) { if (!br.have(7)) return -2; v = 0; rep = 11 + (int)br.get(7); }
        if (n + rep > nlen + ndist) return -1;
        for (int r = 0; r < rep; r++, n++) {
            if (n < nlen) { lc[v]++; if (n == 256) eob = v; if (lens) lens[n] = (uint8_t)v; }
            else { dc[v]++; if (lens) lens[288 + n - nlen] = (uint8_t)v; }
        }
        prev = v;
    }
    if (!eob) return -1;
    if (lens) {
        for (int i = nlen; i < 288; i++) lens[i] = 0;
        for (int i = ndist; i < 32; i++) lens[288 + i] = 0;
        return 0;
    }
    return ht2z_complete(lc) && (ht2z_complete(dc) || (uint32_t)(ndist - dc[0]) <= 1) ? 0 : -1;
}

HT2_HD void ht2z_fixed(uint8_t* lens)
{
    for (int i = 0; i < 320; i++) lens[i] = (uint8_t)(i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : i < 288 ? 8 : 5);
}

// CRC-32 (reflected 0xedb88320), one table
HT2_HD uint32_t ht2z_crc_byte(uint32_t c) { for (int k = 0; k < 8; k++) c = c & 1 ? (c >> 1) ^ 0xedb88320u : c >> 1; return c; }
HT2_HD uint32_t ht2z_crc(uint32_t crc, const uint8_t* p, uint64_t n, const uint32_t* tab)
{
    crc = ~crc;
    for (uint64_t i = 0; i < n; i++) crc = tab[(crc ^ p[i]) & 0xff] ^ (crc >> 8);
    return ~crc;
}

// The header of a gzip member at byte 'at'.  1 ok (*endByte = the first byte of its DEFLATE data), 0 not a member
// header, -1 a member header that is malformed, -2 the input ends inside it.
HT2_HD int ht2z_member_header(const uint8_t* p, uint64_t base, uint64_t end, uint64_t at, uint64_t* endByte)
{
    if (at + 10 > end) return at + 3 <= end && (p[at - base] != 0x1f || p[at + 1 - base] != 0x8b || p[at + 2 - base] != 8) ? 0 : -2;
    const uint8_t* h = p + (at - base);
    if (h[0] != 0x1f || h[1] != 0x8b || h[2] != 8) return 0;
    const uint32_t flg = h[3];
    if (flg & 0xe0) return -1;
    uint64_t q = at + 10;
    if (flg & 4) {
        if (q + 2 > end) return -2;
        q += 2 + (p[q - base] | (uint32_t)p[q + 1 - base] << 8);
        if (q > end) return -2;
    }
    for (uint32_t f = 8; f <= 16; f <<= 1) if (flg & f) {
        while (q < end && p[q - base]) q++;
        if (q >= end) return -2;
        q++;
    }
    if (flg & 2) {
        if (q + 2 > end) return -2;
        uint32_t c = 0xffffffffu;
        for (uint64_t i = at; i < q; i++) c = ht2z_crc_byte((c ^ p[i - base]) & 0xff) ^ (c >> 8);
        if ((~c & 0xffff) != (p[q - base] | (uint32_t)p[q + 1 - base] << 8)) return -1;
        q += 2;
    }
    *endByte = q;
    return 1;
}

// ---------------------------------------------------------------------------------------------------------------------
// 1. find: is there a block or member start at 'bit'?  Returns its kind.  The previous chunk stops at the first
//    boundary at or past ht2z_cand_key: a stored header starts 3 to 10 bits before its LEN
// ---------------------------------------------------------------------------------------------------------------------
HT2_HD uint32_t ht2z_candidate(const uint8_t* p, uint64_t base, uint64_t end, uint64_t bit)
{
    if ((bit & 7) == 0) {
        const uint64_t b = bit >> 3;
        if (b + 3 <= end && p[b - base] == 0x1f && p[b + 1 - base] == 0x8b && p[b + 2 - base] == 8 &&
            (b + 4 > end || !(p[b + 3 - base] & 0xe0)))
            return HT2Z_K_MEMBER;
        if (b > base && b + 4 <= end && !(p[b - 1 - base] & 0xe0)) {
            const uint32_t len = p[b - base] | (uint32_t)p[b + 1 - base] << 8, nlen = p[b + 2 - base] | (uint32_t)p[b + 3 - base] << 8;
            if (len == (~nlen & 0xffff)) return HT2Z_K_STORED;
        }
    }
    Ht2zBits br;
    br.init(p, base, end, bit);
    if (!br.have(3) || br.get(3) != 4) return HT2Z_K_NONE;   // BFINAL 0, BTYPE 2
    return ht2z_dynamic(br, NULL) == 0 ? HT2Z_K_BLOCK : HT2Z_K_NONE;
}
HT2_HD uint64_t ht2z_cand_key(uint64_t bit, uint32_t kind) { return kind == HT2Z_K_STORED ? bit - 10 : bit; }

// Set a chunk up to start decoding at a candidate (kind, bit) found by the block finder.
HT2_HD void ht2z_chunk_at(Ht2zChunk& c, uint32_t kind, uint64_t bit, const uint8_t* p, uint64_t base, uint64_t end)
{
    c.kind = kind; c.cand = bit; c.nout = 0; c.nev = 0; c.nblk = 0; c.base = -(int32_t)HT2Z_WSIZE; c.lastStart = -1;
    c.st.bit = bit; c.st.last = 0; c.st.stored = 0;
    c.st.phase = kind == HT2Z_K_MEMBER ? HT2Z_PH_MEMBER : HT2Z_PH_BLOCK;
    if (kind == HT2Z_K_STORED) {
        const uint64_t b = bit >> 3;
        c.st.phase = HT2Z_PH_STORED; c.st.stored = p[b - base] | (uint32_t)p[b + 1 - base] << 8; c.st.bit = (b + 4) * 8;
        c.nblk = 1;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// 2. decode: run chunk c from c.st, appending to out[c.nout .. c.cap), until the first boundary at or past c.stopBit,
//    the end of the input, a full output or trailer list, or an error (c.status)
// ---------------------------------------------------------------------------------------------------------------------
struct Ht2zTables { Ht2zHuff<288, HT2Z_LFAST> lit; Ht2zHuff<32, HT2Z_DFAST> dist; };

HT2_NI void ht2z_run(Ht2zChunk& c, const uint8_t* p, uint64_t base, uint64_t end, bool srcFinal, uint16_t* out, Ht2zTables& T)
{
    const uint32_t cap = c.cap;
    const Ht2zConst& K = ht2z_k();
    Ht2zBits br;
    br.init(p, base, end, c.st.bit);
    uint32_t phase = c.st.phase, last = c.st.last, stored = c.st.stored, n = c.nout, nblk = c.nblk;
    int32_t mbase = c.base;
    const uint64_t stop = c.stopBit;
    uint32_t status = HT2Z_STOP;
    if (phase == HT2Z_PH_HUFF &&
        (!ht2z_build(T.lit, c.st.lens, 288, true) || !ht2z_build(T.dist, c.st.lens + 288, 32, true))) { status = HT2Z_E_CODES; goto done; }
    for (;;) {
        if (phase == HT2Z_PH_MEMBER || phase == HT2Z_PH_BLOCK) {
            if (br.pos() >= stop) { status = HT2Z_STOP; break; }
        }
        if (phase == HT2Z_PH_MEMBER) {
            const uint64_t at = br.pos() >> 3;
            if (at >= end) { status = srcFinal ? HT2Z_END : HT2Z_NEED_INPUT; break; }
            if (p[at - base] == 0) { status = HT2Z_PAD; break; }
            uint64_t q = 0;
            const int r = ht2z_member_header(p, base, end, at, &q);
            if (r == -2) { status = HT2Z_NEED_INPUT; break; }
            if (r == 0) { status = HT2Z_E_GARBAGE; break; }
            if (r < 0) { status = HT2Z_E_HEADER; break; }
            br.init(p, base, end, q * 8);
            mbase = (int32_t)n; c.lastStart = (int32_t)n;
            phase = HT2Z_PH_BLOCK;
        } else if (phase == HT2Z_PH_BLOCK) {
            const uint64_t at = br.pos();
            if (!br.have(3)) { status = HT2Z_NEED_INPUT; break; }
            last = br.get(1);
            const uint32_t type = br.get(2);
            if (type == 0) {
                br.align();
                if (!br.have(32)) { br.init(p, base, end, at); status = HT2Z_NEED_INPUT; break; }
                stored = br.get(16);
                if (stored != (~br.get(16) & 0xffff)) { status = HT2Z_E_STORED; break; }
                phase = HT2Z_PH_STORED;
            } else if (type == 1) {
                ht2z_fixed(c.st.lens);
                ht2z_build(T.lit, c.st.lens, 288, true); ht2z_build(T.dist, c.st.lens + 288, 32, true);
                phase = HT2Z_PH_HUFF;
            } else if (type == 2) {
                const int r = ht2z_dynamic(br, c.st.lens);
                if (r == -2) { br.init(p, base, end, at); status = HT2Z_NEED_INPUT; break; }
                if (r < 0 || !ht2z_build(T.lit, c.st.lens, 288, true) || !ht2z_build(T.dist, c.st.lens + 288, 32, true)) {
                    status = HT2Z_E_CODES; break;
                }
                phase = HT2Z_PH_HUFF;
            } else { status = HT2Z_E_BTYPE; break; }
            nblk++;
        } else if (phase == HT2Z_PH_STORED) {
            while (stored) {
                if (n == cap) { status = HT2Z_OUT_FULL; goto done; }
                if (!br.have(8)) { status = HT2Z_NEED_INPUT; goto done; }
                out[n++] = (uint16_t)br.get(8); stored--;
            }
            phase = last ? HT2Z_PH_TRAILER : HT2Z_PH_BLOCK;
        } else if (phase == HT2Z_PH_TRAILER) {
            if (c.nev == HT2Z_EV) { status = HT2Z_EV_FULL; break; }
            const uint64_t at = br.pos();
            br.align();
            if (!br.have(32)) { br.init(p, base, end, at); status = HT2Z_NEED_INPUT; break; }
            Ht2zEvent& e = c.ev[c.nev];
            e.crc = br.get(32);
            if (!br.have(32)) { br.init(p, base, end, at); status = HT2Z_NEED_INPUT; break; }
            e.isize = br.get(32); e.pos = n; e.pad = 0;
            c.nev++;
            phase = HT2Z_PH_MEMBER;
        } else {   // PH_HUFF
            for (;;) {
                const uint64_t at = br.pos();
                const int s = ht2z_decode(br, T.lit);
                if (s < 0) { if (s == -2) { br.init(p, base, end, at); status = HT2Z_NEED_INPUT; } else status = HT2Z_E_SYMBOL; goto done; }
                if (s < 256) {
                    if (n == cap) { br.init(p, base, end, at); status = HT2Z_OUT_FULL; goto done; }
                    out[n++] = (uint16_t)s;
                    continue;
                }
                if (s == 256) break;
                if (s > 285) { status = HT2Z_E_SYMBOL; goto done; }
                const uint32_t le = K.lext[s - 257];
                if (!br.have(le)) { br.init(p, base, end, at); status = HT2Z_NEED_INPUT; goto done; }
                const uint32_t len = K.lbase[s - 257] + br.get(le);
                const int d = ht2z_decode(br, T.dist);
                if (d < 0) { if (d == -2) { br.init(p, base, end, at); status = HT2Z_NEED_INPUT; } else status = HT2Z_E_SYMBOL; goto done; }
                if (d > 29) { status = HT2Z_E_DIST; goto done; }
                const uint32_t de = K.dext[d];
                if (!br.have(de)) { br.init(p, base, end, at); status = HT2Z_NEED_INPUT; goto done; }
                const uint32_t dist = K.dbase[d] + br.get(de);
                if ((int64_t)dist > (int64_t)n - mbase) { status = HT2Z_E_DIST; goto done; }
                if (len > cap - n) { br.init(p, base, end, at); status = HT2Z_OUT_FULL; goto done; }
                if (dist > n && dist >= len) {   // (part of) the source lies before the chunk: markers
                    for (uint32_t i = 0; i < len; i++, n++) {
                        const int64_t q = (int64_t)n - dist;
                        out[n] = q < 0 ? (uint16_t)(256 + HT2Z_WSIZE + q) : out[q];
                    }
                    continue;
                }
                if (dist >= len) {   // no overlap: eight independent loads before their stores
                    const uint16_t* q = out + (n - dist);
                    uint16_t* o = out + n;
                    uint32_t i = 0;
                    for (; i + 8 <= len; i += 8) {
                        uint16_t v[8];
                        for (int k = 0; k < 8; k++) v[k] = q[i + k];
                        for (int k = 0; k < 8; k++) o[i + k] = v[k];
                    }
                    for (; i < len; i++) o[i] = q[i];
                    n += len;
                } else if (dist <= n) {
                    for (uint32_t i = 0; i < len; i++, n++) out[n] = out[n - dist];
                } else {
                    for (uint32_t i = 0; i < len; i++, n++) {
                        const int64_t q = (int64_t)n - dist;
                        out[n] = q < 0 ? (uint16_t)(256 + HT2Z_WSIZE + q) : out[q];
                    }
                }
            }
            phase = last ? HT2Z_PH_TRAILER : HT2Z_PH_BLOCK;
        }
    }
done:
    c.st.bit = br.pos(); c.st.phase = phase; c.st.last = last; c.st.stored = stored;
    c.nout = n; c.nblk = nblk; c.base = mbase; c.status = status;
}

// ---------------------------------------------------------------------------------------------------------------------
// 4 / 5. markers: symbol s of a chunk whose preceding window is win (of which the last 'valid' bytes belong to the
// current member) -> its byte; *bad is set for a reference before the member's start
// ---------------------------------------------------------------------------------------------------------------------
HT2_HD uint8_t ht2z_sym(uint16_t s, const uint8_t* win, uint32_t valid, uint32_t* bad)
{
    if (s < 256) return (uint8_t)s;
    const uint32_t i = s - 256u;
    if (i < HT2Z_WSIZE - valid) { *bad = 1; return 0; }
    return win[i];
}
// byte i of the window after a chunk of n symbols
HT2_HD uint8_t ht2z_next_win(uint32_t i, const uint16_t* sym, uint32_t n, const uint8_t* win, uint32_t valid, uint32_t* bad)
{
    if (n >= HT2Z_WSIZE) return ht2z_sym(sym[n - HT2Z_WSIZE + i], win, valid, bad);
    return i < HT2Z_WSIZE - n ? win[i + n] : ht2z_sym(sym[i - (HT2Z_WSIZE - n)], win, valid, bad);
}

// ---------------------------------------------------------------------------------------------------------------------
// CRC-32 combination (GF(2) polynomial arithmetic modulo the CRC polynomial, reflected)
// ---------------------------------------------------------------------------------------------------------------------
inline uint32_t ht2z_multmodp(uint32_t a, uint32_t b)
{
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) { p ^= b; if ((a & (m - 1)) == 0) break; }
        m >>= 1;
        b = b & 1 ? (b >> 1) ^ 0xedb88320u : b >> 1;
    }
    return p;
}
// x^(8 n) modulo the polynomial
struct Ht2zPowers {                 // x^(2^k) modulo the polynomial
    uint32_t pw[64];
    Ht2zPowers() { pw[0] = 1u << 30; for (int k = 1; k < 64; k++) pw[k] = ht2z_multmodp(pw[k - 1], pw[k - 1]); }
};
inline uint32_t ht2z_x8n(uint64_t n)
{
    static const Ht2zPowers P;      // initialised once, thread-safely: mate files are inflated on concurrent threads
    uint32_t p = 1u << 31;
    int k = 3;
    while (n) { if (n & 1) p = ht2z_multmodp(P.pw[k & 63], p); n >>= 1; k++; }
    return p;
}
inline uint32_t ht2z_crc_combine(uint32_t crc1, uint32_t crc2, uint64_t len2)
{
    static const uint32_t piece = ht2z_x8n(HT2Z_PIECE);
    return ht2z_multmodp(len2 == HT2Z_PIECE ? piece : ht2z_x8n(len2), crc1) ^ crc2;
}
struct Ht2zPiece { uint64_t off; uint32_t len, pad; };   // a range of the window's output whose CRC-32 is computed

// ---------------------------------------------------------------------------------------------------------------------
// the driver, over a backend that holds the buffers and runs the phases (device: ht2_inflate.cu; host: below)
// ---------------------------------------------------------------------------------------------------------------------
struct Ht2zGeom {
    uint32_t maxChunks;             // chunks per window
    uint64_t symBudget;             // 16-bit symbols over all chunks of a window
    uint64_t maxWindowIn;           // compressed bytes per window
    uint64_t lookahead;             // compressed bytes past the window end the last chunk may read
};
static const Ht2zGeom HT2Z_GEOM = {512, (uint64_t)64 << 20, (uint64_t)32 << 20, (uint64_t)1 << 20};

inline const char* ht2z_status_msg(uint32_t s)
{
    switch (s) {
    case HT2Z_E_HEADER: return "invalid gzip member header";
    case HT2Z_E_BTYPE: return "invalid block type";
    case HT2Z_E_STORED: return "invalid stored block lengths";
    case HT2Z_E_CODES: return "invalid code lengths in a block header";
    case HT2Z_E_SYMBOL: return "invalid literal/length or distance code";
    case HT2Z_E_DIST: return "invalid distance too far back";
    case HT2Z_E_GARBAGE: return "trailing garbage after the last gzip member";
    default: return "corrupt gzip data";
    }
}

// Where the output goes.  grow makes room for 'need' bytes in all and returns the buffer (it may move it); landed
// says that bytes [0, len) are written (their members' CRC-32 is checked when each member ends) and returns false to
// stop the inflate.
struct Ht2zOut {
    virtual ~Ht2zOut() {}
    virtual char* grow(size_t need) = 0;
    virtual bool landed(size_t) { return true; }
};
// A malloc'ed buffer (ht2gpu_gunzip's *out), first sized from the last member's ISIZE -- the whole size of a
// single-member file under 4 GiB -- but to at most 16 times the input before anything is verified.
struct Ht2zMallocOut : Ht2zOut {
    char* p = NULL;
    size_t cap = 0, first = 0;
    Ht2zMallocOut(const uint8_t* src, size_t n)
    {
        const uint64_t hint = n < 18 ? 0 : src[n - 4] | (uint64_t)src[n - 3] << 8 | (uint64_t)src[n - 2] << 16 | (uint64_t)src[n - 1] << 24;
        first = hint > 16 * (uint64_t)n ? 16 * n : hint > 4 * (uint64_t)n ? (size_t)hint : 4 * n;
        if (first < 4096) first = 4096;
    }
    ~Ht2zMallocOut() { free(p); }
    char* grow(size_t need)
    {
        if (p && need <= cap) return p;
        size_t c = cap ? cap : first;
        while (c < need) c *= 2;
        char* q = (char*)realloc(p, c);
        if (!q) return NULL;
        p = q; cap = c;
        return p;
    }
    char* release() { char* q = p ? p : (char*)malloc(1); p = NULL; return q; }
};

// Per window the backend sees: setSrc (the compressed bytes [base, end)), find (candidates of chunks 1..n-1: the bit
// of the first start in [wb + k C, wb + (k+1) C), or HT2Z_NONE, and its kind), decode (run the listed chunks, chunk k
// writing from symbol k * slice; the chunk array is mirrored both ways), resolve (windows and bytes of the listed
// chunks, in order, and the CRC-32 of each piece; the bytes land at out; returns nonzero for a reference before a
// member's start), carry (the last resolved window becomes the first of the next window).
template <class B>
int ht2z_gunzip_to(B& be, const uint8_t* src, size_t n, uint32_t chunkBytes, Ht2zOut& O, size_t* outLen,
                   ht2gpu_gunzip_stats_t& S, std::string& err)
{
    const Ht2zGeom& G = HT2Z_GEOM;
    *outLen = 0;
    if (n < 2 || src[0] != 0x1f || src[1] != 0x8b) { err = "not in gzip format"; return HT2GPU_ERR_DATA; }
    size_t len = 0;
    auto fail = [&](const std::string& m) { err = m; return HT2GPU_ERR_DATA; };
    std::vector<Ht2zChunk> ch(G.maxChunks);
    std::vector<uint64_t> keys(G.maxChunks);
    std::vector<uint32_t> kinds(G.maxChunks);
    Ht2zState st; memset(&st, 0, sizeof(st));
    st.phase = HT2Z_PH_MEMBER;
    uint32_t valid = 0;             // bytes of the carried window inside the current member
    uint32_t crc = 0; uint64_t isize = 0;
    double ratio = 4.0;
    bool first = true;
    for (;;) {
        const uint64_t wb = st.bit >> 3;
        // expected output of C compressed bytes, with a margin: a chunk's slice of the symbol buffer must hold it
        const double grow = 1.5 * ratio;
        uint64_t C = chunkBytes < G.maxWindowIn ? chunkBytes : G.maxWindowIn;
        if (!C) {   // aim at chunks whose output fills two thirds of their share of the symbol buffer
            const double c = (double)(G.symBudget / G.maxChunks) / grow;
            C = c < 4096 ? 4096 : c > (1 << 20) ? (1 << 20) : ((uint64_t)c & ~(uint64_t)4095);
        }
        if ((double)C * grow > (double)G.symBudget) C = (uint64_t)((double)G.symBudget / grow) + 1;
        uint64_t nc = (n - wb + C - 1) / C;
        if (nc > G.maxChunks) nc = G.maxChunks;
        if (nc * C > G.maxWindowIn) nc = G.maxWindowIn / C;
        if ((double)nc * C * grow > (double)G.symBudget) nc = (uint64_t)((double)G.symBudget / ((double)C * grow));
        if (nc < 1) nc = 1;
        const uint64_t we = wb + nc * C < n ? wb + nc * C : n;
        const uint64_t srcEnd = we + G.lookahead < n ? we + G.lookahead : n;
        const bool final = srcEnd == n;
        const uint32_t slice = (uint32_t)(G.symBudget / nc);
        S.windows++; S.chunk_bytes = (uint32_t)C;
        be.setSrc(src + wb, wb, srcEnd);
        be.find(wb, C, (uint32_t)nc, we, keys.data(), kinds.data());
        // the list of chunks with a start: chunk 0 resumes the carried state
        std::vector<int> L;
        Ht2zChunk& c0 = ch[0];
        c0.st = st; c0.kind = first ? HT2Z_K_MEMBER : HT2Z_K_RESUME; c0.cand = st.bit; c0.nout = 0; c0.nev = 0; c0.nblk = 0;
        c0.base = -(int32_t)valid; c0.lastStart = -1;
        L.push_back(0);
        for (uint32_t k = 1; k < nc; k++)
            if (kinds[k] != HT2Z_K_NONE && keys[k] > st.bit) {
                ht2z_chunk_at(ch[k], kinds[k], keys[k], src + wb, wb, srcEnd);
                L.push_back((int)k);
            }
        for (size_t i = 0; i < L.size(); i++)
            ch[L[i]].stopBit = i + 1 < L.size() ? ht2z_cand_key(ch[L[i + 1]].cand, ch[L[i + 1]].kind) : (final && we == n ? HT2Z_NONE : we * 8);
        // a chunk B is confirmed when its predecessor A stopped exactly on B's start
        auto linked = [&](const Ht2zChunk& A, const Ht2zChunk& Bc) {
            if (A.status != HT2Z_STOP) return false;
            if (Bc.kind == HT2Z_K_STORED) {
                if (A.st.phase != HT2Z_PH_BLOCK || ((A.st.bit + 3 + 7) >> 3) != (Bc.cand >> 3)) return false;
                const uint64_t b = A.st.bit;   // the header there must be BFINAL 0, BTYPE 0
                uint32_t v = 0;
                for (int i = 0; i < 3; i++) v |= ((src[(b + i) >> 3] >> ((b + i) & 7)) & 1) << i;
                return v == 0;
            }
            return A.st.bit == Bc.cand && A.st.phase == (Bc.kind == HT2Z_K_MEMBER ? (uint32_t)HT2Z_PH_MEMBER : (uint32_t)HT2Z_PH_BLOCK);
        };
        // a chunk may fill its own slice of the symbol buffer and those of the chunks up to the next one in the list
        auto setCaps = [&]() { for (size_t i = 0; i < L.size(); i++) ch[L[i]].cap = ((i + 1 < L.size() ? (uint32_t)L[i + 1] : (uint32_t)nc) - (uint32_t)L[i]) * slice; };
        setCaps();
        std::vector<int> run = L;
        for (;;) {
            be.decode(ch.data(), (uint32_t)nc, run, slice, final);
            S.decode_rounds++;
            run.clear();
            // merge every chunk whose predecessor stopped past its (false) start into that predecessor
            for (size_t i = 0; i + 1 < L.size(); i++) {
                Ht2zChunk& A = ch[L[i]];
                if (A.status != HT2Z_STOP || linked(A, ch[L[i + 1]])) continue;
                A.stopBit = ch[L[i + 1]].stopBit;
                L.erase(L.begin() + (ptrdiff_t)i + 1);
                S.chunks_merged_false_positive++;
                run.push_back(L[i]);
            }
            if (run.empty()) break;
            setCaps();
        }
        size_t T = 0;
        while (T + 1 < L.size() && linked(ch[L[T]], ch[L[T + 1]])) T++;
        L.resize(T + 1);
        const Ht2zChunk& E = ch[L[T]];
        for (size_t i = 1; i < L.size(); i++) S.chunks_confirmed++;
        for (uint32_t k = 1; k < nc; k++)   // chunks without a start that the kept ones decoded into
            if (kinds[k] == HT2Z_K_NONE && (wb + k * C) * 8 < E.st.bit) S.chunks_merged_no_candidate++;
        S.chunks += L.size();
        if (E.status == HT2Z_OUT_FULL || E.status == HT2Z_EV_FULL) S.windows_cut++;
        if (E.status >= HT2Z_E_HEADER) return fail(ht2z_status_msg(E.status));
        if (E.status == HT2Z_NEED_INPUT && final) return fail("unexpected end of the compressed input");
        // output of the accepted chunks
        std::vector<uint64_t> off(L.size() + 1, 0);
        std::vector<uint32_t> vld(L.size() + 1);
        vld[0] = valid;
        for (size_t i = 0; i < L.size(); i++) {
            const Ht2zChunk& c = ch[L[i]];
            off[i + 1] = off[i] + c.nout;
            const uint64_t v = c.lastStart >= 0 ? (uint64_t)(c.nout - (uint32_t)c.lastStart) : (uint64_t)vld[i] + c.nout;
            vld[i + 1] = v > HT2Z_WSIZE ? HT2Z_WSIZE : (uint32_t)v;
            S.blocks += c.nblk; S.members += c.nev;
        }
        const uint64_t total = off[L.size()];
        char* out = O.grow(len + total);
        if (!out) return fail("out of host memory");
        // CRC-32 pieces: the output of each member inside each chunk, cut every HT2Z_PIECE bytes
        std::vector<Ht2zPiece> pcs;
        for (size_t i = 0; i < L.size(); i++) {
            const Ht2zChunk& c = ch[L[i]];
            uint32_t at = 0;
            for (uint32_t e = 0; e <= c.nev; e++) {
                const uint32_t to = e < c.nev ? c.ev[e].pos : c.nout;
                for (uint32_t a = at; a < to; a += HT2Z_PIECE) pcs.push_back({off[i] + a, to - a < HT2Z_PIECE ? to - a : HT2Z_PIECE, 0});
                at = to;
            }
        }
        std::vector<uint32_t> pcrc(pcs.size());
        if (be.resolve(ch.data(), L, off, vld, slice, out + len, pcs, pcrc.data())) return fail(ht2z_status_msg(HT2Z_E_DIST));
        size_t pi = 0;
        for (size_t i = 0; i < L.size(); i++) {
            const Ht2zChunk& c = ch[L[i]];
            uint32_t at = 0;
            for (uint32_t e = 0; e <= c.nev; e++) {
                const uint32_t to = e < c.nev ? c.ev[e].pos : c.nout;
                for (uint32_t a = at; a < to; a += HT2Z_PIECE, pi++) crc = ht2z_crc_combine(crc, pcrc[pi], pcs[pi].len);
                isize += to - at; at = to;
                if (e < c.nev) {
                    if (crc != c.ev[e].crc) return fail("crc error: a gzip member's CRC-32 does not match its data");
                    if ((uint32_t)isize != c.ev[e].isize) return fail("length error: a gzip member's ISIZE does not match its data");
                    crc = 0; isize = 0;
                }
            }
        }
        len += total;
        S.in_bytes = n; S.out_bytes = len;
        if (!O.landed(len)) return fail("stopped");
        be.carry((uint32_t)L.size());
        const uint64_t before = st.bit;
        st = E.st; valid = vld[L.size()];
        first = false;
        if (E.status == HT2Z_END) break;
        if (E.status == HT2Z_PAD) {
            for (uint64_t i = st.bit >> 3; i < n; i++) if (src[i]) return fail(ht2z_status_msg(HT2Z_E_GARBAGE));
            break;
        }
        if (st.bit == before && total == 0) return fail("a gzip header field is too long");
        const double r = (double)total / (double)((st.bit >> 3) - wb + 1);
        ratio = r > 1.0 ? r : 1.0;
    }
    if (S.members == 0) return fail("unexpected end of the compressed input");
    *outLen = len;
    return HT2GPU_OK;
}
// The same into a malloc'ed buffer (*outP, free with free()).
template <class B>
int ht2z_gunzip(B& be, const uint8_t* src, size_t n, uint32_t chunkBytes, char** outP, size_t* outLen,
                ht2gpu_gunzip_stats_t& S, std::string& err)
{
    *outP = NULL;
    Ht2zMallocOut O(src, n);
    const int rc = ht2z_gunzip_to(be, src, n, chunkBytes, O, outLen, S, err);
    if (rc == HT2GPU_OK) *outP = O.release();
    return rc;
}

// The host backend: the same phases as loops (tests, and the reference the device backend is compared against).
struct Ht2zHostBackend {
    const uint8_t* src = NULL;
    uint64_t base = 0, end = 0;
    std::vector<uint16_t> sym;
    std::vector<uint8_t> win, carryWin;
    uint32_t tab[256];
    Ht2zHostBackend() : carryWin(HT2Z_WSIZE, 0) { for (uint32_t i = 0; i < 256; i++) tab[i] = ht2z_crc_byte(i); }
    void setSrc(const uint8_t* p, uint64_t b, uint64_t e) { src = p; base = b; end = e; }
    void find(uint64_t wb, uint64_t C, uint32_t nc, uint64_t we, uint64_t* keys, uint32_t* kinds)
    {
        for (uint32_t k = 1; k < nc; k++) {
            keys[k] = HT2Z_NONE; kinds[k] = HT2Z_K_NONE;
            const uint64_t r1 = wb + (k + 1) * C < we ? wb + (k + 1) * C : we;
            for (uint64_t bit = (wb + k * C) * 8; bit < r1 * 8; bit++) {
                const uint32_t kind = ht2z_candidate(src, base, end, bit);
                if (kind) { keys[k] = bit; kinds[k] = kind; break; }
            }
        }
    }
    void decode(Ht2zChunk* ch, uint32_t nc, const std::vector<int>& ids, uint32_t slice, bool final)
    {
        if (sym.size() < (size_t)nc * slice) sym.resize((size_t)nc * slice);
        Ht2zTables* T = new Ht2zTables;
        for (int id : ids) ht2z_run(ch[id], src, base, end, final, sym.data() + (size_t)id * slice, *T);
        delete T;
    }
    int resolve(const Ht2zChunk* ch, const std::vector<int>& L, const std::vector<uint64_t>& off, const std::vector<uint32_t>& vld,
                uint32_t slice, char* out, const std::vector<Ht2zPiece>& pcs, uint32_t* pcrc)
    {
        const size_t m = L.size();
        win.assign((m + 1) * HT2Z_WSIZE, 0);
        memcpy(win.data(), carryWin.data(), HT2Z_WSIZE);
        uint32_t bad = 0;
        for (size_t i = 0; i < m; i++) {
            const uint16_t* s = sym.data() + (size_t)L[i] * slice;
            for (uint32_t j = 0; j < HT2Z_WSIZE; j++)
                win[(i + 1) * HT2Z_WSIZE + j] = ht2z_next_win(j, s, ch[L[i]].nout, win.data() + i * HT2Z_WSIZE, vld[i], &bad);
        }
        for (size_t i = 0; i < m; i++) {
            const Ht2zChunk& c = ch[L[i]];
            const uint16_t* s = sym.data() + (size_t)L[i] * slice;
            uint8_t* o = (uint8_t*)out + off[i];
            for (uint32_t j = 0; j < c.nout; j++) o[j] = ht2z_sym(s[j], win.data() + i * HT2Z_WSIZE, vld[i], &bad);
        }
        for (size_t k = 0; k < pcs.size(); k++) pcrc[k] = ht2z_crc(0, (const uint8_t*)out + pcs[k].off, pcs[k].len, tab);
        memcpy(carryWin.data(), win.data() + m * HT2Z_WSIZE, HT2Z_WSIZE);
        return (int)bad;
    }
    void carry(uint32_t) {}
};

#endif
