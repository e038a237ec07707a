// ht2_reads.cpp -- see ht2_reads.h.
#include "ht2_reads.h"

#include <fcntl.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

// ---------------------------------------------------------------------------
// thread pool
// ---------------------------------------------------------------------------
Ht2ThreadPool::Ht2ThreadPool(unsigned n) : n_(n < 1 ? 1 : n), fn_(NULL), gen_(0), pending_(0), stop_(false)
{
    for (unsigned t = 1; t < n_; t++) th_.emplace_back(&Ht2ThreadPool::worker, this, t);
}
Ht2ThreadPool::~Ht2ThreadPool()
{
    { std::lock_guard<std::mutex> lk(mu_); stop_ = true; }
    cvWork_.notify_all();
    for (auto& x : th_) x.join();
}
void Ht2ThreadPool::worker(unsigned t)
{
    uint64_t seen = 0;
    for (;;) {
        const std::function<void(unsigned)>* fn;
        {
            std::unique_lock<std::mutex> lk(mu_);
            cvWork_.wait(lk, [&] { return stop_ || gen_ != seen; });
            if (stop_) return;
            seen = gen_; fn = fn_;
        }
        (*fn)(t);
        { std::lock_guard<std::mutex> lk(mu_); if (--pending_ == 0) cvDone_.notify_all(); }
    }
}
void Ht2ThreadPool::run(const std::function<void(unsigned)>& fn)
{
    if (n_ == 1) { fn(0); return; }
    { std::lock_guard<std::mutex> lk(mu_); fn_ = &fn; pending_ = n_ - 1; gen_++; }
    cvWork_.notify_all();
    fn(0);
    std::unique_lock<std::mutex> lk(mu_);
    cvDone_.wait(lk, [&] { return pending_ == 0; });
}

// ---------------------------------------------------------------------------
// sources
// ---------------------------------------------------------------------------
bool ht2_source_open(Ht2ReadSource& s, const char* path, std::string& err)
{
    if (strcmp(path, "-") != 0) {
        int fd = open(path, O_RDONLY);
        if (fd < 0) { err = std::string("could not open reads file ") + path; return false; }
        struct stat st;
        if (fstat(fd, &st) == 0 && S_ISREG(st.st_mode)) {
            s.size = (size_t)st.st_size;
            if (s.size == 0) { close(fd); s.data = ""; return true; }
            void* m = mmap(NULL, s.size, PROT_READ, MAP_PRIVATE, fd, 0);
            close(fd);
            if (m == MAP_FAILED) { err = std::string("could not map reads file ") + path; return false; }
            madvise(m, s.size, MADV_SEQUENTIAL | MADV_WILLNEED);
            s.map = m; s.mapLen = s.size; s.data = (const char*)m;
            return true;
        }
        // pipes, character devices: read to the end
        char buf[1 << 16]; ssize_t k;
        while ((k = read(fd, buf, sizeof(buf))) > 0) s.own.insert(s.own.end(), buf, buf + k);
        close(fd);
    } else {
        char buf[1 << 16]; size_t k;
        while ((k = fread(buf, 1, sizeof(buf), stdin)) > 0) s.own.insert(s.own.end(), buf, buf + k);
    }
    s.data = s.own.data(); s.size = s.own.size();
    return true;
}
void ht2_source_memory(Ht2ReadSource& s, const char* data, size_t n) { s.data = data; s.size = n; }
void ht2_source_close(Ht2ReadSource& s)
{
    if (s.map) munmap(s.map, s.mapLen);
    s.map = NULL; s.stream = NULL; s.data = NULL; s.size = 0; s.own.clear(); s.rec.clear(); s.scanPos = 0; s.scanDone = false; s.lineCarry = 0; s.strictFastq = true;
}

// Scan the next block of the input for record starts (appended to s.rec).  Blocks are scanned by all threads; the
// pipeline calls this only as far ahead as the next batch needs, so that indexing overlaps the device work instead
// of preceding it.  When the end of the input is reached the sentinel (== size) is appended and scanDone is set.
// A source whose bytes are still arriving is scanned as far as they go, less one byte (so that the byte after each
// newline scanned is there to be looked at); the sentinel waits for the last byte.
bool ht2_source_scan(Ht2ReadSource& s, bool fastq, Ht2ThreadPool& pool, size_t blockBytes, std::string& err)
{
    if (s.scanDone) return true;
    bool more = false;
    if (s.stream) {
        Ht2SourceStream& q = *s.stream;
        std::unique_lock<std::mutex> lk(q.mu);
        q.cv.wait(lk, [&] { return q.done || q.avail > s.scanPos + 1; });
        if (q.rc) { err = q.err; return false; }
        if (!q.done && fastq && !s.strictFastq) q.cv.wait(lk, [&] { return q.done; });   // the sequential scan below reads to the end
        if (q.rc) { err = q.err; return false; }
        s.size = q.avail; more = !q.done;
    }
    const char* d = s.data; const size_t n = s.size;
    const size_t lim = more ? n - 1 : n;
    const size_t b0 = s.scanPos, b1 = (blockBytes == 0 || lim - b0 <= blockBytes) ? lim : b0 + blockBytes;
    const size_t len = b1 - b0;
    const unsigned T = (len < (1u << 20)) ? 1 : pool.size();
    std::vector<std::vector<uint64_t> > part(T);
    auto chunk = [&](unsigned t, size_t& c0, size_t& c1) { c0 = b0 + len / T * t; c1 = (t + 1 == T) ? b1 : b0 + len / T * (t + 1); };
    auto finish = [&]() { s.scanPos = b1; if (b1 == n && !more) { s.rec.push_back(n); s.scanDone = true; } return true; };
    if (!fastq) {
        // a record starts at a '>' that begins a line
        auto scan = [&](unsigned t) {
            if (t >= T) return;
            size_t c0, c1; chunk(t, c0, c1);
            std::vector<uint64_t>& v = part[t];
            const char* p = d + c0; const char* e = d + c1;
            while (p < e) {
                const char* q = (const char*)memchr(p, '>', (size_t)(e - p));
                if (!q) break;
                if (q == d || q[-1] == '\n' || q[-1] == '\r') v.push_back((uint64_t)(q - d));
                p = q + 1;
            }
        };
        if (T == 1) scan(0); else pool.run(scan);
        const bool hadNone = s.rec.empty();
        for (auto& v : part) s.rec.insert(s.rec.end(), v.begin(), v.end());
        if (hadNone && (!s.rec.empty() || (b1 == n && !more))) {
            // what precedes the first record may only be blank or comment lines (pat.cpp:741-756)
            size_t p = 0; const size_t first = s.rec.empty() ? n : (size_t)s.rec[0];
            while (p < first) {
                if (d[p] == '#' || d[p] == ';') { while (p < first && d[p] != '\n') p++; }
                else if (d[p] == '\n' || d[p] == '\r') p++;
                else { err = "reads file does not look like a FASTA file"; return false; }
            }
        }
        return finish();
    }
    if (s.strictFastq) {
        // strict 4-line records start at lines 0, 4, 8, ...: count newlines per chunk, then emit and verify
        std::vector<uint64_t> nl(T + 1, 0);
        auto count = [&](unsigned t) {
            if (t >= T) return;
            size_t c0, c1; chunk(t, c0, c1);
            uint64_t k = 0;
            const char* p = d + c0; const char* e = d + c1;
            while (p < e) { const char* q = (const char*)memchr(p, '\n', (size_t)(e - p)); if (!q) break; k++; p = q + 1; }
            nl[t + 1] = k;
        };
        if (T == 1) count(0); else pool.run(count);
        nl[0] = s.lineCarry;
        for (unsigned t = 0; t < T; t++) nl[t + 1] += nl[t];
        std::vector<uint8_t> bad(T, 0);
        auto emit = [&](unsigned t) {
            if (t >= T) return;
            size_t c0, c1; chunk(t, c0, c1);
            std::vector<uint64_t>& v = part[t];
            uint64_t line = nl[t];          // the line that starts after the next newline at or after c0 has index line + 1
            const char* p = d + c0; const char* e = d + c1;
            if (c0 == 0) { if (n > 0) { if (d[0] == '@') v.push_back(0); else bad[t] = 1; } }
            while (p < e) {
                const char* q = (const char*)memchr(p, '\n', (size_t)(e - p));
                if (!q) break;
                line++;
                const size_t st = (size_t)(q - d) + 1;
                if ((line & 3) == 0 && st < n) {
                    if (d[st] == '@') v.push_back(st);
                    else {   // trailing blank lines are fine, anything else is not strict 4-line FASTQ
                        size_t z = st; while (z < n && (d[z] == '\n' || d[z] == '\r')) z++;
                        if (z < n) bad[t] = 1;
                    }
                }
                p = q + 1;
            }
        };
        if (T == 1) emit(0); else pool.run(emit);
        bool ok = true;
        for (unsigned t = 0; t < T; t++) if (bad[t]) ok = false;
        if (ok) {
            for (auto& v : part) s.rec.insert(s.rec.end(), v.begin(), v.end());
            s.lineCarry = nl[T];
            return finish();
        }
        s.strictFastq = false;   // blank lines between records: fall through to the sequential scan of the rest
        if (more) return ht2_source_scan(s, fastq, pool, blockBytes, err);   // once all the bytes are there
    }
    {
        // blank lines between records (FastqPatternSource skips them): one sequential pass over the rest, from the
        // end of the last complete record
        size_t p = s.rec.empty() ? 0 : (size_t)s.rec.back();
        auto skipLine = [&]() { while (p < n && d[p] != '\n') p++; if (p < n) p++; };
        if (!s.rec.empty()) { skipLine(); skipLine(); skipLine(); skipLine(); }
        while (p < n) {
            while (p < n && (d[p] == '\n' || d[p] == '\r')) p++;
            if (p >= n) break;
            if (d[p] != '@') { err = "reads file does not look like a FASTQ file"; return false; }
            s.rec.push_back(p);
            skipLine(); skipLine(); skipLine(); skipLine();
        }
        s.scanPos = n; s.rec.push_back(n); s.scanDone = true;
        return true;
    }
}

bool ht2_source_index(Ht2ReadSource& s, bool fastq, Ht2ThreadPool& pool, std::string& err)
{
    s.rec.clear(); s.scanPos = 0; s.scanDone = false; s.lineCarry = 0; s.strictFastq = true;
    while (!s.scanDone) if (!ht2_source_scan(s, fastq, pool, 0, err)) return false;
    return true;
}

// ---------------------------------------------------------------------------
// batches
// ---------------------------------------------------------------------------
void Ht2HostBatch::freeAll()
{
    void* ps[6] = {seq, qual, offs, seeds, names, nameOffs};
    for (void* q : ps) if (q) { if (release) release(q); else free(q); }
    seq = qual = NULL; offs = NULL; seeds = NULL; names = NULL; nameOffs = NULL; capBases = capReads = capNames = 0;
}

namespace {

// solexaToPhred (qual.h:46-50): Solexa -10 .. 255 to Phred, round(10 log10(10^(sol/10) + 1)); below -10 is 0
struct SolexaTable {
    uint8_t phred[266];
    SolexaTable() { for (int s = -10; s <= 255; s++) phred[s + 10] = (uint8_t)(10.0 * log10(pow(10.0, s / 10.0) + 1.0) + 0.5); }
    int operator()(int sol) const { return sol < -10 ? 0 : phred[(sol > 255 ? 255 : sol) + 10]; }
};
static const SolexaTable kSolexa;

struct Tables {
    uint8_t isBase[256];   // FASTA: asc2dnacat > 0 (alphabet.cpp)
    uint8_t isAlpha[256];  // FASTQ: letters, and '.' which reads as N (pat.cpp:1030-1290)
    uint8_t code[256];     // asc2dna; '.' -> 4
    Tables() {
        memset(isBase, 0, sizeof(isBase)); memset(isAlpha, 0, sizeof(isAlpha)); memset(code, 0, sizeof(code));
        for (const char* c = "ACGTacgtBDHKMNRSVWXYbdhkmnrsvwxy-"; *c; c++) isBase[(uint8_t)*c] = 1;
        for (int c = 'a'; c <= 'z'; c++) { isAlpha[c] = 1; isAlpha[c - 32] = 1; }
        isAlpha[(uint8_t)'.'] = 1;
        code[(uint8_t)'C'] = code[(uint8_t)'c'] = 1; code[(uint8_t)'G'] = code[(uint8_t)'g'] = 2;
        code[(uint8_t)'T'] = code[(uint8_t)'t'] = 3; code[(uint8_t)'N'] = code[(uint8_t)'n'] = 4; code[(uint8_t)'.'] = 4;
    }
};
const Tables TB;

struct RawBuf {   // grow-only byte buffer written through raw pointers (no per-byte capacity checks, no zero fill)
    uint8_t* p; size_t n, cap;
    RawBuf() : p(NULL), n(0), cap(0) {}
    ~RawBuf() { free(p); }
    RawBuf(const RawBuf&) = delete;
    RawBuf& operator=(const RawBuf&) = delete;
    RawBuf(RawBuf&& o) : p(o.p), n(o.n), cap(o.cap) { o.p = NULL; o.n = o.cap = 0; }
    void need(size_t extra) {
        if (n + extra <= cap) return;
        size_t c = (n + extra) * 3 / 2 + 4096;
        p = (uint8_t*)realloc(p, c); cap = c;
    }
};

struct Local {   // one thread's share of a batch
    RawBuf seq, qual, names;
    std::vector<uint32_t> len, nameLen, seed;
    std::string err;
    void clear() { seq.n = qual.n = names.n = 0; len.clear(); nameLen.clear(); seed.clear(); err.clear(); }
};

// genRandSeed (pat.h:55-91)
inline uint32_t genSeed(const uint8_t* sq, const uint8_t* ql, uint32_t n, const char* name, size_t nameLen, uint32_t seed)
{
    uint32_t rseed = (seed + 101) * 59 * 61 * 67 * 71 * 73 * 79 * 83;
    for (uint32_t i = 0; i < n; i++) rseed ^= ((uint32_t)sq[i] << ((i & 15) << 1));
    if (ql) for (uint32_t i = 0; i < n; i++) rseed ^= ((uint32_t)ql[i] << ((i & 3) << 3));
    else {   // FASTA: every quality is 'I'; byte lane k of the word collects one 'I' per i with i % 4 == k
        for (uint32_t k = 0; k < 4; k++) if (((n + 3 - k) >> 2) & 1u) rseed ^= ((uint32_t)'I' << (k << 3));
    }
    for (size_t i = 0; i < nameLen; i++) {
        const int p = (int)name[i];
        if (p == '/') break;
        rseed ^= ((uint32_t)p << ((i & 3) << 3));
    }
    return rseed;
}

// Parse record r of 'src' and append it to L.  mate: 0 unpaired, 1 / 2 = fix the mate name.  rdid is the read's
// ordinal in its stream (the files of one kind back to back), the default name of an unnamed read.
bool parseRecord(const Ht2ReadSource& src, uint64_t r, uint64_t rdid, int mate, const Ht2ReadsOpts& o, Local& L)
{
    const char* d = src.data;
    size_t p = (size_t)src.rec[r]; const size_t e = (size_t)src.rec[r + 1];
    const size_t span = e - p;
    L.seq.need(span + 8); L.names.need(span + 32);
    if (o.fastq) L.qual.need(span + 8);
    uint8_t* sq = L.seq.p + L.seq.n;
    char* nm = (char*)L.names.p + L.names.n;
    size_t nl = 0;
    p++;   // '>' or '@'
    {   // the name: up to the end of the line
        const char* q = (const char*)memchr(d + p, '\n', e - p);
        size_t le = q ? (size_t)(q - d) : e;
        size_t ne = le;
        const char* cr = (const char*)memchr(d + p, '\r', le - p);
        if (cr) ne = (size_t)(cr - d);
        nl = ne - p;
        memcpy(nm, d + p, nl);
        p = le;
    }
    size_t n = 0;
    if (!o.fastq) {
        for (; p < e; p++) { const uint8_t c = (uint8_t)d[p]; sq[n] = TB.code[c]; n += TB.isBase[c]; }
        if (o.trim5 > 0) { const size_t t5 = (size_t)o.trim5 < n ? (size_t)o.trim5 : n; memmove(sq, sq + t5, n - t5); n -= t5; }
        n -= (size_t)o.trim3 < n ? (size_t)o.trim3 : n;
    } else {
        if (p < e) p++;   // the newline that ends the name line
        for (; p < e && d[p] != '\n'; p++) { const uint8_t c = (uint8_t)d[p]; sq[n] = TB.code[c]; n += TB.isAlpha[c]; }
        if (p < e) p++;
        if (p >= e || d[p] != '+') { L.err = "reads file does not look like a FASTQ file"; return false; }
        { const char* q = (const char*)memchr(d + p, '\n', e - p); p = q ? (size_t)(q - d) + 1 : e; }
        const size_t t5 = (size_t)o.trim5 < n ? (size_t)o.trim5 : n;
        if (t5) { memmove(sq, sq + t5, n - t5); n -= t5; }
        const size_t t3 = (size_t)o.trim3 < n ? (size_t)o.trim3 : n;
        n -= t3;
        // qualities: the line's characters (minus '\r'), trimmed like the bases, converted to Phred+33
        uint8_t* ql = L.qual.p + L.qual.n;
        size_t qn = 0;
        if (o.intQuals) {   // pat.cpp:997-1030: tokenize(line, " ") keeps a leading empty token (atoi gives 0)
            const size_t l0 = p; while (p < e && d[p] != '\n') p++;
            size_t l1 = p; while (l1 > l0 && d[l1 - 1] == '\r') l1--;
            size_t nTok = 0;
            for (size_t k = l0; l1 > l0;) {   // an empty line has no tokens
                size_t k1 = k; while (k1 < l1 && d[k1] != ' ') k1++;
                if (k1 > k || k == l0) {
                    char tok[32]; size_t tl = 0;
                    for (size_t j = k; j < k1 && tl < sizeof(tok) - 1; j++) tok[tl++] = d[j];
                    tok[tl] = '\0';
                    const int v = atoi(tok);   // intToPhred33 (qual.h:143-165); Solexa values above 255 read as 255
                    const int pq = o.solexa ? kSolexa(v) + 33 : (v <= 93 ? v : 93) + 33;
                    if (pq < 33) { L.err = "negative Phred quality " + std::to_string(pq - 33) + " in read " + std::string(nm, nl); return false; }
                    if (nTok++ >= (size_t)o.trim5) ql[qn++] = (uint8_t)(pq <= 126 ? pq : 126);
                }
                if (k1 >= l1) break;
                k = k1 + 1;
            }
            qn -= (size_t)o.trim3 < qn ? (size_t)o.trim3 : qn;   // trimEnd(gTrim3); one value more than bases is cut
            if (qn < n || qn > n + 1) {
                L.err = std::string(qn < n ? "fewer" : "more") + " quality values than bases for read " + std::string(nm, nl);
                return false;
            }
        } else {
            for (; p < e && d[p] != '\n'; p++) { const uint8_t c = (uint8_t)d[p]; ql[qn] = c; qn += (c != '\r'); }
            const size_t qkeep = qn > (size_t)o.trim5 + t3 ? qn - (size_t)o.trim5 - t3 : 0;
            if (qkeep != n) {
                L.err = std::string(qkeep < n ? "fewer" : "more") + " quality values than bases for read " + std::string(nm, nl);
                return false;
            }
            if (o.trim5 > 0) memmove(ql, ql + o.trim5, n);
        }
        if (o.solexa && !o.intQuals) {   // charToPhred33 (qual.h:106-141): the character is a signed char
            for (size_t i = 0; i < n; i++) {
                if (ql[i] == ' ') { L.err = "space in the quality values of read " + std::string(nm, nl) + "; integer qualities need --int-quals"; return false; }
                ql[i] = (uint8_t)(kSolexa((int)(int8_t)ql[i] - 64) + 33);
            }
        } else if (o.phred64 && !o.intQuals) {
            for (size_t i = 0; i < n; i++) { if (ql[i] < 64) { L.err = "quality value below Phred+64 range in read " + std::string(nm, nl); return false; } ql[i] = (uint8_t)(ql[i] - 31); }
        }
        uint8_t lo = 255;
        for (size_t i = 0; i < n; i++) lo = ql[i] < lo ? ql[i] : lo;
        if (n && lo < 33) { L.err = "quality value below Phred+33 range in read " + std::string(nm, nl); return false; }
        L.qual.n += n;
    }
    if (nl == 0) nl = (size_t)snprintf(nm, 24, "%llu", (unsigned long long)rdid);   // unnamed read: the read ordinal
    if (mate) {   // Read::fixMateName (read.h:171-196)
        const char want = mate == 1 ? '1' : '2';
        if (nl < 2 || nm[nl - 2] != '/' || nm[nl - 1] != want) { nm[nl++] = '/'; nm[nl++] = want; }
    }
    L.seed.push_back(genSeed(sq, o.fastq ? L.qual.p + (L.qual.n - n) : NULL, (uint32_t)n, nm, nl, o.seed));
    nm[nl] = '\0';
    L.seq.n += n; L.names.n += nl + 1;
    L.len.push_back((uint32_t)n);
    L.nameLen.push_back((uint32_t)nl + 1);
    return true;
}

template <typename T> bool ensure(Ht2HostBatch& b, T*& p, size_t count)
{
    void* q = b.alloc ? b.alloc(count * sizeof(T)) : malloc(count * sizeof(T));
    if (!q) return false;
    if (p) { if (b.release) b.release(p); else free(p); }
    p = (T*)q;
    return true;
}

} // namespace

Ht2ParseScratch::Ht2ParseScratch() : impl(new std::vector<Local>()) {}
Ht2ParseScratch::~Ht2ParseScratch() { delete (std::vector<Local>*)impl; }

bool ht2_parse_batch(const Ht2ReadSource& a, const Ht2ReadSource* b, uint64_t r0, uint64_t r1, const Ht2ReadsOpts& o,
                     Ht2HostBatch& out, Ht2ThreadPool& pool, Ht2ParseScratch& scratch, std::string& err)
{
    const Ht2BatchPiece pc = {&a, b, r0, r0, r1 - r0, r0};
    return ht2_parse_pieces(&pc, 1, o, out, pool, scratch, err);
}

bool ht2_parse_pieces(const Ht2BatchPiece* pcs, size_t npc, const Ht2ReadsOpts& o, Ht2HostBatch& out, Ht2ThreadPool& pool,
                      Ht2ParseScratch& scratch, std::string& err)
{
    uint64_t nrec = 0;
    for (size_t k = 0; k < npc; k++) nrec += pcs[k].n;
    const unsigned T = nrec < 2048 ? 1 : pool.size();
    std::vector<Local>& loc = *(std::vector<Local>*)scratch.impl;
    if (loc.size() < T) loc.resize(T);
    auto parse = [&](unsigned t) {
        if (t >= T) return;
        Local& L = loc[t];
        L.clear();
        uint64_t q0 = nrec * t / T, q1 = nrec * (t + 1) / T;   // units of the batch, over the pieces in order
        for (size_t k = 0, at = 0; k < npc && q0 < q1; at += pcs[k].n, k++) {
            const Ht2BatchPiece& pc = pcs[k];
            if (q0 >= at + pc.n) continue;
            const uint64_t e = q1 < at + pc.n ? q1 : at + pc.n;
            for (uint64_t u = q0 - at; u < e - at; u++) {
                if (!parseRecord(*pc.a, pc.ra + u, pc.rdid + u, pc.b ? 1 : 0, o, L)) return;
                if (pc.b && !parseRecord(*pc.b, pc.rb + u, pc.rdid + u, 2, o, L)) return;
            }
            q0 = e;
        }
    };
    if (T == 1) parse(0); else pool.run(parse);
    std::vector<uint64_t> baseAt(T + 1, 0), readAt(T + 1, 0), nameAt(T + 1, 0);
    for (unsigned t = 0; t < T; t++) {
        if (!loc[t].err.empty()) { err = loc[t].err; return false; }
        baseAt[t + 1] = baseAt[t] + loc[t].seq.n; readAt[t + 1] = readAt[t] + loc[t].len.size(); nameAt[t + 1] = nameAt[t] + loc[t].names.n;
    }
    const size_t nb = (size_t)baseAt[T], nr = (size_t)readAt[T], nn = (size_t)nameAt[T];
    if (nr > 0xfffffff0ull || nn > 0xfffffff0ull) { err = "batch too large"; return false; }
    if (nb + 16 > out.capBases || !out.seq) {
        const size_t cap = nb + nb / 8 + 4096;
        if (!ensure(out, out.seq, cap) || !ensure(out, out.qual, cap)) { err = "out of (pinned) host memory"; return false; }
        out.capBases = cap;
    }
    if (nr + 2 > out.capReads || !out.offs) {
        const size_t cap = nr + nr / 8 + 1024;
        if (!ensure(out, out.offs, cap) || !ensure(out, out.seeds, cap) || !ensure(out, out.nameOffs, cap)) { err = "out of (pinned) host memory"; return false; }
        out.capReads = cap;
    }
    if (nn + 16 > out.capNames || !out.names) {
        const size_t cap = nn + nn / 8 + 4096;
        if (!ensure(out, out.names, cap)) { err = "out of (pinned) host memory"; return false; }
        out.capNames = cap;
    }
    auto place = [&](unsigned t) {
        if (t >= T) return;
        const Local& L = loc[t];
        if (L.seq.n) memcpy(out.seq + baseAt[t], L.seq.p, L.seq.n);
        if (o.fastq && L.qual.n) memcpy(out.qual + baseAt[t], L.qual.p, L.qual.n);
        if (L.names.n) memcpy(out.names + nameAt[t], L.names.p, L.names.n);
        uint64_t bo = baseAt[t], no = nameAt[t];
        const size_t k0 = (size_t)readAt[t];
        for (size_t k = 0; k < L.len.size(); k++) {
            out.offs[k0 + k] = bo; out.nameOffs[k0 + k] = (uint32_t)no; out.seeds[k0 + k] = L.seed[k];
            bo += L.len[k]; no += L.nameLen[k];
        }
    };
    if (T == 1) place(0); else pool.run(place);
    out.offs[nr] = nb; out.nameOffs[nr] = (uint32_t)nn;
    out.n_reads = (uint32_t)nr; out.namesBytes = nn; out.haveQual = o.fastq;
    return true;
}
