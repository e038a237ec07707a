// ht2_pipeline.cpp -- reads in, SAM out: the overlapped host pipeline around the device path.
//
// Replaces the reference's worker loop as a whole (multiseedSearchWorker_hisat2, hisat2.cpp:3278-3696: every
// thread pulls one read under a lock, aligns it, formats it, hands the text to the OutputQueue, outq.cpp:51-99)
// with three overlapped stages over batches of reads:
//     parse batch i+1 (all host threads, ht2_reads.cpp)
//  || H2D -> align kernel -> SAM kernels -> D2H of batch i (ht2gpu_submit_sam / ht2gpu_wait_sam, one slot each)
//  || hand the SAM text of batch i-1 to the caller's sink, in read order (= --reorder)
// Host code only parses and moves bytes; selection, MAPQ and SAM formatting run on the device.
#include <stdio.h>
#include <string.h>

#include <chrono>
#include <functional>
#include <condition_variable>
#include <mutex>
#include <string>
#include <thread>

#include "../../include/ht2gpu.h"
#include "ht2_inflate.h"
#include "ht2_reads.h"

#include <sys/mman.h>
#include <atomic>
#include <memory>

bool ht2_same_sam_output(const ht2gpu_handle_t* a, const ht2gpu_handle_t* b);   // ht2_gpu.cu
int ht2_handle_device(const ht2gpu_handle_t* h);                                  // ht2_gpu.cu
int ht2_gunzip_to(int device, const void* src, size_t n, uint32_t chunkBytes, Ht2zOut& out, size_t* outLen,
                  ht2gpu_gunzip_stats_t* stats, std::string& err);               // ht2_inflate.cu

namespace {
double nowS() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// What a handle keeps between ht2gpu_run_reads calls: the parser's thread pool, its per-thread buffers and the
// pinned staging buffers of every slot (allocating pinned memory costs more than parsing a batch).
struct PipeCtx {
    Ht2ThreadPool* pool;
    Ht2ParseScratch scratch;
    std::vector<Ht2HostBatch> stage;
    std::mutex mu;               // one run at a time per handle
    ht2gpu_gunzip_stats_t gz;    // inflate stats of the last run's gzip inputs
    PipeCtx() : pool(NULL) { memset(&gz, 0, sizeof(gz)); }
    ~PipeCtx() { for (auto& hb : stage) hb.freeAll(); delete pool; }
};
void freeCtx(void* p) { delete (PipeCtx*)p; }
PipeCtx* ctxOf(ht2gpu_handle_t* h, unsigned nth, int nSlots)
{
    PipeCtx* c = (PipeCtx*)ht2gpu_ctx_get(h);
    if (!c) { c = new PipeCtx(); ht2gpu_ctx_set(h, c, freeCtx); }
    if (!c->pool || c->pool->size() != nth) { delete c->pool; c->pool = new Ht2ThreadPool(nth); }
    if ((int)c->stage.size() != nSlots) {
        for (auto& hb : c->stage) hb.freeAll();
        c->stage.assign((size_t)nSlots, Ht2HostBatch());
        for (auto& hb : c->stage) { hb.alloc = ht2gpu_host_alloc; hb.release = ht2gpu_host_free; }
    }
    return c;
}

// Compressed input is recognised by its magic bytes, not by a file name suffix.
bool isGzip(const Ht2ReadSource& s) { return s.size >= 2 && (uint8_t)s.data[0] == 0x1f && (uint8_t)s.data[1] == 0x8b; }
bool isBzip2(const Ht2ReadSource& s) { return s.size >= 3 && memcmp(s.data, "BZh", 3) == 0; }
const char* kBzip2Msg = "bzip2-compressed reads are not supported: decompress them through a pipe (bzip2 -dc reads.bz2 | ... -U -)";

void addGunzipStats(ht2gpu_gunzip_stats_t& acc, const ht2gpu_gunzip_stats_t& g)
{
    acc.in_bytes += g.in_bytes; acc.out_bytes += g.out_bytes; acc.members += g.members; acc.blocks += g.blocks; acc.chunks += g.chunks;
    acc.chunks_confirmed += g.chunks_confirmed; acc.chunks_merged_no_candidate += g.chunks_merged_no_candidate;
    acc.chunks_merged_false_positive += g.chunks_merged_false_positive; acc.windows += g.windows; acc.decode_rounds += g.decode_rounds;
    acc.peak_device_bytes += g.peak_device_bytes;   // the mate files are inflated at the same time
    acc.windows_cut += g.windows_cut;
    acc.chunk_bytes = g.chunk_bytes;
    acc.ms_find += g.ms_find; acc.ms_decode += g.ms_decode; acc.ms_window += g.ms_window; acc.ms_replace += g.ms_replace;
    acc.ms_crc += g.ms_crc; acc.ms_copy += g.ms_copy;
}

struct InputSpec { const char* path; const char* data; size_t len; };
bool openSpec(Ht2ReadSource& s, const InputSpec& sp, std::string& err)
{
    if (!sp.path) { ht2_source_memory(s, sp.data, sp.len); return true; }
    return ht2_source_open(s, sp.path, err);
}
// One input of a stream: a file (or memory range) and its record index; the consumer verifies and releases it.  A gzip
// source is inflated on the device, on a thread of its own, into an address range reserved for the largest output
// DEFLATE allows (1032 bytes per input byte); pages are committed as the windows land, so the text never moves and the
// producer indexes and parses it while later windows are still being decoded.  The compressed input is kept until the
// inflate has finished.  The consumer hands no SAM and routes no read before every member's CRC-32 and ISIZE are
// verified (verify), so corrupt input never produces output.
struct InFile : Ht2zOut {
    Ht2ReadSource src;
    bool gzip = false;
    bool started = false;                // plain, or inflate started: src holds the text
    bool released = false;
    std::atomic<bool> exhausted{false};  // producer: moved past its last record, never touches it again
    std::atomic<int64_t> lastBatch{-1};  // the last batch holding records of it
    Ht2ReadSource comp;                  // gzip: the compressed bytes
    Ht2SourceStream stream;
    char* base = NULL;
    size_t reserved = 0, committed = 0;
    std::atomic<bool> stop{false};
    ht2gpu_gunzip_stats_t st;
    std::thread th;
    ~InFile() { if (th.joinable()) { stop = true; th.join(); } }
    bool open(const InputSpec& sp, std::string& err) { return openSpec(src, sp, err); }
    bool detect(std::string& err)
    {
        if (isBzip2(src)) { err = kBzip2Msg; return false; }
        started = !(gzip = isGzip(src));
        return true;
    }
    char* grow(size_t need)
    {
        if (need > reserved) return NULL;
        if (need > committed) {
            size_t c = committed + ((size_t)64 << 20) > need ? committed + ((size_t)64 << 20) : need;
            c = (c + 4095) & ~(size_t)4095;
            if (c > reserved) c = reserved;
            if (mprotect(base + committed, c - committed, PROT_READ | PROT_WRITE) != 0) return NULL;
            committed = c;
        }
        return base;
    }
    bool landed(size_t len) { stream.publish(len); return !stop.load(); }
    // takes over src's compressed bytes; src becomes the (growing) decompressed text
    bool startInflate(int device, std::string& err)
    {
        if (started) return true;
        started = true;
        memset(&st, 0, sizeof(st));
        std::swap(comp.data, src.data); std::swap(comp.size, src.size); std::swap(comp.map, src.map); std::swap(comp.mapLen, src.mapLen);
        std::swap(comp.own, src.own);
        if (comp.own.size()) comp.data = comp.own.data();
        const size_t n = comp.size;
        reserved = n > ((size_t)1 << 40) / 1032 ? (size_t)1 << 40 : n * 1032 + ((size_t)1 << 20);
        void* m = mmap(NULL, reserved, PROT_NONE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
        if (m == MAP_FAILED) { err = "gzip input: could not reserve address space for the decompressed reads"; return false; }
        base = (char*)m;
        src.data = base; src.size = 0; src.map = m; src.mapLen = reserved; src.stream = &stream;
        th = std::thread([this, device]() {
            std::string e;
            size_t len = 0;
            const int rc = ht2_gunzip_to(device, comp.data, comp.size, 0, *this, &len, &st, e);
            stream.finish(rc, rc == HT2GPU_OK ? std::string() : "gzip input: " + e);
        });
        return true;
    }
    // HT2GPU_OK when the text is all there and every member verified (wait: for the inflate to finish), or while
    // the inflate runs (!wait)
    int verify(std::string& err, bool wait = true)
    {
        if (!gzip || !started) return HT2GPU_OK;
        std::unique_lock<std::mutex> lk(stream.mu);
        if (wait) stream.cv.wait(lk, [&] { return stream.done; });
        if (stream.done && stream.rc) err = stream.err;
        return stream.done ? stream.rc : HT2GPU_OK;
    }
    void release(ht2gpu_gunzip_stats_t& gzStats)
    {
        if (released) return;
        if (th.joinable()) { stop = true; th.join(); }
        if (gzip && started) addGunzipStats(gzStats, st);
        ht2_source_close(comp);
        ht2_source_close(src);
        released = true;
    }
};
// ht2gpu_parse_reads / ht2gpu_route_reads are host-only: compressed input is refused, not inflated on the CPU
bool refuseCompressed(const Ht2ReadSource& s, std::string& err)
{
    if (isBzip2(s)) { err = kBzip2Msg; return true; }
    if (isGzip(s)) { err = "gzip-compressed reads: this call is host-only; inflate them with ht2gpu_gunzip first"; return true; }
    return false;
}
unsigned threadCount(const ht2gpu_reads_input_t* in)
{
    const unsigned n = in->threads > 0 ? (unsigned)in->threads : std::thread::hardware_concurrency();
    return n < 1 ? 1 : n > 64 ? 64 : n;
}
Ht2ReadsOpts readsOpts(const ht2gpu_reads_input_t* in)
{
    Ht2ReadsOpts ro; ro.fastq = in->format == 1; ro.trim5 = in->trim5; ro.trim3 = in->trim3; ro.phred64 = in->phred64 != 0; ro.seed = in->seed;
    ro.solexa = in->solexa_quals != 0; ro.intQuals = in->int_quals != 0;
    return ro;
}

// Routes records to the read files of ht2gpu_read_routes_t by their units' outcomes.  Each of the nine streams
// (output x mate) keeps one pending span; a record that continues it in the same input extends it, anything else
// flushes it first, so a run of consecutive records with the same destination reaches the callback as one span
// straight from the input.
struct Router {
    ht2gpu_read_routes_t* R;
    bool fastq;
    const char* pd[HT2GPU_READS_N * 2];
    uint64_t pb[HT2GPU_READS_N * 2], pe[HT2GPU_READS_N * 2];
    int rc;
    Router(ht2gpu_read_routes_t* r, bool fq) : R(r), fastq(fq), rc(0)
    {
        for (int k = 0; k < HT2GPU_READS_N * 2; k++) { pd[k] = NULL; pb[k] = pe[k] = 0; }
    }
    void flush(int k)
    {
        if (pe[k] > pb[k] && rc == 0) {
            const int which = k >> 1, mate = which < HT2GPU_READS_UN_CONC ? 0 : (k & 1) + 1;
            R->n_spans++; R->bytes += pe[k] - pb[k];
            if (R->write(R->ctx, which, mate, pd[k] + pb[k], (size_t)(pe[k] - pb[k])) != 0) rc = 1;
        }
        pb[k] = pe[k] = 0;
    }
    void put(int which, int m, const char* d, uint64_t b, uint64_t e)   // m: 0 mate 1 / unpaired, 1 mate 2
    {
        if (!(R->mask & (1u << which))) return;
        const int k = which * 2 + m;
        if (pd[k] != d || pe[k] != b || pe[k] == pb[k]) { flush(k); pd[k] = d; pb[k] = b; }
        pe[k] = e;
    }
    // Read::readOrigBuf of record r (rec[r] .. rec[r + 1]) of its file: the FASTQ parser keeps the blank lines before
    // each file's first record (pat.cpp:867-874), and FileBuf keeps at most LASTN_BUF_SZ = 8192 bytes (filebuf.h:109, 262)
    void span(const uint64_t* rec, uint64_t i, uint64_t r, uint64_t& b, uint64_t& e) const
    {
        b = (fastq && r == 0) ? 0 : rec[i]; e = rec[i + 1];
        if (e - b > 8192) e = b + 8192;
    }
    // units whose records are ra, ra + 1, ... of input da (and rb, rb + 1, ... of db for pairs): recA / recB hold the
    // record starts rec[ra .. ra + n] / rec[rb .. rb + n] of the two inputs
    void batch(const char* da, const uint64_t* recA, uint64_t ra, const char* db, const uint64_t* recB, uint64_t rb, uint64_t n,
               const uint8_t* out)
    {
        for (uint64_t i = 0; i < n && rc == 0; i++) {
            const uint8_t o = out[i];
            uint64_t b1, e1; span(recA, i, ra + i, b1, e1);
            if (!recB) { put((o & HT2GPU_OUTCOME_AL1) ? HT2GPU_READS_AL : HT2GPU_READS_UN, 0, da, b1, e1); continue; }
            uint64_t b2, e2; span(recB, i, rb + i, b2, e2);
            const int conc = (o & HT2GPU_OUTCOME_CONC) ? HT2GPU_READS_AL_CONC : HT2GPU_READS_UN_CONC;
            put(conc, 0, da, b1, e1); put(conc, 1, db, b2, e2);
            if (o & (HT2GPU_OUTCOME_AL1 | HT2GPU_OUTCOME_AL2)) { put(HT2GPU_READS_AL_CONC_DISC, 0, da, b1, e1); put(HT2GPU_READS_AL_CONC_DISC, 1, db, b2, e2); }
        }
    }
    void finish() { for (int k = 0; k < HT2GPU_READS_N * 2; k++) flush(k); }
};
}
extern "C" int ht2gpu_run_reads(ht2gpu_handle_t* h, const ht2gpu_reads_input_t* in, ht2gpu_sink_fn sink, void* ctx, ht2gpu_run_stats_t* st)
{
    return ht2gpu_run_reads_routed(&h, 1, in, sink, ctx, NULL, st);
}

extern "C" int ht2gpu_run_reads_multi(ht2gpu_handle_t** hs, int nDev, const ht2gpu_reads_input_t* in, ht2gpu_sink_fn sink, void* ctx,
                                      ht2gpu_run_stats_t* st)
{
    return ht2gpu_run_reads_routed(hs, nDev, in, sink, ctx, NULL, st);
}

namespace {
// The reads of one kind: pairs (files[0] the -1 files, files[1] the -2 files) or unpaired reads (files[0]).  Record k
// of the stream is record k of its files back to back; the mates of a pair have the same ordinal, wherever the files end.
struct StreamSpec { bool paired; std::vector<InputSpec> files[2]; };

struct Stream {
    bool paired = false;
    std::vector<std::unique_ptr<InFile> > f[2];
    // a gzip file is inflated from the time the producer reaches the file before it (or the run starts), so that the
    // next file's text is landing while the current one is read
    bool startAhead(int k, size_t fi, int device, std::string& e)
    {
        for (size_t j = fi; j < fi + 2 && j < f[k].size(); j++) if (!f[k][j]->startInflate(device, e)) return false;
        return true;
    }
};
// A submitted batch as the consumer needs it after its wait: its pieces and, per piece and mate, the file and, when
// routing, a copy of the record starts rec[ra .. ra + n] (the producer keeps appending to the files' indexes meanwhile).
struct RecPiece { InFile* f[2]; std::vector<uint64_t> rec[2]; };
struct SlotBatch { std::vector<Ht2BatchPiece> pcs; std::vector<RecPiece> recs; };

// The producer's place in a stream: per mate, the file (cf) and the record in that file (cp) of the next unit.
struct StreamCursor {
    Stream& S;
    Stream* after;   // the next stream: its first file starts inflating when this stream reaches its last one
    const int device;
    const bool fastq;
    Ht2ThreadPool& pool;
    size_t cf[2];
    uint64_t cp[2];
    int nm() const { return S.paired ? 2 : 1; }
    // the n units [r, r + want) that are there (0 at the end of the stream); a pair with only one mate is an error
    bool next(uint64_t r, uint64_t want, uint64_t rEnd, uint64_t& n, std::string& e)
    {
        uint64_t av[2] = {0, 0}; bool ended[2] = {false, false};
        n = ~(uint64_t)0;
        for (int k = 0; k < nm(); k++) { if (!indexAhead(k, want, av[k], ended[k], e)) return false; if (av[k] < n) n = av[k]; }
        if (S.paired && av[0] != av[1] && ended[av[0] < av[1] ? 0 : 1] && r + n < rEnd) {
            e = av[0] < av[1] ? "fewer reads in file specified with -1 than in file specified with -2"
                              : "fewer reads in file specified with -2 than in file specified with -1";
            return false;
        }
        return true;
    }
    // Moves past units [rdid, rdid + n) of batch bi, cut into the pieces in which every mate stays in one file (b ==
    // NULL: skipped records).  A file's last batch is set before the file is marked exhausted, so that the consumer
    // never lets go of a file this batch still has to parse.
    bool take(uint64_t rdid, uint64_t n, SlotBatch* b, int64_t bi, bool route, std::string& e)
    {
        size_t q = 0;
        if (b) b->pcs.clear();
        for (uint64_t u = 0; u < n;) {
            uint64_t m = n - u;
            bool moved = false;
            for (int k = 0; k < nm() && !moved; k++) {
                if (cf[k] >= S.f[k].size()) { e = "read front end: a batch ran past the end of its input"; return false; }
                InFile& F = *S.f[k][cf[k]];
                const uint64_t rem = F.src.nRecords() - cp[k];
                if (rem == 0 && F.src.scanDone) { F.exhausted = true; cf[k]++; cp[k] = 0; moved = true; }
                else if (rem < m) m = rem;
            }
            if (moved) continue;
            if (b) {
                if (q == b->recs.size()) b->recs.emplace_back();
                RecPiece& rp = b->recs[q++];
                for (int k = 0; k < 2; k++) {
                    InFile* F = rp.f[k] = k < nm() ? S.f[k][cf[k]].get() : NULL;
                    if (F) F->lastBatch = bi;
                    if (F && route) rp.rec[k].assign(F->src.rec.begin() + (ptrdiff_t)cp[k], F->src.rec.begin() + (ptrdiff_t)(cp[k] + m) + 1);
                }
                b->pcs.push_back({&rp.f[0]->src, rp.f[1] ? &rp.f[1]->src : NULL, cp[0], rp.f[1] ? cp[1] : 0, m, rdid + u});
            }
            for (int k = 0; k < nm(); k++) cp[k] += m;
            u += m;
        }
        if (b) b->recs.resize(q);
        for (int k = 0; k < nm(); k++)   // a file read to its end is let go at once
            while (cf[k] < S.f[k].size() && S.f[k][cf[k]]->src.scanDone && cp[k] == S.f[k][cf[k]]->src.nRecords()) {
                S.f[k][cf[k]]->exhausted = true; cf[k]++; cp[k] = 0;
            }
        return true;
    }
    // Index mate k's files from the cursor on until `want` records are known, the files end (ended), or a file still
    // being inflated holds a quarter of them, so that the first batches are aligned while the rest is decoded.  have:
    // the number of records known, at most want.
    bool indexAhead(int k, uint64_t want, uint64_t& have, bool& ended, std::string& e)
    {
        size_t fi = cf[k]; uint64_t pos = cp[k];
        have = 0;
        for (;;) {
            if (fi >= S.f[k].size()) { ended = true; return true; }
            if (!S.startAhead(k, fi, device, e)) return false;
            if (fi + 1 == S.f[k].size() && after && !after->startAhead(0, 0, device, e)) return false;
            Ht2ReadSource& src = S.f[k][fi]->src;
            while (!src.scanDone && src.nRecords() < pos + (want - have) && !(src.stream && have + src.nRecords() - pos >= (want + 3) / 4))
                if (!ht2_source_scan(src, fastq, pool, (size_t)256 << 20, e)) return false;
            have += src.nRecords() - pos < want - have ? src.nRecords() - pos : want - have;
            if (have == want || !src.scanDone) return true;
            fi++; pos = 0;
        }
    }
};

// One call of the pipeline over a run's streams, in order (pairs before unpaired reads).  rdid, -s and -u count per
// stream, as the reference's per-source read counters do (pat.h:224, hisat2.cpp:1959-1964, 3319); the read loop ends
// for good at the first unit with rdid >= skip + upto (hisat2.cpp:3634), so a later stream is read only if the earlier
// one ended before that.  A batch never holds units of two streams.  The producer thread indexes, parses and submits
// batches; the caller's thread waits for them in order.  What the two share is under mu, the run's first failure too.
struct Run {
    Run(ht2gpu_handle_t** hs, int nDev, const ht2gpu_reads_input_t* in, ht2gpu_sink_fn sink, void* ctx, ht2gpu_read_routes_t* routes)
        : hs(hs), nDev(nDev), in(in), sink(sink), ctx(ctx), routes(routes), route(routes && routes->mask), ro(readsOpts(in)),
          r0(in->skip), rEnd(in->upto ? in->skip + in->upto : ~(uint64_t)0),
          perRead(in->batch_reads ? in->batch_reads : 4000000),   // large batches amortise the drain of the pool kernel's last reads
          router(routes, ro.fastq) { memset(&S, 0, sizeof(S)); }
    int exec(const std::vector<StreamSpec>& specs, ht2gpu_run_stats_t* st)
    {
        if (route && !routes->write) return HT2GPU_ERR_ARG;
        if (routes) { routes->n_spans = 0; routes->bytes = 0; routes->s_route = 0; }
        for (int i = 1; i < nDev; i++)
            if (!ht2_same_sam_output(hs[0], hs[i])) { ht2gpu_set_error(hs[0], "ht2gpu_run_reads_multi: the handles' SAM output, mate orientation, N-ceiling or spliced-alignment settings differ"); return HT2GPU_ERR_ARG; }
        const double t0 = nowS();
        nSlots = ht2gpu_sam_slots(hs[0]) * nDev;   // stage k: device k % nDev, device slot k / nDev
        C = ctxOf(hs[0], threadCount(in), nSlots);
        std::lock_guard<std::mutex> runLock(C->mu);
        memset(&C->gz, 0, sizeof(C->gz));
        device = ht2_handle_device(hs[0]);
        state.assign((size_t)nSlots, 0);
        batches.resize((size_t)nSlots);
        if (open(specs)) {
            std::thread producer([this] { produce(); std::lock_guard<std::mutex> lk(mu); prodDone = true; cv.notify_all(); });
            consume();
            producer.join();
        }
        return finish(t0, st);
    }
    ht2gpu_handle_t** const hs;
    const int nDev;
    const ht2gpu_reads_input_t* const in;
    const ht2gpu_sink_fn sink; void* const ctx;
    ht2gpu_read_routes_t* const routes; const bool route;
    const Ht2ReadsOpts ro;
    const uint64_t r0, rEnd, perRead;   // -s / -u (hisat2.cpp:1959-1964, 3319): records [skip, skip + upto) of each stream
    int nSlots = 0, device = 0;
    PipeCtx* C = NULL;
    std::vector<Stream> streams;
    std::vector<InFile*> files;          // every file of every stream, in order
    std::vector<SlotBatch> batches;      // per slot
    Router router;                       // consumer
    ht2gpu_run_stats_t S;                // consumer
    double parseS = 0, submitS = 0, indexS = 0, waitS = 0, sinkS = 0, routeS = 0;
    std::mutex mu;
    std::condition_variable cv;
    std::vector<int> state;              // per slot: 0 free, 1 submitted
    uint64_t submitted = 0; bool prodDone = false;
    int rc = HT2GPU_OK;                  // the first failure of either thread
    std::string err;

    // Keeps the first failure and wakes both threads; returns false.
    bool fail(int code, const std::string& m)
    {
        std::lock_guard<std::mutex> lk(mu);
        if (rc == HT2GPU_OK) { rc = code; err = m; }
        cv.notify_all();
        return false;
    }

    // Every file is opened (mapped) up front, so that a missing one fails the run before anything is aligned.
    bool open(const std::vector<StreamSpec>& specs)
    {
        std::string e;
        for (int i = 0; i < nDev && route; i++) { const int orc = ht2gpu_record_outcomes(hs[i], 1); if (orc) return fail(orc, ht2gpu_last_error(hs[i])); }
        streams.resize(specs.size());
        for (size_t s = 0; s < specs.size(); s++) {
            streams[s].paired = specs[s].paired;
            for (int k = 0; k < (specs[s].paired ? 2 : 1); k++)
                for (const InputSpec& sp : specs[s].files[k]) {
                    streams[s].f[k].emplace_back(new InFile());
                    files.push_back(streams[s].f[k].back().get());
                    if (!files.back()->open(sp, e)) return fail(HT2GPU_ERR_ARG, e);
                }
        }
        for (InFile* F : files) if (!F->detect(e)) return fail(HT2GPU_ERR_ARG, e);
        for (int k = 0; k < 2 && !streams.empty(); k++) if (!streams[0].startAhead(k, 0, device, e)) return fail(HT2GPU_ERR_ARG, e);
        return true;
    }

    bool index(StreamCursor& cur, uint64_t r, uint64_t want, uint64_t& n)
    {
        const double ti = nowS();
        std::string e;
        const bool ok = cur.next(r, want, rEnd, n, e);
        indexS += nowS() - ti;
        return ok || fail(HT2GPU_ERR_ARG, e);
    }

    // The producer indexes the input only as far ahead as the next batch needs (so that indexing overlaps the device
    // work), parses the batch on all threads and submits it.  The first batch is a quarter of the others: the device
    // starts early, the later batches are large.
    void produce()
    {
        uint64_t i = 0, n = 0;
        std::string e;
        for (size_t s = 0; s < streams.size(); s++) {
            StreamCursor cur{streams[s], s + 1 < streams.size() ? &streams[s + 1] : NULL, device, ro.fastq, *C->pool, {0, 0}, {0, 0}};
            const uint64_t perBatch = streams[s].paired ? (perRead + 1) / 2 : perRead;   // batch_reads counts reads, a unit here may be a pair
            uint64_t r = 0;
            while (r < r0) {   // -s: the skipped records are indexed, not parsed
                if (!index(cur, r, r0 - r < perBatch ? r0 - r : perBatch, n)) return;
                if (n == 0) break;
                if (!cur.take(r, n, NULL, 0, false, e)) { fail(HT2GPU_ERR_ARG, e); return; }
                r += n;
            }
            bool more = true;   // the stream has units left
            while (r >= r0) {
                const int slot = (int)(i % (uint64_t)nSlots);
                { std::unique_lock<std::mutex> lk(mu); cv.wait(lk, [&] { return state[slot] == 0 || rc != HT2GPU_OK; }); if (rc != HT2GPU_OK) return; }
                uint64_t want = (i == 0 && perBatch >= 8) ? perBatch / 4 : perBatch;
                if (r + want > rEnd) want = rEnd > r ? rEnd - r : 0;
                n = 0;
                if (want && !index(cur, r, want, n)) return;
                if (n == 0) { more = want == 0; break; }   // cut by -u, or nothing left
                SlotBatch& b = batches[slot];
                if (!cur.take(r, n, &b, (int64_t)i, route, e)) { fail(HT2GPU_ERR_ARG, e); return; }
                Ht2HostBatch& hb = C->stage[slot];
                const double tp = nowS();
                const bool parsed = ht2_parse_pieces(b.pcs.data(), b.pcs.size(), ro, hb, *C->pool, C->scratch, e);
                parseS += nowS() - tp;
                if (!parsed) { fail(HT2GPU_ERR_ARG, e); return; }
                ht2gpu_read_batch_t rb; memset(&rb, 0, sizeof(rb));
                rb.n_reads = hb.n_reads; rb.paired = streams[s].paired ? 1 : 0; rb.seq = hb.seq; rb.qual = hb.haveQual ? hb.qual : NULL; rb.offs = hb.offs; rb.seeds = hb.seeds;
                const double ts = nowS();
                const int src = ht2gpu_submit_sam(hs[slot % nDev], slot / nDev, &rb, hb.names, hb.nameOffs, hb.namesBytes);
                submitS += nowS() - ts;
                if (src != HT2GPU_OK) { fail(src, ht2gpu_last_error(hs[slot % nDev])); return; }
                { std::lock_guard<std::mutex> lk(mu); state[slot] = 1; submitted = ++i; cv.notify_all(); }
                r += n;
            }
            // cut by -u: the read loop ends at the first unit with rdid >= skip + upto, if there is one
            if (more && s + 1 < streams.size() && (!index(cur, r, 1, n) || n > 0)) return;
        }
    }

    // The caller's thread waits for the batches in order, hands their SAM to the sink (nothing of a gzip file before
    // the file is verified), routes their records and lets go of the files the producer has left.
    void consume()
    {
        for (uint64_t i = 0; ; i++) {
            const int slot = (int)(i % (uint64_t)nSlots);
            ht2gpu_handle_t* hd = hs[slot % nDev];
            {
                std::unique_lock<std::mutex> lk(mu);
                cv.wait(lk, [&] { return submitted > i || rc != HT2GPU_OK || prodDone; });
                if (submitted <= i) return;   // the producer has finished (or failed)
            }
            ht2gpu_sam_result_t r;
            const double tw = nowS();
            const int wrc = ht2gpu_wait_sam(hd, slot / nDev, &r);
            waitS += nowS() - tw;
            if (wrc != HT2GPU_OK) { fail(wrc, ht2gpu_last_error(hd)); return; }
            S.n_batches++; S.n_units += r.n_units; S.n_reads += C->stage[slot].n_reads; S.sam_bytes += r.sam_len; S.n_err_reads += r.n_err_reads;
            S.ms_align += r.ms_align; S.ms_sam += r.ms_sam; S.ms_h2d += r.ms_h2d; S.ms_d2h += r.ms_d2h;
            S.h2d_bytes += r.h2d_bytes; S.d2h_bytes += r.d2h_bytes; S.n_launches += r.n_launches;
            const SlotBatch& b = batches[slot];
            bool ok = true;
            std::string e;
            for (const RecPiece& rp : b.recs)
                for (InFile* F : rp.f) { const int v = ok && F ? F->verify(e) : HT2GPU_OK; if (v) ok = fail(v, e); }
            const double tk = nowS();
            if (ok && sink && r.sam_len && sink(ctx, r.sam, r.sam_len) != 0) ok = fail(HT2GPU_ERR_ARG, "the SAM sink reported an error");
            sinkS += nowS() - tk;
            if (route && ok) {
                const double tr = nowS();
                const uint8_t* ob = NULL; uint32_t nu = 0;
                const int orc = ht2gpu_unit_outcomes(hd, slot / nDev, &ob, &nu);
                if (orc != HT2GPU_OK) ok = fail(orc, ht2gpu_last_error(hd));
                for (uint64_t q = 0, u = 0; ok && q < b.pcs.size() && u + b.pcs[q].n <= nu; u += b.pcs[q++].n) {
                    const Ht2BatchPiece& pc = b.pcs[q];
                    router.batch(pc.a->data, b.recs[q].rec[0].data(), pc.ra, pc.b ? pc.b->data : NULL, pc.b ? b.recs[q].rec[1].data() : NULL,
                                 pc.rb, pc.n, ob + u);
                }
                if (ok && router.rc) ok = fail(HT2GPU_ERR_ARG, "the read-file writer reported an error");
                routeS += nowS() - tr;
            }
            // files the producer has left whose last batch is done: their text (and address space) is let go
            bool flushed = false;
            for (InFile* F : files)
                if (!F->released && F->exhausted && F->lastBatch <= (int64_t)i) {
                    if (route && !flushed) { router.finish(); flushed = true; }   // no pending span may point into it
                    F->release(C->gz);
                }
            { std::lock_guard<std::mutex> lk(mu); state[slot] = 0; cv.notify_all(); }
            if (!ok) return;
        }
    }

    // After both threads: the gzip files read from are verified, the router finished, the batches still in flight
    // after an error drained, every file let go and the stats filled.
    int finish(double t0, ht2gpu_run_stats_t* st)
    {
        std::string e;
        // a gzip file that was read from (or read to its end) is verified before the run succeeds; one whose records
        // were never needed (-u) is stopped
        for (InFile* F : files)
            if (rc == HT2GPU_OK && !F->released && (F->exhausted || F->lastBatch >= 0)) { const int v = F->verify(e); if (v) fail(v, e); }
        if (rc != HT2GPU_OK)   // a failed inflate explains a failed run better than what the parser made of its bytes
            for (InFile* F : files) { const int z = F->verify(e, false); if (z) { std::lock_guard<std::mutex> lk(mu); rc = z; err = e; } }
        if (rc != HT2GPU_OK)   // drain the batches still in flight (a handle refuses to stop recording outcomes before)
            for (int s = 0; s < nSlots; s++) if (state[s] == 1) { ht2gpu_sam_result_t r; ht2gpu_wait_sam(hs[s % nDev], s / nDev, &r); }
        if (route) {
            const double tr = nowS();
            router.finish();
            if (router.rc) fail(HT2GPU_ERR_ARG, "the read-file writer reported an error");
            routeS += nowS() - tr;
            routes->s_route = routeS;
            for (int i = 0; i < nDev; i++) ht2gpu_record_outcomes(hs[i], 0);
        }
        for (InFile* F : files) F->release(C->gz);
        S.s_index = indexS; S.s_parse = parseS; S.s_submit = submitS; S.s_wait = waitS; S.s_sink = sinkS; S.s_total = nowS() - t0;
        if (st) *st = S;
        if (rc != HT2GPU_OK) ht2gpu_set_error(hs[0], err.empty() ? "ht2gpu_run_reads failed" : err.c_str());
        return rc;
    }
};
}

// The same pipeline over several devices of one process (hisat2-b200 --gpus N): batch i goes to handle i % n,
// the sink still receives the batches in input order.  The index is replicated (ht2gpu_open_peer), reads are the
// only thing that is sharded, no data-path collective.  Context (thread pool, pinned staging) lives in hs[0].
// With routes, every device records its units' outcomes and the records of batch i are routed right after its wait.
extern "C" int ht2gpu_run_reads_routed(ht2gpu_handle_t** hs, int nDev, const ht2gpu_reads_input_t* in, ht2gpu_sink_fn sink, void* ctx,
                                       ht2gpu_read_routes_t* routes, ht2gpu_run_stats_t* st)
{
    if (!hs || nDev < 1 || !in) return HT2GPU_ERR_ARG;
    for (int i = 0; i < nDev; i++) if (!hs[i]) return HT2GPU_ERR_ARG;
    if (!in->path1 && !in->data1) { ht2gpu_set_error(hs[0], "ht2gpu_run_reads: no input"); return HT2GPU_ERR_ARG; }
    std::vector<StreamSpec> ss(1);
    ss[0].paired = in->path2 || in->data2;
    ss[0].files[0].push_back({in->path1, in->data1, in->len1});
    if (ss[0].paired) ss[0].files[1].push_back({in->path2, in->data2, in->len2});
    return Run(hs, nDev, in, sink, ctx, routes).exec(ss, st);
}

// Read-file lists: every -1 / -2 file back to back as one paired stream, then every -U file as one unpaired stream.
extern "C" int ht2gpu_run_reads_files(ht2gpu_handle_t** hs, int nDev, const ht2gpu_reads_files_t* files, const ht2gpu_reads_input_t* in,
                                      ht2gpu_sink_fn sink, void* ctx, ht2gpu_read_routes_t* routes, ht2gpu_run_stats_t* st)
{
    if (!hs || nDev < 1 || !in || !files) return HT2GPU_ERR_ARG;
    for (int i = 0; i < nDev; i++) if (!hs[i]) return HT2GPU_ERR_ARG;
    auto refuse = [&](const std::string& m) { ht2gpu_set_error(hs[0], m.c_str()); return HT2GPU_ERR_ARG; };
    if (in->path1 || in->path2 || in->data1 || in->data2) return refuse("ht2gpu_run_reads_files: the paths and data of ht2gpu_reads_input_t must be NULL");
    if (files->n1 != files->n2)   // hisat2.cpp:1911-1913
        return refuse(std::to_string(files->n1) + " mate files/sequences were specified with -1, but " + std::to_string(files->n2) +
                      "\nmate files/sequences were specified with -2.  The same number of mate files/\nsequences must be specified with -1 and -2.");
    if (files->n1 + files->n_u == 0) return refuse("ht2gpu_run_reads_files: no input");
    std::vector<StreamSpec> ss;
    if (files->n1) ss.push_back(StreamSpec{true, {}});
    if (files->n_u) ss.push_back(StreamSpec{false, {}});
    int stdinUses = 0;
    const char* const* lists[3] = {files->paths1, files->paths2, files->paths_u};
    const uint32_t counts[3] = {files->n1, files->n2, files->n_u};
    for (int l = 0; l < 3; l++) {
        if (counts[l] && !lists[l]) return refuse("ht2gpu_run_reads_files: a list with entries is NULL");
        for (uint32_t j = 0; j < counts[l]; j++) {
            const char* p = lists[l][j];
            if (!p || !*p) return refuse("ht2gpu_run_reads_files: an empty read file name");
            if (strcmp(p, "-") == 0 && ++stdinUses > 1) return refuse("standard input ('-') can be read only once");
            (l < 2 ? ss[0].files[l] : ss.back().files[0]).push_back({p, NULL, 0});
        }
    }
    return Run(hs, nDev, in, sink, ctx, routes).exec(ss, st);
}

namespace {
// The whole input of the host-only calls: opened, indexed, mate counts checked, and the units [r0, r1) after -s / -u.
struct WholeInput {
    Ht2ThreadPool pool;
    Ht2ReadSource a, b;
    const bool paired;
    uint64_t r0 = 0, r1 = 0;
    explicit WholeInput(const ht2gpu_reads_input_t* in) : pool(threadCount(in)), paired(in->path2 != NULL || in->data2 != NULL) {}
    ~WholeInput() { ht2_source_close(a); ht2_source_close(b); }
    bool open(const ht2gpu_reads_input_t* in, std::string& err)
    {
        if (!in->path1 && !in->data1) { err = "no input"; return false; }
        if (!openSpec(a, {in->path1, in->data1, in->len1}, err) || (paired && !openSpec(b, {in->path2, in->data2, in->len2}, err))) return false;
        if (refuseCompressed(a, err) || refuseCompressed(b, err)) return false;
        if (!ht2_source_index(a, in->format == 1, pool, err) || (paired && !ht2_source_index(b, in->format == 1, pool, err))) return false;
        if (paired && a.nRecords() != b.nRecords()) { err = "mate files have different numbers of reads"; return false; }
        r0 = in->skip < a.nRecords() ? in->skip : a.nRecords(); r1 = a.nRecords();
        if (in->upto && r0 + in->upto < r1) r1 = r0 + in->upto;
        return true;
    }
};
int errOut(char* errbuf, size_t errbuf_len, const std::string& m)
{
    if (errbuf && errbuf_len) { strncpy(errbuf, m.c_str(), errbuf_len - 1); errbuf[errbuf_len - 1] = 0; }
    return HT2GPU_ERR_ARG;
}
}

// Host-only: parse a whole input into ONE batch (malloc'ed buffers).  No device is touched: this is the read
// front end on its own (tests, callers that batch for themselves).
extern "C" int ht2gpu_parse_reads(const ht2gpu_reads_input_t* in, ht2gpu_parsed_reads_t* out, char* errbuf, size_t errbuf_len)
{
    if (!in || !out) return HT2GPU_ERR_ARG;
    memset(out, 0, sizeof(*out));
    WholeInput w(in);
    std::string err;
    if (!w.open(in, err)) return errOut(errbuf, errbuf_len, err);
    Ht2HostBatch* hb = new Ht2HostBatch();
    Ht2ParseScratch scratch;
    if (!ht2_parse_batch(w.a, w.paired ? &w.b : NULL, w.r0, w.r1, readsOpts(in), *hb, w.pool, scratch, err)) { hb->freeAll(); delete hb; return errOut(errbuf, errbuf_len, err); }
    out->batch.n_reads = hb->n_reads; out->batch.paired = w.paired ? 1 : 0; out->batch.seq = hb->seq; out->batch.qual = hb->haveQual ? hb->qual : NULL;
    out->batch.offs = hb->offs; out->batch.seeds = hb->seeds;
    out->names = hb->names; out->name_offs = hb->nameOffs; out->names_bytes = hb->namesBytes; out->priv = hb;
    return HT2GPU_OK;
}
// Host-only routing of a whole input by given outcomes (ht2gpu_unit_outcomes of callers that batch for themselves).
extern "C" int ht2gpu_route_reads(const ht2gpu_reads_input_t* in, const uint8_t* outcomes, uint64_t n_units, ht2gpu_read_routes_t* routes,
                                  char* errbuf, size_t errbuf_len)
{
    if (!in || !routes || (n_units && !outcomes) || (routes->mask && !routes->write)) return HT2GPU_ERR_ARG;
    routes->n_spans = 0; routes->bytes = 0; routes->s_route = 0;
    const double t0 = nowS();
    WholeInput w(in);
    std::string err;
    bool ok = w.open(in, err);
    if (ok && w.r1 - w.r0 != n_units) { ok = false; err = "the outcomes do not cover the input's " + std::to_string(w.r1 - w.r0) + " units"; }
    if (ok && routes->mask) {
        Router router(routes, in->format == 1);
        router.batch(w.a.data, w.a.rec.data() + w.r0, w.r0, w.b.data, w.paired ? w.b.rec.data() + w.r0 : NULL, w.r0, w.r1 - w.r0, outcomes);
        router.finish();
        if (router.rc) { ok = false; err = "the read-file writer reported an error"; }
    }
    routes->s_route = nowS() - t0;
    return ok ? HT2GPU_OK : errOut(errbuf, errbuf_len, err);
}

extern "C" void ht2gpu_free_parsed(ht2gpu_parsed_reads_t* p)
{
    if (p && p->priv) { Ht2HostBatch* hb = (Ht2HostBatch*)p->priv; hb->freeAll(); delete hb; p->priv = NULL; }
}

extern "C" int ht2gpu_run_gunzip_stats(ht2gpu_handle_t* h, ht2gpu_gunzip_stats_t* st)
{
    if (!h || !st) return HT2GPU_ERR_ARG;
    PipeCtx* c = (PipeCtx*)ht2gpu_ctx_get(h);
    if (c) { std::lock_guard<std::mutex> lk(c->mu); *st = c->gz; }
    else memset(st, 0, sizeof(*st));
    return HT2GPU_OK;
}
