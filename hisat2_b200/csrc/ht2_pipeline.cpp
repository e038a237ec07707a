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
void* pinAlloc(size_t n) { return ht2gpu_host_alloc(n); }
void pinFree(void* p) { ht2gpu_host_free(p); }

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
        for (auto& hb : c->stage) { hb.alloc = pinAlloc; hb.release = pinFree; }
    }
    return c;
}

// Compressed input is recognised by its magic bytes, not by a file name suffix.
bool isGzip(const Ht2ReadSource& s) { return s.size >= 2 && (uint8_t)s.data[0] == 0x1f && (uint8_t)s.data[1] == 0x8b; }
bool isBzip2(const Ht2ReadSource& s) { return s.size >= 3 && memcmp(s.data, "BZh", 3) == 0; }
const char* kBzip2Msg = "bzip2-compressed reads are not supported: decompress them through a pipe (bzip2 -dc reads.bz2 | ... -U -)";

// A gzip source is inflated on the device, on a thread of its own, into an address range reserved for the largest
// output DEFLATE allows (1032 bytes per input byte); pages are committed as the windows land, so the text never moves
// and the producer indexes and parses it while later windows are still being decoded.  The compressed input is kept
// until the inflate has finished.  The consumer hands no SAM and routes no read before every member's CRC-32 and
// ISIZE are verified (Inflater::verified), so corrupt input never produces output.
struct Inflater : Ht2zOut {
    Ht2ReadSource comp;                 // the compressed bytes
    Ht2SourceStream stream;
    char* base = NULL;
    size_t reserved = 0, committed = 0;
    std::atomic<bool> stop{false};
    ht2gpu_gunzip_stats_t st;
    std::thread th;
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
    // takes over s's compressed bytes; s becomes the (growing) decompressed text
    bool start(Ht2ReadSource& s, int device, std::string& err)
    {
        memset(&st, 0, sizeof(st));
        std::swap(comp.data, s.data); std::swap(comp.size, s.size); std::swap(comp.map, s.map); std::swap(comp.mapLen, s.mapLen);
        std::swap(comp.own, s.own);
        if (comp.own.size()) comp.data = comp.own.data();
        const size_t n = comp.size;
        reserved = n > ((size_t)1 << 40) / 1032 ? (size_t)1 << 40 : n * 1032 + ((size_t)1 << 20);
        void* m = mmap(NULL, reserved, PROT_NONE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
        if (m == MAP_FAILED) { err = "gzip input: could not reserve address space for the decompressed reads"; return false; }
        base = (char*)m;
        s.data = base; s.size = 0; s.map = m; s.mapLen = reserved; s.stream = &stream;
        th = std::thread([this, device]() {
            std::string e;
            size_t len = 0;
            const int rc = ht2_gunzip_to(device, comp.data, comp.size, 0, *this, &len, &st, e);
            stream.finish(rc, rc == HT2GPU_OK ? std::string() : "gzip input: " + e);
        });
        return true;
    }
    // waits for the inflate; HT2GPU_OK when all of it is there and verified
    int verified(std::string& err)
    {
        std::unique_lock<std::mutex> lk(stream.mu);
        stream.cv.wait(lk, [&] { return stream.done; });
        if (stream.rc) err = stream.err;
        return stream.rc;
    }
    void join() { if (th.joinable()) { stop = true; th.join(); } ht2_source_close(comp); }
    ~Inflater() { join(); }
};

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
// ht2gpu_parse_reads / ht2gpu_route_reads are host-only: compressed input is refused, not inflated on the CPU
bool refuseCompressed(const Ht2ReadSource& s, std::string& err)
{
    if (isBzip2(s)) { err = kBzip2Msg; return true; }
    if (isGzip(s)) { err = "gzip-compressed reads: this call is host-only; inflate them with ht2gpu_gunzip first"; return true; }
    return false;
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
// One input of a stream: a file (or memory range), its record index, and its inflate when it is gzip.
struct InFile {
    Ht2ReadSource src;
    std::unique_ptr<Inflater> gz;        // gzip input: created when opened, started when the producer comes near it
    bool started = false;                // plain, or inflate started: src holds the text
    bool verified = false;               // consumer: every gzip member checked
    bool closed = false;
    std::atomic<bool> exhausted{false};  // producer: moved past its last record, never touches it again
    std::atomic<int64_t> lastBatch{-1};  // the last batch holding records of it
};
// The reads of one kind: pairs (f[0] the -1 files, f[1] the -2 files) or unpaired reads (f[0]).  Record k of the
// stream is record k of its files back to back; the mates of a pair have the same ordinal, wherever the files end.
struct Stream {
    bool paired = false;
    std::vector<std::unique_ptr<InFile> > f[2];
};
struct InputSpec { const char* path; const char* data; size_t len; };

// The pipeline over a run's streams, in order (pairs before unpaired reads).  rdid, -s and -u count per stream, as
// the reference's per-source read counters do (pat.h:224, hisat2.cpp:1959-1964, 3319); the read loop ends for good at
// the first unit with rdid >= skip + upto (hisat2.cpp:3634), so a later stream is read only if the earlier one ended
// before that.  A batch never holds units of two streams.
int runStreams(ht2gpu_handle_t** hs, int nDev, const std::vector<InputSpec>* specs, int nStreams, bool pairedFirst,
               const ht2gpu_reads_input_t* in, ht2gpu_sink_fn sink, void* ctx, ht2gpu_read_routes_t* routes, ht2gpu_run_stats_t* st)
{
    ht2gpu_handle_t* h = hs[0];
    const bool route = routes && routes->mask;
    if (route && !routes->write) return HT2GPU_ERR_ARG;
    if (routes) { routes->n_spans = 0; routes->bytes = 0; routes->s_route = 0; }
    for (int i = 1; i < nDev; i++)
        if (!ht2_same_sam_output(h, hs[i])) { ht2gpu_set_error(h, "ht2gpu_run_reads_multi: the handles' SAM output settings differ"); return HT2GPU_ERR_ARG; }
    ht2gpu_run_stats_t S; memset(&S, 0, sizeof(S));
    const double t0 = nowS();
    unsigned nth = in->threads > 0 ? (unsigned)in->threads : std::thread::hardware_concurrency();
    if (nth < 1) nth = 1;
    if (nth > 64) nth = 64;
    const int perDev = ht2gpu_sam_slots(h);
    const int nSlots = perDev * nDev;          // stage k: device k % nDev, device slot k / nDev
    PipeCtx* C = ctxOf(h, nth, nSlots);
    std::lock_guard<std::mutex> runLock(C->mu);
    Ht2ThreadPool& pool = *C->pool;
    std::vector<Ht2HostBatch>& stage = C->stage;
    std::string err;
    const int device = ht2_handle_device(h);
    std::vector<Stream> streams((size_t)nStreams);
    auto eachFile = [&](const std::function<void(InFile&)>& fn) { for (auto& s : streams) for (auto& v : s.f) for (auto& F : v) fn(*F); };
    memset(&C->gz, 0, sizeof(C->gz));
    auto closeFile = [&](InFile& F) {   // the producer is done with it
        if (F.closed) return;
        if (F.gz) { F.gz->join(); if (F.started) addGunzipStats(C->gz, F.gz->st); }
        ht2_source_close(F.src);
        F.closed = true;
    };
    auto fail = [&](int rc, const std::string& m) { ht2gpu_set_error(h, m.c_str()); eachFile(closeFile); if (st) *st = S; return rc; };
    if (route) for (int i = 0; i < nDev; i++) { const int rc = ht2gpu_record_outcomes(hs[i], 1); if (rc) return fail(rc, ht2gpu_last_error(hs[i])); }
    // every file is opened (mapped) up front, so that a missing one fails the run before anything is aligned
    for (int s = 0; s < nStreams; s++) {
        streams[s].paired = pairedFirst && s == 0;
        for (int k = 0; k < (streams[s].paired ? 2 : 1); k++)
            for (const InputSpec& sp : specs[s * 2 + k]) {
                streams[s].f[k].emplace_back(new InFile());
                InFile& F = *streams[s].f[k].back();
                if (sp.path) { if (!ht2_source_open(F.src, sp.path, err)) return fail(HT2GPU_ERR_ARG, err); }
                else ht2_source_memory(F.src, sp.data, sp.len);
            }
    }
    for (int s = 0; s < nStreams; s++)
        for (auto& v : streams[s].f)
            for (auto& F : v) {
                if (isBzip2(F->src)) return fail(HT2GPU_ERR_ARG, kBzip2Msg);
                if (isGzip(F->src)) F->gz.reset(new Inflater()); else F->started = true;
            }
    // a gzip file is inflated from the time the producer reaches the file before it (or the run starts), so that
    // the next file's text is landing while the current one is read
    auto startFile = [&](Stream& S, int k, size_t fi, std::string& e) {
        for (size_t j = fi; j < fi + 2 && j < S.f[k].size(); j++) {
            InFile& F = *S.f[k][j];
            if (!F.started) { F.started = true; if (!F.gz->start(F.src, device, e)) return false; }
        }
        return true;
    };
    for (int k = 0; k < 2 && nStreams > 0; k++) if (!startFile(streams[0], k, 0, err)) return fail(HT2GPU_ERR_ARG, err);
    const bool fastq = in->format == 1;
    // -s / -u (hisat2.cpp:1959-1964, 3319): records [skip, skip + upto) of each stream
    const uint64_t r0 = in->skip;
    const uint64_t rEnd = in->upto ? r0 + in->upto : ~(uint64_t)0;
    const uint64_t perRead = in->batch_reads ? in->batch_reads : 4000000;   // large batches amortise the drain of the pool kernel's last reads
    Ht2ReadsOpts ro; ro.fastq = fastq; ro.trim5 = in->trim5; ro.trim3 = in->trim3; ro.phred64 = in->phred64 != 0; ro.seed = in->seed;

    // slot states: 0 free, 1 submitted
    std::mutex mu; std::condition_variable cv;
    std::vector<int> state((size_t)nSlots, 0);
    uint64_t submitted = 0;
    int prodRc = HT2GPU_OK; std::string prodErr; bool prodDone = false;
    double parseS = 0, submitS = 0, waitS = 0, sinkS = 0, indexS = 0;
    // the pieces of each submitted batch, with their record starts when routing (the producer keeps appending to the
    // sources' indexes meanwhile)
    struct RecPiece { InFile* fa; InFile* fb; const char* da; const char* db; uint64_t ra, rb, n; std::vector<uint64_t> a, b; };
    struct SlotRecs { bool paired; std::vector<RecPiece> pcs; };
    std::vector<SlotRecs> recs((size_t)nSlots);

    // The producer indexes the input only as far ahead as the next batch needs (so that indexing overlaps the device
    // work), parses the batch on all threads and submits it.  The first batch is a quarter of the others: the device
    // starts early, the later batches are large.
    std::thread producer([&]() {
        uint64_t i = 0;
        int rc = HT2GPU_OK;
        std::string e;
        std::vector<Ht2BatchPiece> pcs;
        for (int s = 0; s < nStreams && rc == HT2GPU_OK; s++) {
            Stream& SM = streams[s];
            const int nm = SM.paired ? 2 : 1;
            uint64_t perBatch = SM.paired ? (perRead + 1) / 2 : perRead;   // batch_reads counts reads, a unit here may be a pair
            if (perBatch < 1) perBatch = 1;
            size_t cf[2] = {0, 0}; uint64_t cp[2] = {0, 0};   // per mate: the cursor's file and its record in that file
            // Index mate k's files from the cursor on until `want` records are known, the files end (ended), or a
            // file still being inflated holds a quarter of them, so that the first batches are aligned while the rest
            // is decoded.  Returns the number of records known, at most want.
            auto indexAhead = [&](int k, uint64_t want, bool& ended) -> uint64_t {
                uint64_t have = 0; size_t fi = cf[k]; uint64_t pos = cp[k];
                ended = false;
                for (;;) {
                    if (fi >= SM.f[k].size()) { ended = true; break; }
                    if (!startFile(SM, k, fi, e)) { rc = HT2GPU_ERR_ARG; break; }
                    if (fi + 1 == SM.f[k].size() && s + 1 < nStreams && !startFile(streams[s + 1], 0, 0, e)) { rc = HT2GPU_ERR_ARG; break; }
                    Ht2ReadSource& src = SM.f[k][fi]->src;
                    while (!src.scanDone && src.nRecords() < pos + (want - have) && !(src.stream && have + src.nRecords() - pos >= (want + 3) / 4))
                        if (!ht2_source_scan(src, fastq, pool, (size_t)256 << 20, e)) { rc = HT2GPU_ERR_ARG; break; }
                    if (rc != HT2GPU_OK) break;
                    const uint64_t got = src.nRecords() - pos < want - have ? src.nRecords() - pos : want - have;
                    have += got;
                    if (have == want || !src.scanDone) break;
                    fi++; pos = 0;
                }
                return have;
            };
            // Units [r, r + n) of batch bi: the pieces in which every mate stays in one file (pieces == NULL: skipped
            // records).  A file's last batch is set before the file is marked exhausted, so that the consumer never
            // lets go of a file this batch still has to parse.
            auto take = [&](uint64_t r, uint64_t n, std::vector<Ht2BatchPiece>* pieces, uint64_t bi) {
                for (uint64_t u = 0; u < n;) {
                    uint64_t m = n - u;
                    bool moved = false;
                        for (int k = 0; k < nm; k++) {
                        if (cf[k] >= SM.f[k].size()) { rc = HT2GPU_ERR_ARG; e = "read front end: a batch ran past the end of its input"; return; }
                        InFile& F = *SM.f[k][cf[k]];
                        const uint64_t rem = F.src.nRecords() - cp[k];
                        if (rem == 0 && F.src.scanDone) { F.exhausted = true; cf[k]++; cp[k] = 0; moved = true; break; }
                        if (rem < m) m = rem;
                    }
                    if (moved) continue;
                    if (pieces) {
                        InFile* fb = SM.paired ? SM.f[1][cf[1]].get() : NULL;
                        SM.f[0][cf[0]]->lastBatch = (int64_t)bi;
                        if (fb) fb->lastBatch = (int64_t)bi;
                        Ht2BatchPiece pc = {&SM.f[0][cf[0]]->src, fb ? &fb->src : NULL, cp[0], SM.paired ? cp[1] : 0, m, r + u};
                        pieces->push_back(pc);
                    }
                    for (int k = 0; k < nm; k++) cp[k] += m;
                    u += m;
                }
                for (int k = 0; k < nm; k++)   // a file read to its end is let go at once
                    while (cf[k] < SM.f[k].size() && SM.f[k][cf[k]]->src.scanDone && cp[k] == SM.f[k][cf[k]]->src.nRecords()) {
                        SM.f[k][cf[k]]->exhausted = true; cf[k]++; cp[k] = 0;
                    }
            };
            // the units [r, r + want) that are there, or 0 at the end of the stream; a pair with only one mate is an error
            auto next = [&](uint64_t r, uint64_t want) -> uint64_t {
                const double ti = nowS();
                uint64_t n = ~(uint64_t)0, av[2] = {0, 0}; bool ended[2] = {false, false};
                for (int k = 0; k < nm && rc == HT2GPU_OK; k++) { av[k] = indexAhead(k, want, ended[k]); if (av[k] < n) n = av[k]; }
                indexS += nowS() - ti;
                if (rc != HT2GPU_OK) return 0;
                if (SM.paired && av[0] != av[1] && ended[av[0] < av[1] ? 0 : 1] && r + n < rEnd) {
                    rc = HT2GPU_ERR_ARG;
                    e = av[0] < av[1] ? "fewer reads in file specified with -1 than in file specified with -2"
                                      : "fewer reads in file specified with -2 than in file specified with -1";
                    return 0;
                }
                return n;
            };
            uint64_t r = 0;
            while (r < r0 && rc == HT2GPU_OK) {   // -s: the skipped records are indexed, not parsed
                const uint64_t want = r0 - r < perBatch ? r0 - r : perBatch;
                const uint64_t n = next(r, want);
                if (n == 0) break;
                take(r, n, NULL, 0);
                r += n;
            }
            bool more = true;   // the stream has units left
            while (rc == HT2GPU_OK && r >= r0) {
                const int slot = (int)(i % (uint64_t)nSlots);
                { std::unique_lock<std::mutex> lk(mu); cv.wait(lk, [&] { return state[slot] == 0 || prodRc != HT2GPU_OK; }); if (prodRc != HT2GPU_OK) { rc = prodRc; break; } }
                uint64_t want = (i == 0 && perBatch >= 8) ? perBatch / 4 : perBatch;
                if (r + want > rEnd) want = rEnd > r ? rEnd - r : 0;
                const uint64_t n = want ? next(r, want) : 0;
                if (rc != HT2GPU_OK) break;
                if (n == 0) { more = want == 0; break; }   // cut by -u, or nothing left
                pcs.clear();
                take(r, n, &pcs, i);
                if (rc == HT2GPU_OK) {
                    const double tp = nowS();
                    if (!ht2_parse_pieces(pcs.data(), pcs.size(), ro, stage[slot], pool, C->scratch, e)) rc = HT2GPU_ERR_ARG;
                    parseS += nowS() - tp;
                }
                if (rc == HT2GPU_OK) {
                    SlotRecs& sr = recs[slot];
                    sr.paired = SM.paired;
                    sr.pcs.resize(pcs.size());
                    // the cursor has moved past these records: find each piece's files again from the sources
                    for (size_t q = 0; q < pcs.size(); q++) {
                        RecPiece& rp = sr.pcs[q];
                        rp.fa = rp.fb = NULL;
                        for (int k = 0; k < nm; k++)
                            for (auto& F : SM.f[k]) if (&F->src == (k ? pcs[q].b : pcs[q].a)) { (k ? rp.fb : rp.fa) = F.get(); break; }
                        rp.da = pcs[q].a->data; rp.db = pcs[q].b ? pcs[q].b->data : NULL;
                        rp.ra = pcs[q].ra; rp.rb = pcs[q].rb; rp.n = pcs[q].n;
                        if (route) {
                            rp.a.assign(pcs[q].a->rec.begin() + (ptrdiff_t)rp.ra, pcs[q].a->rec.begin() + (ptrdiff_t)(rp.ra + rp.n) + 1);
                            if (pcs[q].b) rp.b.assign(pcs[q].b->rec.begin() + (ptrdiff_t)rp.rb, pcs[q].b->rec.begin() + (ptrdiff_t)(rp.rb + rp.n) + 1);
                        }
                    }
                }
                if (rc == HT2GPU_OK) {
                    Ht2HostBatch& hb = stage[slot];
                    ht2gpu_read_batch_t rb; memset(&rb, 0, sizeof(rb));
                    rb.n_reads = hb.n_reads; rb.paired = SM.paired ? 1 : 0; rb.seq = hb.seq; rb.qual = hb.haveQual ? hb.qual : NULL; rb.offs = hb.offs; rb.seeds = hb.seeds;
                    const double ts = nowS();
                    rc = ht2gpu_submit_sam(hs[slot % nDev], slot / nDev, &rb, hb.names, hb.nameOffs, hb.namesBytes);
                    submitS += nowS() - ts;
                    if (rc != HT2GPU_OK) e = ht2gpu_last_error(hs[slot % nDev]);
                }
                if (rc != HT2GPU_OK) break;
                std::lock_guard<std::mutex> lk(mu);
                state[slot] = 1; submitted = ++i;
                r += n;
                cv.notify_all();
            }
            // cut by -u: the read loop ends at the first unit with rdid >= skip + upto, if there is one
            if (rc == HT2GPU_OK && more && s + 1 < nStreams && next(r, 1) > 0) break;
        }
        std::lock_guard<std::mutex> lk(mu);
        if (rc != HT2GPU_OK && prodRc == HT2GPU_OK) { prodRc = rc; prodErr = e; }
        prodDone = true;
        cv.notify_all();
    });

    int rc = HT2GPU_OK;
    double routeS = 0;
    Router router(routes, fastq);
    for (uint64_t i = 0; ; i++) {
        const int slot = (int)(i % (uint64_t)nSlots);
        {
            std::unique_lock<std::mutex> lk(mu);
            cv.wait(lk, [&] { return submitted > i || prodRc != HT2GPU_OK || prodDone; });
            if (submitted <= i) { rc = prodRc; break; }   // the producer has finished (or failed)
        }
        ht2gpu_sam_result_t r;
        const double tw = nowS();
        rc = ht2gpu_wait_sam(hs[slot % nDev], slot / nDev, &r);
        waitS += nowS() - tw;
        if (rc != HT2GPU_OK) { prodErr = ht2gpu_last_error(hs[slot % nDev]); break; }
        S.n_batches++; S.n_units += r.n_units; S.n_reads += stage[slot].n_reads; S.sam_bytes += r.sam_len; S.n_err_reads += r.n_err_reads;
        S.ms_align += r.ms_align; S.ms_sam += r.ms_sam; S.ms_h2d += r.ms_h2d; S.ms_d2h += r.ms_d2h;
        S.h2d_bytes += r.h2d_bytes; S.d2h_bytes += r.d2h_bytes; S.n_launches += r.n_launches;
        const SlotRecs& sr = recs[slot];
        for (const RecPiece& rp : sr.pcs)   // nothing of a gzip file leaves the run before the file is verified
            for (InFile* F : {rp.fa, rp.fb})
                if (F && F->gz && !F->verified && rc == HT2GPU_OK) { rc = F->gz->verified(prodErr); F->verified = rc == HT2GPU_OK; }
        const double tk = nowS();
        if (rc == HT2GPU_OK && sink && r.sam_len) { if (sink(ctx, r.sam, r.sam_len) != 0) { rc = HT2GPU_ERR_ARG; prodErr = "the SAM sink reported an error"; } }
        sinkS += nowS() - tk;
        if (route && rc == HT2GPU_OK) {
            const double tr = nowS();
            const uint8_t* ob = NULL; uint32_t nu = 0;
            rc = ht2gpu_unit_outcomes(hs[slot % nDev], slot / nDev, &ob, &nu);
            if (rc != HT2GPU_OK) prodErr = ht2gpu_last_error(hs[slot % nDev]);
            else {
                uint64_t u = 0;
                for (const RecPiece& rp : sr.pcs) {
                    if (u + rp.n > nu) break;
                    router.batch(rp.da, rp.a.data(), rp.ra, rp.db, sr.paired ? rp.b.data() : NULL, rp.rb, rp.n, ob + u);
                    u += rp.n;
                }
                if (router.rc) { rc = HT2GPU_ERR_ARG; prodErr = "the read-file writer reported an error"; }
            }
            routeS += nowS() - tr;
        }
        // files the producer has left whose last batch is done: their text (and address space) is let go
        bool flushed = false;
        for (auto& sm : streams)
            for (auto& v : sm.f)
                for (auto& F : v)
                    if (!F->closed && F->exhausted && F->lastBatch <= (int64_t)i) {
                        if (route && !flushed) { router.finish(); flushed = true; }   // no pending span may point into it
                        closeFile(*F);
                    }
        { std::lock_guard<std::mutex> lk(mu); state[slot] = 0; if (rc != HT2GPU_OK) prodRc = rc; cv.notify_all(); }
        if (rc != HT2GPU_OK) break;
    }
    { std::lock_guard<std::mutex> lk(mu); if (rc != HT2GPU_OK && prodRc == HT2GPU_OK) prodRc = rc; cv.notify_all(); }
    producer.join();
    if (rc == HT2GPU_OK && prodRc != HT2GPU_OK) { rc = prodRc; }
    // a gzip file that was read from (or read to its end) is verified before the run succeeds; one whose records were
    // never needed (-u) is stopped
    eachFile([&](InFile& F) {
        if (rc == HT2GPU_OK && F.gz && F.started && !F.closed && !F.verified && (F.exhausted || F.lastBatch >= 0)) rc = F.gz->verified(prodErr);
    });
    eachFile([&](InFile& F) {   // a failed inflate explains a failed run better than what the parser made of its bytes
        if (F.gz && F.started && rc != HT2GPU_OK) {
            std::lock_guard<std::mutex> lk(F.gz->stream.mu);
            if (F.gz->stream.done && F.gz->stream.rc) { rc = F.gz->stream.rc; prodErr = F.gz->stream.err; }
        }
    });
    if (route) {
        const double tr = nowS();
        router.finish();
        if (router.rc && rc == HT2GPU_OK) { rc = HT2GPU_ERR_ARG; prodErr = "the read-file writer reported an error"; }
        routeS += nowS() - tr;
        routes->s_route = routeS;
        for (int i = 0; i < nDev; i++) ht2gpu_record_outcomes(hs[i], 0);
    }
    // drain anything still in flight after an error
    if (rc != HT2GPU_OK) for (int s = 0; s < nSlots; s++) if (state[s] == 1) { ht2gpu_sam_result_t r; ht2gpu_wait_sam(hs[s % nDev], s / nDev, &r); }
    eachFile(closeFile);
    S.s_index = indexS; S.s_parse = parseS; S.s_submit = submitS; S.s_wait = waitS; S.s_sink = sinkS; S.s_total = nowS() - t0;
    if (st) *st = S;
    if (rc != HT2GPU_OK) ht2gpu_set_error(h, prodErr.empty() ? "ht2gpu_run_reads failed" : prodErr.c_str());
    return rc;
}
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
    std::vector<InputSpec> sp[2];
    sp[0].push_back({in->path1, in->data1, in->len1});
    if (in->path2 || in->data2) sp[1].push_back({in->path2, in->data2, in->len2});
    return runStreams(hs, nDev, sp, 1, !sp[1].empty(), in, sink, ctx, routes, st);
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
    std::vector<InputSpec> sp[4];
    int stdinUses = 0;
    const char* const* lists[3] = {files->paths1, files->paths2, files->paths_u};
    const uint32_t counts[3] = {files->n1, files->n2, files->n_u};
    for (int l = 0; l < 3; l++) {
        if (counts[l] && !lists[l]) return refuse("ht2gpu_run_reads_files: a list with entries is NULL");
        for (uint32_t j = 0; j < counts[l]; j++) {
            const char* p = lists[l][j];
            if (!p || !*p) return refuse("ht2gpu_run_reads_files: an empty read file name");
            if (strcmp(p, "-") == 0 && ++stdinUses > 1) return refuse("standard input ('-') can be read only once");
            sp[files->n1 ? l : 0].push_back({p, NULL, 0});
        }
    }
    return runStreams(hs, nDev, sp, (files->n1 ? 1 : 0) + (files->n_u ? 1 : 0), files->n1 != 0, in, sink, ctx, routes, st);
}

// Host-only: parse a whole input into ONE batch (malloc'ed buffers).  No device is touched: this is the read
// front end on its own (tests, callers that batch for themselves).
extern "C" int ht2gpu_parse_reads(const ht2gpu_reads_input_t* in, ht2gpu_parsed_reads_t* out, char* errbuf, size_t errbuf_len)
{
    if (!in || !out) return HT2GPU_ERR_ARG;
    memset(out, 0, sizeof(*out));
    auto fail = [&](const std::string& m) { if (errbuf && errbuf_len) { strncpy(errbuf, m.c_str(), errbuf_len - 1); errbuf[errbuf_len - 1] = 0; } return HT2GPU_ERR_ARG; };
    unsigned nth = in->threads > 0 ? (unsigned)in->threads : std::thread::hardware_concurrency();
    if (nth < 1) nth = 1;
    if (nth > 64) nth = 64;
    Ht2ThreadPool pool(nth);
    Ht2ReadSource a, b;
    std::string err;
    const bool paired = in->path2 != NULL || in->data2 != NULL;
    if (in->path1) { if (!ht2_source_open(a, in->path1, err)) return fail(err); }
    else if (in->data1) ht2_source_memory(a, in->data1, in->len1);
    else return fail("no input");
    if (in->path2) { if (!ht2_source_open(b, in->path2, err)) { ht2_source_close(a); return fail(err); } }
    else if (in->data2) ht2_source_memory(b, in->data2, in->len2);
    if (refuseCompressed(a, err) || refuseCompressed(b, err)) { ht2_source_close(a); ht2_source_close(b); return fail(err); }
    const bool fastq = in->format == 1;
    bool ok = ht2_source_index(a, fastq, pool, err) && (!paired || ht2_source_index(b, fastq, pool, err));
    if (ok && paired && a.nRecords() != b.nRecords()) { ok = false; err = "mate files have different numbers of reads"; }
    Ht2HostBatch* hb = new Ht2HostBatch();
    if (ok) {
        uint64_t r0 = in->skip, r1 = a.nRecords();
        if (r0 > r1) r0 = r1;
        if (in->upto && r0 + in->upto < r1) r1 = r0 + in->upto;
        Ht2ReadsOpts ro; ro.fastq = fastq; ro.trim5 = in->trim5; ro.trim3 = in->trim3; ro.phred64 = in->phred64 != 0; ro.seed = in->seed;
        Ht2ParseScratch scratch;
        ok = ht2_parse_batch(a, paired ? &b : NULL, r0, r1, ro, *hb, pool, scratch, err);
    }
    ht2_source_close(a); ht2_source_close(b);
    if (!ok) { hb->freeAll(); delete hb; return fail(err); }
    out->batch.n_reads = hb->n_reads; out->batch.paired = paired ? 1 : 0; out->batch.seq = hb->seq; out->batch.qual = hb->haveQual ? hb->qual : NULL;
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
    auto fail = [&](const std::string& m) { if (errbuf && errbuf_len) { strncpy(errbuf, m.c_str(), errbuf_len - 1); errbuf[errbuf_len - 1] = 0; } return HT2GPU_ERR_ARG; };
    const double t0 = nowS();
    unsigned nth = in->threads > 0 ? (unsigned)in->threads : std::thread::hardware_concurrency();
    if (nth < 1) nth = 1;
    if (nth > 64) nth = 64;
    Ht2ThreadPool pool(nth);
    Ht2ReadSource a, b;
    std::string err;
    const bool paired = in->path2 != NULL || in->data2 != NULL;
    if (in->path1) { if (!ht2_source_open(a, in->path1, err)) return fail(err); }
    else if (in->data1) ht2_source_memory(a, in->data1, in->len1);
    else return fail("no input");
    if (in->path2) { if (!ht2_source_open(b, in->path2, err)) { ht2_source_close(a); return fail(err); } }
    else if (in->data2) ht2_source_memory(b, in->data2, in->len2);
    if (refuseCompressed(a, err) || refuseCompressed(b, err)) { ht2_source_close(a); ht2_source_close(b); return fail(err); }
    const bool fastq = in->format == 1;
    bool ok = ht2_source_index(a, fastq, pool, err) && (!paired || ht2_source_index(b, fastq, pool, err));
    if (ok && paired && a.nRecords() != b.nRecords()) { ok = false; err = "mate files have different numbers of reads"; }
    uint64_t r0 = in->skip, r1 = a.nRecords();
    if (r0 > r1) r0 = r1;
    if (in->upto && r0 + in->upto < r1) r1 = r0 + in->upto;
    if (ok && r1 - r0 != n_units) { ok = false; err = "the outcomes do not cover the input's " + std::to_string(r1 - r0) + " units"; }
    int rc = HT2GPU_OK;
    if (ok && routes->mask) {
        Router router(routes, fastq);
        router.batch(a.data, a.rec.data() + r0, r0, b.data, paired ? b.rec.data() + r0 : NULL, r0, r1 - r0, outcomes);
        router.finish();
        if (router.rc) { rc = HT2GPU_ERR_ARG; err = "the read-file writer reported an error"; }
    }
    ht2_source_close(a); ht2_source_close(b);
    routes->s_route = nowS() - t0;
    if (!ok) return fail(err);
    if (rc) return fail(err);
    return HT2GPU_OK;
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
