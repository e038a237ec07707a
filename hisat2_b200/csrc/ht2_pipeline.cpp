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
// (output x mate) keeps one pending span; a record that continues it extends it, anything else flushes it first, so a
// run of consecutive records with the same destination reaches the callback as one span straight from the input.
struct Router {
    ht2gpu_read_routes_t* R;
    bool fastq;
    const char* data[2];             // mate 1 / unpaired, mate 2
    uint64_t pb[HT2GPU_READS_N * 2], pe[HT2GPU_READS_N * 2];
    int rc;
    Router(ht2gpu_read_routes_t* r, bool fq, const char* d1, const char* d2) : R(r), fastq(fq), rc(0)
    {
        data[0] = d1; data[1] = d2;
        for (int k = 0; k < HT2GPU_READS_N * 2; k++) pb[k] = pe[k] = 0;
    }
    void flush(int k)
    {
        if (pe[k] > pb[k] && rc == 0) {
            const int which = k >> 1, mate = which < HT2GPU_READS_UN_CONC ? 0 : (k & 1) + 1;
            R->n_spans++; R->bytes += pe[k] - pb[k];
            if (R->write(R->ctx, which, mate, data[k & 1] + pb[k], (size_t)(pe[k] - pb[k])) != 0) rc = 1;
        }
        pb[k] = pe[k] = 0;
    }
    void put(int which, int m, uint64_t b, uint64_t e)   // m: 0 mate 1 / unpaired, 1 mate 2
    {
        if (!(R->mask & (1u << which))) return;
        const int k = which * 2 + m;
        if (pe[k] != b || pe[k] == pb[k]) { flush(k); pb[k] = b; }
        pe[k] = e;
    }
    // Read::readOrigBuf of record r (rec[r] .. rec[r + 1]): the FASTQ parser keeps the blank lines before the first
    // record (pat.cpp:867-874), and FileBuf keeps at most LASTN_BUF_SZ = 8192 bytes (filebuf.h:109, 262)
    void span(const uint64_t* rec, uint64_t i, uint64_t r, uint64_t& b, uint64_t& e) const
    {
        b = (fastq && r == 0) ? 0 : rec[i]; e = rec[i + 1];
        if (e - b > 8192) e = b + 8192;
    }
    // units [r0, r0 + n): recA / recB hold the record starts rec[r0 .. r0 + n] of the two inputs
    void batch(const uint64_t* recA, const uint64_t* recB, uint64_t r0, uint64_t n, const uint8_t* out)
    {
        for (uint64_t i = 0; i < n && rc == 0; i++) {
            const uint8_t o = out[i];
            uint64_t b1, e1; span(recA, i, r0 + i, b1, e1);
            if (!recB) { put((o & HT2GPU_OUTCOME_AL1) ? HT2GPU_READS_AL : HT2GPU_READS_UN, 0, b1, e1); continue; }
            uint64_t b2, e2; span(recB, i, r0 + i, b2, e2);
            const int conc = (o & HT2GPU_OUTCOME_CONC) ? HT2GPU_READS_AL_CONC : HT2GPU_READS_UN_CONC;
            put(conc, 0, b1, e1); put(conc, 1, b2, e2);
            if (o & (HT2GPU_OUTCOME_AL1 | HT2GPU_OUTCOME_AL2)) { put(HT2GPU_READS_AL_CONC_DISC, 0, b1, e1); put(HT2GPU_READS_AL_CONC_DISC, 1, b2, e2); }
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

// The same pipeline over several devices of one process (hisat2-b200 --gpus N): batch i goes to handle i % n,
// the sink still receives the batches in input order.  The index is replicated (ht2gpu_open_peer), reads are the
// only thing that is sharded, no data-path collective.  Context (thread pool, pinned staging) lives in hs[0].
// With routes, every device records its units' outcomes and the records of batch i are routed right after its wait.
extern "C" int ht2gpu_run_reads_routed(ht2gpu_handle_t** hs, int nDev, const ht2gpu_reads_input_t* in, ht2gpu_sink_fn sink, void* ctx,
                                       ht2gpu_read_routes_t* routes, ht2gpu_run_stats_t* st)
{
    if (!hs || nDev < 1 || !in) return HT2GPU_ERR_ARG;
    for (int i = 0; i < nDev; i++) if (!hs[i]) return HT2GPU_ERR_ARG;
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
    Ht2ReadSource a, b;
    std::string err;
    const bool paired = in->path2 != NULL || in->data2 != NULL;
    std::unique_ptr<Inflater> gzs[2];   // gzip inputs being inflated into a / b
    auto joinInflate = [&]() { for (auto& g : gzs) if (g) g->join(); };
    auto fail = [&](int rc, const std::string& m) {
        ht2gpu_set_error(h, m.c_str()); joinInflate(); ht2_source_close(a); ht2_source_close(b); if (st) *st = S; return rc;
    };
    if (route) for (int i = 0; i < nDev; i++) { const int rc = ht2gpu_record_outcomes(hs[i], 1); if (rc) return fail(rc, ht2gpu_last_error(hs[i])); }
    // the record starts of each submitted batch (the producer keeps appending to the sources' indexes meanwhile)
    struct SlotRecs { uint64_t r0; std::vector<uint64_t> a, b; };
    std::vector<SlotRecs> recs(route ? (size_t)nSlots : 0);
    if (in->path1) { if (!ht2_source_open(a, in->path1, err)) return fail(HT2GPU_ERR_ARG, err); }
    else if (in->data1) ht2_source_memory(a, in->data1, in->len1);
    else return fail(HT2GPU_ERR_ARG, "ht2gpu_run_reads: no input");
    if (in->path2) { if (!ht2_source_open(b, in->path2, err)) return fail(HT2GPU_ERR_ARG, err); }
    else if (in->data2) ht2_source_memory(b, in->data2, in->len2);
    memset(&C->gz, 0, sizeof(C->gz));
    for (int k = 0; k < 2; k++) {   // the mate files are inflated at the same time, and while they are read
        Ht2ReadSource& src = k ? b : a;
        if (isBzip2(src)) return fail(HT2GPU_ERR_ARG, kBzip2Msg);
        if (!isGzip(src)) continue;
        gzs[k].reset(new Inflater());
        if (!gzs[k]->start(src, ht2_handle_device(h), err)) return fail(HT2GPU_ERR_ARG, err);
    }
    bool gzChecked = !gzs[0] && !gzs[1];
    const bool fastq = in->format == 1;
    // -s / -u (hisat2.cpp:1959-1964, 3319): records [skip, skip + upto)
    const uint64_t r0 = in->skip;
    const uint64_t rEnd = in->upto ? r0 + in->upto : ~(uint64_t)0;
    uint64_t perBatch = in->batch_reads ? in->batch_reads : 4000000;   // large batches amortise the drain of the pool kernel's last reads
    if (paired) perBatch = (perBatch + 1) / 2;   // batch_reads counts reads, a record here is a pair
    if (perBatch < 1) perBatch = 1;
    Ht2ReadsOpts ro; ro.fastq = fastq; ro.trim5 = in->trim5; ro.trim3 = in->trim3; ro.phred64 = in->phred64 != 0; ro.seed = in->seed;

    // slot states: 0 free, 1 submitted
    std::mutex mu; std::condition_variable cv;
    std::vector<int> state((size_t)nSlots, 0);
    uint64_t submitted = 0;
    int prodRc = HT2GPU_OK; std::string prodErr; bool prodDone = false;
    double parseS = 0, submitS = 0, waitS = 0, sinkS = 0, indexS = 0;

    // The producer indexes the input only as far ahead as the next batch needs (so that indexing overlaps the device
    // work), parses the batch on all threads and submits it.  The first batch is a quarter of the others: the device
    // starts early, the later batches are large.
    std::thread producer([&]() {
        uint64_t r = r0;
        for (uint64_t i = 0; ; i++) {
            const int slot = (int)(i % (uint64_t)nSlots);
            { std::unique_lock<std::mutex> lk(mu); cv.wait(lk, [&] { return state[slot] == 0 || prodRc != HT2GPU_OK; }); if (prodRc != HT2GPU_OK) break; }
            std::string e;
            int rc = HT2GPU_OK;
            uint64_t want = (i == 0 && perBatch >= 8) ? perBatch / 4 : perBatch;
            if (r + want > rEnd) want = rEnd > r ? rEnd - r : 0;
            // make sure the records [r, r + want) -- and the start of the one after -- are indexed in every source
            const double ti = nowS();
            for (int k = 0; k < (paired ? 2 : 1) && rc == HT2GPU_OK; k++) {
                Ht2ReadSource& src = k ? b : a;
                // a source still being inflated hands over what has landed once it holds a quarter of a batch, so
                // that the first batches are aligned while the rest is decoded
                while (!src.scanDone && src.nRecords() < r + want && !(src.stream && src.nRecords() >= r + (want + 3) / 4))
                    if (!ht2_source_scan(src, fastq, pool, (size_t)256 << 20, e)) { rc = HT2GPU_ERR_ARG; break; }
            }
            indexS += nowS() - ti;
            uint64_t avail = a.nRecords();
            if (paired && b.nRecords() < avail) avail = b.nRecords();
            uint64_t q1 = r + want < avail ? r + want : avail;
            if (rc == HT2GPU_OK && paired && a.scanDone && b.scanDone && a.nRecords() != b.nRecords() && q1 >= avail && q1 < rEnd) {
                rc = HT2GPU_ERR_ARG;
                e = a.nRecords() < b.nRecords() ? "fewer reads in file specified with -1 than in file specified with -2"
                                                : "fewer reads in file specified with -2 than in file specified with -1";
            }
            if (rc == HT2GPU_OK && q1 <= r) break;   // nothing left
            if (rc == HT2GPU_OK) {
                const double tp = nowS();
                if (!ht2_parse_batch(a, paired ? &b : NULL, r, q1, ro, stage[slot], pool, C->scratch, e)) rc = HT2GPU_ERR_ARG;
                parseS += nowS() - tp;
            }
            if (rc == HT2GPU_OK && route) {
                SlotRecs& sr = recs[slot];
                sr.r0 = r;
                sr.a.assign(a.rec.begin() + (ptrdiff_t)r, a.rec.begin() + (ptrdiff_t)q1 + 1);
                if (paired) sr.b.assign(b.rec.begin() + (ptrdiff_t)r, b.rec.begin() + (ptrdiff_t)q1 + 1);
            }
            if (rc == HT2GPU_OK) {
                Ht2HostBatch& hb = stage[slot];
                ht2gpu_read_batch_t rb; memset(&rb, 0, sizeof(rb));
                rb.n_reads = hb.n_reads; rb.paired = paired ? 1 : 0; rb.seq = hb.seq; rb.qual = hb.haveQual ? hb.qual : NULL; rb.offs = hb.offs; rb.seeds = hb.seeds;
                const double ts = nowS();
                rc = ht2gpu_submit_sam(hs[slot % nDev], slot / nDev, &rb, hb.names, hb.nameOffs, hb.namesBytes);
                submitS += nowS() - ts;
                if (rc != HT2GPU_OK) e = ht2gpu_last_error(hs[slot % nDev]);
            }
            std::lock_guard<std::mutex> lk(mu);
            if (rc != HT2GPU_OK) { prodRc = rc; prodErr = e; cv.notify_all(); break; }
            state[slot] = 1; submitted = i + 1;
            r = q1;
            cv.notify_all();
        }
        std::lock_guard<std::mutex> lk(mu);
        prodDone = true;
        cv.notify_all();
    });

    int rc = HT2GPU_OK;
    double routeS = 0;
    Router router(routes, fastq, a.data, b.data);
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
        if (!gzChecked) {   // nothing leaves the run before the gzip inputs are verified
            for (auto& g : gzs) if (g && rc == HT2GPU_OK && (rc = g->verified(prodErr)) != HT2GPU_OK) break;
            gzChecked = true;
        }
        const double tk = nowS();
        if (rc == HT2GPU_OK && sink && r.sam_len) { if (sink(ctx, r.sam, r.sam_len) != 0) { rc = HT2GPU_ERR_ARG; prodErr = "the SAM sink reported an error"; } }
        sinkS += nowS() - tk;
        if (route && rc == HT2GPU_OK) {
            const double tr = nowS();
            const uint8_t* ob = NULL; uint32_t nu = 0;
            rc = ht2gpu_unit_outcomes(hs[slot % nDev], slot / nDev, &ob, &nu);
            if (rc != HT2GPU_OK) prodErr = ht2gpu_last_error(hs[slot % nDev]);
            else {
                const SlotRecs& sr = recs[slot];
                router.batch(sr.a.data(), paired ? sr.b.data() : NULL, sr.r0, nu, ob);
                if (router.rc) { rc = HT2GPU_ERR_ARG; prodErr = "the read-file writer reported an error"; }
            }
            routeS += nowS() - tr;
        }
        { std::lock_guard<std::mutex> lk(mu); state[slot] = 0; if (rc != HT2GPU_OK) prodRc = rc; cv.notify_all(); }
        if (rc != HT2GPU_OK) break;
    }
    { std::lock_guard<std::mutex> lk(mu); if (rc != HT2GPU_OK && prodRc == HT2GPU_OK) prodRc = rc; cv.notify_all(); }
    producer.join();
    if (!gzChecked && rc == HT2GPU_OK) for (auto& g : gzs) if (g && rc == HT2GPU_OK) rc = g->verified(prodErr);
    for (auto& g : gzs)   // a failed inflate explains a failed run better than what the parser made of its bytes
        if (g && rc != HT2GPU_OK) { std::lock_guard<std::mutex> lk(g->stream.mu); if (g->stream.done && g->stream.rc) { rc = g->stream.rc; prodErr = g->stream.err; } }
    joinInflate();
    for (auto& g : gzs) if (g) addGunzipStats(C->gz, g->st);
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
    ht2_source_close(a); ht2_source_close(b);
    S.s_index = indexS; S.s_parse = parseS; S.s_submit = submitS; S.s_wait = waitS; S.s_sink = sinkS; S.s_total = nowS() - t0;
    if (st) *st = S;
    if (rc != HT2GPU_OK) ht2gpu_set_error(h, prodErr.empty() ? "ht2gpu_run_reads failed" : prodErr.c_str());
    return rc;
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
        Router router(routes, fastq, a.data, b.data);
        router.batch(a.rec.data() + r0, paired ? b.rec.data() + r0 : NULL, r0, r1 - r0, outcomes);
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
