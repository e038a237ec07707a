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
#include "ht2_reads.h"

bool ht2_same_sam_output(const ht2gpu_handle_t* a, const ht2gpu_handle_t* b);   // ht2_gpu.cu

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
    PipeCtx() : pool(NULL) {}
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
}

extern "C" int ht2gpu_run_reads(ht2gpu_handle_t* h, const ht2gpu_reads_input_t* in, ht2gpu_sink_fn sink, void* ctx, ht2gpu_run_stats_t* st)
{
    return ht2gpu_run_reads_multi(&h, 1, in, sink, ctx, st);
}

// The same pipeline over several devices of one process (hisat2-b200 --gpus N): batch i goes to handle i % n,
// the sink still receives the batches in input order.  The index is replicated (ht2gpu_open_peer), reads are the
// only thing that is sharded, no data-path collective.  Context (thread pool, pinned staging) lives in hs[0].
extern "C" int ht2gpu_run_reads_multi(ht2gpu_handle_t** hs, int nDev, const ht2gpu_reads_input_t* in, ht2gpu_sink_fn sink, void* ctx,
                                      ht2gpu_run_stats_t* st)
{
    if (!hs || nDev < 1 || !in) return HT2GPU_ERR_ARG;
    for (int i = 0; i < nDev; i++) if (!hs[i]) return HT2GPU_ERR_ARG;
    ht2gpu_handle_t* h = hs[0];
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
    auto fail = [&](int rc, const std::string& m) { ht2gpu_set_error(h, m.c_str()); ht2_source_close(a); ht2_source_close(b); if (st) *st = S; return rc; };
    if (in->path1) { if (!ht2_source_open(a, in->path1, err)) return fail(HT2GPU_ERR_ARG, err); }
    else if (in->data1) ht2_source_memory(a, in->data1, in->len1);
    else return fail(HT2GPU_ERR_ARG, "ht2gpu_run_reads: no input");
    if (in->path2) { if (!ht2_source_open(b, in->path2, err)) return fail(HT2GPU_ERR_ARG, err); }
    else if (in->data2) ht2_source_memory(b, in->data2, in->len2);
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
                while (!src.scanDone && src.nRecords() < r + want)
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
        const double tk = nowS();
        if (sink && r.sam_len) { if (sink(ctx, r.sam, r.sam_len) != 0) { rc = HT2GPU_ERR_ARG; prodErr = "the SAM sink reported an error"; } }
        sinkS += nowS() - tk;
        { std::lock_guard<std::mutex> lk(mu); state[slot] = 0; if (rc != HT2GPU_OK) prodRc = rc; cv.notify_all(); }
        if (rc != HT2GPU_OK) break;
    }
    { std::lock_guard<std::mutex> lk(mu); if (rc != HT2GPU_OK && prodRc == HT2GPU_OK) prodRc = rc; cv.notify_all(); }
    producer.join();
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
extern "C" void ht2gpu_free_parsed(ht2gpu_parsed_reads_t* p)
{
    if (p && p->priv) { Ht2HostBatch* hb = (Ht2HostBatch*)p->priv; hb->freeAll(); delete hb; p->priv = NULL; }
}
