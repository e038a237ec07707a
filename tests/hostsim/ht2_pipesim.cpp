// ht2_pipesim.cpp -- TEST-ONLY host build of the read pipeline (ht2_pipeline.cpp + ht2_reads.cpp) against a fake device.
//
// The pipeline reaches the device only through the slot calls (ht2gpu_sam_slots / _submit_sam / _wait_sam), the outcome
// bytes, pinned memory, the handle's context and error slots, and ht2_gunzip_to.  This file defines those symbols:
//   - gzip input is inflated by the host backend of the same decoder source (Ht2zHostBackend);
//   - ht2gpu_wait_sam formats the batch from the caller's staging when it is waited for, not when it is submitted: the
//     staging must stay valid until the wait, so a pipeline that reuses it too early writes wrong reads.  One line per
//     read: name, sequence (ACGTN), qualities or '*', seed, tab-separated;
//   - ht2gpu_unit_outcomes gives unit u the outcome FNV-1a(name of its first read) & 7;
//   - ht2gpu_record_outcomes is refused while a slot of the handle holds a batch, as the library refuses it.
//
//   ht2_pipesim [-1 a,b -2 c,d] [-U e,f] [-f|-q] [-s N] [-u N] [--batch N] [-p N] [--gpus N] [--slots N]
//               [--un P] [--al P] [--un-conc P] [--al-conc P] [--al-conc-disc P]       ('%' in a -conc path: 1 / 2)
//               [--fail-wait K] [--sleep SEED] [--routed] -S out.txt [--log batches.txt]
//       runs ht2gpu_run_reads_files (ht2gpu_run_reads_routed on a single -U file or -1/-2 pair with --routed), writes
//       the reads, the read files and one line per waited batch ("device slot paired n_reads"), and prints the run's
//       stats, the summed gunzip stats and, per handle i, outcomes_i (recording on) and busy_i (slots holding a batch)
//       as "key=value" pairs.  --fail-wait K: the wait of batch K fails; where the handles have another slot, it first
//       waits (up to 5 s) until a later batch is in flight, and in_flight_at_fail is 1 if one was.  --sleep: each
//       wait sleeps a pseudo-random 0..500 us.  Exit 1 with the run's message on stderr when the run fails.
//   ht2_pipesim --parse [-1 a -2 b | -U a] [-f|-q] [-s N] [-u N] -S out.txt
//       the same lines from ht2gpu_parse_reads (the whole input as one batch).
//   ht2_pipesim --route [-1 a -2 b | -U a] [-f|-q] [-s N] [-u N] --outcomes F [--un P ...]
//       ht2gpu_route_reads of the input by the outcome bytes in F.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <chrono>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/ht2gpu.h"
#include "../../hisat2_b200/csrc/ht2_inflate.h"

namespace {
int gSlots = 2, gGpus = 1;
int64_t gFailWait = -1;
std::atomic<int> gBusy{0};   // slots of every handle that hold a batch
bool gInFlightAtFail = false;
uint64_t gSleepSeed = 0;
bool gSleep = false;
std::atomic<int64_t> gWaits{0};
std::mutex gLogMu;
std::vector<std::string> gLog;

uint32_t fnv1a(const char* s)
{
    uint32_t h = 2166136261u;
    for (; *s; s++) { h ^= (uint8_t)*s; h *= 16777619u; }
    return h;
}

void formatReads(const ht2gpu_read_batch_t& b, const char* names, const uint32_t* nameOffs, std::string& out)
{
    static const char kBase[] = "ACGTN";
    for (uint32_t i = 0; i < b.n_reads; i++) {
        out += names + nameOffs[i];
        out += '\t';
        for (uint64_t k = b.offs[i]; k < b.offs[i + 1]; k++) out += b.seq[k] < 5 ? kBase[b.seq[k]] : '?';
        out += '\t';
        if (b.qual) out.append((const char*)b.qual + b.offs[i], (size_t)(b.offs[i + 1] - b.offs[i]));
        else out += '*';
        out += '\t' + std::to_string(b.seeds[i]) + '\n';
    }
}
}

struct ht2gpu_handle {
    int device = 0;
    bool outcomes = false;
    struct Slot {
        bool busy = false;
        ht2gpu_read_batch_t rb;
        const char* names = NULL;
        const uint32_t* nameOffs = NULL;
        std::string sam;
        std::vector<uint8_t> out;
    };
    std::vector<Slot> slots;
    void* ctx = NULL;
    void (*release)(void*) = NULL;
    std::mutex errMu;
    std::string err;
};

extern "C" {
int ht2gpu_sam_slots(const ht2gpu_handle_t* h) { return (int)h->slots.size(); }
int ht2gpu_submit_sam(ht2gpu_handle_t* h, int slot, const ht2gpu_read_batch_t* batch, const char* names, const uint32_t* name_offs,
                      size_t names_bytes)
{
    if (slot < 0 || slot >= (int)h->slots.size() || h->slots[slot].busy) { ht2gpu_set_error(h, "fake device: slot in use"); return HT2GPU_ERR_ARG; }
    if (name_offs[batch->n_reads] != names_bytes) { ht2gpu_set_error(h, "fake device: names_bytes"); return HT2GPU_ERR_ARG; }
    ht2gpu_handle::Slot& s = h->slots[slot];
    s.busy = true; s.rb = *batch; s.names = names; s.nameOffs = name_offs;
    gBusy++;
    return HT2GPU_OK;
}
int ht2gpu_wait_sam(ht2gpu_handle_t* h, int slot, ht2gpu_sam_result_t* out)
{
    if (slot < 0 || slot >= (int)h->slots.size() || !h->slots[slot].busy) { ht2gpu_set_error(h, "fake device: nothing submitted"); return HT2GPU_ERR_ARG; }
    ht2gpu_handle::Slot& s = h->slots[slot];
    const int64_t k = gWaits++;
    if (k == gFailWait && gSlots * gGpus > 1) {   // fail with a later batch in flight, where the producer has one
        for (int t = 0; t < 5000 && gBusy < 2; t++) std::this_thread::sleep_for(std::chrono::milliseconds(1));
        gInFlightAtFail = gBusy >= 2;
    }
    s.busy = false;
    gBusy--;
    if (gSleep) {
        uint64_t x = (gSleepSeed + (uint64_t)k) * 0x9E3779B97F4A7C15ull;
        x ^= x >> 29;
        std::this_thread::sleep_for(std::chrono::microseconds(x % 500));
    }
    if (k == gFailWait) { ht2gpu_set_error(h, ("fake device: the wait of batch " + std::to_string(k) + " failed").c_str()); return HT2GPU_ERR_CUDA; }
    s.sam.clear();
    formatReads(s.rb, s.names, s.nameOffs, s.sam);
    const uint32_t per = s.rb.paired ? 2 : 1;
    s.out.clear();
    for (uint32_t i = 0; i < s.rb.n_reads; i += per) s.out.push_back((uint8_t)(fnv1a(s.names + s.nameOffs[i]) & 7));
    {
        std::lock_guard<std::mutex> lk(gLogMu);
        gLog.push_back(std::to_string(h->device) + " " + std::to_string(slot) + " " + std::to_string(s.rb.paired) + " " +
                       std::to_string(s.rb.n_reads));
    }
    memset(out, 0, sizeof(*out));
    out->sam = &s.sam[0]; out->sam_len = s.sam.size(); out->n_units = (uint32_t)s.out.size();
    return HT2GPU_OK;
}
int ht2gpu_record_outcomes(ht2gpu_handle_t* h, int enable)
{
    for (const ht2gpu_handle::Slot& s : h->slots)
        if (s.busy) { ht2gpu_set_error(h, "fake device: ht2gpu_record_outcomes: a batch is in flight"); return HT2GPU_ERR_ARG; }
    h->outcomes = enable != 0;
    return HT2GPU_OK;
}
int ht2gpu_unit_outcomes(ht2gpu_handle_t* h, int slot, const uint8_t** bytes, uint32_t* n_units)
{
    if (!h->outcomes || slot < 0 || slot >= (int)h->slots.size()) { ht2gpu_set_error(h, "fake device: outcomes are off"); return HT2GPU_ERR_ARG; }
    *bytes = h->slots[slot].out.data(); *n_units = (uint32_t)h->slots[slot].out.size();
    return HT2GPU_OK;
}
void* ht2gpu_host_alloc(size_t bytes) { return malloc(bytes ? bytes : 1); }
void ht2gpu_host_free(void* p) { free(p); }
void* ht2gpu_ctx_get(ht2gpu_handle_t* h) { return h->ctx; }
void ht2gpu_ctx_set(ht2gpu_handle_t* h, void* ctx, void (*release)(void*)) { h->ctx = ctx; h->release = release; }
void ht2gpu_set_error(ht2gpu_handle_t* h, const char* msg) { std::lock_guard<std::mutex> lk(h->errMu); h->err = msg; }
const char* ht2gpu_last_error(const ht2gpu_handle_t* h) { return h->err.c_str(); }
}

bool ht2_same_sam_output(const ht2gpu_handle_t*, const ht2gpu_handle_t*) { return true; }
int ht2_handle_device(const ht2gpu_handle_t* h) { return h->device; }
int ht2_gunzip_to(int, const void* src, size_t n, uint32_t chunkBytes, Ht2zOut& out, size_t* outLen, ht2gpu_gunzip_stats_t* stats,
                  std::string& err)
{
    ht2gpu_gunzip_stats_t S;
    memset(&S, 0, sizeof(S));
    Ht2zHostBackend be;
    const int rc = ht2z_gunzip_to(be, (const uint8_t*)src, n, chunkBytes, out, outLen, S, err);
    if (stats) *stats = S;
    return rc;
}

namespace {
struct ReadFiles {
    std::string path[HT2GPU_READS_N][2];
    FILE* f[HT2GPU_READS_N][2] = {};
    uint32_t mask = 0;
    void set(int which, const std::string& p)
    {
        mask |= 1u << which;
        const size_t pc = p.find('%');
        for (int m = 0; m < 2; m++)
            path[which][m] = which < HT2GPU_READS_UN_CONC ? p : pc == std::string::npos ? p + "." + std::to_string(m + 1)
                                                                                     : p.substr(0, pc) + std::to_string(m + 1) + p.substr(pc + 1);
    }
    bool open()
    {
        for (int w = 0; w < HT2GPU_READS_N; w++)
            for (int m = 0; m < (w < HT2GPU_READS_UN_CONC ? 1 : 2); m++)
                if ((mask >> w & 1) && !(f[w][m] = fopen(path[w][m].c_str(), "wb"))) return false;
        return true;
    }
    void close() { for (auto& w : f) for (FILE*& x : w) if (x) { fclose(x); x = NULL; } }
    static int write(void* ctx, int which, int mate, const char* data, size_t len)
    {
        FILE* x = ((ReadFiles*)ctx)->f[which][mate == 2 ? 1 : 0];
        return x && fwrite(data, 1, len, x) == len ? 0 : 1;
    }
};

std::vector<std::string> splitList(const char* s)
{
    std::vector<std::string> v;
    std::string cur;
    for (const char* p = s;; p++) {
        if (*p == ',' || !*p) { if (!cur.empty()) v.push_back(cur); cur.clear(); if (!*p) break; }
        else cur += *p;
    }
    return v;
}

int usage() { fprintf(stderr, "usage: see the comment at the top of ht2_pipesim.cpp\n"); return 2; }
}

int main(int argc, char** argv)
{
    std::vector<std::string> m1, m2, us;
    ht2gpu_reads_input_t in;
    memset(&in, 0, sizeof(in));
    ReadFiles rf;
    const char* samPath = NULL; const char* logPath = NULL; const char* outcomesPath = NULL;
    int gpus = 1, mode = 0;   // 0 run, 1 --parse, 2 --route
    bool routed = false;
    static const char* kReadOpt[HT2GPU_READS_N] = {"--un", "--al", "--un-conc", "--al-conc", "--al-conc-disc"};
    for (int i = 1; i < argc; i++) {
        const std::string a = argv[i];
        const bool hasVal = i + 1 < argc;
        auto val = [&]() { return argv[++i]; };
        if (a == "-f") in.format = 0;
        else if (a == "-q") in.format = 1;
        else if (a == "--parse") mode = 1;
        else if (a == "--route") mode = 2;
        else if (a == "--routed") routed = true;
        else if (!hasVal) return usage();
        else if (a == "-1") { for (auto& s : splitList(val())) m1.push_back(s); }
        else if (a == "-2") { for (auto& s : splitList(val())) m2.push_back(s); }
        else if (a == "-U") { for (auto& s : splitList(val())) us.push_back(s); }
        else if (a == "-s") in.skip = strtoull(val(), NULL, 10);
        else if (a == "-u") in.upto = strtoull(val(), NULL, 10);
        else if (a == "--batch") in.batch_reads = (uint32_t)strtoul(val(), NULL, 10);
        else if (a == "-p") in.threads = atoi(val());
        else if (a == "--gpus") gGpus = gpus = atoi(val());
        else if (a == "--slots") gSlots = atoi(val());
        else if (a == "--fail-wait") gFailWait = atoll(val());
        else if (a == "--sleep") { gSleep = true; gSleepSeed = strtoull(val(), NULL, 10); }
        else if (a == "-S") samPath = val();
        else if (a == "--log") logPath = val();
        else if (a == "--outcomes") outcomesPath = val();
        else {
            int w = 0;
            while (w < HT2GPU_READS_N && a != kReadOpt[w]) w++;
            if (w == HT2GPU_READS_N) return usage();
            rf.set(w, val());
        }
    }
    if (m1.size() != m2.size() || gpus < 1 || gSlots < 1) return usage();
    const bool single = (m1.empty() && us.size() == 1) || (us.empty() && m1.size() == 1);
    if (single) { in.path1 = m1.empty() ? us[0].c_str() : m1[0].c_str(); in.path2 = m1.empty() ? NULL : m2[0].c_str(); }
    if ((mode || routed) && !single) return usage();
    char err[1024] = "";

    if (mode == 1) {
        ht2gpu_parsed_reads_t p;
        if (ht2gpu_parse_reads(&in, &p, err, sizeof(err)) != HT2GPU_OK) { fprintf(stderr, "error: %s\n", err); return 1; }
        std::string text;
        formatReads(p.batch, p.names, p.name_offs, text);
        ht2gpu_free_parsed(&p);
        FILE* o = samPath ? fopen(samPath, "wb") : NULL;
        if (!o || fwrite(text.data(), 1, text.size(), o) != text.size() || fclose(o) != 0) return 2;
        return 0;
    }
    if (!rf.open()) { fprintf(stderr, "cannot open a read file\n"); return 2; }
    ht2gpu_read_routes_t routes;
    memset(&routes, 0, sizeof(routes));
    routes.mask = rf.mask; routes.write = ReadFiles::write; routes.ctx = &rf;
    if (mode == 2) {
        std::vector<uint8_t> oc;
        FILE* f = outcomesPath ? fopen(outcomesPath, "rb") : NULL;
        if (!f) return usage();
        for (int c; (c = fgetc(f)) != EOF;) oc.push_back((uint8_t)c);
        fclose(f);
        const int rc = ht2gpu_route_reads(&in, oc.data(), oc.size(), &routes, err, sizeof(err));
        rf.close();
        if (rc != HT2GPU_OK) { fprintf(stderr, "error: %s\n", err); return 1; }
        return 0;
    }

    FILE* fo = samPath ? fopen(samPath, "wb") : NULL;
    if (!fo) return usage();
    std::vector<ht2gpu_handle*> hs;
    for (int g = 0; g < gpus; g++) { hs.push_back(new ht2gpu_handle()); hs.back()->device = g; hs.back()->slots.resize((size_t)gSlots); }
    std::vector<const char*> p1, p2, pu;
    for (auto& s : m1) p1.push_back(s.c_str());
    for (auto& s : m2) p2.push_back(s.c_str());
    for (auto& s : us) pu.push_back(s.c_str());
    auto sink = [](void* ctx, const char* sam, size_t len) -> int { return fwrite(sam, 1, len, (FILE*)ctx) == len ? 0 : 1; };
    ht2gpu_run_stats_t st;
    memset(&st, 0, sizeof(st));
    int rc;
    if (routed) rc = ht2gpu_run_reads_routed(hs.data(), gpus, &in, sink, fo, &routes, &st);
    else {
        ht2gpu_reads_files_t lists;
        lists.paths1 = p1.data(); lists.n1 = (uint32_t)p1.size(); lists.paths2 = p2.data(); lists.n2 = (uint32_t)p2.size();
        lists.paths_u = pu.data(); lists.n_u = (uint32_t)pu.size();
        rc = ht2gpu_run_reads_files(hs.data(), gpus, &lists, &in, sink, fo, &routes, &st);
    }
    fclose(fo);
    rf.close();
    if (logPath) {
        FILE* lf = fopen(logPath, "wb");
        if (!lf) return 2;
        for (const std::string& l : gLog) fprintf(lf, "%s\n", l.c_str());
        fclose(lf);
    }
    ht2gpu_gunzip_stats_t gz;
    ht2gpu_run_gunzip_stats(hs[0], &gz);
    printf("n_reads=%llu n_units=%llu n_batches=%llu sam_bytes=%llu n_spans=%llu route_bytes=%llu gz_in_bytes=%llu gz_out_bytes=%llu "
           "gz_members=%llu\n",
           (unsigned long long)st.n_reads, (unsigned long long)st.n_units, (unsigned long long)st.n_batches,
           (unsigned long long)st.sam_bytes, (unsigned long long)routes.n_spans, (unsigned long long)routes.bytes,
           (unsigned long long)gz.in_bytes, (unsigned long long)gz.out_bytes, (unsigned long long)gz.members);
    for (int g = 0; g < gpus; g++) {
        int busy = 0;
        for (const ht2gpu_handle::Slot& s : hs[g]->slots) busy += s.busy;
        printf("outcomes_%d=%d busy_%d=%d\n", g, (int)hs[g]->outcomes, g, busy);
    }
    printf("in_flight_at_fail=%d\n", (int)gInFlightAtFail);
    if (rc != HT2GPU_OK) fprintf(stderr, "error: %s\n", ht2gpu_last_error(hs[0]));
    for (ht2gpu_handle* h : hs) { if (h->release) h->release(h->ctx); delete h; }
    return rc == HT2GPU_OK ? 0 : 1;
}
