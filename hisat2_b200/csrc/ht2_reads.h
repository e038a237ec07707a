// ht2_reads.h -- batched, multi-threaded read front end (host C++).
//
// The reference hands reads to its workers one at a time under a lock (PairedDualPatternSource::nextReadPair,
// pat.cpp:215-290; FastaPatternSource::read :725-849; FastqPatternSource::read :852-1290).  At GPU rates that
// is the bottleneck, so this front end works on whole files: the input is mapped (or given in memory), the
// record starts are indexed once by all threads, and each batch of records is parsed by all threads straight
// into the structure-of-arrays layout the device consumes (ht2gpu_read_batch_t): base codes 0..4, qualities as
// Phred+33 ASCII, per-read offsets, names, and the per-read pseudo-random seed (genRandSeed, pat.h:55-91).
// What it reproduces of the reference: alphabet (asc2dnacat / asc2dna), -5 / -3 trimming, --phred64,
// default names for unnamed reads (the read ordinal), mate-name fixing (Read::fixMateName, read.h:171-196),
// -s / -u (hisat2.cpp:1959-1964, 3319).
#ifndef HT2_READS_H_
#define HT2_READS_H_

#include <stdint.h>
#include <stddef.h>

#include <condition_variable>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

// A fixed pool of worker threads with a fork-join parallelFor.
class Ht2ThreadPool {
public:
    explicit Ht2ThreadPool(unsigned n);
    ~Ht2ThreadPool();
    unsigned size() const { return n_; }
    // runs fn(t) for t in [0, size()) on the pool's threads (the caller runs t = 0) and waits for all of them
    void run(const std::function<void(unsigned)>& fn);
private:
    unsigned n_;
    std::vector<std::thread> th_;
    std::mutex mu_;
    std::condition_variable cvWork_, cvDone_;
    const std::function<void(unsigned)>* fn_;
    uint64_t gen_;
    unsigned pending_;
    bool stop_;
    void worker(unsigned t);
};

// The bytes of a source that are still arriving (a gzip input being inflated): ht2_source_scan waits for them.
struct Ht2SourceStream {
    std::mutex mu;
    std::condition_variable cv;
    size_t avail = 0;           // bytes of the source written so far
    bool done = false;          // all written (or failed)
    int rc = 0;                 // nonzero: the source failed, err says why
    std::string err;
    void publish(size_t n) { { std::lock_guard<std::mutex> lk(mu); avail = n; } cv.notify_all(); }
    void finish(int r, const std::string& e) { { std::lock_guard<std::mutex> lk(mu); done = true; rc = r; err = e; } cv.notify_all(); }
};

struct Ht2ReadSource {          // one input file (or memory range) and its record index
    const char* data;
    size_t      size;
    void*       map;            // mmap base (NULL when not mapped)
    size_t      mapLen;
    std::vector<char> own;      // slurped input (stdin)
    Ht2SourceStream* stream;    // not NULL while the bytes are still arriving: size grows up to stream->avail
    std::vector<uint64_t> rec;  // offsets of the record starts found so far; a final sentinel == size once scanDone
    size_t      scanPos;        // incremental index: bytes scanned so far
    bool        scanDone;
    uint64_t    lineCarry;      // FASTQ: newlines before scanPos
    bool        strictFastq;    // FASTQ: still in the 4-lines-per-record fast path
    Ht2ReadSource() : data(NULL), size(0), map(NULL), mapLen(0), stream(NULL), scanPos(0), scanDone(false), lineCarry(0), strictFastq(true) {}
    // records whose END is known: record k spans [rec[k], rec[k+1])
    uint64_t nRecords() const { return rec.empty() ? 0 : rec.size() - 1; }
};

bool ht2_source_open(Ht2ReadSource& s, const char* path, std::string& err);        // "-" = stdin
void ht2_source_memory(Ht2ReadSource& s, const char* data, size_t n);
bool ht2_source_index(Ht2ReadSource& s, bool fastq, Ht2ThreadPool& pool, std::string& err);   // the whole input
// the next blockBytes (0 = the rest) of the input; appends to s.rec, sets s.scanDone at the end
bool ht2_source_scan(Ht2ReadSource& s, bool fastq, Ht2ThreadPool& pool, size_t blockBytes, std::string& err);
void ht2_source_close(Ht2ReadSource& s);

struct Ht2ReadsOpts {
    bool     fastq;
    int      trim5, trim3;      // -5 / -3
    bool     phred64;           // --phred64
    bool     solexa;            // --solexa-quals (wins over phred64, as charToPhred33 tests it first)
    bool     intQuals;          // --int-quals: space-separated integer qualities
    uint32_t seed;              // --seed
    Ht2ReadsOpts() : fastq(false), trim5(0), trim3(0), phred64(false), solexa(false), intQuals(false), seed(0) {}
};

// Host staging of one batch.  Buffers come from alloc / release (pinned memory when the CUDA side provides them).
struct Ht2HostBatch {
    uint8_t*  seq;  uint8_t* qual; uint64_t* offs; uint32_t* seeds; char* names; uint32_t* nameOffs;
    size_t    capBases, capReads, capNames;
    uint32_t  n_reads;
    size_t    namesBytes;
    bool      haveQual;
    void* (*alloc)(size_t);
    void  (*release)(void*);
    Ht2HostBatch() : seq(NULL), qual(NULL), offs(NULL), seeds(NULL), names(NULL), nameOffs(NULL), capBases(0), capReads(0), capNames(0),
                     n_reads(0), namesBytes(0), haveQual(false), alloc(NULL), release(NULL) {}
    void freeAll();
};

// Per-thread parse buffers, kept across batches (and across runs) so that steady-state parsing touches no fresh memory.
struct Ht2ParseScratch {
    void* impl;
    Ht2ParseScratch();
    ~Ht2ParseScratch();
};

// Parse records [r0, r1) of 'a' (and, for pairs, the same records of 'b': reads are interleaved mate 1, mate 2).
bool ht2_parse_batch(const Ht2ReadSource& a, const Ht2ReadSource* b, uint64_t r0, uint64_t r1, const Ht2ReadsOpts& o,
                     Ht2HostBatch& out, Ht2ThreadPool& pool, Ht2ParseScratch& scratch, std::string& err);

// A run of a batch's units that lies in one file per mate: records [ra, ra + n) of 'a' (with records [rb, rb + n) of
// 'b' for pairs), whose first unit has ordinal rdid in its stream.  A batch over several files is a list of pieces.
struct Ht2BatchPiece {
    const Ht2ReadSource* a;
    const Ht2ReadSource* b;
    uint64_t ra, rb, n, rdid;
};
bool ht2_parse_pieces(const Ht2BatchPiece* pcs, size_t npc, const Ht2ReadsOpts& o, Ht2HostBatch& out, Ht2ThreadPool& pool,
                      Ht2ParseScratch& scratch, std::string& err);

#endif
