// ht2_host.h -- host-side front end (read preparation, per-read parameters)
// and back end (AlnSinkWrap::finishRead-equivalent selection, MAPQ, SAM text)
// that sit either side of the device hot path.  These reproduce, outside the
// kernels, the reference steps SURVEY.md §9 lists as deciding byte equality:
//   hisat2.cpp:3360-3470 (minsc, filters, RNG seed), pat.h:55-91 (genRandSeed)
//   aln_sink.h:1939-2560 (finishRead), :2680-2755 (selectByScore)
//   unique.h:170-420 (BowtieMapq2), aln_sink.h:3024-3250 (appendMate)
//   sam.h:525-1010 (optional flags), aligner_result.cpp:660-1000 (StackedAln)
#ifndef HT2_HOST_H_
#define HT2_HOST_H_

#include <string>
#include <vector>

#include "ht2_core.h"
#include "ht2_index.h"
#include "../../include/ht2gpu.h"

struct Ht2HostRead {
    std::string name;
    std::vector<uint8_t> seq;   // codes 0..4
    std::vector<uint8_t> qual;  // raw ASCII
    uint32_t seed;
    int mate;                   // 0 unpaired, 1, 2
};

struct Ht2ReadFilters {
    bool nfilt, scfilt, lenfilt, qcfilt; // true = passes
    bool pass() const { return nfilt && scfilt && lenfilt && qcfilt; }
};

void ht2_default_params(Ht2Params& P, const Ht2Image& img, bool noSplicedAlignment);

// Per-read preprocessing (hisat2.cpp:3387-3467)
int64_t ht2_minsc(const Ht2Params& P, uint32_t rdlen);
// --score-min <type>,<const>,<coeff>: type one of C, L, S, G (simple_func.h)
bool ht2_set_score_min(Ht2Params& P, char type, double C, double L);
// --n-ceil <type>,<const>,<coeff> into P.nCeilTab; type one of C, L, S, G
bool ht2_set_n_ceil(Ht2Params& P, char type, double C, double L);
// --pen-canintronlen (which 0) / --pen-noncanintronlen (1) <type>,<const>,<coeff> into P.intronPen over the intron
// lengths 1 .. maxLen; false for a bad type or a function with more than HT2_INTRON_RUNS values there
bool ht2_set_intron_pen(Ht2Params& P, int which, char type, double C, double L, uint32_t maxLen);
// The longest intron the spliced scorer can be given: a novel intron is at most --max-intronlen (canCombine) and
// what a splice edit holds
inline uint32_t ht2_intron_cover(const Ht2ParamsCore& P) { return P.maxIntronLen < HT2_MAX_SPL_LEN ? P.maxIntronLen : HT2_MAX_SPL_LEN; }
// The spliced-alignment settings of o (penalties, intron bounds, --dta, --no-anchorstop, --tmo, --avoid-pseudogene)
// into P, as ht2gpu_open applies them; P.noSplicedAlignment must already be set.  Returns the refusal message of a
// configuration the device cannot reproduce, or NULL.
const char* ht2_apply_spliced_options(Ht2Params& P, const ht2gpu_options_t& o);
// nCeilTab: Ht2Params::nCeilTab; NULL = the default N ceiling
Ht2ReadFilters ht2_filters(const Ht2HostRead& rd, int64_t minsc, const int32_t* nCeilTab = NULL);
uint32_t ht2_gen_rand_seed(const Ht2HostRead& rd, uint32_t seed);
void ht2_fill_read(Ht2Read& dst, const Ht2HostRead& src);

// FASTA reader following FastaPatternSource::read (pat.cpp:725-849)
bool ht2_read_fasta(const char* path, std::vector<Ht2HostRead>& out, int mate, std::string& err);
bool ht2_read_fastq(const char* path, std::vector<Ht2HostRead>& out, int mate, std::string& err);
bool ht2_read_reads(const char* path, std::vector<Ht2HostRead>& out, int mate, std::string& err);  // by first character

// SAM output settings of a handle (ht2gpu_set_sam_output): --no-unal, --omit-sec-seq, --no-sq, --rg-id, --rg,
// --rna-strandness, --sam-no-qname-trunc, --no-templatelen-adjustment
struct Ht2SamOutput {
    bool noUnal = false, omitSecSeq = false, noSq = false;
    std::string rgId;                 // empty = no read group
    std::vector<std::string> rg;      // extra @RG fields, in the given order
    uint32_t rnaStrandness = 0;       // 0 unknown, 1 F, 2 R, 3 FR, 4 RF
    bool noQnameTrunc = false, noTlenAdj = false;
    std::string rgTag() const { return rgId.empty() ? std::string() : "RG:Z:" + rgId; }
    bool operator==(const Ht2SamOutput& o) const {
        return noUnal == o.noUnal && omitSecSeq == o.omitSecSeq && noSq == o.noSq && rgId == o.rgId && rg == o.rg &&
               rnaStrandness == o.rnaStrandness && noQnameTrunc == o.noQnameTrunc && noTlenAdj == o.noTlenAdj;
    }
};

// SAM.  refNames: the handle's reference names (ht2_index.h); NULL = the index's own
void ht2_sam_header(std::string& o, const Ht2Image& img, const Ht2SamOutput* so = NULL, const Ht2RefNames* refNames = NULL);
// ht2gpu_format_sam's body: host-only, shared with the test build.  counts != NULL: the units' outcomes are added
// to it (ReportingMetrics, the counting pass of ht2_sam.h)
bool ht2_format_batch(const Ht2Image& img, const Ht2Params& P, const ht2gpu_read_batch_t* b, const char* names,
                      const ht2gpu_result_batch_t* res, char** out, size_t* out_len, unsigned nthreads, const uint8_t* ssT = NULL,
                      uint32_t* colCount = NULL, struct Ht2SsRec* colRecs = NULL, uint32_t colCap = 0,
                      const Ht2SamOutput* so = NULL, ht2gpu_align_counts_t* counts = NULL, uint8_t* unitOut = NULL,
                      const Ht2RefNames* refNames = NULL);
// AlnSink::printAlSumm (aln_sink.h:1613-1816) with canRep = false (mhits is always 0, hisat2.cpp:1882-1884)
void ht2_format_align_summary(std::string& o, const ht2gpu_align_counts_t& c, bool newStyle, bool discord, bool mixed);

#endif
