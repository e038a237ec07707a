/* ht2gpu.h -- C ABI of the H100 HISAT2 alignment hot path.
 *
 * The reference has no FFI for alignment ("Alignment APIs: TODO",
 * hisat2lib/ht2.h:133-138); its seam is the per-thread C++ call
 *     HI_Aligner::initRead(s) + HI_Aligner::go(...)   hi_aligner.h:3992-4067
 * invoked once per read (pair) from multiseedSearchWorker_hisat2
 * (hisat2.cpp:3532-3559), whose outputs are the AlnRes objects handed to
 * AlnSinkWrap::report (aln_sink.h:2565) and finally printed by
 * AlnSinkWrap::finishRead (aln_sink.h:1939).  This library replaces that seam
 * with a batched call in the style of ht2.h (opaque handle, int error codes,
 * plain pointers and sizes, caller-visible result buffers):
 *
 *   ht2gpu_open          <-> HGFM ctor + loadIntoMemory      hisat2.cpp:3779-3825
 *                            BitPairReference ctor           hisat2.cpp:4040-4060
 *   ht2gpu_align_batch   <-> nextReadPair .. go() per read   hisat2.cpp:3278-3559
 *   ht2gpu_format_sam    <-> AlnSinkWrap::finishRead         aln_sink.h:1939-2560
 *   ht2gpu_close         <-> destructors
 *
 * No CPU fallback exists: every entry point that needs the device fails with
 * HT2GPU_ERR_CUDA when no CUDA device is usable.
 */
#ifndef HT2GPU_H_
#define HT2GPU_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HT2GPU_OK            0
#define HT2GPU_ERR_ARG      -1
#define HT2GPU_ERR_INDEX    -2   /* index files missing / malformed */
#define HT2GPU_ERR_CUDA     -3   /* no usable CUDA device or a CUDA call failed */
#define HT2GPU_ERR_CAPACITY -4   /* a result did not fit its container (seed search); per-read capacity overruns of the
                                   alignment path are reported per read, see ht2gpu_result_batch_t.n_err_reads */
#define HT2GPU_ERR_UNSUPPORTED -5

typedef struct ht2gpu_handle ht2gpu_handle_t;

/* Options mirror the hisat2 command line (hisat2.cpp:541-764).  Zero-initialise
 * and call ht2gpu_default_options, then override. */
typedef struct {
    int32_t  device;                 /* CUDA device ordinal */
    int32_t  no_spliced_alignment;   /* --no-spliced-alignment (must be 1 in this build) */
    int32_t  khits;                  /* -k; 0 = index default (5 linear / 10 graph) */
    int32_t  max_seeds;              /* --max-seeds; 0 = max(5, 2k) */
    int32_t  secondary;              /* --secondary */
    int32_t  mp_max, mp_min;         /* --mp 6,2 */
    int32_t  sp_max, sp_min;         /* --sp 2,1 */
    int32_t  np;                     /* --np 1 */
    int32_t  rdg_const, rdg_linear;  /* --rdg 5,3 */
    int32_t  rfg_const, rfg_linear;  /* --rfg 5,3 */
    int32_t  ignore_quals;           /* --ignore-quals WITHOUT --mp: the reference turns "--mp a,b" into MMP=Q,a,b, which
                                        re-enables quality-aware penalties (aligner_seed_policy.cpp:396-418); the CLI
                                        clears this flag when --mp is given */
    int32_t  nofw, norc;             /* --nofw / --norc */
    int32_t  min_frag, max_frag;     /* -I / -X */
    int32_t  no_mixed, no_discordant;
    uint32_t seed;                   /* --seed */
    int32_t  threads_per_block;      /* 0 = default */
    int32_t  blocks_per_sm;          /* 0 = default */
    int32_t  slots_per_lane;         /* state-regrouping mode: read slots per lane (2,4,8,16); 0 = default */
    int32_t  warp_per_read;          /* execution mode: 0/5 = block-shared slot pool (default), 2 = per-warp state regrouping, 4 = block-synchronous regrouping, 1 = one warp per read, 3 = one lane per read */
    /* --bowtie2-dp (hisat2.cpp:293, 1770; SplicedAligner::hybridSearch spliced_aligner.h:209-297): 0 = off,
     * 1 = dynamic-programming extension when the anchor search found nothing >= the minimum score, 2 = always.
     * The presets are spelled out by the caller exactly as hisat2.cpp:1892-1909 does:
     *   --sensitive      = bowtie2_dp 1 (unless given), khits raised to 10 only when -k < 10 was GIVEN, score-min L,0,-0.5
     *   --very-sensitive = bowtie2_dp 2, khits = max(k, 30), score-min L,0,-1 */
    int32_t  bowtie2_dp;
    int32_t  gbar;                   /* --gbar 4: no gaps within this many positions of either read end (DP only) */
    int32_t  score_min_type;         /* --score-min <type>,<const>,<coeff>: 'C', 'L', 'S' (sqrt) or 'G' (log); default L,0,-0.2 */
    double   score_min_const;
    double   score_min_coeff;
    /* The reference names the handle prints (@SQ, RNAME, RNEXT) and matches splice-site files against
     * (ht2gpu_load_splicesites, ht2gpu_write_novel_splicesites), hisat2.cpp:3957-3976: HT2GPU_CHR_NAMES_INDEX (0) as in
     * the index, _REMOVE (--remove-chrname) drops a leading "chr", _ADD (--add-chrname) puts "chr" before every name
     * that does not start with it.  Both flags together, or any other value, is HT2GPU_ERR_ARG before a device is
     * used (both: the reference's "--remove-chrname and --add-chrname cannot be used at the same time").
     * ht2gpu_open_peer takes the source handle's setting.  ht2gpu_ref_name and the ht2_* compatibility calls keep the
     * index's own names, as the reference's hisat2lib does: it has no such option. */
    int32_t  chr_names;
    /* --fr / --rf / --ff (hisat2.cpp:1166-1168, 3227-3236): the orientations of mate 1 and mate 2 on the forward strand
     * of a concordant pair.  HT2GPU_PE_FR (0) mate 1 forward, mate 2 reverse-complement; _RF the opposite; _FF both
     * forward.  Any other value is HT2GPU_ERR_ARG. */
    int32_t  pe_orient;
    /* --n-ceil <type>,<const>,<coeff> (NCEIL, aligner_seed_policy.cpp:547-549): the most Ns a read of length x may hold
     * (reads with more are filtered, YF:Z:NS) and the N ceiling of the --bowtie2-dp extension, as
     * max(0, const + coeff * F(x)) with F as for score_min_type.  0 = the default L,0,0.15. */
    int32_t  n_ceil_type;
    double   n_ceil_const;
    double   n_ceil_coeff;
    /* Spliced alignment (hisat2.cpp:1631-1728, 4075-4084).  A negative penalty, an intron bound below 20 or
     * min_intronlen > max_intronlen is HT2GPU_ERR_ARG before a device is used.
     *   pen_cansplice / pen_noncansplice / pen_conflictsplice: --pen-cansplice 0, --pen-noncansplice 12,
     *     --pen-conflictsplice 1000000 (a read spliced in both senses).
     *   can_intronlen_* / noncan_intronlen_*: --pen-canintronlen / --pen-noncanintronlen <type>,<const>,<coeff>, the
     *     intron-length penalty max(0, (int)(const + coeff * F(len))) of novel canonical and non-canonical junctions,
     *     F as for score_min_type.  Type 0 = the default G,-8,1.  A function that takes more than 1024 distinct
     *     values over the intron lengths up to max_intronlen is HT2GPU_ERR_UNSUPPORTED.
     *   min_intronlen / max_intronlen: --min-intronlen 20 / --max-intronlen 500000.  max_intronlen also bounds the
     *     distance of concordant mates under --no-spliced-alignment, as in the reference.
     *   dta: HT2GPU_DTA_STRINGTIE (--dta) needs anchors of 15 (canonical) / 20 (non-canonical) bases for long
     *     introns and makes the non-canonical function G,-8,2 whatever noncan_intronlen_* say; HT2GPU_DTA_CUFFLINKS
     *     (--dta-cufflinks) does the same and drops spliced alignments of unknown or conflicting sense.
     *   no_anchorstop: --no-anchorstop, partial searches do not stop at a unique anchor.
     *   tmo: --tmo, only alignments spliced through known sites (ht2gpu_load_splicesites) are reported.
     *   avoid_pseudogene: --avoid-pseudogene, in spliced mode an unspliced alignment within 10 000 bases of a loaded
     *     splice site ranks like a spliced one when the primary alignment is chosen (the SAM formatter's key).  No
     *     effect without a loaded DB.
     * ht2gpu_open_peer takes the source handle's settings. */
    int32_t  pen_cansplice, pen_noncansplice, pen_conflictsplice;
    int32_t  can_intronlen_type;
    double   can_intronlen_const, can_intronlen_coeff;
    int32_t  noncan_intronlen_type;
    double   noncan_intronlen_const, noncan_intronlen_coeff;
    int32_t  min_intronlen, max_intronlen;
    int32_t  dta;
    int32_t  no_anchorstop;
    int32_t  tmo;
    int32_t  avoid_pseudogene;
} ht2gpu_options_t;
enum { HT2GPU_CHR_NAMES_INDEX = 0, HT2GPU_CHR_NAMES_REMOVE = 1, HT2GPU_CHR_NAMES_ADD = 2 };
enum { HT2GPU_PE_FR = 0, HT2GPU_PE_RF = 1, HT2GPU_PE_FF = 2 };
enum { HT2GPU_DTA_NONE = 0, HT2GPU_DTA_STRINGTIE = 1, HT2GPU_DTA_CUFFLINKS = 2 };

/* A batch of reads, structure-of-arrays, host memory.  Read i occupies
 * seq[offs[i] .. offs[i+1]).  Bases are codes 0..4 (A,C,G,T,N) exactly as
 * Read::patFw holds them (read.h:47); qual is raw ASCII (NULL = all 'I', what
 * the FASTA parser assigns, pat.cpp:828).  seeds[i] is Read::seed
 * (pat.h:55-91).  When paired != 0 reads 2j and 2j+1 are mate 1 / mate 2. */
typedef struct {
    uint32_t        n_reads;
    int32_t         paired;
    const uint8_t*  seq;
    const uint8_t*  qual;
    const uint64_t* offs;     /* n_reads + 1 entries */
    const uint32_t* seeds;    /* n_reads entries (mate seeds are combined by the library) */
} ht2gpu_read_batch_t;

/* One nucleotide edit of an alignment: Edit (edit.h:41), positions in the
 * 5'->3' orientation of the read, relative to the soft-trimmed 5' end
 * (AlnRes::ned, aligner_result.cpp:111-118). */
typedef struct {
    uint32_t pos;
    uint8_t  chr;      /* reference char, '-' for a reference gap */
    uint8_t  qchr;     /* read char, '-' for a read gap */
    uint8_t  type;     /* 1 read gap, 2 ref gap, 3 mismatch, 5 splice (spliced mode; not produced by this build yet) */
    uint8_t  pad;      /* 0; splice: intron length bits 16-19, direction (1 unknown, 2 +, 3 -, 4 semi +, 5 semi -) in bits 4-6 */
    uint32_t snp_id;   /* ALT index or 0xffffffff; splice: IEEE-754 bits of the site's donor/acceptor probability.
                          A splice edit keeps the low 16 bits of the intron length in chr | qchr << 8 */
} ht2gpu_edit_t;

/* One reported alignment == the arguments reportHit gives AlnRes::init
 * (hi_aligner.h:6129-6166). */
typedef struct {
    uint32_t tidx;       /* reference id */
    uint32_t toff;       /* 0-based leftmost reference offset */
    int32_t  score;      /* AS:i */
    uint8_t  fw;         /* aligned to forward strand */
    uint8_t  mate;       /* 0 = mate 1 / unpaired, 1 = mate 2 */
    uint16_t n_edits;
    uint16_t trim5;      /* soft-trimmed bases at the read's 5' end */
    uint16_t trim3;
    uint32_t ref_extent; /* # reference chars covered */
    uint32_t edit_off;   /* first edit in ht2gpu_result_batch_t.edits */
} ht2gpu_aln_t;

/* Per-read (pair) summary.  alns[aln_off .. aln_off+n_aln[0]) are mate-1 /
 * unpaired alignments in the order the reference's sink received them
 * (rs1u_), followed by n_aln[1] mate-2 alignments (rs2u_).  Concordant pairs
 * (rs1_/rs2_) are index pairs into those two lists. */
typedef struct {
    uint32_t aln_off;
    uint16_t n_aln[2];
    uint32_t pair_off;
    uint32_t n_pairs;
    uint32_t rng_state;  /* RandomSource::last after go(); finishRead continues from it */
    uint32_t err;        /* 0, or HT2_ERR_* capacity bits: results unreliable */
    uint32_t n_lf;       /* LF-mapping steps executed (roofline accounting) */
    uint32_t alg_bytes;  /* algorithmic bytes touched: sides*sideSz + ftab + SA samples + 2-bit ref */
    uint32_t filt;       /* bit0 mate1 passed filters, bit1 mate2 passed filters; bits 4.. = YF reasons */
} ht2gpu_read_result_t;

typedef struct {
    uint32_t              n_reads;   /* reads (SE) or pairs (PE) */
    ht2gpu_read_result_t* reads;
    uint32_t              n_alns;
    ht2gpu_aln_t*         alns;
    uint32_t              n_edits;
    ht2gpu_edit_t*        edits;
    uint32_t              n_pairs;
    uint16_t*             pairs;     /* 2 entries per pair */
    /* timings of the last call, milliseconds (CUDA events on the launch stream) */
    float                 ms_h2d, ms_kernel, ms_d2h;
    uint64_t              h2d_bytes, d2h_bytes;
    uint32_t              n_launches;
    uint32_t              n_err_reads; /* reads (pairs) whose reads[i].err != 0: a fixed device-side capacity was exceeded,
                                          their results are unreliable; the call itself still returns HT2GPU_OK */
    void*                 priv;      /* owned by the library */
} ht2gpu_result_batch_t;

void ht2gpu_default_options(ht2gpu_options_t* opt);

/* Parse <index_base>.[1-8].ht2, build the packed image, upload it to HBM. */
int ht2gpu_open(const char* index_base, const ht2gpu_options_t* opt, ht2gpu_handle_t** out);
/* Same, from an image produced by another rank (see ht2gpu_image_*): host copy. */
int ht2gpu_open_image(const void* image, size_t bytes, const ht2gpu_options_t* opt, ht2gpu_handle_t** out);
/* Same, adopting an image that already sits in device memory (e.g. the
 * destination buffer of an NCCL broadcast).  The caller keeps ownership of
 * dev_image and must keep it alive until ht2gpu_close. host_image_prefix is the
 * leading part (at least the header) of the same image in host memory. */
int ht2gpu_open_device_image(const void* dev_image, size_t bytes, const void* host_image_prefix, size_t prefix_bytes,
                             const ht2gpu_options_t* opt, ht2gpu_handle_t** out);
/* Parse only (no device needed): returns a malloc'ed image the caller frees with ht2gpu_free_image. */
int ht2gpu_build_image(const char* index_base, void** image, size_t* bytes, char* errbuf, size_t errbuf_len);
void ht2gpu_free_image(void* image);
const void* ht2gpu_image_data(const ht2gpu_handle_t* h);   /* host copy of the image */
size_t ht2gpu_image_bytes(const ht2gpu_handle_t* h);
const void* ht2gpu_device_image(const ht2gpu_handle_t* h); /* device pointer */

/* Align a batch held in host memory: H2D copy, kernels, D2H copy. */
int ht2gpu_align_batch(ht2gpu_handle_t* h, const ht2gpu_read_batch_t* batch, ht2gpu_result_batch_t* res);
/* Upload a batch once and run the alignment kernels 'iters' times on the
 * resident copy (device-timed throughput; results of the last iteration). */
int ht2gpu_align_resident(ht2gpu_handle_t* h, const ht2gpu_read_batch_t* batch, int iters,
                          ht2gpu_result_batch_t* res);
void ht2gpu_free_results(ht2gpu_result_batch_t* res);

/* ---- SAM straight from the device -------------------------------------------
 * The whole per-batch pipeline of the reference's worker loop -- nextReadPair .. go() .. AlnSinkWrap::finishRead
 * (hisat2.cpp:3278-3559, aln_sink.h:1939-2560) -- on the GPU: H2D copy of the reads and their names, the
 * alignment kernel, the SAM kernels (selectByScore, MAPQ, CIGAR / MD:Z and the optional fields, csrc/ht2_sam.h),
 * D2H copy of the SAM text into pinned host memory.  Records are in read order (= --reorder) and byte-identical
 * to the reference's.  names: '\0'-terminated read names, concatenated; name_offs[i] = offset of read i's name,
 * name_offs[n_reads] = names_bytes.
 *
 * ht2gpu_submit_sam enqueues a batch on one of ht2gpu_sam_slots() slots and returns; ht2gpu_wait_sam blocks
 * until that batch is done and hands back its text (valid until the next submit on the same slot).  Slots have
 * their own streams and buffers, so the copies of one batch overlap the kernels of another; the host buffers
 * of a submitted batch must stay valid (ideally pinned) until its wait returns; a failed submit leaves the slot
 * free and nothing of it running.  One thread at a time per slot; ht2gpu_align_batch / _align_sam / _seed_search use slot 0. */
typedef struct {
    char*    sam;          /* pinned host memory owned by the library, '\0'-terminated */
    size_t   sam_len;
    uint32_t n_units;      /* reads (SE) or pairs (PE) of the batch */
    uint32_t n_alns;       /* alignments the kernel reported (before selection) */
    uint32_t n_err_reads;  /* units that exceeded a device-side capacity (their records are unreliable) */
    uint32_t n_launches;   /* kernels launched for this batch */
    float    ms_h2d, ms_align, ms_sam, ms_d2h;   /* CUDA events on the slot's stream */
    uint64_t h2d_bytes, d2h_bytes;
    uint32_t sam_unplanned; /* 1: the batch's records did not fit the SAM plan's arena and were printed one unit per thread */
    uint32_t pad;
} ht2gpu_sam_result_t;

int ht2gpu_sam_slots(const ht2gpu_handle_t* h);
int ht2gpu_submit_sam(ht2gpu_handle_t* h, int slot, const ht2gpu_read_batch_t* batch, const char* names,
                      const uint32_t* name_offs, size_t names_bytes);
int ht2gpu_wait_sam(ht2gpu_handle_t* h, int slot, ht2gpu_sam_result_t* out);
/* submit + wait on slot 0 */
int ht2gpu_align_sam(ht2gpu_handle_t* h, const ht2gpu_read_batch_t* batch, const char* names, const uint32_t* name_offs,
                     size_t names_bytes, ht2gpu_sam_result_t* out);

/* ---- reads in, SAM out ---------------------------------------------------------
 * The reference's whole worker loop (multiseedSearchWorker_hisat2 + PatternSource + OutputQueue,
 * hisat2.cpp:3278-3696, pat.cpp:215-290, outq.cpp:51-99) as one call: FASTA / FASTQ bytes (files or host
 * memory) are parsed by all host threads, aligned and formatted on the device in overlapped batches, and the SAM
 * text is handed to 'sink' batch by batch, in read order (= --reorder).  sink receives pointers into pinned
 * host memory that are valid only during the call; it returns 0 to continue. */
typedef int (*ht2gpu_sink_fn)(void* ctx, const char* sam, size_t len);
typedef struct {
    const char* path1;      /* -U / -1 file ("-" = stdin), or NULL to use data1 */
    const char* path2;      /* -2 file, or NULL */
    const char* data1;      /* reads already in host memory */
    size_t      len1;
    const char* data2;
    size_t      len2;
    int32_t     format;     /* 0 = FASTA (-f), 1 = FASTQ (-q) */
    int32_t     trim5, trim3;   /* -5 / -3 */
    int32_t     phred64;    /* --phred64 */
    uint32_t    seed;       /* --seed (per-read seeds, pat.h:55-91) */
    uint64_t    skip;       /* -s */
    uint64_t    upto;       /* -u; 0 = no limit */
    uint32_t    batch_reads;/* reads per device batch; 0 = 4,000,000 */
    int32_t     threads;    /* host parser threads (-p); 0 = all cores, at most 64 */
    /* --solexa-quals: FASTQ qualities are Solexa-scaled, 64-based (qual.h:46-50, 106-136); wins over phred64.
     * --int-quals: the quality line is space-separated integers (pat.cpp:997-1030), Phred unless solexa_quals; one
     * value more than bases is cut, fewer or more is an error.  Qualities are converted before the per-read seed. */
    int32_t     solexa_quals;
    int32_t     int_quals;
} ht2gpu_reads_input_t;
typedef struct {
    uint64_t n_reads, n_units, sam_bytes, n_err_reads, n_batches;
    double   s_index, s_parse, s_total;          /* host wall clock: record indexing, batch parsing (overlapped), whole call */
    double   s_submit, s_wait, s_sink;           /* host wall clock inside ht2gpu_submit_sam / ht2gpu_wait_sam / the sink */
    float    ms_h2d, ms_align, ms_sam, ms_d2h;   /* summed CUDA-event times of the batches */
    uint64_t h2d_bytes, d2h_bytes;
    uint32_t n_launches, pad;
} ht2gpu_run_stats_t;
int ht2gpu_run_reads(ht2gpu_handle_t* h, const ht2gpu_reads_input_t* in, ht2gpu_sink_fn sink, void* ctx, ht2gpu_run_stats_t* stats);
/* The same over several devices of ONE process (hisat2 -p N + --reorder, hisat2.cpp:3657-3696, outq.cpp:51-99, with
 * GPUs in place of threads): batch i runs on hs[i % n], the sink receives the batches in input order.  Every handle
 * holds a replica of the same index (ht2gpu_open_peer); reads are the only thing that is sharded.  Handles whose
 * SAM output settings (ht2gpu_set_sam_output) differ are refused with HT2GPU_ERR_ARG. */
int ht2gpu_run_reads_multi(ht2gpu_handle_t** hs, int n, const ht2gpu_reads_input_t* in, ht2gpu_sink_fn sink, void* ctx,
                           ht2gpu_run_stats_t* stats);

/* ---- reads routed to files by their outcome (--un, --al, --un-conc, --al-conc, --al-conc-disc) -----------------
 * The hisat2 wrapper's read files (hisat2:546-650), decided from the same choices that set the SAM FLAGs of each read's
 * primary records.  With ht2gpu_record_outcomes(h, 1) the SAM counting pass stores one byte per unit (read or pair);
 * ht2gpu_unit_outcomes hands back the bytes of the slot's last ht2gpu_wait_sam (valid until the next submit on that
 * slot).  Off by default, and refused while a batch is in flight. */
#define HT2GPU_OUTCOME_AL1  1   /* mate 1 / the unpaired read has an alignment (its primary record has FLAG & 4 clear) */
#define HT2GPU_OUTCOME_AL2  2   /* mate 2 has an alignment */
#define HT2GPU_OUTCOME_CONC 4   /* the primary records are concordant (FLAG & 2) */
int ht2gpu_record_outcomes(ht2gpu_handle_t* h, int enable);
int ht2gpu_unit_outcomes(ht2gpu_handle_t* h, int slot, const uint8_t** bytes, uint32_t* n_units);

/* The five outputs; bit (1 << which) of ht2gpu_read_routes_t.mask selects one.  Unpaired reads go to UN / AL, pairs to
 * UN_CONC / AL_CONC (mate 1 and mate 2 to separate files) and AL_CONC_DISC (both mates of every pair with at least
 * one aligned mate).  write receives the records' original input text, runs of consecutive records with the same
 * destination as one span straight from the input (mate 0 = unpaired, 1 / 2); it returns 0 to continue.  What is
 * written is what the reference's parser keeps of a record (Read::readOrigBuf): the bytes from its '>' / '@' up to
 * the next record's, with the blank lines before the first FASTQ record, and at most its first 8192 bytes. */
enum { HT2GPU_READS_UN = 0, HT2GPU_READS_AL, HT2GPU_READS_UN_CONC, HT2GPU_READS_AL_CONC, HT2GPU_READS_AL_CONC_DISC, HT2GPU_READS_N };
typedef int (*ht2gpu_reads_fn)(void* ctx, int which, int mate, const char* data, size_t len);
typedef struct {
    uint32_t        mask;
    ht2gpu_reads_fn write;
    void*           ctx;
    /* filled by the call */
    uint64_t        n_spans, bytes;
    double          s_route;        /* host wall clock spent routing, write calls included */
} ht2gpu_read_routes_t;
/* ht2gpu_run_reads_multi that also routes every batch's records by their outcomes, in read order; routes = NULL or a
 * zero mask is ht2gpu_run_reads_multi. */
int ht2gpu_run_reads_routed(ht2gpu_handle_t** hs, int n, const ht2gpu_reads_input_t* in, ht2gpu_sink_fn sink, void* ctx,
                            ht2gpu_read_routes_t* routes, ht2gpu_run_stats_t* stats);
/* Lists of read files (hisat2 -1 a1,a2 -2 b1,b2 -U u1,u2).  The -1 files back to back and the -2 files back to back
 * are one stream of pairs: record k of the one goes with record k of the other, wherever the files end.  The -U
 * files back to back are one stream of unpaired reads, aligned after every pair (PairedDualPatternSource,
 * pat.cpp:234-304).  Each file keeps its own records and is detected as plain or gzip on its own.  "-" (stdin) may
 * appear once over all lists. */
typedef struct {
    const char* const* paths1;  uint32_t n1;    /* -1 */
    const char* const* paths2;  uint32_t n2;    /* -2: as many as -1 */
    const char* const* paths_u; uint32_t n_u;   /* -U */
} ht2gpu_reads_files_t;
/* ht2gpu_run_reads_routed over lists of files.  Format, trims, --phred64, seed, batch size and threads come from
 * 'in', whose path and data fields must be NULL.  Read ids, default names of unnamed reads, -s and -u count per stream
 * (the first unpaired read is rdid 0 again); the read loop ends at the first unit with rdid >= skip + upto, so with -u
 * below the number of pairs no unpaired read is aligned.  A batch holds units of one stream only.  Pairs are routed to
 * the -conc outputs, unpaired reads to UN / AL.  Different -1 and -2 counts are HT2GPU_ERR_ARG with the reference's
 * message (hisat2.cpp:1911-1913). */
int ht2gpu_run_reads_files(ht2gpu_handle_t** hs, int n, const ht2gpu_reads_files_t* files, const ht2gpu_reads_input_t* in,
                           ht2gpu_sink_fn sink, void* ctx, ht2gpu_read_routes_t* routes, ht2gpu_run_stats_t* stats);
/* Host only (no device): route the records of an input (after -s / -u) by outcomes[0 .. n_units), e.g. the bytes of
 * ht2gpu_unit_outcomes of callers that batch through ht2gpu_align_sam.  n_units must equal the input's units. */
int ht2gpu_route_reads(const ht2gpu_reads_input_t* in, const uint8_t* outcomes, uint64_t n_units, ht2gpu_read_routes_t* routes,
                       char* errbuf, size_t errbuf_len);

/* ---- gzip input, inflated on the device --------------------------------------------------------------------------
 * ht2gpu_gunzip inflates a complete gzip file (one or more RFC 1952 members: gzip, pigz, BGZF, `cat a.gz b.gz`) on a
 * device: the compressed input is cut into chunks that are decoded in parallel from the first block start found in each
 * (DESIGN.md 5.2).  Every member's CRC-32 and ISIZE are checked; trailing zero bytes are ignored, anything else after the
 * last member is an error.  Corrupt input returns HT2GPU_ERR_DATA with no output (ht2gpu_gunzip_error has the reason).
 * Device memory is a fixed cap (ht2gpu_gunzip_stats_t.peak_device_bytes) whatever the file size, all freed on return.
 * *out is malloc'ed (free with ht2gpu_free_text).
 * ht2gpu_run_reads(_multi, _routed) inflate a path or data1 / data2 buffer that begins with 1f 8b this way, on the
 * first handle's device, while its reads are parsed and aligned; no SAM reaches the sink before every member is
 * verified.  ht2gpu_parse_reads and ht2gpu_route_reads refuse such input. */
#define HT2GPU_ERR_DATA -6   /* compressed input that is not valid gzip */
typedef struct {
    uint32_t chunk_bytes;   /* compressed bytes per chunk; 0 = chosen per window from the compression ratio */
    uint32_t reserved;
} ht2gpu_gunzip_opts_t;
typedef struct {
    uint64_t in_bytes, out_bytes;
    uint64_t members, blocks;
    uint64_t chunks;                        /* chunks whose output was kept, each counted once */
    uint64_t chunks_confirmed;              /* of those, decoded speculatively from a confirmed start */
    uint64_t chunks_merged_no_candidate;    /* chunks in which no block start was found, decoded by their predecessor */
    uint64_t chunks_merged_false_positive;  /* chunks whose start was not a real one, decoded by their predecessor */
    uint64_t windows, decode_rounds;        /* windows of compressed input; launches of the chunk decoder */
    uint64_t windows_cut;                   /* windows ended early because a chunk's output (or its list of member
                                               ends) was full: the rest of such a window is decoded again */
    uint64_t peak_device_bytes;             /* device memory the call allocates; all of it is allocated up front */
    uint32_t chunk_bytes, pad;              /* chunk size of the last window */
    float    ms_find, ms_decode, ms_window, ms_replace, ms_crc, ms_copy;   /* CUDA-event time per phase */
} ht2gpu_gunzip_stats_t;
int ht2gpu_gunzip(int device, const void* src, size_t n, const ht2gpu_gunzip_opts_t* opts, char** out, size_t* out_len,
                  ht2gpu_gunzip_stats_t* stats);
/* The reason the calling thread's last ht2gpu_gunzip (or gzip input of a run) failed. */
const char* ht2gpu_gunzip_error(void);
/* The summed inflate stats of the gzip inputs of the handle's last ht2gpu_run_reads(_multi, _routed) (zero when its
 * inputs were plain text). */
int ht2gpu_run_gunzip_stats(ht2gpu_handle_t* h, ht2gpu_gunzip_stats_t* stats);

/* Replicate an open index onto another device of this process: the packed image is copied device to device
 * (cudaMemcpyPeer: NVLink / NVSwitch when peer access exists), options as given (opt->device = the target). */
int ht2gpu_open_peer(const ht2gpu_handle_t* src, const ht2gpu_options_t* opt, ht2gpu_handle_t** out);

/* The read front end on its own, host only (no device): the whole input as ONE batch in the layout
 * ht2gpu_align_batch / ht2gpu_submit_sam take (FastaPatternSource / FastqPatternSource + genRandSeed +
 * fixMateName, pat.cpp:725-1290, pat.h:55-91, read.h:171-196). */
typedef struct {
    ht2gpu_read_batch_t batch;
    char*     names;        /* '\0'-terminated names, concatenated */
    uint32_t* name_offs;    /* batch.n_reads + 1 entries */
    size_t    names_bytes;
    void*     priv;
} ht2gpu_parsed_reads_t;
int ht2gpu_parse_reads(const ht2gpu_reads_input_t* in, ht2gpu_parsed_reads_t* out, char* errbuf, size_t errbuf_len);
void ht2gpu_free_parsed(ht2gpu_parsed_reads_t* p);

/* Pinned host memory for batches handed to ht2gpu_submit_sam (asynchronous H2D copies need it). */
void* ht2gpu_host_alloc(size_t bytes);
void ht2gpu_host_free(void* p);
void ht2gpu_set_error(ht2gpu_handle_t* h, const char* msg);
/* An opaque per-handle context slot (the pipeline keeps its thread pool and pinned staging there); freed by ht2gpu_close. */
void* ht2gpu_ctx_get(ht2gpu_handle_t* h);
void ht2gpu_ctx_set(ht2gpu_handle_t* h, void* ctx, void (*release)(void*));

/* ---- seed search on its own (linear AND graph/SNP indexes) -------------------
 * For every read and strand (fw first): the chain of partial searches
 * HI_Aligner::partialSearch produces when driven like nextBWT (hi_aligner.h:
 * 6361-6601, 4720-4751), i.e. the BWTHit list of ReadBWTHit (hi_aligner.h:108-
 * 391), and for hits whose node range is <= max_range the joined/text
 * coordinate of every element (GFM::getOffset gfm.h:5682, joinedToTextOff
 * :5527; element i = first BW row of node i, group_walk.h:545-560).
 * Uses the batch's seq/offs only (unpaired view). */
typedef struct {
    uint32_t read;                   /* index into the batch */
    uint8_t  fw;                     /* 1 = forward strand of the read */
    uint8_t  hit_type;               /* 1 candidate, 2 pseudogene, 3 anchor (hi_aligner.h:96-100) */
    uint8_t  pseudogene_stop, anchor_stop;
    uint32_t bwoff, len;             /* offset from the read's 3' end, # bases consumed */
    uint32_t top, bot;               /* BW row range; 0xffffffff = blank hit */
    uint32_t node_top, node_bot;     /* node range (== row range on linear indexes) */
    uint32_t n_iedges, iedge_off;    /* in-edge list: pairs (node index in range, # extra incoming edges) */
    uint32_t n_coords, coord_off;
} ht2gpu_seed_hit_t;

typedef struct {
    uint32_t row;                    /* BW row the walk started from */
    uint32_t joined_off;             /* offset in the joined reference */
    uint32_t tidx, toff;             /* 0xffffffff tidx: not inside a reference fragment */
} ht2gpu_seed_coord_t;

typedef struct {
    uint32_t             n_reads;
    uint32_t*            first_hit;  /* n_reads + 1 entries: hits of read i are [first_hit[i], first_hit[i+1]) */
    uint32_t             n_hits;
    ht2gpu_seed_hit_t*   hits;
    uint32_t             n_iedges;
    uint16_t*            iedges;     /* 2 entries per pair */
    uint32_t             n_coords;
    ht2gpu_seed_coord_t* coords;
    uint64_t             n_lf;       /* LF steps (boundary ranks) executed */
    uint64_t             alg_bytes;  /* algorithmic bytes of those steps (DESIGN.md 4) */
    float                ms_kernel;  /* both passes (count, fill) */
    uint32_t             err;        /* reads with capacity errors */
    void*                priv;
} ht2gpu_seed_result_t;

int ht2gpu_seed_search(ht2gpu_handle_t* h, const ht2gpu_read_batch_t* batch, uint32_t max_range,
                       ht2gpu_seed_result_t* res);
void ht2gpu_free_seed_results(ht2gpu_seed_result_t* res);
/* 1 when the opened index is a graph index: built with SNPs, splice sites or exons (hisat2-build --snp / --ss /
 * --exon: the _snp, _tran and _snp_tran indexes).  Alignment crosses SNP, indel and splice-site ALTs; an index with
 * splice sites or exons also brings its own splice-site DB (ht2gpu_load_splicesites).  ALT_SNP_ALT records, which the
 * reference never handles either, make alignment calls fail with HT2GPU_ERR_UNSUPPORTED. */
int ht2gpu_index_is_graph(const ht2gpu_handle_t* h);

/* Host back end: selection, MAPQ and SAM text for a batch (finishRead).
 * names: n_reads '\0'-terminated read names, concatenated.  The returned
 * buffer is malloc'ed; free with ht2gpu_free_text. */
int ht2gpu_format_sam(ht2gpu_handle_t* h, const ht2gpu_read_batch_t* batch, const char* names,
                      const ht2gpu_result_batch_t* res, char** out, size_t* out_len);
/* @HD, @SQ (unless no_sq) and @RG (when a read-group id is set) of ht2gpu_set_sam_output: SamConfig::printHeader
 * (sam.h:446-463) without @PG. */
int ht2gpu_sam_header(ht2gpu_handle_t* h, char** out, size_t* out_len);
void ht2gpu_free_text(char* p);

/* ---- SAM output settings and the alignment summary ------------------------------
 * SAM output settings of a handle (AlnSinkSam::appendMate aln_sink.h:3040, 3190-3215; sam.h:446-463, 780, 1102):
 *   no_unal       --no-unal: no record for a read (mate) without an alignment; its aligned mate keeps its record
 *   omit_sec_seq  --omit-sec-seq: SEQ and QUAL are '*' in non-primary records
 *   no_sq         --no-sq: ht2gpu_sam_header prints no @SQ lines
 *   rg_id         --rg-id: "@RG\tID:<rg_id>" (+ "\t<rg[i]>" for every --rg field) in the header, "RG:Z:<rg_id>" in
 *                 every record; NULL or "" = no read group (the rg fields are then not printed either)
 *   rna_strandness  --rna-strandness: 0 unknown, 1 F, 2 R, 3 FR, 4 RF (read.h:30-36).  When known, every aligned
 *                 record gets XS:A:+ or - from the library's strand, the mate and the alignment's orientation
 *                 (sam.h:938-963); it replaces the splice-motif sense of spliced records.  Single-end reads and
 *                 mate 1 take the mate-1 rule, mate 2 the mate-2 rule, whatever the read layout (F or R on pairs
 *                 prints '+' for every mate 2, as the reference does)
 *   no_qname_trunc  --sam-no-qname-trunc: QNAME is the whole name line, not cut at white space or at 255 characters
 *                 (sam.h:238-256); a trailing /1 or /2 of a mate is still left out
 *   no_templatelen_adjustment  --no-templatelen-adjustment: the TLEN of concordant pairs is not shortened by a known
 *                 intron between the mates (aln_sink.h:2068-2076)
 * All off by default.  Set between batches, like ht2gpu_load_splicesites (refused while a batch is in flight). */
typedef struct {
    int32_t no_unal, omit_sec_seq, no_sq;
    const char* rg_id;
    const char* const* rg;
    int32_t n_rg;
    int32_t rna_strandness, no_qname_trunc, no_templatelen_adjustment;
} ht2gpu_sam_output_t;
int ht2gpu_set_sam_output(ht2gpu_handle_t* h, const ht2gpu_sam_output_t* cfg);

/* Per-read outcome counts of ReportingMetrics (aln_sink.h:2007-2012, 2100-2110, 2191-2192, 2271-2346), tallied by the
 * SAM kernels for every read (pair) formatted through ht2gpu_wait_sam (ht2gpu_align_sam, ht2gpu_run_reads(_multi)).
 * Reads that fail the length / N / score filters count as unaligned; reads skipped by -s / -u are not counted. */
typedef struct {
    uint64_t nread, npaired, nunpaired;
    uint64_t nconcord_0, nconcord_uni1, nconcord_uni2, ndiscord;
    uint64_t nunp_0_0, nunp_0_uni1, nunp_0_uni2;   /* mates of pairs without a concordant / discordant alignment */
    uint64_t nunp_0, nunp_uni1, nunp_uni2;         /* unpaired reads */
} ht2gpu_align_counts_t;
/* The sum over hs[0..n) of the counts since open (or since the last reset); reset != 0 zeroes them afterwards. */
int ht2gpu_align_counts(ht2gpu_handle_t** hs, int n, int reset, ht2gpu_align_counts_t* out);
/* Host only (no device): the alignment summary hisat2 prints at the end of a run, AlnSink::printAlSumm
 * (aln_sink.h:1613-1816).  new_style = --new-summary; discordant / mixed = 0 under --no-discordant / --no-mixed
 * (the classic format then leaves out that section).  Free *out with ht2gpu_free_text. */
int ht2gpu_format_align_summary(const ht2gpu_align_counts_t* c, int new_style, int discordant, int mixed,
                                char** out, size_t* out_len);

/* Reference-sequence names and lengths (ht2_index_getrefnames, ht2.h:108): the index's own names, whatever chr_names. */
uint32_t ht2gpu_num_refs(const ht2gpu_handle_t* h);
const char* ht2gpu_ref_name(const ht2gpu_handle_t* h, uint32_t i);
uint32_t ht2gpu_ref_len(const ht2gpu_handle_t* h, uint32_t i);

/* Per-read seed exactly as the reference derives it (pat.h:55-91). */
uint32_t ht2gpu_read_seed(const uint8_t* seq, const uint8_t* qual, uint32_t len,
                          const char* name, uint32_t global_seed);

/* The run's read-only splice-site DB (spliced mode): the index's own splice sites and exons when it was built with
 * --ss / --exon (known sites, inserted first; SpliceSiteDB::read splice_site.cpp:653-720), then the sites of
 * --known-splicesite-infile and --novel-splicesite-infile ("<chr> <left> <right> <+|->" per line, 0-based;
 * hisat2.cpp:4093-4116, splice_site.cpp:727-775; either path may be NULL; a site already present is dropped).  Such an
 * index's handle holds its DB from ht2gpu_open on (also replicas made by ht2gpu_open_peer or from a device image), and
 * ht2gpu_load_splicesites(h, NULL, NULL) returns to it; on other indexes that call empties the DB.  Without spliced
 * alignment the index's sites are left out, as the reference does.  With a DB loaded, alignment runs the
 * three `if(!ssdb.empty())` branches of hybridSearch_recur (spliced_aligner.h:409-668, 685-811, 1365-1494):
 * short exon ends next to a listed site are aligned across it, and the template length of a concordant pair
 * excludes the longest listed intron between the mates (aligner_result.h:1631-1690).  Replaces a DB loaded
 * earlier; refused (HT2GPU_ERR_ARG) while a batch is in flight.  Temporary sites (learned while aligning) are not
 * modelled: the reference's own output depends on thread timing there (DESIGN.md). */
int ht2gpu_load_splicesites(ht2gpu_handle_t* h, const char* known_path, const char* novel_path, uint32_t* n_sites);

/* --novel-splicesite-outfile (hisat2.cpp:4092; aln_sink.h:1571-1580; SpliceSiteDB::addSpliceSite / print,
 * splice_site.cpp:190-350, 565-651): while enabled, the SAM kernel records the junctions of every printed alignment
 * (anchors >= 15 bases + 2 per mismatch, + 6 without a canonical motif; soft-trimmed alignments skipped) and
 * ht2gpu_wait_sam aggregates them per handle; ht2gpu_write_novel_splicesites merges the handles of a run and writes
 * "<chr> <left> <right> <+|-|.>" with the reference's read-count cutoffs and near-duplicate suppression -- the
 * first pass of the two-pass use (second pass: ht2gpu_load_splicesites(h, NULL, file)).  Refused while a DB is
 * loaded: the reference would let such sites steer later reads, i.e. depend on read order.  So it is always refused on
 * an index built with splice sites / exons in spliced mode, whose DB is always loaded; the message names the index. */
int ht2gpu_collect_splicesites(ht2gpu_handle_t* h, int enable);
int ht2gpu_write_novel_splicesites(ht2gpu_handle_t** hs, int n, const char* path, uint64_t* n_written);

/* Diagnostics: the warp-wide fill of the --bowtie2-dp score planes against the single-lane fill on n random
 * problems (aligner_swsse_ee_u8.cpp:791-1163 restated twice, ht2_sw.h).  out[0] = mismatching cells / scores
 * (must be 0), out[1] = problems run, out[2] = cells compared per plane, out[3] = problems with a valid best. */
int ht2gpu_sw_selftest(int device, uint32_t n, uint32_t seed, uint64_t out[4]);
/* Diagnostics: the --bowtie2-dp seed extension (the dp block of SplicedAligner::hybridSearch) on n jobs, one per
 * lane, with the handle's options and (linear) index.  Job i aligns the read at seq / qual[read_off, + read_len)
 * (codes 0..4, Phred+33) on strand fw, framed by the anchor (tidx, toff, rdoff, len), with minsc and a
 * RandomSource seeded with seed.  warp_fill != 0 runs the pool kernel's DP round (the warp fills the planes of
 * one problem after the other), 0 the lane fill.  res[i]: found, the per-read error bits, the hit's toff and
 * score, the best last-row score (INT64_MIN when the DP did not run or nothing reached minsc), n_edits and the
 * first draw of the RandomSource afterwards; its edits (the reference's convention) are at
 * edits[i * HT2GPU_SW_MAX_EDITS].  Device temporaries are sized for the n jobs and freed before returning. */
#define HT2GPU_SW_MAX_EDITS 128
typedef struct {
    uint32_t fw, tidx, toff, rdoff, len;
    uint32_t seed;
    int64_t  minsc;
    uint64_t read_off;
    uint32_t read_len, pad;
} ht2gpu_sw_job_t;
typedef struct {
    uint32_t found, err, toff, n_edits;
    int64_t  score, best;
    uint32_t rnd_next, pad;
} ht2gpu_sw_result_t;
int ht2gpu_sw_extend(ht2gpu_handle_t* h, uint32_t n, const ht2gpu_sw_job_t* jobs, const uint8_t* seq, const uint8_t* qual,
                     int warp_fill, ht2gpu_sw_result_t* res, ht2gpu_edit_t* edits);
/* Diagnostics: the geometry of the handle's alignment kernel.  out[0] = warps per block, out[1] = read slots per
 * lane, out[2] = blocks per SM.  The slots can differ from the options: a default handle on a device without room
 * for the 4-slot workspace, or in a process that already holds the 2-slot one, runs with 2. */
int ht2gpu_launch_geometry(const ht2gpu_handle_t* h, int32_t out[3]);

const char* ht2gpu_last_error(const ht2gpu_handle_t* h);
int ht2gpu_close(ht2gpu_handle_t* h);

#ifdef __cplusplus
}
#endif
#endif /* HT2GPU_H_ */
