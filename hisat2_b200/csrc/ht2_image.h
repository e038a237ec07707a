// ht2_image.h -- the packed, device-resident HISAT2 index image.
//
// One contiguous, 128-byte aligned blob holds everything the alignment hot
// path reads: the global (graph) FM index, the SA sample, all local 16-bit
// FM indexes, the 2-bit reference and the ALT table.  The same blob is
// uploaded to HBM (and NCCL-broadcast to the other ranks) unchanged; all
// cross references are byte offsets from the blob base so the image is
// position independent.
//
// Reference formats this replaces (parsed in ht2_index.cpp):
//   global index  .1/.2.ht2  gfm.h:5917-6458   (GFM::readIntoMemory)
//   local indexes .5/.6.ht2  hgfm.h:2582-2590, 1106-1530
//   2-bit ref     .3/.4.ht2  reference.cpp:30-390
//   geometry                 gfm.h:134-176     (GFMParams::init)
#ifndef HT2_IMAGE_H_
#define HT2_IMAGE_H_

#include <stdint.h>

#if defined(__CUDACC__)
#define HT2_HD __host__ __device__ __forceinline__
#define HT2_HDN __host__ __device__ inline
#define HT2_NI __host__ __device__ __noinline__   /* big functions: keep ONE copy (I-cache) */
#else
#define HT2_HD inline
#define HT2_HDN inline
#define HT2_NI inline
#endif

// Spliced alignment (the reference's default mode) is compiled in unless HT2_DISABLE_SPLICED is given.
#if !defined(HT2_DISABLE_SPLICED) && !defined(HT2_ENABLE_SPLICED)
#define HT2_ENABLE_SPLICED
#endif

#define HT2_MAGIC 0x42325448u /* "HT2B" */
#define HT2_IMAGE_VERSION 6u

// Local-index constants (hier_idx_common.h:23-41).
#define HT2_LOCAL_INDEX_SIZE     57344u
#define HT2_LOCAL_INDEX_OVERLAP  1024u
#define HT2_LOCAL_INDEX_INTERVAL 56320u

// Linear FM indexes (global and local) are NOT kept in the .ht2 side format
// (48/56 B of BWT + 4 occ entries, 192/224 rows per side, a div/mod per LF
// step).  The image re-lays them as 32-byte "rank sides", one DRAM sector each:
//     [ 64 BW chars, 2 bit each = 16 B ][ u32 occ[4] ]
// occ[c] = fchr[c] + #c in rows [0, sideStart), '$' not counted, so that
// LF(row,c) = occ[c] + popcount(matches among the first row&63 chars) and the
// side of a row is row>>6.  (ht2_index.cpp:relayLinear, ht2_fm.h:ht2_lf.)
// Graph (GBWT) indexes use 64-byte rank sides, also 64 rows each (Ht2GSide in ht2_graph.h):
//     [16 B BW chars][u64 F bits][u64 M bits][u32 occ[4]][u32 M_occ][u32 F_loc][8 B pad]
// M_occ = rank1(M, sideStart), F_loc = select1(F, M_occ) (row of the M_occ-th set F bit), which is
// what the .ht2 trailer pair (F_loc, M_occ) of gfm.h:3790-3807 encodes for 208-row sides.
#define HT2_GSIDE_BYTES 64u
#define HT2_SIDE_SHIFT 6u
#define HT2_SIDE_CHARS 64u
#define HT2_SIDE_BYTES 32u

// Geometry + array locations of one FM index (global: 32-bit entries,
// local: 16-bit entries).  Mirrors GFMParams (gfm.h:115-299).
struct Ht2Gfm {
    uint32_t len;          // # unambiguous reference bases
    uint32_t gbwtLen;      // # BW rows
    uint32_t numNodes;     // # graph nodes (== gbwtLen for linear)
    uint32_t eftabLen;
    uint32_t linearFM;     // 1 iff len+1 == gbwtLen
    uint32_t sideSz;       // bytes per side: 32 for linear indexes, 64 for graph indexes (re-laid "rank sides")
    uint32_t sideGbwtSz;   // BWT bytes per side (16 linear)
    uint32_t sideGbwtLen;  // BW chars per side (64 linear)
    uint32_t numSides;
    uint32_t offRate;
    uint32_t offMask;      // all-ones << offRate, truncated to entry width
    uint32_t ftabChars;
    uint32_t ftabLen;      // 4^ftabChars + 1
    uint32_t offsLen;
    uint32_t nPat;
    uint32_t nFrag;
    uint32_t nzOffs;
    uint32_t ftabCmp;      // linear ? len : gbwtLen  (gfm.h:2600, 2621)
    uint32_t fchr[5];
    uint32_t entryBytes;   // 4 (global) or 2 (local)
    // local-index placement (zero for the global index)
    uint32_t tidx;
    uint32_t localOffset;
    uint32_t joinedOffset;
    uint32_t zOff0;        // first (linear: only) row whose BW char is '$'
    // byte offsets from blob base
    uint64_t o_gfm;
    uint64_t o_ftab;
    uint64_t o_eftab;
    uint64_t o_offs;
    uint64_t o_zoffs;
    uint64_t o_rstarts;
    uint64_t o_plen;
};

// One unambiguous stretch of a reference (ref_read.h:73-103).
struct Ht2RefRecord {
    uint32_t off;   // # Ns skipped before the stretch
    uint32_t len;   // # unambiguous bases
    uint32_t first; // 1 = first record of a reference
    uint32_t pad;
};

// ALT record (alt.h:43-204); 'left'/'right' alias pos/len for splice sites and exons.  As in the
// reference's union, the low byte of 'seq' doubles as the 'reversed' flag of the deletion copies the
// loader appends (gfm.h:856-872) and as the strand ('fw') of a splice site; 'reversed' mirrors it for
// deletions only.  A splice site is stored twice: as read (left < right) and as the loader's reversed
// copy with left and right swapped (left > right), which the leftward ALT extension walks.
#define HT2_ALT_NONE 0u
#define HT2_ALT_SNP_SGL 1u
#define HT2_ALT_SNP_INS 2u
#define HT2_ALT_SNP_DEL 3u
#define HT2_ALT_SNP_ALT 4u
#define HT2_ALT_SPLICESITE 5u
#define HT2_ALT_EXON 6u
struct Ht2Alt {
    uint32_t pos;
    uint32_t type;
    uint32_t len;
    uint32_t reversed;
    uint64_t seq;
};

struct Ht2ImageHeader {
    uint32_t magic;
    uint32_t version;
    uint64_t totalBytes;
    Ht2Gfm   global;
    // local indexes
    uint32_t nLocal;
    uint32_t nRefs;        // # references (== global.nPat)
    uint64_t o_localGfm;   // Ht2Gfm[nLocal]
    uint64_t o_localFirst; // uint32[nRefs+1]: first local index of each ref
    // 2-bit reference
    uint32_t nRecs;
    uint32_t pad1;
    uint64_t o_recs;       // Ht2RefRecord[nRecs]
    uint64_t o_refRecOffs; // uint32[nRefs+1]
    uint64_t o_refOffs;    // uint64[nRefs+1]  base offset into 2-bit buffer
    uint64_t o_refLens;    // uint32[nRefs]    approxLen (reference.cpp:142-160)
    uint64_t o_refBuf;     // packed 2-bit bases
    uint64_t refBufBytes;
    // ALTs
    uint32_t nAlts;
    uint32_t nSpliceSites;    // ALT_SPLICESITE records of the .7.ht2 (each also has its reversed copy in the table)
    uint64_t o_alts;       // Ht2Alt[nAlts]: augmented with reversed deletions and splice sites, sorted like the reference's loader
    uint64_t o_altNames;   // '\0'-separated, nAlts entries (host side: Zs:Z)
    uint64_t altNamesBytes;
    uint32_t altsUnsupported; // 1 when the ALT list holds ALT_SNP_ALT records (which the reference never handles either)
    uint32_t nExons;          // ALT_EXON records of the .7.ht2
    // reference names (host side only, for SAM headers)
    uint64_t o_names;      // '\0'-separated, nRefs entries
    uint64_t namesBytes;
    // name-offset tables (the SAM back end runs on the device: no linear walks over the name blobs)
    uint64_t o_nameOffs;    // uint32[nRefs + 1]: reference i's name starts at o_names + nameOffs[i]
    uint64_t o_altNameOffs; // uint32[nAlts + 1]: ALT i's name starts at o_altNames + altNameOffs[i]
};

#endif // HT2_IMAGE_H_
