// ht2_index.h -- host-side owner of a packed index image (see ht2_image.h).
#ifndef HT2_INDEX_H_
#define HT2_INDEX_H_

#include <string>
#include <vector>
#include <map>
#include <tuple>

#include "ht2_image.h"
#include "../../include/ht2gpu.h"

struct Ht2Image {
    std::vector<uint8_t> blob;
    const Ht2ImageHeader* header() const { return (const Ht2ImageHeader*)blob.data(); }
    const char* refName(uint32_t i) const {
        return (const char*)blob.data() + header()->o_names + ((const uint32_t*)(blob.data() + header()->o_nameOffs))[i];
    }
    uint32_t refPlen(uint32_t i) const {
        return ((const uint32_t*)(blob.data() + header()->global.o_plen))[i];
    }
};

// Parse <base>.[1-8].ht2 into an image.  Returns NULL and sets 'err' on failure.
Ht2Image* ht2_image_load(const char* base, std::string& err);

// The reference names a handle prints (@SQ, RNAME, RNEXT) and matches splice-site files against, made once when the
// handle opens (ht2gpu_options_t::chr_names, hisat2.cpp:3957-3976): the index's own names, with --remove-chrname a
// leading "chr" dropped, with --add-chrname "chr" put before every name that does not start with it.  Names keep
// their comments (what follows the first white space); every user reads a name up to its first white space.
// blob: one uint32 offset per name from the blob's start, then the '\0'-terminated names.  The SAM formatter reads
// the blob as it is, on the host and on the device.
struct Ht2RefNames {
    std::vector<uint8_t> blob;
    void build(const Ht2Image& img, int chrNames);
    const char* operator[](uint32_t i) const { return (const char*)blob.data() + ((const uint32_t*)blob.data())[i]; }
    std::string token(uint32_t i) const;   // name i up to its first white space
};

// The read-only splice-site DB of a run (ht2_ssdb.h): first the splice sites (unless indexSites is false, as under
// --no-spliced-alignment, where the reference does not load them: gfm.h:760-771) and exons of the index
// (SpliceSiteDB::read(gfm, alts), splice_site.cpp:653-720: each site known, at left - 1 / right + 1, each exon widened
// by 10 bases at both ends), then the sites of the text files of --known-splicesite-infile ('known' = true)
// and --novel-splicesite-infile (false): "<chr> <left> <right> <+|->" per site, 0-based, as hisat2_extract_splice_sites.py
// writes them (SpliceSiteDB::read, splice_site.cpp:727-775: names compared up to the first white space, unknown
// names skipped, a site already present is dropped).  Files are read in the order given.  An unreadable file is
// skipped like the reference does (hisat2.cpp:4101-4116); a malformed one is an error.
struct Ht2SsFile { std::string path; bool known; };
// --novel-splicesite-outfile: junction records of printed alignments (Ht2SsRec, ht2_ssdb.h) aggregated like
// SpliceSiteDB::addSpliceSite does (number of alignments per site, smallest edit distance), and written like
// SpliceSiteDB::print (splice_site.cpp:565-651): read-count cutoffs from the distribution over all sites, sites
// within 10 bases of a better-supported neighbour suppressed.  The result does not depend on the order of 'add'.
struct Ht2NovelSites {
    std::map<std::tuple<uint32_t, uint32_t, uint32_t, uint32_t>, std::pair<uint32_t, uint32_t>> sites;   // (ref, left, right, dir) -> (numreads, editdist)
    void add(const struct Ht2SsRec* recs, size_t n);
    void merge(const Ht2NovelSites& o);
    // names: the handle's reference names; NULL = the index's own
    bool write(const Ht2Image& img, const char* path, uint64_t* nWritten, std::string& err, const Ht2RefNames* names = NULL) const;
};
bool ht2_ssdb_build(const Ht2Image& img, const std::vector<Ht2SsFile>& files, std::vector<uint8_t>& blob, uint32_t& nSites, std::string& err,
                    const Ht2RefNames* names = NULL, bool indexSites = true);

#endif
