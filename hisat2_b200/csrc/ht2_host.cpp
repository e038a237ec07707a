// ht2_host.cpp -- see ht2_host.h.
#include "ht2_host.h"

#include <stdio.h>
#include <string.h>
#include <math.h>

#include <algorithm>
#include <limits>
#include <functional>
#include <thread>

#include "ht2_sam.h"

// decimal append without a temporary std::string
static inline void appendInt(std::string& o, int64_t v) {
    char buf[24]; int n = 0;
    uint64_t u = v < 0 ? (uint64_t)0 - (uint64_t)v : (uint64_t)v;
    do { buf[n++] = (char)('0' + u % 10); u /= 10; } while (u);
    if (v < 0) o.push_back('-');
    while (n) o.push_back(buf[--n]);
}

// ---------------------------------------------------------------------------
// parameters
// ---------------------------------------------------------------------------
void ht2_default_params(Ht2Params& P, const Ht2Image& img, bool noSplicedAlignment)
{
    memset(&P, 0, sizeof(P));
    const Ht2ImageHeader* H = img.header();
    P.mmpMax = 6; P.mmpMin = 2; P.scpMax = 2; P.scpMin = 1; P.npen = 1;
    P.rdGapConst = 5; P.rdGapLinear = 3; P.rfGapConst = 5; P.rfGapLinear = 3;
    P.mmcostConstant = 0;
    P.canSplPen = 0;
    P.khits = H->global.linearFM ? 5 : 10;              // hisat2.cpp:3903-3906
    P.kseeds = std::max<uint32_t>(5, P.khits * 2);      // hisat2.cpp:3174-3176
    P.secondary = 0;
    P.minIntronLen = 20; P.maxIntronLen = 500000;
    P.minAnchorLen = 7; P.minAnchorLenNoncan = 14;
    P.noSplicedAlignment = noSplicedAlignment ? 1 : 0;
    P.maxAltsTried = 16;
    P.anchorStop = 1;
    uint32_t genomeLen = H->global.len;                 // hi_aligner.h:3979-3985
    P.minK = 0;
    while (genomeLen > 0) { genomeLen >>= 2; P.minK++; }
    P.minKLocal = 8;
    P.pePolicy = 2; P.minFrag = 0; P.maxFrag = 1000;
    P.gMate1fw = 1; P.gMate2fw = 0;
    P.nofw = 0; P.norc = 0; P.mixed = 1; P.discord = 1;
    P.bowtie2Dp = 0; P.gapbar = 4;                      // hisat2.cpp:529, 419
#ifdef HT2_ENABLE_SPLICED
    P.noncanSplPen = 12;                                // hisat2.cpp:494
#endif
    ht2_set_score_min(P, 'L', (double)0.0f, (double)-0.2f);   // hisat2.cpp:441
    // hisat2.cpp:443 initialises 2 + 0.1 len, but SeedAlignmentPolicy::parseString -- always called, hisat2.cpp:1849 --
    // resets it to DEFAULT_N_CEIL_CONST / LINEAR = 0.0 / 0.15 (aligner_seed_policy.cpp:293-296, scoring.h:65-67)
    ht2_set_n_ceil(P, 'L', (double)0.0f, (double)0.15f);
    // --pen-canintronlen / --pen-noncanintronlen G,-8,1 (hisat2.cpp:496-497) over the lengths the scorer can be given
    const uint32_t cover = ht2_intron_cover(P);
    ht2_set_intron_pen(P, 0, 'G', -8.0, 1.0, cover);
    ht2_set_intron_pen(P, 1, 'G', -8.0, 1.0, cover);
#ifdef HT2_ENABLE_SPLICED
    P.conflictSplPen = 1000000;                         // hisat2.cpp:495
#endif
}

// SimpleFunc::f<TAlScore> (simple_func.h:86-108) with min = -DBL_MAX, max = DBL_MAX
// (SimpleFunc::init(type, C, L)), tabulated for every supported read length.
bool ht2_set_score_min(Ht2Params& P, char type, double C, double L)
{
    if (type != 'C' && type != 'L' && type != 'S' && type != 'G') return false;
    for (uint32_t len = 0; len <= HT2_PARAMS_MAX_RDLEN; len++) {
        double x = (double)len, X;
        if (type == 'C') X = 0.0; else if (type == 'L') X = x; else if (type == 'S') X = sqrt(x); else X = log(x);
        double v = std::max(-1.7976931348623157e308, std::min(1.7976931348623157e308, C + L * X));
        if (!(v == v)) v = 0.0;
        if (v > 2147483647.0) v = 2147483647.0;
        if (v < -2147483648.0) v = -2147483648.0;
        P.minscTab[len] = (int32_t)(int64_t)v;
    }
    return true;
}

// SimpleFunc::f<int> (simple_func.h:86-108) with min = 0 and max = DBL_MAX, as the reference's nCeil.  The value is
// converted as x86-64 does: DBL_MAX gives INT_MAX, anything else at or above 2^31 gives INT_MIN.
bool ht2_set_n_ceil(Ht2Params& P, char type, double C, double L)
{
    if (type != 'C' && type != 'L' && type != 'S' && type != 'G') return false;
    const double dmax = 1.7976931348623157e308;
    for (uint32_t len = 0; len <= HT2_PARAMS_MAX_RDLEN; len++) {
        double x = (double)len, X;
        if (type == 'C') X = 0.0; else if (type == 'L') X = x; else if (type == 'S') X = sqrt(x); else X = log(x);
        const double v = std::max(0.0, std::min(dmax, C + L * X));
        P.nCeilTab[len] = v == dmax ? 2147483647 : v >= 2147483648.0 ? (int32_t)0x80000000u : (int32_t)v;
    }
    return true;
}

// The runs of max(0, SimpleFunc::f<int>(x)) (simple_func.h:86-108, min -DBL_MAX, max DBL_MAX; scoring.h:473-487) for
// the intron lengths x = 1 .. maxLen, into P.intronPen[which]; length 0 scores 0.  The value is converted as x86-64
// converts it: DBL_MAX gives INT_MAX, DBL_MIN and anything outside int's range INT_MIN, which the max makes 0.
// False for a bad type, or when the function takes more than HT2_INTRON_RUNS values over the range.
bool ht2_set_intron_pen(Ht2Params& P, int which, char type, double C, double L, uint32_t maxLen)
{
    if (type != 'C' && type != 'L' && type != 'S' && type != 'G') return false;
    Ht2IntronPen& t = P.intronPen[which];
    const double dmax = std::numeric_limits<double>::max(), dmin = std::numeric_limits<double>::min();
    t.n = 1; t.start[0] = 0; t.pen[0] = 0;
    for (uint32_t len = 1; len <= maxLen; len++) {
        const double x = (double)len;
        double X;
        if (type == 'C') X = 0.0; else if (type == 'L') X = x; else if (type == 'S') X = sqrt(x); else X = log(x);
        const double v = std::max(-dmax, std::min(dmax, C + L * X));
        int32_t pen = v == dmax ? 2147483647 : v == dmin ? (int32_t)0x80000000u
                    : (v >= -2147483648.0 && v < 2147483648.0) ? (int32_t)v : (int32_t)0x80000000u;
        if (pen < 0) pen = 0;
        if (pen == t.pen[t.n - 1]) continue;
        if (t.n == HT2_INTRON_RUNS) return false;
        t.start[t.n] = len; t.pen[t.n] = pen; t.n++;
    }
    return true;
}

const char* ht2_apply_spliced_options(Ht2Params& P, const ht2gpu_options_t& o)
{
    // hisat2.cpp:1631-1728, 3920-3922, 4075-4084.  maxIntronLen also bounds concordant pairs without spliced
    // alignment (ht2_pair.h).
    P.minIntronLen = (uint32_t)o.min_intronlen; P.maxIntronLen = (uint32_t)o.max_intronlen;
    P.anchorStop = o.no_anchorstop ? 0 : 1;
    P.canSplPen = o.pen_cansplice;
#ifdef HT2_ENABLE_SPLICED
    P.noncanSplPen = o.pen_noncansplice; P.conflictSplPen = o.pen_conflictsplice;
#endif
    P.tranFilter = (o.dta == HT2GPU_DTA_CUFFLINKS ? HT2_TRAN_XS_ONLY : 0u) | (o.tmo ? HT2_TRAN_TMO : 0u) |
                   (o.avoid_pseudogene ? HT2_TRAN_AVOID_PSEUDOGENE : 0u);
    if (o.dta != HT2GPU_DTA_NONE) { P.minAnchorLen = 15; P.minAnchorLenNoncan = 20; }
    // the intron-length functions: tokens left out keep G,-8,1; --dta sets the non-canonical one to G,-8,2 after
    // everything else was parsed.  No splice is scored without spliced alignment.
    const uint32_t cover = P.noSplicedAlignment ? 0u : ht2_intron_cover(P);
    const bool can = o.can_intronlen_type != 0, noncan = o.noncan_intronlen_type != 0 && o.dta == HT2GPU_DTA_NONE;
    if (!ht2_set_intron_pen(P, 0, can ? (char)o.can_intronlen_type : 'G', can ? o.can_intronlen_const : -8.0, can ? o.can_intronlen_coeff : 1.0, cover))
        return "--pen-canintronlen takes more distinct values over the intron lengths up to --max-intronlen than the device holds (1024)";
    if (!ht2_set_intron_pen(P, 1, noncan ? (char)o.noncan_intronlen_type : 'G', noncan ? o.noncan_intronlen_const : -8.0,
                            noncan ? o.noncan_intronlen_coeff : o.dta != HT2GPU_DTA_NONE ? 2.0 : 1.0, cover))
        return "--pen-noncanintronlen takes more distinct values over the intron lengths up to --max-intronlen than the device holds (1024)";
    return NULL;
}

int64_t ht2_minsc(const Ht2Params& P, uint32_t rdlen)
{
    // scoreMin.f(rdlen) (default L,0,-0.2, hisat2.cpp:441); clamped to <= 0 in end-to-end mode (:3395-3402)
    int64_t m = P.minscTab[rdlen <= HT2_PARAMS_MAX_RDLEN ? rdlen : HT2_PARAMS_MAX_RDLEN];
    if (m > 0) m = 0;
    return m;
}

Ht2ReadFilters ht2_filters(const Ht2HostRead& rd, int64_t minsc, const int32_t* nCeilTab)
{
    Ht2ReadFilters f;
    size_t rdlen = rd.seq.size();
    // Scoring::nFilter (scoring.cpp:104-117)
    const size_t maxns = (uint32_t)ht2_nceil(nCeilTab, (uint32_t)rdlen);
    size_t ns = 0;
    f.nfilt = true;
    for (size_t i = 0; i < rdlen; i++) {
        if (rd.seq[i] == 4) { ns++; if (ns > maxns) { f.nfilt = false; break; } }
    }
    f.scfilt = (0 >= minsc);                 // Scoring::scoreFilter with match bonus 0
    f.lenfilt = true;
    if (rdlen <= 0 /*multiseedMms*/ || rdlen < 2) f.lenfilt = false;
    f.qcfilt = true;
    return f;
}

uint32_t ht2_gen_rand_seed(const Ht2HostRead& rd, uint32_t seed)
{
    uint32_t rseed = (seed + 101) * 59 * 61 * 67 * 71 * 73 * 79 * 83;
    size_t qlen = rd.seq.size();
    for (size_t i = 0; i < qlen; i++) {
        int p = (int)rd.seq[i];
        size_t off = ((i & 15) << 1);
        rseed ^= ((uint32_t)p << off);
    }
    for (size_t i = 0; i < qlen; i++) {
        int p = (int)rd.qual[i];
        size_t off = ((i & 3) << 3);
        rseed ^= ((uint32_t)p << off);
    }
    for (size_t i = 0; i < rd.name.size(); i++) {
        int p = (int)rd.name[i];
        if (p == '/') break;
        size_t off = ((i & 3) << 3);
        rseed ^= ((uint32_t)p << off);
    }
    return rseed;
}

void ht2_fill_read(Ht2Read& dst, const Ht2HostRead& src)
{
    uint32_t n = (uint32_t)src.seq.size();
    if (n > HT2_MAX_RDLEN) n = HT2_MAX_RDLEN;
    dst.len = n;
    for (uint32_t i = 0; i < n; i++) {
        dst.seq[0][i] = src.seq[i];
        dst.qual[0][i] = src.qual[i];
        uint8_t c = src.seq[n - i - 1];
        dst.seq[1][i] = c < 4 ? (uint8_t)(c ^ 3) : (uint8_t)4;
        dst.qual[1][i] = src.qual[n - i - 1];
    }
    ht2_pack_bases(dst.pk[0], dst.seq[0], n);
    ht2_pack_bases(dst.pk[1], dst.seq[1], n);
}

// ---------------------------------------------------------------------------
// FASTA (pat.cpp:725-849; alphabet.cpp asc2dnacat / asc2dna)
// ---------------------------------------------------------------------------
static int dnacat(int c) {
    switch (c) {
        case 'A': case 'C': case 'G': case 'T': case 'a': case 'c': case 'g': case 't': return 1;
        case 'B': case 'D': case 'H': case 'K': case 'M': case 'N': case 'R': case 'S': case 'V': case 'W': case 'X': case 'Y':
        case 'b': case 'd': case 'h': case 'k': case 'm': case 'n': case 'r': case 's': case 'v': case 'w': case 'x': case 'y': return 2;
        case '-': return 3;
        default: return 0;
    }
}
static uint8_t asc2dna(int c) {
    switch (c) {
        case 'C': case 'c': return 1;
        case 'G': case 'g': return 2;
        case 'T': case 't': return 3;
        case 'N': case 'n': return 4;
        default: return 0;
    }
}

bool ht2_read_fasta(const char* path, std::vector<Ht2HostRead>& out, int mate, std::string& err)
{
    FILE* f = fopen(path, "rb");
    if (!f) { err = std::string("could not open reads file ") + path; return false; }
    std::vector<char> buf;
    {
        fseek(f, 0, SEEK_END); long sz = ftell(f); fseek(f, 0, SEEK_SET);
        buf.resize((size_t)sz);
        if (sz > 0 && fread(buf.data(), 1, (size_t)sz, f) != (size_t)sz) { fclose(f); err = "short read"; return false; }
        fclose(f);
    }
    size_t p = 0, n = buf.size();
    uint64_t readCnt = 0;
    while (p < n) {
        // skip comment / blank lines
        while (p < n && (buf[p] == '#' || buf[p] == ';' || buf[p] == '\r' || buf[p] == '\n')) {
            if (buf[p] == '#' || buf[p] == ';') { while (p < n && buf[p] != '\n') p++; }
            else p++;
        }
        if (p >= n) break;
        if (buf[p] != '>') { err = "reads file does not look like a FASTA file"; return false; }
        p++;
        Ht2HostRead r;
        r.mate = mate;
        while (p < n && buf[p] != '\n' && buf[p] != '\r') r.name.push_back(buf[p++]);
        while (p < n && (buf[p] == '\n' || buf[p] == '\r')) p++;
        while (p < n && buf[p] != '>') {
            int c = (unsigned char)buf[p++];
            if (dnacat(c) > 0) { r.seq.push_back(asc2dna(c)); r.qual.push_back('I'); }
        }
        if (r.name.empty()) r.name = std::to_string(readCnt);
        readCnt++;
        // an empty record stays in the stream: the reference reports it as unaligned with YF:Z:LN
        out.push_back(r);
    }
    return true;
}

// FastqPatternSource::parse (pat.cpp:1030-1290) for well-formed 4-line Phred+33 records:
// '@name', bases ('.' reads as N, letters only), '+...', qualities kept as raw ASCII.
bool ht2_read_fastq(const char* path, std::vector<Ht2HostRead>& out, int mate, std::string& err)
{
    FILE* f = fopen(path, "rb");
    if (!f) { err = std::string("could not open reads file ") + path; return false; }
    std::vector<char> buf;
    {
        fseek(f, 0, SEEK_END); long sz = ftell(f); fseek(f, 0, SEEK_SET);
        buf.resize((size_t)sz);
        if (sz > 0 && fread(buf.data(), 1, (size_t)sz, f) != (size_t)sz) { fclose(f); err = "short read"; return false; }
        fclose(f);
    }
    size_t p = 0, n = buf.size();
    uint64_t readCnt = 0;
    auto line = [&](std::string& o) {
        o.clear();
        while (p < n && buf[p] != '\n') { if (buf[p] != '\r') o.push_back(buf[p]); p++; }
        if (p < n) p++;
    };
    std::string l1, l2, l3, l4;
    while (p < n) {
        while (p < n && (buf[p] == '\n' || buf[p] == '\r')) p++;
        if (p >= n) break;
        line(l1); line(l2); line(l3); line(l4);
        if (l1.empty() || l1[0] != '@' || l3.empty() || l3[0] != '+') { err = "reads file does not look like a FASTQ file"; return false; }
        Ht2HostRead r;
        r.mate = mate;
        r.name = l1.substr(1);
        for (size_t i = 0; i < l2.size(); i++) {
            int c = (unsigned char)l2[i];
            if (c == '.') c = 'N';
            if (isalpha(c)) r.seq.push_back(asc2dna(c));
        }
        if (l4.size() < r.seq.size()) { err = "fewer quality values than bases for read " + r.name; return false; }
        if (l4.size() > r.seq.size()) { err = "more quality values than bases for read " + r.name; return false; }
        for (size_t i = 0; i < r.seq.size(); i++) {
            if ((unsigned char)l4[i] < 33) { err = "quality value below Phred+33 range in read " + r.name; return false; }
            r.qual.push_back((uint8_t)l4[i]);
        }
        if (r.name.empty()) r.name = std::to_string(readCnt);
        readCnt++;
        out.push_back(r);
    }
    return true;
}

// FASTA or FASTQ by the first record character (the CLI's -f / -q select explicitly).
bool ht2_read_reads(const char* path, std::vector<Ht2HostRead>& out, int mate, std::string& err)
{
    FILE* f = fopen(path, "rb");
    if (!f) { err = std::string("could not open reads file ") + path; return false; }
    int c;
    while ((c = fgetc(f)) != EOF && (c == '\n' || c == '\r')) {}
    fclose(f);
    return c == '@' ? ht2_read_fastq(path, out, mate, err) : ht2_read_fasta(path, out, mate, err);
}

// ---------------------------------------------------------------------------
// SAM back end
// ---------------------------------------------------------------------------
// SamConfig::printHeader (sam.h:446-463) without @PG: @HD, @SQ unless --no-sq, @RG when a read-group id is set
void ht2_sam_header(std::string& o, const Ht2Image& img, const Ht2SamOutput* so, const Ht2RefNames* refNames)
{
    o += "@HD\tVN:1.0\tSO:unsorted\n";
    const Ht2ImageHeader* H = img.header();
    Ht2RefNames own;
    if (!refNames) { own.build(img, HT2GPU_CHR_NAMES_INDEX); refNames = &own; }
    for (uint32_t i = 0; !(so && so->noSq) && i < H->nRefs; i++) {
        o += "@SQ\tSN:";
        o += refNames->token(i);
        o += "\tLN:";
        appendInt(o, img.refPlen(i));
        o += "\n";
    }
    if (so && !so->rgId.empty()) {
        o += "@RG\tID:";
        o += so->rgId;
        for (const std::string& f : so->rg) { o += "\t"; o += f; }
        o += "\n";
    }
}

// printPct (aln_sink.h:1613-1622): fixed, two decimals, 0.00% for a zero denominator
static void appendPct(std::string& o, uint64_t num, uint64_t denom)
{
    double pct = 0.0f;
    if (denom != 0) pct = 100.0 * (double)num / (double)denom;
    char buf[64];
    snprintf(buf, sizeof(buf), "%.2f%%", pct);
    o += buf;
}

void ht2_format_align_summary(std::string& o, const ht2gpu_align_counts_t& m, bool newStyle, bool discord, bool mixed)
{
    auto num = [&](uint64_t v) { appendInt(o, (int64_t)v); };
    // "<n> (<pct>)" as most lines of the summary print it
    auto np = [&](uint64_t v, uint64_t denom) { num(v); o += " ("; appendPct(o, v, denom); o += ")"; };
    const uint64_t totread = m.nread, totpair = m.npaired, totunpair = m.nunpaired;
    const uint64_t tot_al_cand = totunpair + totpair * 2;
    const uint64_t tot_al = (m.nconcord_uni1 + m.nconcord_uni2) * 2 + m.ndiscord * 2 + m.nunp_0_uni1 + m.nunp_0_uni2 + m.nunp_uni1 + m.nunp_uni2;
    const uint64_t ncondiscord_0 = m.nconcord_0 - m.ndiscord;
    if (newStyle) {
        o += "HISAT2 summary stats:\n";
        if (totpair > 0) {
            o += "\tTotal pairs: "; num(totpair); o += "\n";
            o += "\t\tAligned concordantly or discordantly 0 time: "; np(ncondiscord_0, m.npaired); o += "\n";
            o += "\t\tAligned concordantly 1 time: "; np(m.nconcord_uni1, m.npaired); o += "\n";
            o += "\t\tAligned concordantly >1 times: "; np(m.nconcord_uni2, m.npaired); o += "\n";
            o += "\t\tAligned discordantly 1 time: "; np(m.ndiscord, m.npaired); o += "\n";
            o += "\tTotal unpaired reads: "; num(ncondiscord_0 * 2); o += "\n";
            o += "\t\tAligned 0 time: "; np(m.nunp_0_0, ncondiscord_0 * 2); o += "\n";
            o += "\t\tAligned 1 time: "; np(m.nunp_0_uni1, ncondiscord_0 * 2); o += "\n";
            o += "\t\tAligned >1 times: "; np(m.nunp_0_uni2, ncondiscord_0 * 2); o += "\n";
        } else {
            o += "\tTotal reads: "; num(totread); o += "\n";
            o += "\t\tAligned 0 time: "; np(m.nunp_0, m.nunpaired); o += "\n";
            o += "\t\tAligned 1 time: "; np(m.nunp_uni1, m.nunpaired); o += "\n";
            o += "\t\tAligned >1 times: "; np(m.nunp_uni2, m.nunpaired); o += "\n";
        }
        o += "\tOverall alignment rate: "; appendPct(o, tot_al, tot_al_cand); o += "\n";
        return;
    }
    num(totread); o += totread > 0 ? " reads; of these:\n" : " reads\n";
    if (totpair > 0) {
        o += "  "; np(totpair, totread); o += " were paired; of these:\n";
        o += "    "; np(m.nconcord_0, m.npaired); o += " aligned concordantly 0 times\n";
        o += "    "; np(m.nconcord_uni1, m.npaired); o += " aligned concordantly exactly 1 time\n";
        o += "    "; np(m.nconcord_uni2, m.npaired); o += " aligned concordantly >1 times\n";
        if (discord) {
            o += "    ----\n";
            o += "    "; num(m.nconcord_0); o += " pairs aligned concordantly 0 times; of these:\n";
            o += "      "; np(m.ndiscord, m.nconcord_0); o += " aligned discordantly 1 time\n";
        }
        if (mixed) {
            o += "    ----\n";
            o += "    "; num(ncondiscord_0); o += " pairs aligned 0 times concordantly or discordantly; of these:\n";
            o += "      "; num(ncondiscord_0 * 2); o += " mates make up the pairs; of these:\n";
            o += "        "; np(m.nunp_0_0, ncondiscord_0 * 2); o += " aligned 0 times\n";
            o += "        "; np(m.nunp_0_uni1, ncondiscord_0 * 2); o += " aligned exactly 1 time\n";
            o += "        "; np(m.nunp_0_uni2, ncondiscord_0 * 2); o += " aligned >1 times\n";
        }
    }
    if (totunpair > 0) {
        o += "  "; np(totunpair, totread); o += " were unpaired; of these:\n";
        o += "    "; np(m.nunp_0, m.nunpaired); o += " aligned 0 times\n";
        o += "    "; np(m.nunp_uni1, m.nunpaired); o += " aligned exactly 1 time\n";
        o += "    "; np(m.nunp_uni2, m.nunpaired); o += " aligned >1 times\n";
    }
    appendPct(o, tot_al, tot_al_cand); o += " overall alignment rate\n";
}

extern "C" int ht2gpu_format_align_summary(const ht2gpu_align_counts_t* c, int new_style, int discordant, int mixed,
                                           char** out, size_t* out_len)
{
    if (!c || !out) return HT2GPU_ERR_ARG;
    std::string s;
    ht2_format_align_summary(s, *c, new_style != 0, discordant != 0, mixed != 0);
    char* p = (char*)malloc(s.size() + 1);
    if (!p) return HT2GPU_ERR_ARG;
    memcpy(p, s.data(), s.size()); p[s.size()] = 0;
    *out = p; if (out_len) *out_len = s.size();
    return HT2GPU_OK;
}

// The SAM back end of one batch (ht2gpu_format_sam) on the host: the formatter of ht2_sam.h -- the same
// source the device kernel runs -- on host threads over contiguous unit ranges: a counting pass, a prefix
// over the ranges, a writing pass straight into the output (records in read order = --reorder).
bool ht2_format_batch(const Ht2Image& img, const Ht2Params& P, const ht2gpu_read_batch_t* b, const char* names,
                      const ht2gpu_result_batch_t* res, char** out, size_t* out_len, unsigned nth, const uint8_t* ssT, uint32_t* colCount, Ht2SsRec* colRecs, uint32_t colCap,
                      const Ht2SamOutput* so, ht2gpu_align_counts_t* counts, uint8_t* unitOut, const Ht2RefNames* refNames)
{
    const std::string rgTag = so ? so->rgTag() : std::string();
    Ht2RefNames own;
    if (!refNames) { own.build(img, HT2GPU_CHR_NAMES_INDEX); refNames = &own; }
    const uint32_t units = b->paired ? b->n_reads / 2 : b->n_reads;
    std::vector<uint32_t> nameOffs((size_t)b->n_reads + 1);
    {
        size_t at = 0;
        for (uint32_t i = 0; i < b->n_reads; i++) { nameOffs[i] = (uint32_t)at; at += strlen(names + at) + 1; }
        nameOffs[b->n_reads] = (uint32_t)at;
    }
    Ht2SamIn in;
    in.blob = img.blob.data(); in.refNames = refNames->blob.data(); in.minscTab = P.minscTab;
    in.seq = b->seq; in.qual = b->qual; in.offs = b->offs; in.names = names; in.nameOffs = nameOffs.data();
    in.n_reads = b->n_reads; in.paired = b->paired;
    in.reads = res->reads; in.alns = res->alns; in.edits = res->edits; in.pairs = res->pairs;
    in.khits = P.khits; in.secondary = P.secondary; in.mixed = P.mixed; in.discord = P.discord;
    in.ssT = so && so->noTlenAdj ? NULL : ssT;
    in.nearSsT = (P.tranFilter & HT2_TRAN_AVOID_PSEUDOGENE) && !P.noSplicedAlignment ? ssT : NULL;
    in.colCount = colCount; in.colRecs = colRecs; in.colCap = colCap;
    in.noUnal = so && so->noUnal; in.omitSecSeq = so && so->omitSecSeq; in.rgTag = rgTag.empty() ? NULL : rgTag.c_str();
    in.rnaStrandness = so ? so->rnaStrandness : 0; in.noQnameTrunc = so && so->noQnameTrunc;
    in.unitOut = unitOut;
    Ht2SamFmt F; F.bind(&in);
    if (nth > 64) nth = 64;
    if (nth < 1 || units < 4096) nth = 1;
    std::vector<uint64_t> bytes(nth, 0), at(nth + 1, 0);
    std::vector<Ht2SamTally> tally(nth);
    auto range = [&](unsigned t, uint32_t& u0, uint32_t& u1) { u0 = (uint32_t)((uint64_t)units * t / nth); u1 = (uint32_t)((uint64_t)units * (t + 1) / nth); };
    auto forThreads = [&](const std::function<void(unsigned)>& fn) {
        if (nth == 1) { fn(0); return; }
        std::vector<std::thread> th;
        for (unsigned t = 0; t < nth; t++) th.emplace_back(fn, t);
        for (auto& x : th) x.join();
    };
    forThreads([&](unsigned t) {
        uint32_t u0, u1; range(t, u0, u1);
        Ht2SamOut<false> o; o.p = NULL; o.n = 0;
        memset(&tally[t], 0, sizeof(Ht2SamTally));
        for (uint32_t u = u0; u < u1; u++) F.unit(o, u, &tally[t]);
        bytes[t] = o.n;
    });
    for (unsigned t = 0; t < nth; t++) at[t + 1] = at[t] + bytes[t];
    if (counts) {
        uint64_t* c = (uint64_t*)counts;   // ht2gpu_align_counts_t: HT2_T_N uint64_t in the order of the tally
        for (unsigned t = 0; t < nth; t++) for (int k = 0; k < HT2_T_N; k++) c[k] += tally[t].c[k];
    }
    const size_t total = (size_t)at[nth];
    char* p = (char*)malloc(total + 1);
    if (!p) return false;
    forThreads([&](unsigned t) {
        uint32_t u0, u1; range(t, u0, u1);
        Ht2SamOut<true> o; o.p = p + at[t]; o.n = 0;
        for (uint32_t u = u0; u < u1; u++) F.unit(o, u);
    });
    p[total] = 0;
    *out = p; if (out_len) *out_len = total;
    return true;
}
