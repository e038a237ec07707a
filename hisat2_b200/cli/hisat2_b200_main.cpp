// hisat2-b200 -- command-line front end with the hisat2-align-s option surface
// (hisat2.cpp:541-764) for the subset that reaches the GPU alignment path.
// Host C++ over the C ABI only (include/ht2gpu.h): ht2gpu_run_reads parses the reads on all host threads,
// aligns and formats them on the device in overlapped batches, and hands back SAM text in read order.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/stat.h>
#include <sys/wait.h>
#include <sstream>
#include <string>
#include <vector>
#include "ht2gpu.h"

// --un / --al / --un-conc / --al-conc / --al-conc-disc and their -gz / -bz2 forms: the read files of the hisat2
// wrapper (hisat2:546-650).  Outputs are opened before the run; compressed ones are piped through gzip -c / bzip2 -c.
static const char* const kReadOpt[HT2GPU_READS_N] = {"un", "al", "un-conc", "al-conc", "al-conc-disc"};
struct ReadFile { FILE* f = NULL; bool pipe = false; std::string path; };
static bool closeReadFile(ReadFile& rf);
struct ReadFiles {
    std::string spec[HT2GPU_READS_N];
    int compress[HT2GPU_READS_N] = {0, 0, 0, 0, 0};   // 0 none, 1 gzip, 2 bzip2
    ReadFile file[HT2GPU_READS_N][2];                // [output][mate 1 or unpaired, mate 2]
    uint32_t mask() const { uint32_t m = 0; for (int w = 0; w < HT2GPU_READS_N; w++) if (!spec[w].empty()) m |= 1u << w; return m; }
    ~ReadFiles() { for (auto& f : file) { closeReadFile(f[0]); closeReadFile(f[1]); } }   // every exit waits for gzip / bzip2
};
// The wrapper's names (File::Spec->splitpath + catpath): a directory (or a path ending in '/') gets <opt>-seqs, or
// <opt>-mate.1 / .2; with -conc a '%' in the name becomes 1 / 2, else .1 / .2 goes in before the last extension, else
// it is appended.
static std::string readFileName(const std::string& spec, int which, int mate)
{
    struct stat st;
    const bool isDir = stat(spec.c_str(), &st) == 0 && S_ISDIR(st.st_mode);
    std::string dir, base;
    if (isDir) dir = spec;
    else { const size_t k = spec.rfind('/'); dir = k == std::string::npos ? "" : spec.substr(0, k + 1); base = spec.substr(dir.size()); }
    const bool conc = which >= HT2GPU_READS_UN_CONC;
    if (base.empty()) base = std::string(kReadOpt[which]) + (conc ? "-mate" : "-seqs");
    else if (!conc) return spec;
    if (conc) {
        const char m = mate == 2 ? '2' : '1';
        const size_t dot = base.rfind('.');
        if (base.find('%') != std::string::npos) { for (char& c : base) if (c == '%') c = m; }
        else if (dot != std::string::npos) base = base.substr(0, dot) + "." + m + base.substr(dot);
        else base += std::string(".") + m;
    }
    if (!dir.empty() && dir.back() != '/') dir += '/';
    return dir + base;
}
static bool openReadFile(ReadFile& rf, const std::string& path, int compress)
{
    rf.path = path;
    FILE* f = fopen(path.c_str(), "wb");   // the wrapper's open(): an unwritable path is an error before anything runs
    if (!f) return false;
    if (!compress) { rf.f = f; return true; }
    fclose(f);
    std::string q = "'";
    for (char c : path) { if (c == '\'') q += "'\\''"; else q += c; }
    q += "'";
    const std::string cmd = std::string(compress == 1 ? "gzip -c > " : "bzip2 -c > ") + q;
    rf.f = popen(cmd.c_str(), "w");
    rf.pipe = true;
    return rf.f != NULL;
}
static bool closeReadFile(ReadFile& rf)
{
    if (!rf.f) return true;
    bool ok = fflush(rf.f) == 0 && !ferror(rf.f);
    if (rf.pipe) { const int st = pclose(rf.f); ok = ok && st != -1 && WIFEXITED(st) && WEXITSTATUS(st) == 0; }
    else ok = fclose(rf.f) == 0 && ok;
    rf.f = NULL;
    return ok;
}

static void usage() {
    fprintf(stderr, "hisat2-b200 -x <index> {-U <r> | -1 <m1> -2 <m2> [-U <r>]} [-S out.sam] [-f|-q] --no-spliced-alignment [-k N]\n"
                    "            [--mp MX,MN] [--sp MX,MN] [--np N] [--rdg C,L] [--rfg C,L] [--ignore-quals] [--nofw] [--norc]\n"
                    "            [-I N] [-X N] [--no-mixed] [--no-discordant] [--seed N] [--batch N] [--device N] [--gpus N] [-p N]\n"
                    "            [-5 N] [-3 N] [-s N] [-u N] [--phred33|--phred64|--solexa-quals] [--int-quals] [--no-temp-splicesite]\n"
                    "            [--known-splicesite-infile F] [--novel-splicesite-infile F] [--novel-splicesite-outfile F]\n"
                    "            [--bowtie2-dp 0|1|2] [--score-min F,C,L] [--gbar N] [--sensitive] [--very-sensitive] [--fast]\n"
                    "            [--no-unal] [--omit-sec-seq] [--no-hd] [--no-sq] [--rg-id ID] [--rg TEXT]...\n"
                    "            [--rna-strandness F|R|FR|RF] [--remove-chrname|--add-chrname] [--no-templatelen-adjustment]\n"
                    "            [--sam-no-qname-trunc] [--fr|--rf|--ff] [--n-ceil F,C,L] [--no-softclip] [--ma N (ignored)]\n"
                    "            [--pen-cansplice N] [--pen-noncansplice N] [--pen-conflictsplice N] [--pen-canintronlen F,C,L]\n"
                    "            [--pen-noncanintronlen F,C,L] [--min-intronlen N] [--max-intronlen N] [--dta|--dta-cufflinks]\n"
                    "            [--no-anchorstop] [--tmo] [--avoid-pseudogene] [--splicesite-db-only (ignored)]\n"
                    "            [--summary-file F] [--new-summary] [--quiet]\n"
                    "            [--un P] [--al P] [--un-conc P] [--al-conc P] [--al-conc-disc P], each also as --<opt>-gz\n"
                    "            and --<opt>-bz2: write unpaired reads that did not / did align, pairs that did not / did align\n"
                    "            concordantly, and pairs with at least one aligned mate (P.1 / P.2, or '%%' in P replaced by 1 / 2)\n"
                    "  Read files (and '-' for stdin) may be gzip-compressed (.gz, BGZF, multi-member); they are recognised by\n"
                    "  their first bytes, whatever their name, and inflated on the GPU.  For bzip2 use a pipe: -U <(bzip2 -dc r.bz2)\n"
                    "  -U, -1 and -2 take comma-separated lists and may be repeated; as many -1 as -2 files.  The -1 / -2 files\n"
                    "  are one stream of pairs, the -U files one stream of unpaired reads, aligned after the pairs\n");
}
static void two(const char* a, int32_t& x, int32_t& y) { sscanf(a, "%d,%d", &x, &y); }
// tokenize() (tokenize.h:33-51): a leading empty token is kept, later runs of the delimiter are one
static std::vector<std::string> refTokens(const std::string& v, char delim)
{
    std::vector<std::string> t;
    for (size_t p = 0, c = v.find(delim); c != std::string::npos || p != std::string::npos;) {
        t.push_back(v.substr(p, c == std::string::npos ? std::string::npos : c - p));
        p = v.find_first_not_of(delim, c);
        c = p == std::string::npos ? p : v.find(delim, p);
    }
    return t;
}
// --n-ceil: one token is C,<x>, two are <type>,<const>, three <type>,<const>,<coeff> (hisat2.cpp:1525-1550, PARSE_FUNC
// aligner_seed_policy.cpp:47-62).  Tokens left out keep the default L,0,0.15.  Returns false after printing the
// reference's error.  A later --n-ceil overrides only the tokens it gives, as the reference appends each to its policy.
static bool nCeil(const std::string& v, ht2gpu_options_t& o)
{
    if (o.n_ceil_type == 0) { o.n_ceil_const = (double)0.0f; o.n_ceil_coeff = (double)0.15f; }
    std::vector<std::string> t = refTokens(v, ',');
    if (t.size() > 3) { fprintf(stderr, "Error: expected 3 or fewer comma-separated arguments to --n-ceil option, got %zu\n", t.size()); return false; }
    if (t.empty()) { fprintf(stderr, "Error: expected at least one argument to --n-ceil option\n"); return false; }
    if (t.size() == 1) { t.insert(t.begin(), "C"); if (t[1].empty()) t.pop_back(); }   // "C,<x>", tokenized once more
    const std::string& ty = t[0];
    if (ty == "C" || ty == "Constant") o.n_ceil_type = 'C'; else if (ty == "L" || ty == "Linear") o.n_ceil_type = 'L';
    else if (ty == "S" || ty == "Sqrt") o.n_ceil_type = 'S'; else if (ty == "G" || ty == "Log") o.n_ceil_type = 'G';
    else {
        fprintf(stderr, "Error: Bad function type '%s'.  Should be C (constant), L (linear), S (square root) or G (natural log).\n", ty.c_str());
        return false;
    }
    if (t.size() > 1) o.n_ceil_const = atof(t[1].c_str());
    if (t.size() > 2) o.n_ceil_coeff = atof(t[2].c_str());
    return true;
}
// parseInt (hisat2.cpp:1016-1039): strtol, then the bounds; a value that is no number reads as 0.  Returns false after
// printing the reference's message.
static bool refInt(const char* arg, int lower, const char* msg, int32_t& out)
{
    const long l = strtol(arg, NULL, 10);
    if (l < lower || l > 2147483647L) { fprintf(stderr, "%s\n", msg); return false; }
    out = (int32_t)l;
    return true;
}
// --pen-canintronlen / --pen-noncanintronlen <type>[,<const>[,<coeff>]] (hisat2.cpp:1643-1680): the first three
// tokens become CANINTRONLEN= / NONCANINTRONLEN= of the policy string, read by PARSE_FUNC (aligner_seed_policy.cpp:47-62,
// 652-659).  Tokens left out keep the previous value, G,-8,1 at first.  An empty first token, which the reference does
// not handle, is refused.
static bool intronFunc(const char* opt, const std::string& v, int32_t& type, double& C, double& L)
{
    std::vector<std::string> t = refTokens(v, ',');
    if (t.empty() || t[0].empty()) { fprintf(stderr, "Error: %s needs a function type as its first comma-separated token\n", opt); return false; }
    if (type == 0) { C = -8.0; L = 1.0; }
    const std::string& ty = t[0];
    if (ty == "C" || ty == "Constant") type = 'C'; else if (ty == "L" || ty == "Linear") type = 'L';
    else if (ty == "S" || ty == "Sqrt") type = 'S'; else if (ty == "G" || ty == "Log") type = 'G';
    else {
        fprintf(stderr, "Error: Bad function type '%s'.  Should be C (constant), L (linear), S (square root) or G (natural log).\n", ty.c_str());
        return false;
    }
    auto num = [](const std::string& x) { double d = 0; std::istringstream ss(x); ss >> d; return d; };   // as PARSE_FUNC reads it
    if (t.size() > 1) C = num(t[1]);
    if (t.size() > 2) L = num(t[2]);
    return true;
}
// -U / -1 / -2 a,b,c: appended to the list, empty names dropped (tokenize, hisat2.cpp:1120-1121, 1621-1626)
static void addFiles(std::vector<std::string>& v, const char* arg)
{
    std::string a = arg;
    for (size_t p = 0; p <= a.size();) {
        size_t c = a.find(',', p);
        if (c == std::string::npos) c = a.size();
        if (c > p) v.push_back(a.substr(p, c - p));
        p = c + 1;
    }
}

int main(int argc, char** argv)
{
    ht2gpu_options_t o; ht2gpu_default_options(&o);
    o.no_spliced_alignment = 0; // must be requested explicitly, like the reference's default is spliced
    const char *idx = NULL, *out = NULL;
    std::vector<std::string> us, m1s, m2s;   // -U, -1, -2
    bool fastq = true; size_t batchSz = 0 /* library default */; uint32_t gseed = 0;
    int trim5 = 0, trim3 = 0, threads = 0, gpus = 1; bool phred64 = false, solexa = false, intQuals = false; uint64_t skip = 0, upto = 0;
    bool sensitive = false, verySensitive = false, fast = false, noTempSpliceSite = false;
    const char *knownSs = NULL, *novelSs = NULL, *novelOut = NULL;   // --known-splicesite-infile / --novel-splicesite-infile (hisat2.cpp:1689-1691)
    // SAM output (hisat2.cpp:601-623, 1342-1343, 1389-1407): --no-hd prints no header at all (no @PG either,
    // hisat2.cpp:4127-4131); --rg ID:<x> sets the read-group id like --rg-id <x>, any other --rg text is an @RG field
    bool noHd = false, newSummary = false, quiet = false;
    int32_t noUnal = 0, omitSecSeq = 0, noSq = 0, rnaStrandness = 0, noQnameTrunc = 0, noTlenAdj = 0;
    std::string rgId; std::vector<std::string> rgFields;
    const char* summaryFile = NULL;
    ReadFiles rfs;
    int maBonus = 0;   // --ma: the last one counts (MA=, aligner_seed_policy.cpp:363-373)
    bool mpGiven = false;   // "--mp a,b" becomes MMP=Q,a,b, which switches the cost model back to quality-aware even
                            // under --ignore-quals (aligner_seed_policy.cpp:396-418)
    for (int i = 1; i < argc; i++) {
        std::string a = argv[i];
        auto next = [&]() -> const char* { if (i + 1 >= argc) { usage(); exit(1); } return argv[++i]; };
        if (a == "-x") idx = next(); else if (a == "-U") addFiles(us, next()); else if (a == "-1") addFiles(m1s, next()); else if (a == "-2") addFiles(m2s, next());
        else if (a == "-S") out = next(); else if (a == "-f") fastq = false; else if (a == "-q") fastq = true;
        else if (a == "--no-spliced-alignment") o.no_spliced_alignment = 1;
        else if (a == "--no-temp-splicesite") noTempSpliceSite = true;   // spliced mode with an empty splice-site DB: the only spliced form a (HT2_SPLICED=1) library build honours
        else if (a == "--known-splicesite-infile") knownSs = next(); else if (a == "--novel-splicesite-infile") novelSs = next();
        else if (a == "--novel-splicesite-outfile") novelOut = next();
        else if (a == "-k") o.khits = atoi(next()); else if (a == "--max-seeds") o.max_seeds = atoi(next());
        else if (a == "--secondary") o.secondary = 1;
        else if (a == "--mp") { two(next(), o.mp_max, o.mp_min); mpGiven = true; } else if (a == "--sp") { two(next(), o.sp_max, o.sp_min); o.sp_min = o.sp_max; /* the reference reads BOTH values from the first number, aligner_seed_policy.cpp:438-441 */ }
        else if (a == "--np") o.np = atoi(next()); else if (a == "--rdg") two(next(), o.rdg_const, o.rdg_linear);
        else if (a == "--rfg") two(next(), o.rfg_const, o.rfg_linear); else if (a == "--ignore-quals") o.ignore_quals = 1;
        else if (a == "--nofw") o.nofw = 1; else if (a == "--norc") o.norc = 1;
        else if (a == "-I" || a == "--minins") o.min_frag = atoi(next()); else if (a == "-X" || a == "--maxins") o.max_frag = atoi(next());
        else if (a == "--no-mixed") o.no_mixed = 1; else if (a == "--no-discordant") o.no_discordant = 1;
        else if (a == "--seed") gseed = (uint32_t)atoi(next()); else if (a == "--batch") batchSz = (size_t)atol(next());
        else if (a == "--device") o.device = atoi(next());
        else if (a == "--gpus") gpus = atoi(next());   // devices device .. device + gpus - 1: batches round-robin, output in input order
        else if (a == "--bowtie2-dp") { o.bowtie2_dp = atoi(next()); if (o.bowtie2_dp < 0 || o.bowtie2_dp > 2) { fprintf(stderr, "Error: --bowtie2-dp arg must be 0, 1, or 2\n"); return 1; } }
        else if (a == "--gbar") o.gbar = atoi(next());
        else if (a == "--score-min" || a == "--min-score") {   // <type>,<const>,<coeff>; missing tokens keep the default (PARSE_FUNC, aligner_seed_policy.cpp:47-62)
            std::string v = next(); size_t c1 = v.find(','), c2 = c1 == std::string::npos ? c1 : v.find(',', c1 + 1);
            if (!v.empty()) o.score_min_type = v[0];
            if (c1 != std::string::npos) o.score_min_const = atof(v.c_str() + c1 + 1);
            if (c2 != std::string::npos) o.score_min_coeff = atof(v.c_str() + c2 + 1);
            if (o.score_min_type != 'C' && o.score_min_type != 'L' && o.score_min_type != 'S' && o.score_min_type != 'G') { fprintf(stderr, "Error: bad function type in --score-min\n"); return 1; }
        }
        else if (a == "--sensitive") sensitive = true; else if (a == "--very-sensitive") verySensitive = true; else if (a == "--fast") fast = true;
        else if (a == "-p" || a == "--threads") threads = atoi(next());   // host parser threads; the alignment itself runs on the GPU
        else if (a == "-5" || a == "--trim5") trim5 = atoi(next()); else if (a == "-3" || a == "--trim3") trim3 = atoi(next());
        else if (a == "-s" || a == "--skip") skip = (uint64_t)atoll(next()); else if (a == "-u" || a == "--upto" || a == "--qupto") upto = (uint64_t)atoll(next());
        else if (a == "--phred64" || a == "--phred64-quals" || a == "--solexa1.3-quals") phred64 = true; else if (a == "--phred33" || a == "--phred33-quals") phred64 = solexa = false;
        else if (a == "--no-unal") noUnal = 1;
        else if (a == "--omit-sec-seq" || a == "--sam-omit-sec-seq") omitSecSeq = 1;
        else if (a == "--no-hd" || a == "--no-head" || a == "--no-HD" || a == "--sam-no-hd" || a == "--sam-no-head" || a == "--sam-nohead" || a == "--sam-noHD") noHd = true;
        else if (a == "--no-sq" || a == "--no-SQ" || a == "--sam-no-sq" || a == "--sam-nosq" || a == "--sam-noSQ") noSq = 1;
        else if (a == "--rg-id" || a == "--sam-rg-id") rgId = next();
        else if (a == "--rg" || a == "--RG" || a == "--sam-rg" || a == "--sam-RG") {
            std::string v = next();
            if (v.compare(0, 3, "ID:") == 0) rgId = v.substr(3); else rgFields.push_back(v);
        }
        else if (a == "--rna-strandness") {   // hisat2.cpp:1694-1705; read.h:30-36 numbering
            const std::string v = next();
            if (v == "F") rnaStrandness = 1; else if (v == "R") rnaStrandness = 2; else if (v == "FR") rnaStrandness = 3; else if (v == "RF") rnaStrandness = 4;
            else { fprintf(stderr, "Error: should be one of F, R, FR, or RF \n"); return 1; }
        }
        else if (a == "--remove-chrname") o.chr_names |= HT2GPU_CHR_NAMES_REMOVE; else if (a == "--add-chrname") o.chr_names |= HT2GPU_CHR_NAMES_ADD;
        else if (a == "--no-templatelen-adjustment") noTlenAdj = 1; else if (a == "--sam-no-qname-trunc") noQnameTrunc = 1;
        else if (a == "--summary-file") summaryFile = next(); else if (a == "--new-summary") newSummary = true;
        else if (a == "--quiet") quiet = true;   // no alignment summary (hisat2.cpp:4165)
        else if (a.compare(0, 2, "--") == 0 && [&]() {
                     for (int w = 0; w < HT2GPU_READS_N; w++)
                         for (int c = 0; c < 3; c++)
                             if (a == std::string("--") + kReadOpt[w] + (c == 1 ? "-gz" : c == 2 ? "-bz2" : "")) { rfs.spec[w] = next(); rfs.compress[w] = c; return true; }
                     return false; }()) {}
        else if (a == "--fr") o.pe_orient = HT2GPU_PE_FR; else if (a == "--rf") o.pe_orient = HT2GPU_PE_RF; else if (a == "--ff") o.pe_orient = HT2GPU_PE_FF;
        else if (a == "--n-ceil") { if (!nCeil(next(), o)) return 1; }
        else if (a == "--ma") {   // the match bonus is always 0 in end-to-end mode: warned about below, then ignored
            const std::string v = next();
            if (refTokens(v, ',').size() != 1) { fprintf(stderr, "Error parsing alignment policy setting MA=%s; RHS must have 1 token\n", v.c_str()); return 1; }
            maBonus = atoi(v.c_str());
        }
        else if (a == "--no-softclip") { o.sp_max = o.sp_min = 2147483647; }   // SCP=Q,INT_MAX,INT_MAX, in order with --sp (hisat2.cpp:1588-1596)
        else if (a == "--solexa-quals") solexa = true;
        else if (a == "--int-quals" || a == "--integer-quals") intQuals = true;
        else if (a == "--pen-cansplice") { if (!refInt(next(), 0, "--pen-cansplice arg must be at least 0", o.pen_cansplice)) return 1; }
        else if (a == "--pen-noncansplice") { if (!refInt(next(), 0, "--pen-noncansplice arg must be at least 0", o.pen_noncansplice)) return 1; }
        else if (a == "--pen-conflictsplice") { if (!refInt(next(), 0, "--pen-conflictsplice arg must be at least 0", o.pen_conflictsplice)) return 1; }
        else if (a == "--pen-canintronlen" || a == "--pen-intronlen") { if (!intronFunc(a.c_str(), next(), o.can_intronlen_type, o.can_intronlen_const, o.can_intronlen_coeff)) return 1; }
        else if (a == "--pen-noncanintronlen") { if (!intronFunc(a.c_str(), next(), o.noncan_intronlen_type, o.noncan_intronlen_const, o.noncan_intronlen_coeff)) return 1; }
        else if (a == "--min-intronlen") { if (!refInt(next(), 20, "--min-intronlen arg must be at least 20", o.min_intronlen)) return 1; }
        else if (a == "--max-intronlen") { if (!refInt(next(), 20, "--max-intronlen arg must be at least 20", o.max_intronlen)) return 1; }
        else if (a == "--dta" || a == "--downstream-transcriptome-assembly") { if (o.dta == HT2GPU_DTA_NONE) o.dta = HT2GPU_DTA_STRINGTIE; }
        else if (a == "--dta-cufflinks") o.dta = HT2GPU_DTA_CUFFLINKS;
        else if (a == "--no-anchorstop") o.no_anchorstop = 1;
        else if (a == "--tmo" || a == "--transcriptome-mapping-only") o.tmo = 1;
        else if (a == "--avoid-pseudogene") o.avoid_pseudogene = 1;
        else if (a == "--reorder" || a == "-t" || a == "--time" || a == "--no-unal-ignored" || a == "--splicesite-db-only") {}
        else if (a == "-h" || a == "--help") { usage(); return 0; }
        else { fprintf(stderr, "Error: option %s is not supported by hisat2-b200\n", a.c_str()); return 1; }
    }
    if (!idx || (us.empty() && m1s.empty() && m2s.empty())) { usage(); return 1; }
    if (m1s.size() != m2s.size()) {   // hisat2.cpp:1911-1913
        fprintf(stderr, "Error: %zu mate files/sequences were specified with -1, but %zu\n"
                        "mate files/sequences were specified with -2.  The same number of mate files/\n"
                        "sequences must be specified with -1 and -2.\n", m1s.size(), m2s.size());
        return 1;
    }
    {
        int nStdin = 0;
        for (const auto* v : {&us, &m1s, &m2s}) for (const std::string& f : *v) nStdin += f == "-";
        if (nStdin > 1) { fprintf(stderr, "Error: standard input ('-') can be read only once\n"); return 1; }
    }
    if (!o.no_spliced_alignment && !noTempSpliceSite)
        fprintf(stderr, "Warning: temporary splice sites (the reference's default) make results depend on the order reads are processed in;\n"
                        "         hisat2-b200 aligns every read independently, i.e. as with --no-temp-splicesite\n");
    if (o.min_intronlen > o.max_intronlen) {   // hisat2.cpp:4278-4283
        fprintf(stderr, "--min-intronlen(%d) should not be greater than --max-intronlen(%d)\n", o.min_intronlen, o.max_intronlen);
        return 1;
    }
    if (mpGiven) o.ignore_quals = 0;
    if (maBonus > 0) fprintf(stderr, "Warning: Match bonus always = 0 in --end-to-end mode; ignoring user setting\n");   // hisat2.cpp:3916-3919
    // presets, spelled out the way hisat2.cpp:1889-1909 applies them after option parsing
    if (fast) {}
    else if (sensitive) {
        if (o.bowtie2_dp == 0) o.bowtie2_dp = 1;
        if (o.khits > 0 && o.khits < 10) o.khits = 10;   // an omitted -k stays "index default": the parse-time default is 10 (hisat2.cpp:336, 3903-3906)
        o.score_min_type = 'L'; o.score_min_const = (double)0.0f; o.score_min_coeff = (double)-0.5f;
    } else if (verySensitive) {
        o.bowtie2_dp = 2;
        if (o.khits < 30) o.khits = 30;
        o.score_min_type = 'L'; o.score_min_const = (double)0.0f; o.score_min_coeff = (double)-1.0f;
    }
    o.seed = gseed;
    // read files: opened before the run starts, like the wrapper
    for (int w = 0; w < HT2GPU_READS_N; w++) {
        if (rfs.spec[w].empty()) continue;
        const int nMates = w >= HT2GPU_READS_UN_CONC ? 2 : 1;
        for (int m = 0; m < nMates; m++) {
            const std::string fn = readFileName(rfs.spec[w], w, nMates == 2 ? m + 1 : 0);
            if (!openReadFile(rfs.file[w][m], fn, rfs.compress[w])) {
                fprintf(stderr, "Error: could not open --%s%s output file '%s'\n", kReadOpt[w], nMates == 2 ? (m ? " mate-2" : " mate-1") : "", fn.c_str());
                return 1;
            }
        }
    }
    ht2gpu_handle_t* h = NULL;
    if (ht2gpu_open(idx, &o, &h) != HT2GPU_OK) { fprintf(stderr, "Error: %s\n", ht2gpu_last_error(h)); return 1; }
    FILE* fo = out ? fopen(out, "wb") : stdout;
    if (!fo) { fprintf(stderr, "Error: cannot write %s\n", out); return 1; }
    std::vector<const char*> rgPtrs;
    for (const std::string& f : rgFields) rgPtrs.push_back(f.c_str());
    ht2gpu_sam_output_t so; memset(&so, 0, sizeof(so));
    so.no_unal = noUnal; so.omit_sec_seq = omitSecSeq; so.no_sq = noSq;
    so.rg_id = rgId.empty() ? NULL : rgId.c_str(); so.rg = rgPtrs.data(); so.n_rg = (int32_t)rgPtrs.size();
    so.rna_strandness = rnaStrandness; so.no_qname_trunc = noQnameTrunc; so.no_templatelen_adjustment = noTlenAdj;
    if (ht2gpu_set_sam_output(h, &so) != HT2GPU_OK) { fprintf(stderr, "Error: %s\n", ht2gpu_last_error(h)); return 1; }
    if (!noHd) {
        char* hd; size_t hl; ht2gpu_sam_header(h, &hd, &hl); fwrite(hd, 1, hl, fo); ht2gpu_free_text(hd);
        fprintf(fo, "@PG\tID:hisat2\tPN:hisat2-b200\tVN:0.2\n");
    }
    ht2gpu_reads_input_t in; memset(&in, 0, sizeof(in));
    std::vector<const char*> p1, p2, pu;
    for (const std::string& f : m1s) p1.push_back(f.c_str());
    for (const std::string& f : m2s) p2.push_back(f.c_str());
    for (const std::string& f : us) pu.push_back(f.c_str());
    ht2gpu_reads_files_t lists;
    lists.paths1 = p1.data(); lists.n1 = (uint32_t)p1.size(); lists.paths2 = p2.data(); lists.n2 = (uint32_t)p2.size();
    lists.paths_u = pu.data(); lists.n_u = (uint32_t)pu.size();
    in.format = fastq ? 1 : 0; in.trim5 = trim5; in.trim3 = trim3; in.phred64 = phred64 ? 1 : 0; in.seed = gseed;
    in.solexa_quals = solexa ? 1 : 0; in.int_quals = intQuals ? 1 : 0;
    in.skip = skip; in.upto = upto; in.batch_reads = (uint32_t)batchSz; in.threads = threads;
    ht2gpu_read_routes_t routes; memset(&routes, 0, sizeof(routes));
    routes.mask = rfs.mask(); routes.ctx = &rfs;
    routes.write = [](void* ctx, int which, int mate, const char* data, size_t len) -> int {
        FILE* f = ((ReadFiles*)ctx)->file[which][mate == 2 ? 1 : 0].f;
        return fwrite(data, 1, len, f) == len ? 0 : 1;
    };
    ht2gpu_run_stats_t st;
    auto sink = [](void* ctx, const char* sam, size_t len) -> int { return fwrite(sam, 1, len, (FILE*)ctx) == len ? 0 : 1; };
    std::vector<ht2gpu_handle_t*> hs(1, h);
    for (int g = 1; g < gpus; g++) {   // replicate the index device to device
        ht2gpu_options_t og = o; og.device = o.device + g;
        ht2gpu_handle_t* hg = NULL;
        if (ht2gpu_open_peer(h, &og, &hg) != HT2GPU_OK) { fprintf(stderr, "Error: device %d: %s\n", og.device, ht2gpu_last_error(hg)); return 1; }
        hs.push_back(hg);
        if (ht2gpu_set_sam_output(hg, &so) != HT2GPU_OK) { fprintf(stderr, "Error: %s\n", ht2gpu_last_error(hg)); return 1; }
    }
    if (knownSs || novelSs) {
        uint32_t ns = 0;
        for (ht2gpu_handle_t* hh : hs)
            if (ht2gpu_load_splicesites(hh, knownSs, novelSs, &ns) != HT2GPU_OK) { fprintf(stderr, "Error: %s\n", ht2gpu_last_error(hh)); return 1; }
    }
    if (novelOut)
        for (ht2gpu_handle_t* hh : hs)
            if (ht2gpu_collect_splicesites(hh, 1) != HT2GPU_OK) { fprintf(stderr, "Error: %s\n", ht2gpu_last_error(hh)); return 1; }
    const int runRc = ht2gpu_run_reads_files(hs.data(), (int)hs.size(), &lists, &in, sink, fo, &routes, &st);
    bool filesOk = true;
    for (int w = 0; w < HT2GPU_READS_N; w++)
        for (int m = 0; m < 2; m++) {
            ReadFile& rf = rfs.file[w][m];
            if (rf.f && !closeReadFile(rf)) { fprintf(stderr, "Error: could not write --%s output file '%s'\n", kReadOpt[w], rf.path.c_str()); filesOk = false; }
        }
    if (runRc != HT2GPU_OK) { fprintf(stderr, "Error: %s\n", ht2gpu_last_error(h)); return 1; }
    if (!filesOk) return 1;
    if (novelOut) {
        uint64_t nw = 0;
        if (ht2gpu_write_novel_splicesites(hs.data(), (int)hs.size(), novelOut, &nw) != HT2GPU_OK) { fprintf(stderr, "Error: %s\n", ht2gpu_last_error(h)); return 1; }
    }
    if (st.n_err_reads)
        fprintf(stderr, "Warning: %llu read(s) exceeded a device-side capacity; their records may differ from hisat2's\n", (unsigned long long)st.n_err_reads);
    if (fo != stdout) fclose(fo);
    if (!quiet) {   // the alignment summary over every device (AlnSink::finish, hisat2.cpp:4165-4185)
        ht2gpu_align_counts_t c;
        char* txt = NULL; size_t tl = 0;
        if (ht2gpu_align_counts(hs.data(), (int)hs.size(), 0, &c) != HT2GPU_OK ||
            ht2gpu_format_align_summary(&c, newSummary ? 1 : 0, o.no_discordant ? 0 : 1, o.no_mixed ? 0 : 1, &txt, &tl) != HT2GPU_OK) {
            fprintf(stderr, "Error: cannot format the alignment summary\n"); return 1;
        }
        fwrite(txt, 1, tl, stderr);
        if (summaryFile) {
            FILE* fs = fopen(summaryFile, "wb");
            if (fs) { fwrite(txt, 1, tl, fs); fclose(fs); }
        }
        ht2gpu_free_text(txt);
    }
    for (size_t g = 1; g < hs.size(); g++) ht2gpu_close(hs[g]);
    ht2gpu_close(h);
    return 0;
}
