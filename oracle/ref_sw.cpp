// oracle/ref_sw.cpp -- TEST INFRASTRUCTURE.  A small driver that links the
// UNMODIFIED reference (headers and objects of the reference sources at
// $(REF), built by oracle/Makefile) and runs the --bowtie2-dp seed extension of
// SplicedAligner::hybridSearch (spliced_aligner.h:209-297) on one job per
// input line: SwAligner::initRead on the read, frameSeedExtensionRect
// (readGaps = refGaps = maxhalf = 10, nceil = 0, trimToRef = false), initRef
// with the arguments of that call site, align, one nextAlignment, and
// invertEdits for the reverse strand.  The job lines are written by
// tools/swjobs.py.
//
// Input (one job per line, whitespace separated):
//   <id> <mp_max> <mp_min> <ignore_quals> <np> <rdg_const> <rdg_linear> <rfg_const> <rfg_linear> <gbar>
//   <fw> <tidx> <toff> <rdoff> <len> <minsc> <seed> <READ> <QUAL>
// Output (one line per job):
//   <id> <found> <coord.off|-> <score|-> <best|-> <rnd.nextU32() after> <edits: pos:type:chr:qchr,...|->
// "found" without an offset is the anchor that already spans the read (no DP); best is "-" when the DP
// was not run or when no last-row cell reached minsc.
// usage: ref_sw <index_base> <jobs.txt>
#include <stdlib.h>
#include <stdint.h>
#include <iostream>
#include <fstream>
#include <sstream>
#include <string>
#include <limits>
#include "alphabet.h"
#include "assert_helpers.h"
#include "ds.h"
#include "read.h"
#include "scoring.h"
#include "simple_func.h"
#include "random_source.h"
#include "reference.h"
#include "dp_framer.h"
#include "aligner_sw.h"
#include "aligner_result.h"

using namespace std;

bool gColor = false, gColorExEnds = false, gReportOverhangs = false, gColorSeq = false, gColorEdit = false,
     gColorQual = false, gNoMaqRound = false, gStrandFix = false, gRangeMode = false;
int gVerbose = 0, gQuiet = 0;
bool gNofw = false, gNorc = false, gMate1fw = true, gMate2fw = false;
int gMinInsert = 0, gMaxInsert = 1000, gTrim5 = 0, gTrim3 = 0, gGapBarrier = 4, gAllowRedundant = 0;

extern void initializeCntLut();
extern void initializeCntBit();
MemoryTally gMemTally;

int main(int argc, char** argv) {
    if(argc < 3) { cerr << "usage: ref_sw index jobs.txt" << endl; return 2; }
    initializeCntLut();
    initializeCntBit();
    BitPairReference ref(argv[1], NULL, false);
    if(!ref.loaded()) { cerr << "ref_sw: cannot load the reference of " << argv[1] << endl; return 1; }
    ifstream in(argv[2]);
    if(!in) { cerr << "ref_sw: cannot open " << argv[2] << endl; return 1; }
    SwAligner swa;
    LinkedEList<EList<Edit> > rawEdits;
    string line;
    while(getline(in, line)) {
        if(line.empty() || line[0] == '#') continue;
        istringstream is(line);
        long long id, mpMax, mpMin, ignq, np, rdc, rdl, rfc, rfl, gbar, fw, tidx, toff, rdoff, len, minsc;
        unsigned long long seed;
        string seq, qual;
        if(!(is >> id >> mpMax >> mpMin >> ignq >> np >> rdc >> rdl >> rfc >> rfl >> gbar >> fw >> tidx >> toff >> rdoff
                >> len >> minsc >> seed >> seq >> qual) || seq.size() != qual.size()) {
            cerr << "ref_sw: malformed job line: " << line << endl;
            return 1;
        }
        gGapBarrier = (int)gbar;
        SimpleFunc scoreMin; scoreMin.init(SIMPLE_FUNC_LINEAR, 0.0f, -0.2f);
        SimpleFunc nCeil; nCeil.init(SIMPLE_FUNC_LINEAR, 0.0f, 0.15f);
        SimpleFunc icp, incp; icp.init(SIMPLE_FUNC_LOG, -8, 1); incp.init(SIMPLE_FUNC_LOG, -8, 1);
        Scoring sc(0, ignq ? DEFAULT_MM_PENALTY_TYPE_IGNORE_QUALS : DEFAULT_MM_PENALTY_TYPE, (int)mpMax, (int)mpMin, 2, 1,
                   scoreMin, nCeil, DEFAULT_N_PENALTY_TYPE, (int)np, false, (int)rdc, (int)rfc, (int)rdl,
                   (int)rfl, (int)gbar, 0, 12, 24, &icp, &incp);
        Read rd;
        rd.name.install("job");
        for(size_t i = 0; i < seq.size(); i++) { rd.patFw.append(asc2dna[(int)seq[i]]); rd.qual.append(qual[i]); }
        rd.finalize();
        rd.constructRevComps();
        rd.constructReverses();
        RandomSource rnd; rnd.init((uint32_t)seed);
        cout << id << " ";
        swa.initRead(rd.patFw, rd.patRc, rd.qual, rd.qualRev, 0, rd.length(), sc);
        if((size_t)len >= rd.length()) {
            cout << "1 - - - " << rnd.nextU32() << " -\n";
            continue;
        }
        DynProgFramer dpframe(false);
        size_t tlen = ref.approxLen((size_t)tidx);
        size_t readGaps = 10, refGaps = 10, nceil = 0, maxhalf = 10;
        uint32_t refoff = toff > rdoff ? (uint32_t)(toff - rdoff) : 0;
        DPRect rect;
        dpframe.frameSeedExtensionRect(refoff, rd.length(), tlen, readGaps, refGaps, nceil, maxhalf, rect);
        size_t cminlen = 2000, cpow2 = 4, nwindow = 10, nsInLeftShift = 0;
        swa.initRef(fw != 0, (TRefId)tidx, rect, ref, tlen, sc, minsc, true, cminlen, cpow2, false, true, nwindow, nsInLeftShift);
        TAlScore best = std::numeric_limits<TAlScore>::min();
        bool found = swa.align(rnd, best);
        SwResult res;
        if(found) {
            res.reset();
            res.alres.init_raw_edits(&rawEdits);
            found = swa.nextAlignment(res, minsc, rnd);
            if(found && fw == 0) res.alres.invertEdits();
        }
        ostringstream bs;
        if(best == std::numeric_limits<TAlScore>::min()) bs << "-"; else bs << best;
        if(!found) {
            cout << "0 - - " << bs.str() << " " << rnd.nextU32() << " -\n";
        } else {
            const EList<Edit>& ned = res.alres.ned();
            cout << "1 " << res.alres.refcoord().off() << " " << res.alres.score().score() << " " << bs.str() << " "
                 << rnd.nextU32() << " ";
            if(ned.empty()) cout << "-";
            for(size_t i = 0; i < ned.size(); i++)
                cout << (i ? "," : "") << ned[i].pos << ":" << (int)ned[i].type << ":" << (char)ned[i].chr << ":" << (char)ned[i].qchr;
            cout << "\n";
        }
        swa.reset();
    }
    return 0;
}
