// ht2_transim.cpp -- TEST-ONLY host build of ht2_sploptsim for indexes built with splice sites / exons
// (hisat2-build --ss / --exon).  In spliced mode (HT2_OPTS spliced=1) the run's splice-site DB always holds the index's
// sites and exons, as ht2gpu_open builds it: with no HT2_SS given, the DB is the index's alone (an empty file name,
// which ht2_ssdb_build skips like any unreadable file).
// usage and every variable as ht2_sploptsim.
#include <stdlib.h>
#include <string.h>

static struct TranDefaultDb {
    TranDefaultDb() {
        const char* o = getenv("HT2_OPTS");
        if (o && strstr(o, "spliced=1") && !getenv("HT2_SS")) setenv("HT2_SS", "", 1);
    }
} g_tranDefaultDb;

#include "ht2_sploptsim.cpp"
