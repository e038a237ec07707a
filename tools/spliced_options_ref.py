#!/usr/bin/env python3
"""Spliced-alignment options against the unmodified reference: --pen-cansplice, --pen-noncansplice,
--pen-conflictsplice, --pen-canintronlen / --pen-noncanintronlen, --min-intronlen / --max-intronlen, --dta /
--dta-cufflinks, --no-anchorstop, --tmo, --avoid-pseudogene and --splicesite-db-only.

  python tools/spliced_options_ref.py      # writes tests/golden/spliced_options_sets.json

The expected values come from oracle/_ref/hisat2-align-s (oracle/Makefile), run with --no-temp-splicesite --reorder
on tools/refsets.py's spliced and DNA sets and on one set of its own (generate_splopt, seeded): junctions whose
intron lengths sit at the steps of the intron-length functions the cases use, at the --min-intronlen /
--max-intronlen bounds of the cases, with the 14 / 15 and 19 / 20-base anchors --dta moves, and with semi- and
non-canonical motifs; and on refsets' repeat reads (windows of tiny.fa that occur twice) with a site file next to
some of them (generate_rep), where --avoid-pseudogene chooses the copy near a site.  The JSON keeps, per case, the md5 of the SAM without @PG (and without the records of refsets'
flagged reads) and the alignment summary the reference prints, and, for the argument errors, the first line it prints
to stderr with its exit status."""
import json
import math
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import refsets  # noqa: E402

GOLDEN = refsets.GOLDEN
OUT = os.path.join(GOLDEN, "spliced_options_sets.json")
SPLOPT_SEED = 23
MIN_I, MAX_I = 50, 2000   # the --min-intronlen / --max-intronlen of the bound cases


def steps(t, c, l, upto, n):
    """The first n intron lengths x >= 2 at which max(0, (int)(c + l * F(x))) changes, below upto."""
    f = lambda x: max(0, int(c + l * {"C": 0.0, "L": float(x), "S": math.sqrt(x), "G": math.log(x)}[t]))
    out, prev = [], f(1)
    for x in range(2, upto):
        v = f(x)
        if v != prev:
            out.append(x)
            prev = v
            if len(out) == n:
                break
    return out


def splopt_lengths():
    """Intron lengths at the boundaries the cases move: each step and the length before it."""
    ls = {MIN_I - 1, MIN_I, MIN_I + 1, MAX_I - 1, MAX_I, MAX_I + 1}
    for fn, n in ((("G", -8.0, 1.0), 2), (("G", -8.0, 2.0), 8), (("L", 0.0, 0.01), 3), (("S", -10.0, 0.5), 3),
                  (("G", -4.0, 1.0), 3), (("S", -5.0, 0.3), 3), (("L", -2.0, 0.001), 2), (("G", -6.0, 1.0), 2)):
        for x in steps(*fn, 30000, n):
            ls |= {x - 1, x}
    return sorted(l for l in ls if l >= 19)


def generate_splopt(d):
    """d/splopt_se.fa (101-base reads, one junction each) and d/splopt_ss.txt (85 % of their introns plus decoys)."""
    se = os.path.join(d, "splopt_se.fa")
    if os.path.exists(se):
        return se
    import splicereads
    from edgereads import load_contigs, write_fasta
    g = splicereads.SpliceGen(load_contigs(os.path.join(GOLDEN, "tiny.fa")), SPLOPT_SEED)
    out = []
    for L in splopt_lengths():   # canonical, semi-canonical and non-canonical introns at every step, both strands
        for m in ("GTAG", "CTAC", "GCAG", "non"):
            for rep in range(2):
                left = int(g.rng.integers(30, 72))
                j = g.junction(L, m, left, 101 - left)
                if j:
                    out.append(("len_%d_%s_%d" % (L, m, rep), g.strand(j[0], rep)))
    for a in (12, 13, 14, 15, 16, 18, 19, 20, 21, 22):   # the anchors --dta requires (15 canonical, 20 otherwise)
        for m in ("GTAG", "CTAC", "ATAC", "non"):
            for side in range(2):
                L = int(g.rng.integers(300, 6000))
                left = a if side == 0 else 101 - a
                j = g.junction(L, m, left, 101 - left)
                if j:
                    out.append(("anchor_%d_%s_%d_%d" % (a, m, side, L), g.strand(j[0], int(g.rng.integers(0, 2)))))
    for k in range(40):   # two junctions, of the same or of opposite sense (--pen-conflictsplice, --dta-cufflinks)
        ms = (("GTAG", "CTAC"), ("GTAG", "GCAG"), ("CTAC", "CTGC"), ("GTAG", "non"))[k % 4]
        r = g.chain(101, ms, mid=(25, 41), lens=(100, 3000))
        if r:
            out.append(("sense_%s_%s_%d" % (ms[0], ms[1], k), g.strand(r, k & 1)))
    write_fasta(se, out)
    open(os.path.join(d, "splopt_ss.txt"), "w").write("\n".join(splicereads.site_lines(g)) + "\n")
    return se


def generate_rep(d):
    """refsets' rep_1.fa (windows of tiny.fa that occur exactly twice) under d, and d/rep_ss.txt: a site a few hundred
    bases right of every 25th of those windows, so that one copy of some repeats lies near a listed site and the other
    may not (--avoid-pseudogene)."""
    refsets.generate_repeats(d)
    ss = os.path.join(d, "rep_ss.txt")
    if not os.path.exists(ss):
        reads = [l[5:].strip() for l in open(os.path.join(d, "rep_1.fa")) if l.startswith(">")]
        with open(ss, "w") as f:
            for name in reads[::25]:
                chrom, pos = name.rsplit("_", 1)
                f.write("%s\t%d\t%d\t+\n" % (chrom, int(pos) + 300, int(pos) + 900))
    return ss


def _c(src, flags, **opts):
    return dict(src=src, flags=list(flags), opts=opts)


SO, SO_SS = ("splopt", "se"), ("splopt", "se_ss")
REP, REP_SS = ("rep", "se"), ("rep", "se_ss")
DTA = dict(dta=1)
CASES = {
    # the default run of every input the cases below use
    "default_rep": _c(REP, []),
    "default_rep_ss": _c(REP_SS, []),
    "default_spliced_edge_se": _c(("spliced", "edge_se"), []),
    "default_spliced_edge_pe": _c(("spliced", "edge_pe"), []),
    "default_spliced_sim_pe": _c(("spliced", "sim_pe"), []),
    "default_spliced_ss_sim_pe": _c(("spliced", "ss_sim_pe"), []),
    "default_spliced_graph_ss_sim_pe": _c(("spliced", "graph_ss_sim_pe"), []),
    "default_spliced_graph_edge_se": _c(("spliced", "graph_edge_se"), []),
    "default_se_reads": _c(("se", "reads"), []),
    "default_paired_reads": _c(("paired", "reads"), []),
    "default_so": _c(SO, []),
    "default_so_ss": _c(SO_SS, []),
    "db_only_so_ss": _c(SO_SS, ["--splicesite-db-only"]),
    "pen_can3_so": _c(SO, ["--pen-cansplice", "3"], pen_cansplice=3),
    "pen_noncan0_so": _c(SO, ["--pen-noncansplice", "0"], pen_noncansplice=0),
    "pen_noncan30_so": _c(SO, ["--pen-noncansplice", "30"], pen_noncansplice=30),
    "pen_conflict0_so": _c(SO, ["--pen-conflictsplice", "0"], pen_conflictsplice=0),
    "pen_conflict0_edge_se": _c(("spliced", "edge_se"), ["--pen-conflictsplice", "0"], pen_conflictsplice=0),
    "can_G2_so": _c(SO, ["--pen-canintronlen", "G,-8,2"], can_intronlen_type="G", can_intronlen_const=-8.0, can_intronlen_coeff=2.0),
    "can_L_so": _c(SO, ["--pen-canintronlen", "L,0,0.01", "--max-intronlen", "50000"], can_intronlen_type="L", can_intronlen_const=0.0,
                   can_intronlen_coeff=0.01, max_intronlen=50000),
    "can_S_so": _c(SO, ["--pen-canintronlen", "S,-10,0.5"], can_intronlen_type="S", can_intronlen_const=-10.0, can_intronlen_coeff=0.5),
    "can_C_two_so": _c(SO, ["--pen-canintronlen", "C,3"], can_intronlen_type="C", can_intronlen_const=3.0, can_intronlen_coeff=1.0),
    "can_type_only_so": _c(SO, ["--pen-intronlen", "G"], can_intronlen_type="G", can_intronlen_const=-8.0, can_intronlen_coeff=1.0),
    "can_four_so": _c(SO, ["--pen-canintronlen", "Log,-6,1,5"], can_intronlen_type="G", can_intronlen_const=-6.0, can_intronlen_coeff=1.0),
    "can_L_small_so": _c(SO, ["--pen-canintronlen", "L,-2,0.001"], can_intronlen_type="L", can_intronlen_const=-2.0, can_intronlen_coeff=0.001),
    "noncan_G_two_so": _c(SO, ["--pen-noncanintronlen", "G,-4"], noncan_intronlen_type="G", noncan_intronlen_const=-4.0, noncan_intronlen_coeff=1.0),
    "noncan_C0_so": _c(SO, ["--pen-noncanintronlen", "C,0"], noncan_intronlen_type="C", noncan_intronlen_const=0.0, noncan_intronlen_coeff=1.0),
    "noncan_S_so": _c(SO, ["--pen-noncanintronlen", "Sqrt,-5,0.3"], noncan_intronlen_type="S", noncan_intronlen_const=-5.0, noncan_intronlen_coeff=0.3),
    "min_intron_so": _c(SO, ["--min-intronlen", str(MIN_I)], min_intronlen=MIN_I),
    "max_intron_so": _c(SO, ["--max-intronlen", str(MAX_I)], max_intronlen=MAX_I),
    "min_max_intron_so_ss": _c(SO_SS, ["--min-intronlen", str(MIN_I), "--max-intronlen", str(MAX_I)], min_intronlen=MIN_I, max_intronlen=MAX_I),
    "max_intron_ss_sim_pe": _c(("spliced", "ss_sim_pe"), ["--max-intronlen", "1000"], max_intronlen=1000),
    "max_intron_dna_pe": _c(("paired", "reads"), ["--max-intronlen", "100"], max_intronlen=100),
    "dta_so": _c(SO, ["--dta"], **DTA),
    "dta_noncan_so": _c(SO, ["--dta", "--pen-noncanintronlen", "C,0"], noncan_intronlen_type="C", noncan_intronlen_const=0.0,
                        noncan_intronlen_coeff=1.0, **DTA),
    "dta_so_ss": _c(SO_SS, ["--downstream-transcriptome-assembly"], **DTA),
    "dta_cufflinks_so": _c(SO, ["--dta-cufflinks"], dta=2),
    "dta_cufflinks_so_ss": _c(SO_SS, ["--dta-cufflinks"], dta=2),
    "dta_cufflinks_edge_pe": _c(("spliced", "edge_pe"), ["--dta-cufflinks"], dta=2),
    "no_anchorstop_k1_so": _c(SO, ["--no-anchorstop", "-k", "1"], no_anchorstop=1, khits=1),
    "no_anchorstop_k1_dna_se": _c(("se", "reads"), ["--no-anchorstop", "-k", "1"], no_anchorstop=1, khits=1),
    "no_anchorstop_sim_pe": _c(("spliced", "sim_pe"), ["--no-anchorstop"], no_anchorstop=1),
    "tmo_so": _c(SO, ["--tmo"], tmo=1),
    "tmo_so_ss": _c(SO_SS, ["--tmo"], tmo=1),
    "tmo_ss_sim_pe": _c(("spliced", "ss_sim_pe"), ["--transcriptome-mapping-only"], tmo=1),
    "tmo_dna_se": _c(("se", "reads"), ["--tmo"], tmo=1),
    "avoid_rep_ss": _c(REP_SS, ["--avoid-pseudogene"], avoid_pseudogene=1),
    "avoid_rep": _c(REP, ["--avoid-pseudogene"], avoid_pseudogene=1),
    "avoid_so_ss": _c(SO_SS, ["--avoid-pseudogene"], avoid_pseudogene=1),
    "avoid_ss_sim_pe": _c(("spliced", "ss_sim_pe"), ["--avoid-pseudogene"], avoid_pseudogene=1),
    "avoid_dna_se": _c(("se", "reads"), ["--avoid-pseudogene"], avoid_pseudogene=1),
    "avoid_k5_rep_ss": _c(REP_SS, ["--avoid-pseudogene", "-k", "5", "--secondary"], avoid_pseudogene=1, khits=5, secondary=1),
    "dta_dp2_so": _c(SO, ["--dta", "--bowtie2-dp", "2"], bowtie2_dp=2, **DTA),
    "can_G2_sensitive_so": _c(SO, ["--pen-canintronlen", "G,-8,2", "--sensitive"], can_intronlen_type="G", can_intronlen_const=-8.0,
                              can_intronlen_coeff=2.0, bowtie2_dp=1, score_min_type=ord("L"), score_min_const=0.0, score_min_coeff=-0.5),
    "dta_cufflinks_k20_sec_ss_sim_pe": _c(("spliced", "ss_sim_pe"), ["--dta-cufflinks", "-k", "20", "--secondary"], dta=2, khits=20, secondary=1),
    "dta_graph_ss_sim_pe": _c(("spliced", "graph_ss_sim_pe"), ["--dta"], **DTA),
    "noncan0_graph_edge_se": _c(("spliced", "graph_edge_se"), ["--pen-noncansplice", "0", "--pen-noncanintronlen", "C,0"],
                                pen_noncansplice=0, noncan_intronlen_type="C", noncan_intronlen_const=0.0, noncan_intronlen_coeff=1.0),
}
# argument errors: reference flags -> the first line of its stderr and its exit status (recorded under "errors")
ERRORS = {
    "pen_cansplice_negative": ["--pen-cansplice", "-1"],
    "pen_noncansplice_negative": ["--pen-noncansplice", "-3"],
    "pen_conflictsplice_negative": ["--pen-conflictsplice", "-1"],
    "min_intronlen_19": ["--min-intronlen", "19"],
    "max_intronlen_not_a_number": ["--max-intronlen", "abc"],
    "min_greater_than_max": ["--min-intronlen", "600", "--max-intronlen", "500"],
    "canintronlen_bad_type": ["--pen-canintronlen", "X,1"],
    "noncanintronlen_bad_type": ["--pen-noncanintronlen", "Q"],
}


def generate(d):
    """Every read set the CASES use under d; returns d."""
    refsets.generate(d, ("reads",))
    refsets.generate_spliced(d)
    generate_splopt(d)
    generate_rep(d)
    return d


def case_input(d, case):
    """(index, read files, format flag, reference flags, Index options, known-splice-site file or None) of a case
    under generate(d)."""
    c = CASES[case]
    if c["src"][0] == "rep":
        ss = generate_rep(d) if c["src"][1] == "se_ss" else None
        return "tiny", [os.path.join(d, "rep_1.fa")], "-f", \
            ["--no-temp-splicesite"] + (["--known-splicesite-infile", ss] if ss else []) + c["flags"], \
            dict(c["opts"], no_spliced_alignment=0), ss
    if c["src"][0] == "splopt":
        ss = os.path.join(d, "splopt_ss.txt") if c["src"][1] == "se_ss" else None
        return "tiny", [os.path.join(d, "splopt_se.fa")], "-f", \
            ["--no-temp-splicesite"] + (["--known-splicesite-infile", ss] if ss else []) + c["flags"], \
            dict(c["opts"], no_spliced_alignment=0), ss
    index, fs, fmt, base, opts, ss = refsets.output_input(d, c["src"])
    return index, fs, fmt, base + c["flags"], dict(opts, **c["opts"]), ss


def flagged(case):
    """The reads of a case's source that hit a fixed device capacity (refsets' `flagged`): no md5 covers their records."""
    src, fl = CASES[case]["src"], refsets.load_expected()["flagged"]
    return fl.get("spliced/" + src[1], []) if src[0] == "spliced" else []


def reference_run(d, case):
    """(SAM, stderr) of the reference on a case (--reorder)."""
    index, fs, fmt, flags, _, _ = case_input(d, case)
    out = os.path.join(d, "ref.sam")
    reads = ["-1", fs[0], "-2", fs[1]] if len(fs) == 2 else ["-U", fs[0]]
    r = subprocess.run([refsets.REFBIN, fmt, "-x", os.path.join(GOLDEN, index)] + flags + reads +
                       ["-S", out, "-p", str(min(16, os.cpu_count() or 1)), "--reorder"], check=True, stderr=subprocess.PIPE)
    return open(out, "rb").read(), r.stderr.decode()


def reference_error(d, flags):
    """(first line of the reference's stderr, exit status) for argument errors on a small input."""
    r = subprocess.run([refsets.REFBIN, "-f", "-x", os.path.join(GOLDEN, "tiny"), "--no-temp-splicesite"] + flags +
                       ["-U", os.path.join(d, "reads_1.fa"), "-S", os.path.join(d, "err.sam")], stderr=subprocess.PIPE)
    return r.stderr.decode().splitlines()[0], r.returncode


def load_expected():
    return json.load(open(OUT))


def main():
    md5, summary, errors = {}, {}, {}
    with tempfile.TemporaryDirectory() as d:
        generate(d)
        for case in sorted(CASES):
            sam, err = reference_run(d, case)
            md5[case] = refsets.sam_md5(sam, flagged(case))
            summary[case] = refsets.summary_text(err.encode())
        for name, flags in sorted(ERRORS.items()):
            errors[name] = reference_error(d, flags)
    json.dump({"md5": md5, "summary": summary, "errors": errors}, open(OUT, "w"), indent=1, sort_keys=True)
    open(OUT, "a").write("\n")


if __name__ == "__main__":
    main()
