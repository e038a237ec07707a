#!/usr/bin/env python3
"""Alignment against splice-site / exon graph indexes (hisat2-build --ss / --exon) against the unmodified reference.

  python tools/tran_index_ref.py fixtures   # writes tests/golden/tiny_tran_exons.txt and the two indexes
  python tools/tran_index_ref.py            # writes tests/golden/tran_index_sets.json

The indexes are tests/golden/tiny_tran and tiny_snp_tran (fixtures(), with oracle/_ref/hisat2-build-s).  The expected values come
from oracle/_ref/hisat2-align-s (oracle/Makefile), run with --reorder on the RNA corpus of make_golden.py known_splice
(tiny_ss_rna.fa, tiny_ss_rna_{1,2}.fa) under each mode of MODES, and on the DNA pairs used with tiny_snp
(tiny_alt_{1,2}.fa) with --no-spliced-alignment.  The JSON keeps, per case, the md5 of the SAM without @PG and the
alignment summary the reference prints."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import refsets  # noqa: E402

GOLDEN = refsets.GOLDEN
OUT = os.path.join(GOLDEN, "tran_index_sets.json")
INDEXES = ("tiny_tran", "tiny_snp_tran")
# mode -> (reference flags after --no-temp-splicesite, Index options, known-splice-site file or None)
MODES = {
    "default": ([], {}, None),
    "nospl": (["--no-spliced-alignment"], dict(no_spliced_alignment=1), None),
    "tmo": (["--tmo"], dict(tmo=1), None),
    "avoid": (["--avoid-pseudogene"], dict(avoid_pseudogene=1), None),
    "dta": (["--dta"], dict(dta=1), None),
    "k20sec": (["-k", "20", "--secondary"], dict(khits=20, secondary=1), None),
    "known": (["--known-splicesite-infile", "tiny_ss_novel.txt"], {}, "tiny_ss_novel.txt"),
}
READS = {"se": ["tiny_ss_rna.fa"], "pe": ["tiny_ss_rna_1.fa", "tiny_ss_rna_2.fa"], "dna_pe": ["tiny_alt_1.fa", "tiny_alt_2.fa"]}


def fixtures():
    """Splice-site / exon graph indexes (hisat2-build --ss / --exon): tiny_tran_exons.txt holds the 150-base flanks of
    every site of tiny_ss_known.txt plus a 400-base exon every 2500 bases of each sequence, so that unspliced hits fall
    both inside and outside exons.  tiny_tran = --ftabchars 7 --ss tiny_ss_known.txt --exon tiny_tran_exons.txt over
    tiny.fa, tiny_snp_tran the same with --snp tiny.snp.  Every other fixture is left as it is."""
    import sim_rna
    lens = {name: len(s) for name, s in sim_rna.load_fasta(os.path.join(GOLDEN, "tiny.fa")).items()}
    ex = set()
    for l in open(os.path.join(GOLDEN, "tiny_ss_known.txt")):
        f = l.split()
        if f[0] not in lens:
            continue
        left, right = int(f[1]), int(f[2])
        ex.add((f[0], max(0, left - 149), left, f[3]))
        ex.add((f[0], right, min(lens[f[0]] - 1, right + 149), f[3]))
    for name, n in sorted(lens.items()):
        for st in range(0, n - 400, 2500):
            ex.add((name, st, st + 399, "+"))
    with open(os.path.join(GOLDEN, "tiny_tran_exons.txt"), "w") as f:
        for e in sorted(ex):
            f.write("%s\t%d\t%d\t%s\n" % e)
    build = os.path.join(os.path.dirname(refsets.REFBIN), "hisat2-build-s")
    for extra, out in (([], "tiny_tran"), (["--snp", "tiny.snp"], "tiny_snp_tran")):
        subprocess.run([build, "-q", "--ftabchars", "7", "--ss", "tiny_ss_known.txt", "--exon", "tiny_tran_exons.txt"] +
                       extra + ["tiny.fa", out], check=True, cwd=GOLDEN, stdout=subprocess.DEVNULL)


def _cases():
    c = {}
    for index in INDEXES:
        for src in ("se", "pe"):
            for mode in MODES:
                c["%s_%s_%s" % (index, src, mode)] = (index, src, mode)
    c["tiny_snp_tran_dna_pe_nospl"] = ("tiny_snp_tran", "dna_pe", "nospl")
    return c


CASES = _cases()


def case_input(case):
    """(index, read files, reference flags, Index options, known-splice-site file or None) of a case; the file paths
    are absolute."""
    index, src, mode = CASES[case]
    flags, opts, ss = MODES[mode]
    flags = ["--no-temp-splicesite"] + [os.path.join(GOLDEN, f) if f == ss else f for f in flags]
    opts = dict(dict(no_spliced_alignment=0), **opts)
    return index, [os.path.join(GOLDEN, f) for f in READS[src]], flags, opts, os.path.join(GOLDEN, ss) if ss else None


def reference_run(case, out):
    """(SAM, stderr) of the reference on a case (--reorder)."""
    index, fs, flags, _, _ = case_input(case)
    reads = ["-1", fs[0], "-2", fs[1]] if len(fs) == 2 else ["-U", fs[0]]
    r = subprocess.run([refsets.REFBIN, "-f", "-x", os.path.join(GOLDEN, index)] + flags + reads +
                       ["-S", out, "-p", str(min(16, os.cpu_count() or 1)), "--reorder"], check=True, stderr=subprocess.PIPE)
    return open(out, "rb").read(), r.stderr.decode()


def load_expected():
    return json.load(open(OUT))


def main():
    import tempfile
    md5, summary = {}, {}
    with tempfile.TemporaryDirectory() as d:
        for case in sorted(CASES):
            sam, err = reference_run(case, os.path.join(d, "ref.sam"))
            md5[case] = refsets.sam_md5(sam)
            summary[case] = refsets.summary_text(err.encode())
    json.dump({"md5": md5, "summary": summary}, open(OUT, "w"), indent=1, sort_keys=True)
    open(OUT, "a").write("\n")


if __name__ == "__main__":
    if sys.argv[1:] == ["fixtures"]:
        fixtures()
    else:
        main()
