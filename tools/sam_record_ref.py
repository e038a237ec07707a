#!/usr/bin/env python3
"""SAM record options against the unmodified reference: --rna-strandness, --remove-chrname / --add-chrname,
--no-templatelen-adjustment and --sam-no-qname-trunc.

  python tools/sam_record_ref.py           # writes tests/golden/sam_record_sets.json
  python tools/sam_record_ref.py --index   # first rebuilds tests/golden/tiny_nochr.*.ht2 (NOCHR_RECIPE)

The expected values come from oracle/_ref/hisat2-align-s (oracle/Makefile), run with --reorder on tools/refsets.py's
read sets (refsets.output_input) and on a seeded read set with hard names (generate_qnames).  The JSON keeps, per
case, the md5 of the SAM without @PG (and without the records of refsets' flagged reads, see flagged); for
--novel-splicesite-outfile cases the file's text; and the first line the reference prints to stderr for the argument
errors, with its exit status."""
import json
import os
import random
import shutil
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import refsets  # noqa: E402

GOLDEN = refsets.GOLDEN
OUT = os.path.join(GOLDEN, "sam_record_sets.json")
REFDIR = os.path.dirname(refsets.REFBIN)

# tests/golden/tiny_nochr.*.ht2: tiny.fa with chrB renamed to B, built like tiny (tests/golden/make_golden.py).  Its
# names are "chrA test contig" and "B", so --add-chrname and --remove-chrname each rename one of them.
NOCHR_RECIPE = ["hisat2-build-s", "-q", "--ftabchars", "7", "tiny_nochr.fa", "tiny_nochr"]

# case -> dict(src: a refsets.output_input source or ("qname", "se_fa" | "pe_fa" | "pe_fq"),
#              index: overrides the source's index, flags: reference flags, out: Index.set_sam_output settings,
#              chr_names: None | "remove" | "add", ss: "renamed" = the source's known-splice-site file with "chr" dropped
#              from its names, novel: also record --novel-splicesite-outfile)
def _strand(src, s):
    return dict(src=src, flags=["--rna-strandness", s], out=dict(rna_strandness=s))


def _qname(kind, whole):
    return dict(src=("qname", kind), flags=["--sam-no-qname-trunc"] if whole else [], out=dict(no_qname_trunc=True) if whole else {})


def _names(src, chr_names, **kw):
    return dict(src=src, flags=["--%s-chrname" % chr_names], chr_names=chr_names, **kw)


ALL_OPTIONS = ["--rna-strandness", "RF", "--remove-chrname", "--sam-no-qname-trunc", "--no-templatelen-adjustment",
               "--no-unal", "--rg-id", "g1"]
CASES = {
    "strand_F_se_reads": _strand(("se", "reads"), "F"),
    "strand_R_se_reads": _strand(("se", "reads"), "R"),
    "strand_F_se_hard20k": _strand(("se", "hard20k"), "F"),
    "strand_R_se_hard20k": _strand(("se", "hard20k"), "R"),
    "strand_FR_pe_hard20k": _strand(("paired", "hard20k"), "FR"),
    "strand_RF_pe_hard20k": _strand(("paired", "hard20k"), "RF"),
    "strand_RF_graph_pe_alt20k": _strand(("graph_pe", "alt20k"), "RF"),
    "strand_RF_spliced_ss_sim_pe": _strand(("spliced", "ss_sim_pe"), "RF"),
    "strand_RF_spliced_edge_se": _strand(("spliced", "edge_se"), "RF"),
    # the layouts the strandness does not describe: the reference prints what its branch gives
    "strand_F_pe_hard20k": _strand(("paired", "hard20k"), "F"),
    "strand_FR_se_hard20k": _strand(("se", "hard20k"), "FR"),
    "qname_se_fa": _qname("se_fa", False),
    "qname_se_fa_whole": _qname("se_fa", True),
    "qname_pe_fa": _qname("pe_fa", False),
    "qname_pe_fa_whole": _qname("pe_fa", True),
    "qname_pe_fq": _qname("pe_fq", False),
    "qname_pe_fq_whole": _qname("pe_fq", True),
    "tlen_spliced_ss_sim_pe": dict(src=("spliced", "ss_sim_pe"), flags=["--no-templatelen-adjustment"], out=dict(no_templatelen_adjustment=True)),
    "tlen_spliced_graph_ss_sim_pe": dict(src=("spliced", "graph_ss_sim_pe"), flags=["--no-templatelen-adjustment"],
                                         out=dict(no_templatelen_adjustment=True)),
    "names_remove_se_reads": _names(("se", "reads"), "remove"),
    "names_remove_pe_reads": _names(("paired", "reads"), "remove"),
    # the known sites in renamed names (TLEN adjusted), and in the index's names (no name matches: no sites)
    "names_remove_ss_renamed": _names(("spliced", "ss_sim_pe"), "remove", ss="renamed"),
    "names_remove_ss_chr": _names(("spliced", "ss_sim_pe"), "remove"),
    "names_remove_novel": _names(("spliced", "sim_pe"), "remove", novel=True),
    "names_add_nochr_se_reads": _names(("se", "reads"), "add", index="tiny_nochr"),
    "names_add_nochr_pe_reads": _names(("paired", "reads"), "add", index="tiny_nochr"),
    "names_remove_nochr_pe_reads": _names(("paired", "reads"), "remove", index="tiny_nochr"),
    "all_spliced_ss_sim_pe": dict(src=("spliced", "ss_sim_pe"), flags=ALL_OPTIONS, chr_names="remove", ss="renamed",
                                  out=dict(rna_strandness="RF", no_qname_trunc=True, no_templatelen_adjustment=True,
                                           no_unal=True, rg_id="g1")),
}
# argument errors: reference flags -> the first line of its stderr and its exit status (recorded under "errors")
ERRORS = {
    "both_chrname": ["--remove-chrname", "--add-chrname"],
    "bad_strandness": ["--rna-strandness", "FF"],
}
QNAME_SEED = 23


def generate_qnames(d):
    """qn_se.fa, qn_1.fa / qn_2.fa and qn_1.fq / qn_2.fq under d: the first 400 pairs of refsets' `reads` set with
    seeded names of 256 to 600 characters (and exactly 255, 256, 257), names with a space or tab comment, mate names
    with /1 /2 before or after a comment, and unnamed reads.  Returns d."""
    if os.path.exists(os.path.join(d, "qn_2.fq")):
        return d
    refsets.generate(d, ("reads",))
    rng = random.Random(QNAME_SEED)
    alpha = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789:_-.|"

    def word(n):
        return "".join(rng.choice(alpha) for _ in range(n))

    def seqs(path):
        return [r.split("\n", 1)[1].replace("\n", "") for r in open(path).read().split(">")[1:]][:400]

    s1, s2 = seqs(os.path.join(d, "reads_1.fa")), seqs(os.path.join(d, "reads_2.fa"))
    names = []   # (mate 1 name, mate 2 name); the single-end set uses the first
    for i in range(len(s1)):
        k = i % 8
        if k == 0:
            n = [255, 256, 257][i // 8 % 3] if i < 24 else rng.randint(256, 600)
            base = word(n)
            names.append((base, base))
        elif k == 1:
            base = "q%d_%s" % (i, word(rng.randint(2, 20)))
            c = rng.choice([" ", "\t"]) + word(rng.randint(1, 30)) + rng.choice(["", " x=1", "\tBC:Z:%s" % word(6)])
            names.append((base + c, base + c))
        elif k == 2:
            base, c = "q%d" % i, rng.choice([" ", "\t"]) + word(rng.randint(1, 12))
            names.append((base + "/1" + c, base + "/2" + c))
        elif k == 3:
            base, c = "q%d" % i, rng.choice([" ", "\t"]) + word(rng.randint(1, 12))
            names.append((base + c + "/1", base + c + "/2"))
        elif k == 4:
            names.append(("", ""))
        elif k == 5:   # long names with a comment and a mate suffix
            base = word(rng.randint(250, 400)) + " " + word(rng.randint(10, 200))
            names.append((base + "/1", base + "/2"))
        else:
            base = "q%d" % i
            names.append((base, base))

    def qual(n):
        return "".join(chr(33 + rng.randint(2, 40)) for _ in range(n))

    with open(os.path.join(d, "qn_se.fa"), "w") as f:
        for (n1, _), s in zip(names, s1):
            f.write(">%s\n%s\n" % (n1, s))
    for m, ss in ((0, s1), (1, s2)):
        with open(os.path.join(d, "qn_%d.fa" % (m + 1)), "w") as fa, open(os.path.join(d, "qn_%d.fq" % (m + 1)), "w") as fq:
            for nm, s in zip(names, ss):
                fa.write(">%s\n%s\n" % (nm[m], s))
                fq.write("@%s\n%s\n+\n%s\n" % (nm[m], s, qual(len(s))))
    return d


def generate(d):
    """Every read set and splice-site file the CASES use, under d; returns d."""
    refsets.generate(d, ("reads", "hard20k", "alt20k"))
    refsets.generate_spliced(d)
    generate_qnames(d)
    return d


def renamed_ss(src, dst):
    """A known-splice-site file with a leading "chr" dropped from every name (what --remove-chrname expects)."""
    with open(src) as f, open(dst, "w") as o:
        for l in f:
            o.write(l[3:] if l.startswith("chr") else l)
    return dst


def case_input(d, case):
    """(index, read files, format flag, reference flags, library options, known-splice-site file or None) of a case
    under generate(d).  The reference flags hold the case's own flags, not --novel-splicesite-outfile."""
    c = CASES[case]
    src = c["src"]
    if src[0] == "qname":
        kind = src[1]
        fs = [os.path.join(d, "qn_se.fa")] if kind == "se_fa" else [os.path.join(d, "qn_%d.%s" % (m, kind[3:])) for m in (1, 2)]
        index, fmt, base, opts, ss = "tiny", "-q" if kind.endswith("fq") else "-f", ["--no-spliced-alignment"], {}, None
    else:
        index, fs, fmt, base, opts, ss = refsets.output_input(d, src)
        if ss and c.get("ss") == "renamed":
            new = renamed_ss(ss, os.path.join(d, "renamed_" + os.path.basename(ss)))
            base = [new if a == ss else a for a in base]
            ss = new
    index = c.get("index", index)
    opts = dict(opts)
    if c.get("chr_names"):
        opts["chr_names"] = c["chr_names"]
    return index, fs, fmt, base + c["flags"], opts, ss


def flagged(case):
    """The reads of a case's source that hit a fixed device capacity (refsets' `flagged`): no md5 covers their records."""
    src = CASES[case]["src"]
    return refsets.load_expected()["flagged"].get("spliced/" + src[1], []) if src[0] == "spliced" else []


def reference_run(d, case):
    """(SAM, --novel-splicesite-outfile text or None) of the reference on a case (--reorder)."""
    index, fs, fmt, flags, _, _ = case_input(d, case)
    out, novel = os.path.join(d, "ref.sam"), os.path.join(d, "novel.txt")
    reads = ["-1", fs[0], "-2", fs[1]] if len(fs) == 2 else ["-U", fs[0]]
    extra = ["--novel-splicesite-outfile", novel] if CASES[case].get("novel") else []
    subprocess.run([refsets.REFBIN, fmt, "-x", os.path.join(GOLDEN, index)] + flags + extra + reads +
                   ["-S", out, "-p", str(min(16, os.cpu_count() or 1)), "--reorder"], check=True, stderr=subprocess.DEVNULL)
    return open(out, "rb").read(), (open(novel).read() if extra else None)


def reference_error(d, flags):
    """(first line of the reference's stderr, exit status) for argument errors on a small input."""
    refsets.generate(d, ("reads",))
    r = subprocess.run([refsets.REFBIN, "-f", "-x", os.path.join(GOLDEN, "tiny"), "--no-spliced-alignment"] + flags +
                       ["-U", os.path.join(d, "reads_1.fa"), "-S", os.path.join(d, "err.sam")], stderr=subprocess.PIPE)
    return r.stderr.decode().splitlines()[0], r.returncode


def build_nochr_index():
    """tests/golden/tiny_nochr.*.ht2 by NOCHR_RECIPE, from tiny.fa with the name line "chrB" made "B"."""
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(GOLDEN, "tiny.fa")) as f, open(os.path.join(d, "tiny_nochr.fa"), "w") as o:
            for l in f:
                o.write(">B\n" if l.rstrip("\n") == ">chrB" else l)
        subprocess.run([os.path.join(REFDIR, NOCHR_RECIPE[0])] + NOCHR_RECIPE[1:], check=True, cwd=d, stdout=subprocess.DEVNULL)
        for k in range(1, 9):
            shutil.copy(os.path.join(d, "tiny_nochr.%d.ht2" % k), GOLDEN)


def load_expected():
    return json.load(open(OUT))


def main(index=False):
    if index:
        build_nochr_index()
    md5, novel, errors = {}, {}, {}
    with tempfile.TemporaryDirectory() as d:
        generate(d)
        for case in sorted(CASES):
            sam, nv = reference_run(d, case)
            md5[case] = refsets.sam_md5(sam, flagged(case))
            if nv is not None:
                novel[case] = nv
        for name, flags in sorted(ERRORS.items()):
            errors[name] = reference_error(d, flags)
    json.dump({"md5": md5, "novel": novel, "errors": errors}, open(OUT, "w"), indent=1, sort_keys=True)
    open(OUT, "a").write("\n")


if __name__ == "__main__":
    main(index="--index" in sys.argv[1:])
