#!/usr/bin/env python3
"""Read sets of the reference-parity GPU tests, generated from the committed tiny fixtures (tests/golden/tiny.fa,
tiny.snp) by the seeded generators tools/simreads.py and tools/altreads.py, so that a checkout needs nothing else.

  python tools/refsets.py        # writes tests/golden/ref_sets.json: md5 of the unmodified reference's SAM per case
  python tools/refsets.py --edge # only the edge/* cases (tools/edgereads.py); also writes tests/golden/edge_se.sam
  python tools/refsets.py --spliced  # only the spliced/* and spliced_novel/* cases (tools/splicereads.py); also
                                     # writes tests/golden/edge_spliced_se.sam (SPLICED_GOLDEN)
  python tools/refsets.py --output   # only tests/golden/output_sets.json: the output/* cases (SAM output options) and
                                     # the alignment summaries summary/* and summary_new/* (verbatim, under "summary")

The expected values come from oracle/_ref/hisat2-align-s (oracle/Makefile).  Cases whose reads can hit a fixed device
capacity list the flagged reads (`flagged`, from a GPU run of the library); their md5 excludes those reads' records."""
import hashlib
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
TOOLS = os.path.join(ROOT, "tools")
REFBIN = os.path.join(ROOT, "oracle", "_ref", "hisat2-align-s")
OUT = os.path.join(GOLDEN, "ref_sets.json")
OUTPUT_OUT = os.path.join(GOLDEN, "output_sets.json")   # --output: SAM output options and alignment summaries

# name -> generator arguments (every set is written as <name>_1.fa / <name>_2.fa)
SETS = {
    "reads": ["simreads", "1000", "--seed", "2", "--paired"],
    "sim10k": ["simreads", "10000", "--seed", "1", "--paired"],
    "hard20k": ["simreads", "20000", "--seed", "3", "--paired", "--indel", "0.004", "--nrate", "0.003", "--sub", "0.02", "--ragged"],
    "len36": ["simreads", "20000", "--seed", "106", "--paired", "--indel", "0.004", "--nrate", "0.002", "--sub", "0.01", "--ragged", "--rdlen", "36"],
    "len150": ["simreads", "20000", "--seed", "220", "--paired", "--indel", "0.004", "--nrate", "0.002", "--sub", "0.01", "--ragged", "--rdlen", "150"],
    "len250": ["simreads", "20000", "--seed", "320", "--paired", "--indel", "0.004", "--nrate", "0.002", "--sub", "0.01", "--ragged", "--rdlen", "250"],
    "len500": ["simreads", "3000", "--seed", "570", "--paired", "--indel", "0.003", "--nrate", "0.002", "--sub", "0.01", "--ragged", "--rdlen", "500"],
    "len1000": ["simreads", "3000", "--seed", "1070", "--paired", "--indel", "0.003", "--nrate", "0.002", "--sub", "0.01", "--ragged", "--rdlen", "1000"],
    "alt20k": ["altreads", "20000", "--seed", "9", "--paired"],
    "sim200k": ["simreads", "200000", "--seed", "5", "--paired"],
}

# --bowtie2-dp / preset cases: (index, set, paired, reference flags, library options)
DP_CASES = [
    ("tiny", "hard20k", False, ["--bowtie2-dp", "2"], dict(bowtie2_dp=2)),
    ("tiny", "hard20k", True, ["--sensitive"], dict(bowtie2_dp=1, score_min_type=ord("L"), score_min_const=0.0, score_min_coeff=-0.5)),
    ("tiny_snp", "alt20k", True, ["--very-sensitive"], dict(bowtie2_dp=2, khits=30, score_min_type=ord("L"), score_min_const=0.0, score_min_coeff=-1.0)),
    ("tiny", "len150", False, ["--bowtie2-dp", "1", "--score-min", "L,0,-0.4", "--gbar", "2"],
     dict(bowtie2_dp=1, gbar=2, score_min_type=ord("L"), score_min_const=0.0, score_min_coeff=-0.4)),
]


def _edge_cases():
    """edge/<case>: the tools/edgereads.py corpus.  case -> (index, files, format flag, reference flags, library options,
    front-end options of ht2gpu_reads_input_t).  Every case but `near` also runs as <case>_dp with --bowtie2-dp 2: on
    near_A0_624 (a 250-base read with an insertion, overhanging the start of chrA) the reference under --bowtie2-dp 2
    asks for a 32 GiB DP matrix and aborts."""
    sys.path.insert(0, TOOLS)
    import edgereads
    cases = {
        "se": ("tiny", ["se.fa"], "-f", [], {}, {}),
        "near": ("tiny", ["near.fa"], "-f", [], {}, {}),
        "pe": ("tiny", ["pe_1.fa", "pe_2.fa"], "-f", [], {}, {}),
        "graph_se": ("tiny_snp", ["se.fa"], "-f", [], {}, {}),
        "fq": ("tiny", ["q.fq"], "-q", [], {}, {}),
        # --mp 42,2 makes a Q41+ mismatch cost more than a Q40 one unless the quality is clamped at 40
        "fq_mp42": ("tiny", ["q.fq"], "-q", ["--mp", "42,2", "--score-min", "L,0,-1.5"],
                    dict(mp_max=42, mp_min=2, score_min_type=ord("L"), score_min_const=0.0, score_min_coeff=-1.5), {}),
        "fq64": ("tiny", ["q64.fq"], "-q", ["--phred64"], {}, dict(phred64=1)),
        "fq_trim": ("tiny", ["q.fq"], "-q", ["-5", "3", "-3", "5"], {}, dict(trim5=3, trim3=5)),
    }
    for i, sm in enumerate(edgereads.SCORE_MIN):
        flag = edgereads.score_min_flag(sm)
        opts = {} if flag is None else dict(score_min_type=ord(sm[0]), score_min_const=sm[1], score_min_coeff=sm[2])
        cases["sc%d" % i] = ("tiny", ["sc%d.fa" % i], "-f", [] if flag is None else ["--score-min", flag], opts, {})
    for k in [k for k in cases if k != "near"]:
        index, fs, fmt, flags, opts, front = cases[k]
        cases[k + "_dp"] = (index, fs, fmt, flags + ["--bowtie2-dp", "2"], dict(opts, bowtie2_dp=2), front)
    return cases


EDGE_CASES = _edge_cases()
EDGE_SEED = 11

# spliced/<case>: the tools/splicereads.py corpus (splice_*) and its tools/sim_rna.py bulk (splice_sim*), aligned in
# spliced mode as the reference's --no-temp-splicesite (splice sites are not carried from read to read, so every read
# aligns on its own, as the library does).  case -> (index, files, format flag, reference flags, library options,
# known-splice-site file or None).
SPLICED_CASES = {
    "edge_se": ("tiny", ["se.fa"], "-f", [], {}, None),
    "edge_pe": ("tiny", ["pe_1.fa", "pe_2.fa"], "-f", [], {}, None),
    "edge_fq": ("tiny", ["q.fq"], "-q", [], {}, None),
    "sim_se": ("tiny", ["sim.fa"], "-f", [], {}, None),
    "sim_pe": ("tiny", ["sim_1.fa", "sim_2.fa"], "-f", [], {}, None),
    "ss_edge_se": ("tiny", ["se.fa"], "-f", [], {}, "ss.txt"),
    "ss_sim_pe": ("tiny", ["sim_1.fa", "sim_2.fa"], "-f", [], {}, "sim_ss.txt"),
    "edge_se_dp": ("tiny", ["se.fa"], "-f", ["--bowtie2-dp", "2"], dict(bowtie2_dp=2), None),
    "graph_edge_se": ("tiny_snp", ["se.fa"], "-f", [], {}, None),
    "graph_ss_sim_pe": ("tiny_snp", ["sim_1.fa", "sim_2.fa"], "-f", [], {}, "sim_ss.txt"),
}
# cases whose --novel-splicesite-outfile is recorded too, as spliced_novel/<case>
SPLICED_NOVEL = ("sim_pe", "edge_se")
SPLICE_SEED = 17
# the reads of spliced/edge_se whose reference records are committed as tests/golden/edge_spliced_se.sam: the intron
# lengths at the rule boundaries and the junctions of opposite sense (the md5 covers the rest of the corpus)
SPLICED_GOLDEN = (b"len_", b"sense_")


# output/<case>: SAM output options (--no-unal, --rg-id / --rg, --omit-sec-seq, --no-sq) on the sets above.
# case -> (input, reference flags, library options, SAM output settings of Index.set_sam_output).  An input is
# ("se" | "paired" | "graph_se" | "graph_pe", <set>), ("edge", <EDGE_CASES key>), ("spliced", <SPLICED_CASES key>) or
# ("dp", <DP_CASES index>).  Only inputs without flagged reads.
RG = ["--rg-id", "g1", "--rg", "SM:s1", "--rg", "PL:ILLUMINA"]
RG_OUT = dict(rg_id="g1", rg=("SM:s1", "PL:ILLUMINA"))
OUTPUT_CASES = {
    "no_unal_se_hard20k": (("se", "hard20k"), ["--no-unal"], {}, dict(no_unal=1)),
    "no_unal_pe_hard20k": (("paired", "hard20k"), ["--no-unal"], {}, dict(no_unal=1)),
    "no_unal_pe_hard20k_no_mixed": (("paired", "hard20k"), ["--no-unal", "--no-mixed"], dict(no_mixed=1), dict(no_unal=1)),
    "no_unal_edge_se": (("edge", "se"), ["--no-unal"], {}, dict(no_unal=1)),
    "no_unal_spliced_edge_pe": (("spliced", "edge_pe"), ["--no-unal"], {}, dict(no_unal=1)),
    "rg_graph_pe_alt20k": (("graph_pe", "alt20k"), RG, {}, RG_OUT),
    "rg_spliced_ss_edge_se": (("spliced", "ss_edge_se"), RG, {}, RG_OUT),
    "rg_id_from_rg_se_reads": (("se", "reads"), ["--rg", "ID:g2", "--rg", "LB:x"], {}, dict(rg_id="g2", rg=("LB:x",))),
    "rg_without_id_se_reads": (("se", "reads"), ["--rg", "SM:only"], {}, dict(rg=("SM:only",))),
    "omit_sec_seq_k30_se_reads": (("se", "reads"), ["--omit-sec-seq", "-k", "30", "--secondary"], dict(khits=30, secondary=1), dict(omit_sec_seq=1)),
    "omit_sec_seq_k5_se_reads": (("se", "reads"), ["--omit-sec-seq", "-k", "5"], dict(khits=5), dict(omit_sec_seq=1)),
    "omit_sec_seq_k30_pe_sim10k": (("paired", "sim10k"), ["--omit-sec-seq", "-k", "30", "--secondary"], dict(khits=30, secondary=1), dict(omit_sec_seq=1)),
    "omit_sec_seq_k5_pe_sim10k": (("paired", "sim10k"), ["--omit-sec-seq", "-k", "5"], dict(khits=5), dict(omit_sec_seq=1)),
    "no_sq_se_reads": (("se", "reads"), ["--no-sq"], {}, dict(no_sq=1)),
}
# summary/<case> and summary_new/<case>: the reference's alignment summary (stderr), classic and --new-summary.
# case -> (input, reference flags, library options, read front-end options of ht2gpu_reads_input_t)
SUMMARY_CASES = {
    "se_reads": (("se", "reads"), [], {}, {}),
    "se_hard20k": (("se", "hard20k"), [], {}, {}),
    "pe_sim10k": (("paired", "sim10k"), [], {}, {}),
    "pe_hard20k": (("paired", "hard20k"), [], {}, {}),
    "graph_se_alt20k": (("graph_se", "alt20k"), [], {}, {}),
    "graph_pe_alt20k": (("graph_pe", "alt20k"), [], {}, {}),
    "edge_se": (("edge", "se"), [], {}, {}),
    "edge_pe": (("edge", "pe"), [], {}, {}),
    "spliced_sim_pe": (("spliced", "sim_pe"), [], {}, {}),
    "spliced_edge_se": (("spliced", "edge_se"), [], {}, {}),
    "pe_hard20k_no_mixed": (("paired", "hard20k"), ["--no-mixed"], dict(no_mixed=1), {}),
    "pe_hard20k_no_discordant": (("paired", "hard20k"), ["--no-discordant"], dict(no_discordant=1), {}),
    "pe_hard20k_no_mixed_no_discordant": (("paired", "hard20k"), ["--no-mixed", "--no-discordant"], dict(no_mixed=1, no_discordant=1), {}),
    "pe_hard20k_k1": (("paired", "hard20k"), ["-k", "1"], dict(khits=1), {}),
    "se_reads_skip100_upto300": (("se", "reads"), ["-s", "100", "-u", "300"], {}, dict(skip=100, upto=300)),
    "dp1_sensitive": (("dp", 1), [], {}, {}),
}
SUMMARY_SETS = ("reads", "sim10k", "hard20k", "alt20k")
# rep_1.fa (generate_repeats): 100-base reads of the segments tiny.fa holds twice.  Under -k 30 --secondary every read
# prints two records, more SAM text than the device's first estimate per read, so the SAM kernels run again
SUMMARY_CASES["rep_k30_secondary"] = (("se", "rep"), ["-k", "30", "--secondary"], dict(khits=30, secondary=1), {})


def generate_repeats(outdir, rdlen=100, n=1000):
    """rep_1.fa under outdir: every fifth of the rdlen-base windows of tiny.fa whose sequence (or reverse complement)
    occurs exactly twice, at most n reads, in reference order.  Deterministic; returns outdir."""
    path = os.path.join(outdir, "rep_1.fa")
    if os.path.exists(path):
        return outdir
    seqs, cur = {}, None
    for l in open(os.path.join(GOLDEN, "tiny.fa")):
        l = l.strip()
        if l.startswith(">"):
            cur = l[1:].split()[0]
            seqs[cur] = []
        elif cur is not None:
            seqs[cur].append(l.upper())
    comp = str.maketrans("ACGT", "TGCA")
    count, order = {}, []
    for name, parts in seqs.items():
        s = "".join(parts)
        for i in range(len(s) - rdlen + 1):
            w = s[i:i + rdlen]
            if "N" in w:
                continue
            key = min(w, w.translate(comp)[::-1])
            count[key] = count.get(key, 0) + 1
            order.append((name, i, w, key))
    reads = [(name, i, w) for name, i, w, key in order if count[key] == 2][::5][:n]
    with open(path, "w") as f:
        for name, i, w in reads:
            f.write(">rep_%s_%d\n%s\n" % (name, i, w))
    return outdir


def generate_output_sets(d):
    """Every read set the OUTPUT_CASES and SUMMARY_CASES use, under d; returns d."""
    generate(d, SUMMARY_SETS)
    generate_repeats(d)
    generate_edge(d)
    generate_spliced(d)
    return d


def output_input(d, src):
    """(index, read files, format flag, reference flags, library options, known-splice-site file or None) of an
    OUTPUT_CASES / SUMMARY_CASES input under d (generate(d, SUMMARY_SETS), generate_edge(d) and generate_spliced(d))."""
    kind, name = src
    if kind in ("se", "paired", "graph_se", "graph_pe"):
        paired = kind in ("paired", "graph_pe")
        fs = [os.path.join(d, name + "_1.fa")] + ([os.path.join(d, name + "_2.fa")] if paired else [])
        return ("tiny_snp" if kind.startswith("graph") else "tiny"), fs, "-f", ["--no-spliced-alignment"], {}, None
    if kind == "edge":
        index, _, fmt, flags, opts, _ = EDGE_CASES[name]
        return index, edge_files(d, name), fmt, ["--no-spliced-alignment"] + flags, dict(opts), None
    if kind == "spliced":
        index, _, fmt, flags, opts, _ = SPLICED_CASES[name]
        fs, ss = spliced_files(d, name)
        return index, fs, fmt, ["--no-temp-splicesite"] + flags + (["--known-splicesite-infile", ss] if ss else []), \
            dict(opts, no_spliced_alignment=0), ss
    index, setname, paired, flags, opts = DP_CASES[name]
    fs = [os.path.join(d, setname + "_1.fa")] + ([os.path.join(d, setname + "_2.fa")] if paired else [])
    return index, fs, "-f", ["--no-spliced-alignment"] + flags, dict(opts), None


def summary_text(stderr):
    """The alignment summary at the end of the reference's stderr (warnings come earlier)."""
    lines = stderr.decode().splitlines(True)
    for i, l in enumerate(lines):
        if re.match(r"^\d+ reads", l) or l.startswith("HISAT2 summary stats:"):
            return "".join(lines[i:])
    raise ValueError("no alignment summary in the reference's stderr")


def reference_run(d, src, flags):
    """(SAM, stderr) of the unmodified reference on an OUTPUT_CASES / SUMMARY_CASES input (--reorder)."""
    index, fs, fmt, base, _, _ = output_input(d, src)
    out = os.path.join(d, "ref.sam")
    reads = ["-1", fs[0], "-2", fs[1]] if len(fs) == 2 else ["-U", fs[0]]
    r = subprocess.run([REFBIN, fmt, "-x", os.path.join(GOLDEN, index)] + base + list(flags) + reads +
                       ["-S", out, "-p", str(min(16, os.cpu_count() or 1)), "--reorder"], check=True, stderr=subprocess.PIPE)
    return open(out, "rb").read(), r.stderr


def load_output_expected():
    return json.load(open(OUTPUT_OUT))


def output_main():
    """Writes OUTPUT_OUT: {"md5": output/<case> md5s, "summary": summary/<case>, summary_new/<case> texts}."""
    md5, summary = {}, {}
    with tempfile.TemporaryDirectory() as d:
        output_reference(d, md5, summary)
    json.dump({"md5": md5, "summary": summary}, open(OUTPUT_OUT, "w"), indent=1, sort_keys=True)
    open(OUTPUT_OUT, "a").write("\n")


def output_reference(d, md5, summary):
    """output/<case> md5s and summary/<case>, summary_new/<case> texts."""
    generate_output_sets(d)
    for case, (src, flags, _, _) in sorted(OUTPUT_CASES.items()):
        sam, _ = reference_run(d, src, flags)
        md5["output/" + case] = sam_md5(sam)
    for case, (src, flags, _, _) in sorted(SUMMARY_CASES.items()):
        summary["summary/" + case] = summary_text(reference_run(d, src, flags)[1])
        summary["summary_new/" + case] = summary_text(reference_run(d, src, flags + ["--new-summary"])[1])


def spliced_golden_lines(sam):
    """The SAM lines (headers without @PG, records of the SPLICED_GOLDEN reads) kept as edge_spliced_se.sam."""
    return [l for l in sam.splitlines(True) if (l.startswith(b"@") and not l.startswith(b"@PG")) or l.startswith(SPLICED_GOLDEN)]


def load_expected():
    return json.load(open(OUT))


def generate(outdir, names=None):
    """Write the read sets (all, or `names`) under outdir; returns outdir."""
    for name in (names or SETS):
        if os.path.exists(os.path.join(outdir, name + "_1.fa")):
            continue
        tool, args = SETS[name][0], SETS[name][1:]
        inputs = [os.path.join(GOLDEN, "tiny.fa")] + ([os.path.join(GOLDEN, "tiny.snp")] if tool == "altreads" else [])
        subprocess.run([sys.executable, os.path.join(TOOLS, tool + ".py")] + inputs + [args[0], os.path.join(outdir, name)] + args[1:],
                       check=True, stdout=subprocess.DEVNULL)
    return outdir


def generate_edge(outdir):
    """The tools/edgereads.py corpus under outdir (edge_*); returns outdir."""
    sys.path.insert(0, TOOLS)
    import edgereads
    if not os.path.exists(os.path.join(outdir, "edge_se.fa")):
        edgereads.generate(os.path.join(GOLDEN, "tiny.fa"), os.path.join(outdir, "edge"), EDGE_SEED)
    return outdir


def edge_files(d, case):
    return [os.path.join(d, "edge_" + f) for f in EDGE_CASES[case][1]]


def generate_spliced(outdir):
    """The tools/splicereads.py corpus under outdir (splice_*); returns outdir."""
    sys.path.insert(0, TOOLS)
    import splicereads
    if not os.path.exists(os.path.join(outdir, "splice_se.fa")):
        splicereads.generate(os.path.join(GOLDEN, "tiny.fa"), os.path.join(outdir, "splice"), SPLICE_SEED)
    return outdir


def spliced_files(d, case):
    """(read files, known-splice-site file or None) of spliced/<case> under d."""
    c = SPLICED_CASES[case]
    return [os.path.join(d, "splice_" + f) for f in c[1]], (os.path.join(d, "splice_" + c[5]) if c[5] else None)


def sam_md5(sam, exclude=()):
    """md5 of the SAM lines without @PG (and without the records of the read names in `exclude`)."""
    if isinstance(sam, str):
        sam = sam.encode()
    ex = set(n.encode() if isinstance(n, str) else n for n in exclude)
    lines = [l for l in sam.splitlines() if not l.startswith(b"@PG") and (l.startswith(b"@") or l.split(b"\t")[0] not in ex)]
    return hashlib.md5(b"\n".join(lines) + b"\n").hexdigest()


def files(d, name, paired):
    f1, f2 = os.path.join(d, name + "_1.fa"), os.path.join(d, name + "_2.fa")
    return ["-1", f1, "-2", f2] if paired else ["-U", f1]


def reference(d, index, name, paired, flags=(), fa=False, fmt="-f"):
    """SAM of the unmodified reference (--reorder).  fmt is -f or -q; flags may hold any of its alignment and input
    options (--score-min, --phred64, -5 / -3, ...)."""
    out = os.path.join(d, "ref.sam")
    subprocess.run([REFBIN, fmt, "-x", os.path.join(GOLDEN, index)] + list(flags or ["--no-spliced-alignment"]) +
                   (fa if fa else files(d, name, paired)) + ["-S", out, "-p", str(min(16, os.cpu_count() or 1)), "--reorder"],
                   check=True, stderr=subprocess.DEVNULL)
    return open(out, "rb").read()


def main(edge_only=False, spliced_only=False, output_only=False):
    if output_only:
        output_main()
        return
    old = json.load(open(OUT)) if os.path.exists(OUT) else {}
    flagged = old.get("flagged", {})
    md5 = {}
    if spliced_only:
        md5 = {k: v for k, v in old.get("md5", {}).items() if not k.startswith(("spliced/", "spliced_novel/"))}
        with tempfile.TemporaryDirectory() as d:
            spliced_reference(d, md5, flagged)
        json.dump({"md5": md5, "flagged": flagged}, open(OUT, "w"), indent=1, sort_keys=True)
        open(OUT, "a").write("\n")
        return
    if edge_only:
        md5 = {k: v for k, v in old.get("md5", {}).items() if not k.startswith("edge/")}
        with tempfile.TemporaryDirectory() as d:
            edge_reference(d, md5, flagged)
        json.dump({"md5": md5, "flagged": flagged}, open(OUT, "w"), indent=1, sort_keys=True)
        open(OUT, "a").write("\n")
        return
    with tempfile.TemporaryDirectory() as d:
        generate(d)
        for name in ("sim10k", "hard20k", "len36", "len150", "len500", "sim200k"):
            md5["paired/" + name] = sam_md5(reference(d, "tiny", name, True))
        for name in ("reads", "hard20k", "sim200k", "len36", "len150", "len250", "len500", "len1000"):
            md5["se/" + name] = sam_md5(reference(d, "tiny", name, False))
        for name, paired in (("reads", False), ("hard20k", False), ("alt20k", False), ("sim200k", False), ("sim10k", True),
                             ("alt20k", True), ("hard20k", True)):
            md5["graph_%s/%s" % ("pe" if paired else "se", name)] = sam_md5(reference(d, "tiny_snp", name, paired))
        for i, (index, name, paired, flags, _) in enumerate(DP_CASES):
            key = "dp/%d" % i
            md5[key] = sam_md5(reference(d, index, name, paired, ["--no-spliced-alignment"] + flags), flagged.get(key, ()))
        for name in ("len250", "len1000"):
            key = "long/" + name
            md5[key] = sam_md5(reference(d, "tiny", name, True), flagged.get(key, ()))
        # the bench workload's own generator (bench.sim_fasta) at full size: 1 M single-end reads, 500 k pairs
        sys.path.insert(0, ROOT)
        import bench
        d1, d2 = bench.sim_fasta(0, 1000000)
        f1, f2 = os.path.join(d, "m1.fa"), os.path.join(d, "m2.fa")
        d1.tofile(f1)
        md5["full/se1M"] = sam_md5(reference(d, "tiny", None, False, fa=["-U", f1]))
        k = 500000
        d1[:k * bench.RECSZ].tofile(f1); d2[:k * bench.RECSZ].tofile(f2)
        md5["full/pe500k"] = sam_md5(reference(d, "tiny", None, True, fa=["-1", f1, "-2", f2]))
        edge_reference(d, md5, flagged)
        spliced_reference(d, md5, flagged)
    json.dump({"md5": md5, "flagged": flagged}, open(OUT, "w"), indent=1, sort_keys=True)
    open(OUT, "a").write("\n")
    output_main()


def spliced_reference(d, md5, flagged):
    """spliced/<case> md5s (reference run with --no-temp-splicesite) and spliced_novel/<case>, the md5 of its
    --novel-splicesite-outfile; the reference records of the SPLICED_GOLDEN reads of spliced/edge_se are also kept as
    tests/golden/edge_spliced_se.sam."""
    generate_spliced(d)
    for case, (index, _, fmt, flags, _, _) in sorted(SPLICED_CASES.items()):
        fs, ss = spliced_files(d, case)
        key = "spliced/" + case
        novel = os.path.join(d, "novel.txt")
        extra = (["--known-splicesite-infile", ss] if ss else []) + (["--novel-splicesite-outfile", novel] if case in SPLICED_NOVEL else [])
        sam = reference(d, index, None, len(fs) == 2, ["--no-temp-splicesite"] + flags + extra, fmt=fmt,
                        fa=["-1", fs[0], "-2", fs[1]] if len(fs) == 2 else ["-U", fs[0]])
        md5[key] = sam_md5(sam, flagged.get(key, ()))
        if case in SPLICED_NOVEL:
            md5["spliced_novel/" + case] = hashlib.md5(open(novel, "rb").read()).hexdigest()
        if case == "edge_se":
            open(os.path.join(GOLDEN, "edge_spliced_se.sam"), "wb").write(b"".join(spliced_golden_lines(sam)))


def edge_reference(d, md5, flagged):
    """edge/<case> md5s; the reference SAM of edge/se is also kept as tests/golden/edge_se.sam."""
    generate_edge(d)
    for case, (index, _, fmt, flags, _, _) in sorted(EDGE_CASES.items()):
        fs = edge_files(d, case)
        key = "edge/" + case
        sam = reference(d, index, None, len(fs) == 2, ["--no-spliced-alignment"] + flags, fmt=fmt,
                        fa=["-1", fs[0], "-2", fs[1]] if len(fs) == 2 else ["-U", fs[0]])
        md5[key] = sam_md5(sam, flagged.get(key, ()))
        if case == "se":
            open(os.path.join(GOLDEN, "edge_se.sam"), "wb").write(b"".join(l for l in sam.splitlines(True) if not l.startswith(b"@PG")))


if __name__ == "__main__":
    main(edge_only="--edge" in sys.argv[1:], spliced_only="--spliced" in sys.argv[1:], output_only="--output" in sys.argv[1:])
