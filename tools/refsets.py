#!/usr/bin/env python3
"""Read sets of the reference-parity GPU tests, generated from the committed tiny fixtures (tests/golden/tiny.fa,
tiny.snp) by the seeded generators tools/simreads.py and tools/altreads.py, so that a checkout needs nothing else.

  python tools/refsets.py        # writes tests/golden/ref_sets.json: md5 of the unmodified reference's SAM per case

The expected values come from oracle/_ref/hisat2-align-s (oracle/Makefile).  Cases whose reads can hit a fixed device
capacity list the flagged reads (`flagged`, from a GPU run of the library); their md5 excludes those reads' records."""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
TOOLS = os.path.join(ROOT, "tools")
REFBIN = os.path.join(ROOT, "oracle", "_ref", "hisat2-align-s")
OUT = os.path.join(GOLDEN, "ref_sets.json")

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


def reference(d, index, name, paired, flags=(), fa=False):
    out = os.path.join(d, "ref.sam")
    subprocess.run([REFBIN, "-f", "-x", os.path.join(GOLDEN, index)] + list(flags or ["--no-spliced-alignment"]) +
                   (fa if fa else files(d, name, paired)) + ["-S", out, "-p", str(min(16, os.cpu_count() or 1)), "--reorder"],
                   check=True, stderr=subprocess.DEVNULL)
    return open(out, "rb").read()


def main():
    old = json.load(open(OUT)) if os.path.exists(OUT) else {}
    flagged = old.get("flagged", {})
    md5 = {}
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
    json.dump({"md5": md5, "flagged": flagged}, open(OUT, "w"), indent=1, sort_keys=True)
    open(OUT, "a").write("\n")


if __name__ == "__main__":
    main()
