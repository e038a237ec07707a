#!/usr/bin/env python3
"""Expected read files of --un, --al, --un-conc, --al-conc and --al-conc-disc, from the unmodified reference.

  python tools/readfiles_ref.py            # writes tests/golden/read_files_sets.json

For every case the reference (oracle/_ref/hisat2-align-s, oracle/Makefile) runs with --passthrough --reorder, the way
the hisat2 wrapper runs it when a read file is asked for: after every SAM record it prints the record's original input
text (Read::readOrigBuf), percent-escaped, on a line of its own.  route() restates the wrapper's loop that sorts those
texts into the files (hisat2:595-650).  The JSON keeps md5, size and record count of every file, and the md5 of the
reference's SAM without @PG, so that a test can tell a routing difference from an alignment difference.

The inputs are the read sets of tools/refsets.py plus a small record-text corpus (corpus()) with the record shapes the
routing has to reproduce byte for byte."""
import hashlib
import json
import os
import random
import re
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import refsets  # noqa: E402

OUT = os.path.join(refsets.GOLDEN, "read_files_sets.json")
FILES = ("un", "al", "un_conc", "al_conc", "al_conc_disc")
CORPUS_SEED = 23

# case -> (input, reference flags, library options, read front-end options of ht2gpu_reads_input_t).  An input is one
# of tools/refsets.py's (see refsets.output_input) or ("corpus", <file name>) from corpus().
CASES = {
    "se_reads": (("se", "reads"), [], {}, {}),
    "edge_se": (("edge", "se"), [], {}, {}),
    "edge_fq": (("edge", "fq"), [], {}, {}),
    "edge_fq64": (("edge", "fq64"), [], {}, dict(phred64=1)),
    "edge_fq_trim": (("edge", "fq"), ["-5", "3", "-3", "2"], {}, dict(trim5=3, trim3=2)),
    "pe_hard20k": (("paired", "hard20k"), [], {}, {}),
    "pe_hard20k_no_mixed": (("paired", "hard20k"), ["--no-mixed"], dict(no_mixed=1), {}),
    "pe_hard20k_no_discordant": (("paired", "hard20k"), ["--no-discordant"], dict(no_discordant=1), {}),
    "pe_hard20k_k1": (("paired", "hard20k"), ["-k", "1"], dict(khits=1), {}),
    "pe_sim10k_k30_secondary": (("paired", "sim10k"), ["-k", "30", "--secondary"], dict(khits=30, secondary=1), {}),
    "graph_pe_alt20k": (("graph_pe", "alt20k"), [], {}, {}),
    "spliced_sim_pe": (("spliced", "sim_pe"), [], {}, {}),
    "se_reads_skip100_upto300": (("se", "reads"), ["-s", "100", "-u", "300"], {}, dict(skip=100, upto=300)),
    "corpus_fq": (("corpus", "corpus.fq"), [], {}, {}),
    "corpus_fa": (("corpus", "corpus.fa"), [], {}, {}),
}


def corpus(d, seed=CORPUS_SEED):
    """corpus.fq and corpus.fa under d: reads drawn from tests/golden/tiny.fa (so that some align and some do not),
    written with the record shapes the read files must keep byte for byte:
      FASTQ: blank lines (LF and CRLF) before the first record and between records, CRLF line ends, '+name' third
      lines, '%' and tabs in names, lower-case bases, a record over 8 KiB (a long name), no final newline;
      FASTA: multi-line sequences, '#' / ';' comment lines before and between records, an empty record, unnamed
      records."""
    rng = random.Random(seed)
    ref = "".join(l.strip() for l in open(os.path.join(refsets.GOLDEN, "tiny.fa")) if not l.startswith(">")).upper()

    def read(i):
        if i % 5 == 4:   # random sequence: does not align
            return "".join(rng.choice("ACGT") for _ in range(rng.randint(60, 120)))
        n = rng.randint(50, 150)
        while True:
            p = rng.randint(0, len(ref) - n)
            s = ref[p:p + n]
            if "N" not in s:
                break
        if rng.random() < 0.5:
            s = s.translate(str.maketrans("ACGT", "TGCA"))[::-1]
        return s

    fq = ["\n", "\r\n"]
    for i in range(40):
        s = read(i)
        nl = "\r\n" if i % 3 == 0 else "\n"
        name = "q%d" % i
        if i % 7 == 1:
            name += "\tdesc with\ttabs"
        if i % 7 == 2:
            name += "%20pct%zz"
        if i == 17:
            name += "_" + "L" * 9000
        if i % 4 == 3:
            s = s.lower()
        q = "".join(chr(33 + rng.randint(2, 40)) for _ in s)
        third = "+" + name if i % 6 == 5 else "+"
        rec = "@" + name + nl + s + nl + third + nl + q
        if i < 39:
            rec += nl + ("\n" if i % 8 == 4 else "") + ("\r\n" if i % 11 == 6 else "")
        fq.append(rec)
    open(os.path.join(d, "corpus.fq"), "w", newline="").write("".join(fq))
    fa = ["# comment before the first record\n", "; another\n", "\n"]
    for i in range(40):
        s = read(i)
        name = "" if i % 9 == 3 else "f%d" % i
        if i == 20:
            fa.append(">empty%d\n" % i)
            continue
        w = 60 if i % 2 else 37
        fa.append(">" + name + "\n" + "".join(s[k:k + w] + "\n" for k in range(0, len(s), w)))
        if i % 10 == 7:
            fa.append("# a comment line between records\n")
        if i % 10 == 8:
            fa.append("; a semicolon comment\n\n")
    open(os.path.join(d, "corpus.fa"), "w", newline="").write("".join(fa))
    return d


def case_input(d, case):
    """(index, read files, format flag, reference flags without the case's own, library options) of a case under d."""
    src = CASES[case][0]
    if src[0] == "corpus":
        return "tiny", [os.path.join(d, src[1])], ("-q" if src[1].endswith(".fq") else "-f"), ["--no-spliced-alignment"], {}
    index, fs, fmt, base, opts, _ = refsets.output_input(d, src)
    return index, fs, fmt, base, opts


def generate(d):
    """Every input the cases use, under d; returns d."""
    refsets.generate_output_sets(d)
    corpus(d)
    return d


def reference_passthrough(d, case):
    """stdout of the reference with --passthrough --reorder (SAM records, each followed by its escaped record text)."""
    index, fs, fmt, base, _ = case_input(d, case)
    reads = ["-1", fs[0], "-2", fs[1]] if len(fs) == 2 else ["-U", fs[0]]
    r = subprocess.run([refsets.REFBIN, fmt, "-x", os.path.join(refsets.GOLDEN, index)] + base + list(CASES[case][1]) + reads +
                       ["-p", str(min(16, os.cpu_count() or 1)), "--reorder", "--passthrough"],
                       check=True, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
    return r.stdout


def route(out):
    """The hisat2 wrapper's read-file loop (hisat2:595-650) over --passthrough output.  Returns (SAM without the record
    lines, {file: [record texts]}) with files un, al, un_conc/1, un_conc/2, al_conc/1, al_conc/2, al_conc_disc/1,
    al_conc_disc/2.  Lines are taken positionally: the record text of a FASTQ read starts with '@', so telling it from
    a header line by its first byte would drop it."""
    files = {k: [] for k in ("un", "al", "un_conc/1", "un_conc/2", "al_conc/1", "al_conc/2", "al_conc_disc/1", "al_conc_disc/2")}
    sam = []
    lines = out.split(b"\n")
    if lines and lines[-1] == b"":
        lines.pop()
    i = 0
    while i < len(lines):
        l = lines[i]
        i += 1
        sam.append(l + b"\n")
        if l.startswith(b"@"):
            continue
        fl = int(l.split(b"\t")[1])
        rec = re.sub(rb"%(..)", lambda m: bytes([int(m.group(1), 16)]), lines[i])
        i += 1
        unal, secondary = fl & 4 != 0, fl & 256 != 0
        mate1, mate2 = fl & 64 != 0, fl & 128 != 0
        if secondary:
            continue
        if not mate1 and not mate2:
            files["un" if unal else "al"].append(rec)
            continue
        m = "1" if mate1 else "2"
        files[("al_conc/" if fl & 2 else "un_conc/") + m].append(rec)
        if fl & 4 == 0 or fl & 8 == 0:
            files["al_conc_disc/" + m].append(rec)
    return b"".join(sam), files


def summarize(files):
    return {k: {"md5": hashlib.md5(b"".join(v)).hexdigest(), "bytes": sum(len(x) for x in v), "records": len(v)}
            for k, v in files.items()}


def load_expected():
    return json.load(open(OUT))


def main():
    res = {}
    with tempfile.TemporaryDirectory() as d:
        generate(d)
        for case in sorted(CASES):
            sam, files = route(reference_passthrough(d, case))
            res[case] = {"files": summarize(files), "sam_md5": refsets.sam_md5(sam)}
    json.dump(res, open(OUT, "w"), indent=1, sort_keys=True)
    open(OUT, "a").write("\n")


if __name__ == "__main__":
    main()
