#!/usr/bin/env python3
"""Expected output of read-file lists (-1 a1,a2 -2 b1,b2 -U u1,u2), from the unmodified reference.

  python tools/multi_input_ref.py          # writes tests/golden/multi_input_sets.json

Every case splits read sets of tests/golden (tiny_*.fq) and tools/refsets.py into several files: the -1 and -2 files
end at different records, and lists mix plain, gzip and BGZF files.  The reference (oracle/_ref/hisat2-align-s) reads
no gzip, so it is given the same files decompressed, as a list; the hisat2 wrapper's pipes give it the same streams.
It runs with --reorder.  The JSON keeps, per case, the md5 of its SAM without @PG, its alignment summary (stderr) and,
for cases with read files, md5, size and record count of every file, routed from a --passthrough run the way
tools/readfiles_ref.py routes them (the wrapper strips --no-unal from the reference's arguments and applies it to the
SAM only, so the read files do not depend on it)."""
import gzip
import hashlib
import json
import os
import struct
import subprocess
import sys
import tempfile
import zlib

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import readfiles_ref  # noqa: E402
import refsets  # noqa: E402

OUT = os.path.join(refsets.GOLDEN, "multi_input_sets.json")

# An input file: (name, source, first record, end record, compression), where source is a FASTA/FASTQ file of
# tests/golden ("golden:<name>") or of tools/refsets.py's sets under the data directory ("set:<file>"), and
# compression is None, "gz" or "bgzf".  "unnamed" as a sixth element blanks the name of every third record.
# case -> dict(index, fmt, m1, m2, u (lists of input files, -U given first when u_first), flags (reference),
#              opts (library), front (ht2gpu_reads_input_t), sam_output, read_files, new_summary)
F_SE, F_PE1, F_PE2 = "golden:tiny_se.fq", "golden:tiny_pe_1.fq", "golden:tiny_pe_2.fq"
MIXED = dict(index="tiny", fmt="-q",
             m1=[("p1a.fq", F_PE1, 0, 60, None), ("p1b.fq.gz", F_PE1, 60, 150, "gz")],
             m2=[("p2a.fq.gz", F_PE2, 0, 95, "gz"), ("p2b.fq", F_PE2, 95, 150, None)],
             u=[("ua.fq", F_SE, 0, 170, None), ("ub.fq.gz", F_SE, 170, 400, "bgzf")])
CASES = {
    "se_fq_plain_gz_bgzf": dict(index="tiny", fmt="-q", m1=[], m2=[],
                                u=[("s1.fq", F_SE, 0, 130, None), ("s2.fq.gz", F_SE, 130, 280, "gz"),
                                   ("s3.fq.bgz", F_SE, 280, 400, "bgzf")]),
    "pe_two_lanes": dict(index="tiny", fmt="-f",
                         m1=[("l1_1.fa", "set:reads_1.fa", 0, 400, None), ("l2_1.fa.gz", "set:reads_1.fa", 400, 1000, "gz")],
                         m2=[("l1_2.fa.gz", "set:reads_2.fa", 0, 650, "gz"), ("l2_2.fa", "set:reads_2.fa", 650, 1000, None)],
                         u=[]),
    "mixed_u_first": dict(MIXED, u_first=True),
    "unnamed_fa": dict(index="tiny", fmt="-f",
                       m1=[("n1a.fa", "set:reads_1.fa", 0, 100, None, "unnamed"), ("n1b.fa", "set:reads_1.fa", 100, 300, None, "unnamed")],
                       m2=[("n2a.fa", "set:reads_2.fa", 0, 200, None, "unnamed"), ("n2b.fa.gz", "set:reads_2.fa", 200, 300, "gz", "unnamed")],
                       u=[("nu.fa", "set:reads_1.fa", 300, 500, None, "unnamed")]),
    "mixed_skip40": dict(MIXED, flags=["-s", "40"], front=dict(skip=40)),
    "mixed_upto100": dict(MIXED, flags=["-u", "100"], front=dict(upto=100)),
    "mixed_upto150": dict(MIXED, flags=["-u", "150"], front=dict(upto=150)),
    "mixed_upto250": dict(MIXED, flags=["-u", "250"], front=dict(upto=250)),
    "mixed_skip30_upto200": dict(MIXED, flags=["-s", "30", "-u", "200"], front=dict(skip=30, upto=200)),
    "mixed_read_files_no_unal_new_summary": dict(MIXED, flags=["--no-unal", "--new-summary"], sam_output=dict(no_unal=1),
                                                 read_files=True, new_summary=True),
    "graph_alt_lanes": dict(index="tiny_snp", fmt="-f",
                            m1=[("g1a.fa", "set:alt20k_1.fa", 0, 700, None), ("g1b.fa.gz", "set:alt20k_1.fa", 700, 2000, "gz")],
                            m2=[("g2a.fa", "set:alt20k_2.fa", 0, 1300, None), ("g2b.fa", "set:alt20k_2.fa", 1300, 2000, None)],
                            u=[("gu.fa.gz", "set:alt20k_1.fa", 2000, 3000, "bgzf")]),
    "spliced_lanes": dict(index="tiny", fmt="-f", spliced=True,
                          m1=[("x1a.fa", "set:splice_sim_1.fa", 0, 150, None), ("x1b.fa", "set:splice_sim_1.fa", 150, 400, None)],
                          m2=[("x2a.fa.gz", "set:splice_sim_2.fa", 0, 280, "gz"), ("x2b.fa", "set:splice_sim_2.fa", 280, 400, None)],
                          u=[("xu.fa", "set:splice_sim_1.fa", 400, 600, None)]),
}


def bgzf(data, level=6, block=65280):
    """BGZF: gzip members of at most `block` input bytes with a BC extra field holding the member size, then the
    empty end-of-file member."""
    def member(part):
        c = zlib.compressobj(level, zlib.DEFLATED, -15)
        raw = c.compress(part) + c.flush()
        bsize = 12 + 6 + len(raw) + 8 - 1
        return (b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff" + struct.pack("<H", 6) + b"BC" + struct.pack("<HH", 2, bsize) +
                raw + struct.pack("<II", zlib.crc32(part), len(part)))
    return b"".join(member(data[i:i + block]) for i in range(0, len(data), block)) + member(b"")


def records(path):
    """The records of a FASTA (by '>') or FASTQ (4 lines) file."""
    data = open(path, "rb").read()
    if path.endswith((".fa", ".fasta")):
        return [b">" + r for r in data.split(b">")[1:]]
    lines = data.splitlines(True)
    return [b"".join(lines[i:i + 4]) for i in range(0, len(lines), 4)]


def generate(d):
    """Every input file of every case under d: <name> as the library and the CLI read it (compressed where the case
    says so) and plain/<name>, the decompressed text the reference reads.  Returns d."""
    refsets.generate(d, ["reads", "alt20k"])
    refsets.generate_spliced(d)
    os.makedirs(os.path.join(d, "plain"), exist_ok=True)
    cache = {}
    for case in CASES.values():
        for f in case["m1"] + case["m2"] + case["u"]:
            name, src, r0, r1, comp = f[:5]
            kind, fn = src.split(":", 1)
            path = os.path.join(refsets.GOLDEN if kind == "golden" else d, fn)
            if path not in cache:
                cache[path] = records(path)
            recs = cache[path][r0:r1]
            if len(f) > 5 and f[5] == "unnamed":
                recs = [r[:1] + r[r.index(b"\n"):] if i % 3 == 1 else r for i, r in enumerate(recs)]
            text = b"".join(recs)
            open(os.path.join(d, "plain", name), "wb").write(text)
            out = gzip.compress(text, 6, mtime=0) if comp == "gz" else bgzf(text) if comp == "bgzf" else text
            open(os.path.join(d, name), "wb").write(out)
    return d


def reads_args(d, case, plain=False):
    """-1 / -2 / -U arguments of a case (file names under d, or under d/plain for the reference)."""
    c = CASES[case]
    p = lambda fs: ",".join(os.path.join(d, "plain", f[0]) if plain else os.path.join(d, f[0]) for f in fs)
    pairs = ["-1", p(c["m1"]), "-2", p(c["m2"])] if c["m1"] else []
    unp = ["-U", p(c["u"])] if c["u"] else []
    return unp + pairs if c.get("u_first") else pairs + unp


def base_flags(case):
    c = CASES[case]
    return ["--no-temp-splicesite"] if c.get("spliced") else ["--no-spliced-alignment"]


def lib_opts(case):
    return dict(no_spliced_alignment=0) if CASES[case].get("spliced") else {}


def reference(d, case, passthrough=False):
    """(stdout, stderr) of the reference on a case; without --no-unal and with --passthrough for the read files."""
    c = CASES[case]
    flags = list(c.get("flags", []))
    if passthrough:
        flags = [f for f in flags if f != "--no-unal"] + ["--passthrough"]
    r = subprocess.run([refsets.REFBIN, c["fmt"], "-x", os.path.join(refsets.GOLDEN, c["index"])] + base_flags(case) + flags +
                       reads_args(d, case, plain=True) + ["-p", "1", "--reorder"],
                       check=True, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    return r.stdout, r.stderr


def load_expected():
    return json.load(open(OUT))


def main():
    res = {}
    with tempfile.TemporaryDirectory() as d:
        generate(d)
        for case in sorted(CASES):
            sam, err = reference(d, case)
            e = {"sam_md5": refsets.sam_md5(sam), "summary": refsets.summary_text(err),
                 "records": sum(1 for l in sam.splitlines() if not l.startswith(b"@"))}
            if CASES[case].get("read_files"):
                _, files = readfiles_ref.route(reference(d, case, passthrough=True)[0])
                e["files"] = readfiles_ref.summarize(files)
            res[case] = e
    json.dump(res, open(OUT, "w"), indent=1, sort_keys=True)
    open(OUT, "a").write("\n")


if __name__ == "__main__":
    main()
