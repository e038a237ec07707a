#!/usr/bin/env python3
"""Cost of reading a run from several files: the same pairs (bench.py's synthetic 2x101 bp set on tests/golden/tiny)
given as one file per mate, as four lane files per mate, and gzip-compressed as one file and as four lane files.
The -1 and -2 lanes end at different records, so batches cross file boundaries at different places in the two mates.

  python tools/multi_input_bench.py [--pairs N] [--repeats R] [--out DIR]

One process, one index, SAM collected by no one (the text still lands in pinned host memory).  Every arm is warmed
up once, then the arms alternate, R runs each.  The time of a run is the library call's own wall clock (s_total of
ht2gpu_run_reads_routed / ht2gpu_run_reads_files): parse, inflate, align, SAM and the wait for the last batch.
Prints one JSON line: reads/s of every run per arm, their medians and spread (max - min over median), the card's name
and power limit, and whether every arm's SAM equals the single file's."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, check=True)
    return q.stdout.decode().strip().splitlines()[0]


def note(msg, t0=time.perf_counter()):
    print("[%7.1f s] %s" % (time.perf_counter() - t0, msg), file=sys.stderr, flush=True)


def gz(src, dst, level=1):
    c = zlib.compressobj(level, zlib.DEFLATED, 31)
    with open(src, "rb") as fi, open(dst, "wb") as fo:
        while True:
            b = fi.read(1 << 24)
            if not b:
                break
            fo.write(c.compress(b))
        fo.write(c.flush())
    return dst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=4000000)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/multi_input_bench.json")
    a = ap.parse_args()
    import hisat2_b200 as h2
    with tempfile.TemporaryDirectory() as d:
        m1, m2 = bench.sim_fasta(0, a.pairs)
        one = [os.path.join(d, "r_1.fa"), os.path.join(d, "r_2.fa")]
        m1.tofile(one[0])
        m2.tofile(one[1])
        lanes = [[], []]
        for k, m in enumerate((m1, m2)):   # four lanes per mate, cut at different records in the two mates
            cuts = [0] + [a.pairs * q // 4 + (k * 997 if q else 0) for q in (1, 2, 3)] + [a.pairs]
            for q in range(4):
                p = os.path.join(d, "l%d_%d.fa" % (q, k + 1))
                m[cuts[q] * bench.RECSZ:cuts[q + 1] * bench.RECSZ].tofile(p)
                lanes[k].append(p)
        del m1, m2
        note("plain files written")
        one_gz = [gz(p, p + ".gz") for p in one]
        lanes_gz = [[gz(p, p + ".gz") for p in v] for v in lanes]
        arms = {"one_file": dict(path1=one[0], path2=one[1]),
                "four_lanes": dict(path1=lanes[0], path2=lanes[1]),
                "one_file_gz": dict(path1=one_gz[0], path2=one_gz[1]),
                "four_lanes_gz": dict(path1=lanes_gz[0], path2=lanes_gz[1])}
        note("gzip files written")
        idx = h2.Index(bench.INDEX, device=0)   # bench.py's options
        md5 = {}
        for k, kw in arms.items():   # warm-up, and the SAM of every arm
            sam, _ = idx.run_reads(**kw)
            md5[k] = hashlib.md5(sam).hexdigest()
            del sam
            note("warm-up " + k)
        rates = {k: [] for k in arms}
        for _ in range(a.repeats):
            for k, kw in arms.items():
                _, st = idx.run_reads(collect=False, **kw)
                rates[k].append(2 * a.pairs / st["s_total"])
                note("%s %.3f s" % (k, st["s_total"]))
        idx.close()
    med = {k: sorted(v)[len(v) // 2] for k, v in rates.items()}
    line = {"gpu": gpu_info(), "pairs": a.pairs, "reads_per_s": rates, "median_reads_per_s": med,
            "spread": {k: (max(v) - min(v)) / med[k] for k, v in rates.items()},
            "four_lanes_vs_one_file": med["four_lanes"] / med["one_file"],
            "four_lanes_gz_vs_one_file_gz": med["four_lanes_gz"] / med["one_file_gz"],
            "same_sam": len(set(md5.values())) == 1}
    print(json.dumps(line))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        json.dump(line, open(os.path.join(a.out, "multi_input_bench.json"), "w"))


if __name__ == "__main__":
    main()
