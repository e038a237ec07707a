#!/usr/bin/env python3
"""End-to-end cost of --un-conc / --al-conc: hisat2-b200 on bench.py's read set (synthetic 2x101 bp pairs on
tests/golden/tiny, -k 5), SAM to /dev/null, without read files and with both written to /dev/null.

  python tools/read_files_bench.py [--pairs N] [--repeats R] [--out DIR]

The two arms alternate, R runs each, in one process; every run is the whole CLI (index load, parse, align, SAM,
routing).  Prints one JSON line: reads/s of every run per arm, their medians, the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

CLI = os.path.join(ROOT, "hisat2_b200", "hisat2-b200")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, check=True)
    return q.stdout.decode().strip().splitlines()[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=4000000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/read_files_bench.json")
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as d:
        f1, f2 = os.path.join(d, "r_1.fa"), os.path.join(d, "r_2.fa")
        m1, m2 = bench.sim_fasta(0, a.pairs)
        m1.tofile(f1)
        m2.tofile(f2)
        for n in ("uc.1", "uc.2", "ac.1", "ac.2"):
            os.symlink("/dev/null", os.path.join(d, n))
        base = [CLI, "-x", bench.INDEX, "-f", "--no-spliced-alignment", "-k", "5", "-1", f1, "-2", f2, "-S", "/dev/null", "--quiet"]
        arms = {"off": base, "un_conc_al_conc": base + ["--un-conc", os.path.join(d, "uc"), "--al-conc", os.path.join(d, "ac")]}
        subprocess.run(base, check=True)   # warm-up: page cache, module load
        rates = {k: [] for k in arms}
        for _ in range(a.repeats):
            for k, cmd in arms.items():
                t0 = time.perf_counter()
                subprocess.run(cmd, check=True)
                rates[k].append(2 * a.pairs / (time.perf_counter() - t0))
    med = {k: sorted(v)[len(v) // 2] for k, v in rates.items()}
    line = {"gpu": gpu_info(), "pairs": a.pairs, "reads_per_s": rates, "median_reads_per_s": med,
            "routing_cost": 1 - med["un_conc_al_conc"] / med["off"]}
    print(json.dumps(line))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        json.dump(line, open(os.path.join(a.out, "read_files_bench.json"), "w"))


if __name__ == "__main__":
    main()
