#!/usr/bin/env python3
"""Informational: the graph alignment kernel's rate on tests/golden/tiny_snp (SNP ALTs only: what existing graph-index
users run) and on tests/golden/tiny_snp_tran (SNP, splice-site and exon ALTs), in spliced mode on RNA-like pairs
(tools/sim_rna.py transcripts over tiny.fa, 25 k distinct pairs x --copies) and without spliced alignment on
bench.py's synthetic DNA pairs.

  python tools/tran_bench.py [--lib-root DIR] [--copies C] [--pairs N] [--repeats R]

--lib-root runs another build of the library (for example a checkout of the parent commit, after its build()) on this
tree's fixtures; an index that build refuses is reported as "refused".  One process; every arm is warmed up once, then
the arms alternate, R runs each.  Prints one JSON line: per arm the kernel reads/s (ms_align + ms_sam of
ht2gpu_run_reads) of every run and their median, and the card's name and power limit.  Not part of bench.py's value."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib-root", default=ROOT)
    ap.add_argument("--copies", type=int, default=8)
    ap.add_argument("--pairs", type=int, default=100000)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    sys.path.insert(0, os.path.abspath(a.lib_root))
    sys.path.insert(1, ROOT)
    sys.path.insert(2, os.path.join(ROOT, "tools"))
    import hisat2_b200 as h2
    import bench
    import sim_rna
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                         check=True).stdout.decode().strip().splitlines()[0]
    _, pairs, _ = sim_rna.sim(sim_rna.load_fasta(os.path.join(GOLDEN, "tiny.fa")), 0, 25000, 7)
    r1 = "".join(">r%dp%d/1\n%s\n" % (r, i, x) for r in range(a.copies) for i, (x, _) in enumerate(pairs)).encode()
    r2 = "".join(">r%dp%d/2\n%s\n" % (r, i, y) for r in range(a.copies) for i, (_, y) in enumerate(pairs)).encode()
    m1, m2 = bench.sim_fasta(0, a.pairs)
    inputs = {"rna": (r1, r2, 2 * a.copies * len(pairs), 0), "dna": (m1.tobytes(), m2.tobytes(), 2 * a.pairs, 1)}
    arms = {}
    for index in ("tiny_snp", "tiny_snp_tran"):
        for kind, (d1, d2, n, nospl) in inputs.items():
            name = "%s_%s" % (index, kind)
            try:
                idx = h2.Index(os.path.join(GOLDEN, index), no_spliced_alignment=nospl)
                idx.run_reads(data1=d1, data2=d2, collect=False)
            except h2.Ht2GpuError as e:
                arms[name] = str(e)
                continue
            arms[name] = (idx, d1, d2, n)
    rates = {k: [] for k, v in arms.items() if not isinstance(v, str)}
    for _ in range(a.repeats):
        for k in rates:
            idx, d1, d2, n = arms[k]
            _, st = idx.run_reads(data1=d1, data2=d2, collect=False)
            rates[k].append(n / ((st["ms_align"] + st["ms_sam"]) / 1e3))
    out = {"gpu": gpu, "lib_root": os.path.abspath(a.lib_root), "kernel_reads_per_s": rates,
           "median": {k: statistics.median(v) for k, v in rates.items()},
           "refused": {k: v for k, v in arms.items() if isinstance(v, str)}}
    for v in arms.values():
        if not isinstance(v, str):
            v[0].close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
