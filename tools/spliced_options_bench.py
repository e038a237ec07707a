#!/usr/bin/env python3
"""Informational: the kernel rate of spliced alignment under --dta, under non-default intron-length functions
(--pen-canintronlen G,-8,2, --pen-noncanintronlen S,-5,0.3) and under --avoid-pseudogene, against the default, on two
slices of bench.py:
  dna_like  its synthetic 2x101 bp pairs on tests/golden/tiny in spliced mode ("spliced_no_temp_splicesite_PE"): few
            junctions, so this mostly shows that the options cost nothing where nothing is spliced;
  rna       its RNA-like pairs ("spliced_known_splicesites_RNA_like_PE"): tools/sim_rna.py transcripts over the
            index's sequence with their site file loaded, where most pairs cross junctions and the intron-length
            penalty is looked up for every novel one.

  python tools/spliced_options_bench.py [--pairs N] [--rna-copies C] [--repeats R]

One process; every arm is warmed up once, then the arms alternate, R runs each.  Prints one JSON line: per slice and arm
the kernel reads/s (ms_align + ms_sam of ht2gpu_run_reads) of every run and their median, and the card's name and power
limit.  Not part of bench.py's value."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

ARMS = {
    "default": {},
    "dta": dict(dta=1),
    "intron_functions": dict(can_intronlen_type="G", can_intronlen_const=-8.0, can_intronlen_coeff=2.0,
                             noncan_intronlen_type="S", noncan_intronlen_const=-5.0, noncan_intronlen_coeff=0.3),
    "avoid_pseudogene": dict(avoid_pseudogene=1),
}


def rna_slice(copies):
    """bench.extra_rna_line's RNA-like pairs (25 k distinct pairs x copies) and their site lines."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import sim_rna
    _, pairs, lines = sim_rna.sim(sim_rna.load_fasta(bench.INDEX + ".fa"), 0, 25000, 7)
    b1 = "".join(">r%dp%d/1\n%s\n" % (r, i, a) for r in range(copies) for i, (a, _) in enumerate(pairs)).encode()
    b2 = "".join(">r%dp%d/2\n%s\n" % (r, i, b) for r in range(copies) for i, (_, b) in enumerate(pairs)).encode()
    return b1, b2, 2 * copies * len(pairs), lines


def run_slice(h2, d1, d2, n_reads, repeats, ss=None):
    idx = {k: h2.Index(bench.INDEX, no_spliced_alignment=0, **o) for k, o in ARMS.items()}
    rates = {k: [] for k in ARMS}
    try:
        for k in ARMS:
            if ss:
                idx[k].load_splicesites(ss)
            idx[k].run_reads(data1=d1, data2=d2, collect=False)
        for _ in range(repeats):
            for k in ARMS:
                _, st = idx[k].run_reads(data1=d1, data2=d2, collect=False)
                rates[k].append(n_reads / ((st["ms_align"] + st["ms_sam"]) / 1e3))
    finally:
        for i in idx.values():
            i.close()
    return {"reads": n_reads, "kernel_reads_per_s": rates, "median": {k: statistics.median(v) for k, v in rates.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=100000)
    ap.add_argument("--rna-copies", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    import hisat2_b200 as h2
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                         check=True).stdout.decode().strip().splitlines()[0]
    m1, m2 = bench.sim_fasta(0, a.pairs)
    out = {"gpu": gpu, "dna_like": run_slice(h2, m1.tobytes(), m2.tobytes(), 2 * a.pairs, a.repeats)}
    r1, r2, n, lines = rna_slice(a.rna_copies)
    with tempfile.NamedTemporaryFile("w", suffix="_ss.txt") as f:
        f.write("\n".join(lines) + "\n")
        f.flush()
        out["rna"] = run_slice(h2, r1, r2, n, a.repeats, f.name)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
