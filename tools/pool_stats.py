#!/usr/bin/env python3
"""Where the alignment pool kernel's rounds go, on a bench-shaped launch.

  python tools/pool_stats.py [--pairs 2000000] [--index tests/golden/tiny] [--spliced]

Aligns one batch of bench.py's synthetic 2x101-bp pairs (the same generator and seed) with HT2GPU_STATS=1 and
prints the pool kernel's per-state round table (rounds, lanes per round, cycles per round, share of the kernel's
cycles) that the library writes to stderr after the batch.  A first, unmeasured pass warms the kernel up.  The
card's name and power limit are printed first: cycle counts are only comparable on the same card and limit.
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["HT2GPU_STATS"] = "1"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=2000000)
    ap.add_argument("--index", default=os.path.join(ROOT, "tests", "golden", "tiny"))
    ap.add_argument("--spliced", action="store_true", help="spliced mode (default: --no-spliced-alignment, like bench.py)")
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, universal_newlines=True)
    print("gpu:", smi.stdout.strip(), flush=True)
    import bench
    import hisat2_b200 as h2
    idx = h2.Index(args.index, device=0, **({"no_spliced_alignment": 0} if args.spliced else {}))   # bench.py's options
    d1, d2 = bench.sim_fasta(0, args.pairs)
    batch = h2.ReadBatch.parse(data1=d1, data2=d2)
    print("warm-up pass (its table follows and is not the measurement)", file=sys.stderr, flush=True)
    idx.align_sam(batch, with_stats=True)
    print("=== measured pass: %d pairs, geometry %s ===" % (args.pairs, idx.geometry()), file=sys.stderr, flush=True)
    _, st = idx.align_sam(batch, with_stats=True)
    sys.stderr.flush()
    print("ms_align %.2f  ms_sam %.2f  pairs/s (align) %.0f" % (st["ms_align"], st["ms_sam"], args.pairs / (st["ms_align"] / 1e3)))


if __name__ == "__main__":
    main()
