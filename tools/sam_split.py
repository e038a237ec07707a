#!/usr/bin/env python3
"""Where the SAM back end's time goes, on a bench-shaped batch.

  python tools/sam_split.py [--pairs 2000000] [--index tests/golden/tiny] [--repeat 3]

Aligns one batch of bench.py's synthetic 2x101-bp pairs (the same generator and seed, default options) with
HT2GPU_SAM_SPLIT=1, which makes the library print, after every batch, the CUDA-event time of each of the three SAM
kernels (counting pass ht2_sam_kernel<false>, block scan ht2_sam_scan_kernel, writing pass ht2_sam_kernel<true>),
the batch's SAM bytes and the bytes per second.  A first, unmeasured pass warms the kernels up; --repeat measured
passes follow.  The card's name and power limit are printed first: times are only comparable on the same card and
limit.
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["HT2GPU_SAM_SPLIT"] = "1"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=2000000)
    ap.add_argument("--index", default=os.path.join(ROOT, "tests", "golden", "tiny"))
    ap.add_argument("--repeat", type=int, default=3)
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, universal_newlines=True)
    print("gpu:", smi.stdout.strip(), flush=True)
    import bench
    import hisat2_b200 as h2
    idx = h2.Index(args.index, device=0)   # bench.py's options
    d1, d2 = bench.sim_fasta(0, args.pairs)
    batch = h2.ReadBatch.parse(data1=d1, data2=d2)
    print("warm-up pass (its line follows and is not the measurement)", file=sys.stderr, flush=True)
    idx.align_sam(batch)
    for r in range(args.repeat):
        print("=== measured pass %d: %d pairs ===" % (r + 1, args.pairs), file=sys.stderr, flush=True)
        sam, st = idx.align_sam(batch, with_stats=True)
        sys.stderr.flush()
        print("ms_align %.2f  ms_sam %.2f  sam bytes %d" % (st["ms_align"], st["ms_sam"], len(sam)), flush=True)


if __name__ == "__main__":
    main()
