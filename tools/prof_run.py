#!/usr/bin/env python3
"""Short run for ncu: align <reads.fa> (default oracle/_ref/data/sim200k_1.fa) `iters` times."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import hisat2_b200 as h2
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
fa = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "oracle", "_ref", "data", "sim200k_1.fa")
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 3
opts = dict(kv.split("=") for kv in sys.argv[3:])
opts = {k: int(v) for k, v in opts.items()}
idx = h2.Index(os.path.join(ROOT, "oracle", "_ref", "data", os.environ.get("HT2_INDEX", "22_20-21M")), **opts)
print("opts", opts)
if fa.startswith("synth"):          # bench.py's synthetic workload, e.g. synth:1000000
    import numpy as np
    sys.path.insert(0, ROOT)
    import bench
    n = int(fa.split(":")[1])                       # synth:N = N single-end reads, synthpe:N = N pairs
    d1, d2 = bench.sim_fasta(0, n, paired=fa.startswith("synthpe:"))
    batch = h2.ReadBatch.parse(data1=d1, data2=d2)
else:
    batch = h2.ReadBatch.from_fasta(fa)
for i in range(iters):
    _, st = idx.align_sam(batch, with_stats=True)
    print("iter", i, "align ms %.2f  sam ms %.2f  reads/s (align) %.0f" % (st["ms_align"], st["ms_sam"], batch.n / (st["ms_align"] / 1e3)))
