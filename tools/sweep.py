#!/usr/bin/env python3
"""Sweep launch configurations on one read set; verify results identical across configs."""
import os, sys, hashlib
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import hisat2_b200 as h2
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
fa = sys.argv[1]
if fa.startswith("synth:"):          # bench.py's synthetic workload, e.g. synth:1000000
    import numpy as np
    sys.path.insert(0, ROOT)
    import bench
    n = int(fa.split(":")[1])
    d1, _ = bench.sim_fasta(0, n, paired=False)
    batch = h2.ReadBatch.parse(data1=d1)
else:
    batch = h2.ReadBatch.from_fasta(fa)
ref = None
for cfg in sys.argv[2:]:
    opts = {k: int(v) for k, v in (kv.split("=") for kv in cfg.split(","))}
    idx = h2.Index(os.path.join(ROOT, "oracle", "_ref", "data", os.environ.get("HT2_INDEX", "22_20-21M")), **opts)
    best = None
    for i in range(3):
        r = idx.align(batch)
        best = r.ms_kernel if best is None else min(best, r.ms_kernel)
        if i < 2: r.close()
    sam = idx.format_sam(batch, r)
    dg = hashlib.md5(sam).hexdigest()
    if ref is None: ref = dg
    print("%-50s kernel %.2f ms  %.2f Mreads/s  same=%s err=%d" % (cfg, best, batch.n / best / 1e3, dg == ref, int((r.reads["err"] != 0).sum())), flush=True)
    r.close(); idx.close()
