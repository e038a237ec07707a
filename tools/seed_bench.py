#!/usr/bin/env python3
"""Time the seed-search kernel alone (ht2gpu_seed_search) on a linear and a graph index."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import hisat2_b200 as h2
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
fa = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "oracle", "_ref", "data", "sim200k_1.fa")
batch = h2.ReadBatch.from_fasta(fa)
for name in ("22_20-21M", "22_20-21M_snp"):
    idx = h2.Index(os.path.join(ROOT, "oracle", "_ref", "data", name))
    best = None
    for i in range(3):
        r = idx.seed_search(batch, max_range=4)
        if best is None or r.ms_kernel < best[0]:
            best = (r.ms_kernel, r.n_lf, r.alg_bytes, len(r.hits), len(r.coords))
        r.close()
    ms, nlf, ab, nh, nc = best
    print("%-14s graph=%d reads=%d: %.2f ms (count+fill passes)  %.1f M reads/s  %.1f LF/read  %.2f G LF/s  alg %.1f GB/s  hits=%d coords=%d"
          % (name, idx.is_graph(), batch.n, ms, batch.n / ms / 1e3, nlf / batch.n, nlf / ms / 1e6, ab / ms / 1e6, nh, nc), flush=True)
    idx.close()
