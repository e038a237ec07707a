#!/usr/bin/env python3
"""How much does grouping similar reads into the same warp help?  Sort the batch by
keys derived from a first run (n_lf, alignment shape) and re-time the kernel."""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import hisat2_b200 as h2
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
fa = sys.argv[1]
batch = h2.ReadBatch.from_fasta(fa)
idx = h2.Index(os.path.join(ROOT, "oracle", "_ref", "data", "22_20-21M"))
def time_batch(b, label):
    best = None
    for i in range(3):
        r = idx.align(b)
        best = r.ms_kernel if best is None else min(best, r.ms_kernel)
        if i < 2: r.close()
    print("%-40s kernel %.2f ms  %.2f Mreads/s" % (label, best, b.n / best / 1e3), flush=True)
    return r
r = time_batch(batch, "input order")
L = 101
def permute(order):
    seq = batch.seq.reshape(-1, L)[order].reshape(-1)
    return h2.ReadBatch(seq, batch.offs, batch.seeds[order], [batch.names[i] for i in order])
nlf = r.reads["n_lf"].astype(np.int64)
time_batch(permute(np.argsort(nlf, kind="stable")), "sorted by n_lf")
fw = np.zeros(batch.n, np.int64); sc = np.zeros(batch.n, np.int64); na = r.reads["n_aln"][:, 0].astype(np.int64)
has = na > 0
first = r.alns[r.reads["aln_off"][has]]
fw[has] = first["fw"]; sc[has] = -first["score"]
key = ((na * 2 + fw) * 64 + sc) * 100000 + nlf
time_batch(permute(np.argsort(key, kind="stable")), "sorted by (n_aln, strand, score, n_lf)")
rng = np.random.default_rng(1)
time_batch(permute(rng.permutation(batch.n)), "random order")
