"""Measure gzip read input: device inflate on its own, and reads/s end to end for plain FASTQ, .fq.gz inflated on the
device, and .fq.gz through `gzip -dc` pipes (the hisat2 wrapper's way).

    python tools/bench_gunzip.py [--pairs 2000000] [--level 6] [--out DIR]

2x101 pairs simulated from the tiny fixture (tools/simreads_fast.c, seed 1) as FASTQ with varied qualities; the
compression (Python zlib, one member) is not timed.  End to end is one Index.run_reads on one handle, from the call
(or from starting the gzip processes) to the last SAM batch, --no-spliced-alignment.  The pipe arm drains both mate
pipes concurrently, as hisat2-align-s would read them.  Prints the card name and power limit beside the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import threading
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def sim_fastq(pairs, seed=1):
    import bench
    a, b = bench.sim_fasta(0, pairs, seed=seed)
    rng = np.random.default_rng(seed)
    out = []
    for buf in (a, b):
        r = np.asarray(buf).reshape(pairs, bench.RECSZ)
        q = np.empty((pairs, 217), np.uint8)
        q[:, 0] = ord("@")
        q[:, 1:113] = r[:, 1:113]                      # name, bases and their newlines
        q[:, 113:115] = np.frombuffer(b"+\n", np.uint8)
        q[:, 115:216] = np.frombuffer(b"FFFF:F,F#:FFFFFF", np.uint8)[rng.integers(0, 16, (pairs, 101))]
        q[:, 216] = ord("\n")
        out.append(q.tobytes())
    return out


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
    return r.stdout.decode().strip().splitlines()[0] if r.returncode == 0 and r.stdout else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=2000000)
    ap.add_argument("--level", type=int, default=6)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import hisat2_b200 as h2
    tmp = tempfile.mkdtemp(prefix="bench_gunzip_")
    texts = sim_fastq(a.pairs)
    plain, gz = [], []
    for i, t in enumerate(texts):
        p = os.path.join(tmp, "r_%d.fq" % (i + 1))
        open(p, "wb").write(t)
        open(p + ".gz", "wb").write(zlib.compress(t, a.level, wbits=31))
        plain.append(p)
        gz.append(p + ".gz")
    res = {"gpu": gpu_info(), "pairs": a.pairs, "level": a.level, "fastq_bytes": [len(t) for t in texts],
           "gz_bytes": [os.path.getsize(p) for p in gz]}
    # inflate only
    data = open(gz[0], "rb").read()
    h2.gunzip(data)                                    # warm-up: module load, first allocations
    runs = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        out, st = h2.gunzip(data)
        runs.append((time.perf_counter() - t0, st))
        assert out == texts[0]
    best = min(runs, key=lambda x: x[0])
    res["inflate"] = {"s_call": [round(r[0], 4) for r in runs], "gb_per_s_out": round(len(texts[0]) / best[0] / 1e9, 3),
                      "stats": best[1]}
    # end to end
    idx = h2.Index(os.path.join(ROOT, "tests", "golden", "tiny"), no_spliced_alignment=1)
    n_reads = 2 * a.pairs
    idx.run_reads(path1=plain[0], path2=plain[1], fastq=True, collect=False, upto=20000)   # warm-up

    def timed(fn):
        t0 = time.perf_counter()
        fn()
        return time.perf_counter() - t0

    def pipe_run():
        procs = [subprocess.Popen(["gzip", "-dc", p], stdout=subprocess.PIPE) for p in gz]
        bufs = [None, None]

        def drain(i):
            bufs[i] = procs[i].stdout.read()
        th = [threading.Thread(target=drain, args=(i,)) for i in range(2)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        for p in procs:
            p.wait()
        idx.run_reads(data1=bufs[0], data2=bufs[1], fastq=True, collect=False)

    e2e = {"plain": [], "gz_device": [], "gz_pipe": []}
    sams = {}
    for _ in range(a.reps):
        e2e["plain"].append(timed(lambda: idx.run_reads(path1=plain[0], path2=plain[1], fastq=True, collect=False)))
        e2e["gz_device"].append(timed(lambda: idx.run_reads(path1=gz[0], path2=gz[1], fastq=True, collect=False)))
        res["run_gunzip_stats"] = idx.gunzip_stats()
        e2e["gz_pipe"].append(timed(pipe_run))
    sams["plain"] = idx.run_reads(path1=plain[0], path2=plain[1], fastq=True, upto=200000)[0]
    sams["gz"] = idx.run_reads(path1=gz[0], path2=gz[1], fastq=True, upto=200000)[0]
    idx.close()
    res["sam_equal_first_200k_pairs"] = sams["plain"] == sams["gz"]
    res["end_to_end_s"] = {k: [round(x, 3) for x in v] for k, v in e2e.items()}
    res["reads_per_s"] = {k: round(n_reads / min(v)) for k, v in e2e.items()}
    res["gz_device_over_pipe"] = round(min(e2e["gz_pipe"]) / min(e2e["gz_device"]), 2)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        open(os.path.join(a.out, "bench_gunzip.json"), "w").write(line + "\n")
    for p in plain + gz:
        os.unlink(p)
    os.rmdir(tmp)


if __name__ == "__main__":
    main()
