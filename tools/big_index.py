#!/usr/bin/env python3
"""HBM-resident regime (SURVEY 8d stand-in for BASELINE configs[3]): a synthetic reference of --mbp Mbp (random
chromosomes of 64 Mbp with a 10 kbp N gap each, plus repeat families), indexed with the reference's own
hisat2-build-s (index construction is out of scope), then
  * parity: 200 k reads / 100 k pairs, SAM byte-compared with the reference binary run on this box;
  * throughput of the alignment path (FASTA -> SAM through ht2gpu_run_reads) and of the seed kernel alone
    (LF mapping: algorithmic GB/s against the HBM copy peak).
Run on a GPU machine:  python tools/big_index.py --mbp 512 --out big_index.json
Everything lands in data_big/ (git- and gpurun-ignored: the index is rebuilt where it is used)."""
import argparse, ctypes, json, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench
import hisat2_b200 as h2

B = os.path.join(ROOT, "data_big")
REFDIR = os.path.join(ROOT, "oracle", "_ref")


def make_reference(mbp, seed=11):
    rng = np.random.default_rng(seed)
    chroms = []
    nchr = max(1, mbp // 64)
    per = mbp * 1000000 // nchr
    fams = [rng.integers(0, 4, 3000, dtype=np.uint8) for _ in range(20)]
    for c in range(nchr):
        s = rng.integers(0, 4, per, dtype=np.uint8)
        for f in fams:                                      # 10 copies per family and chromosome, 2 % divergence
            for _ in range(10):
                p = int(rng.integers(0, per - 4000))
                cp = f.copy()
                m = rng.random(len(cp)) < 0.02
                cp[m] = (cp[m] + rng.integers(1, 4, int(m.sum()), dtype=np.uint8)) & 3
                s[p:p + len(cp)] = cp
        a = np.frombuffer(b"ACGT", dtype=np.uint8)[s]
        g = per // 2
        a[g:g + 10000] = ord("N")
        chroms.append(a)
    return chroms


def write_fasta(path, chroms):
    with open(path, "wb") as f:
        for i, a in enumerate(chroms):
            f.write(b">chr%d synthetic\n" % (i + 1))
            n = len(a) // 60 * 60
            body = np.empty((n // 60, 61), dtype=np.uint8)
            body[:, :60] = a[:n].reshape(-1, 60)
            body[:, 60] = 10
            f.write(body.tobytes())
            if n < len(a):
                f.write(a[n:].tobytes() + b"\n")


def sim(chroms, n_per_chr, paired):
    """FASTA text of reads simulated from every chromosome (fragments never span chromosomes)."""
    lib = bench.sim_lib()
    outs1, outs2 = [], []
    first = 0
    for a in chroms:
        ref = a.tobytes()
        b1 = np.empty(n_per_chr * bench.RECSZ, np.uint8)
        b2 = np.empty(n_per_chr * bench.RECSZ, np.uint8) if paired else None
        lib.ht2_simreads(ref, len(ref), first, n_per_chr, 7, bench.RDLEN, 200, 400, 0.005, bench.DIGITS, b1.ctypes.data,
                         b2.ctypes.data if paired else None)
        outs1.append(b1)
        if paired:
            outs2.append(b2)
        first += n_per_chr
    return np.concatenate(outs1), (np.concatenate(outs2) if paired else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mbp", type=int, default=512)
    ap.add_argument("--out", default=None)
    ap.add_argument("--threads", type=int, default=min(64, os.cpu_count() or 1))
    args = ap.parse_args()
    os.makedirs(B, exist_ok=True)
    base = os.path.join(B, "synth%d" % args.mbp)
    res = {"what": "HBM-resident regime: %d Mbp synthetic reference (random 64-Mbp chromosomes, N gaps, 20 repeat families), "
                   "hisat2-build-s default parameters" % args.mbp, "gpu": bench.gpu_info(0)}
    t0 = time.time()
    chroms = make_reference(args.mbp)
    if not os.path.exists(base + ".1.ht2"):
        write_fasta(base + ".fa", chroms)
        res["generate_s"] = round(time.time() - t0, 1)
        t0 = time.time()
        subprocess.run([os.path.join(REFDIR, "hisat2-build-s"), "-q", "-p", str(args.threads), base + ".fa", base], check=True, stdout=subprocess.DEVNULL)
        res["hisat2_build_s"] = round(time.time() - t0, 1)
    t0 = time.time()
    idx = h2.Index(base)
    res["open_s"] = round(time.time() - t0, 1)
    res["image_MB"] = round(idx.image().nbytes / 1e6, 1)
    res["l2_MB"] = 50
    hdr = idx.sam_header()
    per = 200000 // len(chroms)
    # ---- parity against the reference on this box
    for paired in (False, True):
        d1, d2 = sim(chroms, per // (2 if paired else 1), paired)
        f1, f2 = os.path.join(B, "q_1.fa"), os.path.join(B, "q_2.fa")
        d1.tofile(f1)
        if paired:
            d2.tofile(f2)
        sam, st = idx.run_reads(data1=d1, data2=d2)
        out = os.path.join(B, "ref.sam")
        best = None
        for p in (8, 16, 32):
            t = time.time()
            subprocess.run([os.path.join(REFDIR, "hisat2-align-s"), "--no-spliced-alignment", "-f", "-x", base] +
                           (["-1", f1, "-2", f2] if paired else ["-U", f1]) + ["-S", out, "-p", str(p), "--reorder"], check=True, stderr=subprocess.DEVNULL)
            dt = time.time() - t
            if best is None or dt < best[0]:
                best = (dt, p)
        want = open(out, "rb").read()
        body = want[want.index(b"\n@PG"):].split(b"\n", 2)[2]
        res["pe_parity" if paired else "se_parity"] = {"reads": int(st["n_reads"]), "sam_identical_to_reference_on_the_same_box": bool(sam == body),
                                                        "capacity_error_reads": int(st["n_err_reads"]),
                                                        "reference_best": "%.2f s at -p %d (%.3f M reads/s incl. index load)" % (best[0], best[1], st["n_reads"] / best[0] / 1e6)}
        print(json.dumps(res["pe_parity" if paired else "se_parity"]), flush=True)
    # ---- throughput: alignment path and the LF-mapping kernel alone
    d1, _ = sim(chroms, 4000000 // len(chroms), False)
    idx.run_reads(data1=d1, collect=False)
    t = time.perf_counter()
    _, st = idx.run_reads(data1=d1, collect=False)
    dt = time.perf_counter() - t
    res["se_4M"] = {"reads": int(st["n_reads"]), "e2e_reads_per_s": st["n_reads"] / dt, "kernel_reads_per_s": st["n_reads"] / ((st["ms_align"] + st["ms_sam"]) / 1e3),
                    "ms_align": st["ms_align"], "note": "same pool kernel and pipeline as the bench; compare with the L2-resident 1 Mbp index"}
    k = 1000000
    sb = h2.ReadBatch.parse(data1=d1[:k * bench.RECSZ])
    best = None
    for _ in range(3):
        sr = idx.seed_search(sb, max_range=4)
        if best is None or sr.ms_kernel < best[0]:
            best = (sr.ms_kernel, sr.n_lf, sr.alg_bytes)
        sr.close()
    peak = 3350.0     # H100 SXM data-sheet HBM3 bandwidth, unless MEASURED_PEAKS.json says otherwise
    pk = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(pk):
        peak = float(json.load(open(pk)).get("hbm_gbs", peak))
    res["lf_map"] = {"kernel": "ht2_seed_kernel (count pass + fill pass)", "reads": k, "ms_two_passes": best[0], "lf_steps_counted_once": int(best[1]),
                     "lf_per_s_per_pass": 2 * best[1] / best[0] * 1e3, "achieved_GBps_per_pass": 2 * best[2] / best[0] / 1e6,
                     "peak_GBps": peak, "frac": 2 * best[2] / best[0] / 1e6 / peak,
                     "note": "algorithmic bytes (sides touched x 32 B + ftab + SA samples) of one pass over half the two-pass time"}
    print(json.dumps(res, indent=1))
    if args.out:
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
