#!/usr/bin/env python3
"""bench.py -- reads/s of the HISAT2 alignment path on H100, FASTA in -> SAM out.

  python bench.py --gpus N --steps K --warmup W            our CUDA path
  python bench.py --impl reference --gpus N --steps K ...  reference CPU path (unmodified hisat2-align-s)
  python bench.py ... --dump-outputs DIR                   also write a sample of the last timed step's SAM as .npy
  python bench.py ... --index oracle/_ref/data/22_20-21M   the same workload shape on another linear index

Workload (config.workload): the shape of BASELINE.json configs[2] on an index that ships with the repository --
the linear tests/golden/tiny index (80 kbp cut from the 22_20-21M example region, chrA carrying a mutated
duplicate), a FIXED set of 10 M synthetic 2x101-bp pairs drawn from its chrA (seeded generator,
tools/simreads_fast.c), --no-spliced-alignment -- sharded over the N ranks by contiguous pair ranges (strong
scaling).  One "step" = one pass of the whole path over the rank's shard, in device batches of 4 M reads.
--index runs the same shape on another linear index: the reads come from the first record of <index>.fa, the graph
extra from <index>_snp (e.g. the 22_20-21M example index that oracle/make_data.sh stages next to the reference).
  e2e   : FASTA bytes in host memory -> SAM bytes in host memory through ht2gpu_run_reads (multi-threaded
          parser, H2D, alignment kernel, SAM kernels, D2H), host wall clock, max over ranks.  THE headline.
  value : the same job counted on the device only: reads / sum of the CUDA-event times of the alignment and
          SAM kernels of every batch (inputs resident in HBM when each timed interval starts).
The only collective is the start-up NCCL broadcast of the index image; every rank keeps its SAM text in host
memory in read order, so the job's output is the rank-order concatenation (= --reorder).
"""
import argparse
import ctypes
import json
import mmap
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

INDEX = os.path.join(ROOT, "tests", "golden", "tiny")
FASTA = INDEX + ".fa"
REFBIN = os.path.join(ROOT, "oracle", "_ref", "hisat2-align-s")
RDLEN = 101
DIGITS = 8
RECSZ = 2 + DIGITS + 1 + RDLEN + 1
WORKLOAD = ("%s linear index, fixed set of %d synthetic 2x101bp pairs from its first sequence (seed 1, --fr, -I 0 -X 1000), "
            "--no-spliced-alignment -k 5, sharded over the ranks by contiguous pair ranges")
L2_NOTE = ("inputs larger than L2: every step streams the whole read set (110 B of FASTA per read in, ~360 B of SAM per read out) through "
           "the device; the index image is L2-resident; no flush between steps")
SAM_SAMPLE_BYTES = 1 << 21     # --dump-outputs: the first 2 MB of SAM text of every batch of the last timed step ...
SAM_SAMPLE_TOTAL = 1 << 24     # ... until 16 MB are taken (about 45 k records, 7 MB of .npy)


def workload_config(pairs):
    """The `config` object, identical for both arms."""
    return {"workload": WORKLOAD % (os.path.relpath(INDEX, ROOT), pairs), "read_len": RDLEN, "pairs_total": pairs, "l2": L2_NOTE}


def huge_buffer(nbytes):
    """Anonymous mapping with transparent huge pages: first-touch of GBs of 4 KiB pages costs tens of seconds in this sandbox."""
    m = mmap.mmap(-1, max(nbytes, 1))
    try:
        m.madvise(mmap.MADV_HUGEPAGE)
    except Exception:
        pass
    return np.frombuffer(m, dtype=np.uint8, count=nbytes)


_sim = None


def sim_lib():
    global _sim
    if _sim is None:
        so = os.path.join(ROOT, "tools", "libsimreads.so")
        src = os.path.join(ROOT, "tools", "simreads_fast.c")
        if not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
            subprocess.run(["gcc", "-O2", "-shared", "-fPIC", "-o", so, src], check=True)
        _sim = ctypes.CDLL(so)
        _sim.ht2_simreads.restype = ctypes.c_uint64
        _sim.ht2_simreads.argtypes = [ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_int,
                                      ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    return _sim


_ref = None


def ref_seq():
    """Upper-case bases of the first record of FASTA: fragments never span two records."""
    global _ref
    if _ref is None:
        _ref = open(FASTA, "rb").read().split(b">")[1].split(b"\n", 1)[1].replace(b"\n", b"").upper()
    return _ref


def sim_fasta(first, n, seed=1, paired=True):
    """FASTA text (uint8 arrays) of fragments [first, first+n) of the synthetic read set: mate-1 file, mate-2 file."""
    ref = ref_seq()
    a = huge_buffer(n * RECSZ)
    b = huge_buffer(n * RECSZ) if paired else None
    sim_lib().ht2_simreads(ref, len(ref), first, n, seed, RDLEN, 200, 400, 0.005, DIGITS, a.ctypes.data, b.ctypes.data if paired else None)
    return a, b


class ClockSampler(object):
    def __init__(self, dev):
        self.dev = dev
        self.rows = []
        self._stop = threading.Event()
        self._t = None

    def start(self):
        def run():
            q = "clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
                "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"
            while not self._stop.is_set():
                try:
                    out = subprocess.run(["nvidia-smi", "-i", str(self.dev), "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=5).stdout.decode().strip()
                    if out:
                        self.rows.append([x.strip() for x in out.split(",")])
                except Exception:
                    pass
                self._stop.wait(0.2)
        self._t = threading.Thread(target=run, daemon=True)
        self._t.start()

    def stop(self):
        self._stop.set()
        if self._t:
            self._t.join(timeout=6)
        if not self.rows:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": []}
        sm = sorted(int(r[0]) for r in self.rows if r[0].isdigit())
        mx = max(int(r[1]) for r in self.rows if r[1].isdigit())
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [names[i] for i in range(4) if any(r[2 + i].lower().startswith("active") for r in self.rows)]
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx, "reasons": reasons}


# ---------------------------------------------------------------------------------------------------------
# reference (CPU) side
# ---------------------------------------------------------------------------------------------------------
def run_reference(f1, f2, threads, extra=()):
    """Time the unmodified reference binary (wall clock: index load + parse + align + SAM to /dev/null)."""
    cmd = [REFBIN, "--no-spliced-alignment", "-f", "-x", INDEX] + (["-1", f1, "-2", f2] if f2 else ["-U", f1]) + \
          ["-S", "/dev/null", "-p", str(threads), "--reorder"] + list(extra)
    t0 = time.time()
    subprocess.run(cmd, check=True, stderr=subprocess.DEVNULL, stdout=subprocess.DEVNULL)
    return time.time() - t0


def reference_sample(n_pairs, tag):
    a, b = sim_fasta(0, n_pairs)
    d = "/dev/shm" if os.path.isdir("/dev/shm") else "/tmp"
    f1, f2 = os.path.join(d, "ht2_bench_%s_%d_1.fa" % (tag, os.getpid())), os.path.join(d, "ht2_bench_%s_%d_2.fa" % (tag, os.getpid()))
    a.tofile(f1); b.tofile(f2)
    return f1, f2


def thread_table(f1, f2, n_reads):
    """reads/s of the reference at every -p candidate, measured on the FULL sample (not a probe)."""
    ncpu = os.cpu_count() or 1
    cands = sorted(set(c for c in (8, 16, 32, 64, 128, ncpu) if c <= ncpu))
    table = {}
    for c in cands:
        table[c] = n_reads / run_reference(f1, f2, c)
    best = max(table, key=lambda c: table[c])
    return best, {str(c): round(v, 1) for c, v in table.items()}


def reference_arm(args, rank):
    if rank != 0:
        return
    if not (os.path.exists(REFBIN) and os.path.exists(INDEX + ".1.ht2")):
        print(json.dumps({"impl": "reference", "unavailable": "oracle/_ref/hisat2-align-s not built"}))
        return
    npairs = args.ref_sample_pairs
    f1, f2 = reference_sample(npairs, "ref")
    nreads = 2 * npairs
    threads, table = thread_table(f1, f2, nreads)
    for _ in range(min(args.warmup, 2)):
        run_reference(f1, f2, threads)
    times = [run_reference(f1, f2, threads) for _ in range(args.steps)]
    os.remove(f1); os.remove(f2)
    tot = sum(times)
    v = nreads * args.steps / tot
    line = {"impl": "reference", "metric": "reads_per_sec_aligned", "value": v, "unit": "reads/s", "n_gpus": args.gpus, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": 1000.0 * tot / args.steps, "higher_is_better": True, "scaling": "strong",
            "vs_baseline": None, "dtype": "u8/u32", "data": "synthetic",
            "config": workload_config(args.pairs),
            "cpu_baseline": {"value": v, "unit": "reads/s", "cores": threads, "kind": "reference",
                             "sample": "first %d pairs (%d reads) of the workload per step, hisat2-align-s -p %d --reorder (fastest of the -p table, "
                                       "measured on this full sample), wall clock incl. index load, FASTA parsing and SAM to /dev/null" % (npairs, nreads, threads),
                             "threads_table_reads_per_s": table, "host_cores": os.cpu_count()},
            "e2e": {"value": v, "unit": "reads/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "gpu_launches": 0}
    print(json.dumps(line))


# ---------------------------------------------------------------------------------------------------------
# our side
# ---------------------------------------------------------------------------------------------------------
def run_steps(idx, d1, d2, steps, batch_reads, threads, last_sink=None):
    """K passes over the shard; returns (wall seconds, summed stats).  `last_sink` sees the SAM text of the last pass."""
    acc = {}
    t0 = time.perf_counter()
    for i in range(steps):
        _, st = idx.run_reads(data1=d1, data2=d2, collect=False, batch_reads=batch_reads, threads=threads,
                              sink=last_sink if i == steps - 1 else None)
        for k, v in st.items():
            acc[k] = acc.get(k, 0) + v
    return time.perf_counter() - t0, acc


class SamSample(object):
    """SAM sink of the last timed step: keeps the first SAM_SAMPLE_BYTES of every batch, cut back to whole records, until
    SAM_SAMPLE_TOTAL bytes are taken (a fixed sample: the same arguments give the same batches), and counts the bytes of
    the whole step.  It runs inside the timed region: one copy of at most 2 MB per batch."""
    def __init__(self):
        self.parts = []
        self.taken = 0
        self.batches = 0
        self.total_bytes = 0

    def __call__(self, ptr, n):
        take = min(n, SAM_SAMPLE_BYTES, SAM_SAMPLE_TOTAL - self.taken)
        if take > 0:
            b = ctypes.string_at(ptr, take)
            self.parts.append(b[:b.rfind(b"\n") + 1])
            self.taken += take
        self.batches += 1
        self.total_bytes += n


def dump_outputs(out_dir, sample, ref_names):
    """The sampled SAM records as float64 columns, one .npy per SAM field, plus a CRC-32 of every whole record.
    Records without an AS:i / NM:i tag (unaligned reads) have 0 there and 0 in has_as / has_nm."""
    import zlib
    rid = {n.encode(): i for i, n in enumerate(ref_names)}
    cols = {k: [] for k in ("read_id", "flag", "ref_id", "pos", "mapq", "rnext_id", "pnext", "tlen", "as_score", "has_as", "nm", "has_nm",
                            "record_crc32")}
    for part in sample.parts:
        for rec in part.splitlines():
            f = rec.split(b"\t")
            tags = dict((t[:2], t[5:]) for t in f[11:] if t[2:5] == b":i:")
            ref = rid.get(f[2], -1)
            for k, v in (("read_id", int(f[0][1:])), ("flag", int(f[1])), ("ref_id", ref), ("pos", int(f[3])), ("mapq", int(f[4])),
                         ("rnext_id", ref if f[6] == b"=" else rid.get(f[6], -1)), ("pnext", int(f[7])), ("tlen", int(f[8])),
                         ("as_score", int(tags.get(b"AS", 0))), ("has_as", int(b"AS" in tags)),
                         ("nm", int(tags.get(b"NM", 0))), ("has_nm", int(b"NM" in tags)),
                         ("record_crc32", zlib.crc32(rec))):
                cols[k].append(v)
    os.makedirs(out_dir, exist_ok=True)
    for k, v in cols.items():
        np.save(os.path.join(out_dir, k + ".npy"), np.asarray(v, dtype=np.float64))
    np.save(os.path.join(out_dir, "step_sam_bytes.npy"), np.asarray([sample.total_bytes, sample.batches], dtype=np.float64))
    return len(cols["flag"])


def gpu_info(dev):
    """Name and power limit of the device the numbers were measured on."""
    import torch
    info = {"name": torch.cuda.get_device_name(dev), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(dev), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=10).stdout.decode().strip()
        info["power_limit_w"] = float(out)
    except Exception:
        pass
    return info


def extra_line(h2, base, d1, d2, n_reads, threads, **opts):
    """Informational: another index / option set on a slice of the same reads (not part of value / e2e)."""
    idx = h2.Index(base, **opts)
    idx.run_reads(data1=d1, data2=d2, collect=False, threads=threads)
    t0 = time.perf_counter()
    _, st = idx.run_reads(data1=d1, data2=d2, collect=False, threads=threads)
    dt = time.perf_counter() - t0
    idx.close()
    return {"reads": n_reads, "e2e_reads_per_s": n_reads / dt, "kernel_reads_per_s": n_reads / ((st["ms_align"] + st["ms_sam"]) / 1e3),
            "ms_align": st["ms_align"], "ms_sam": st["ms_sam"], "capacity_error_reads": st["n_err_reads"]}


def extra_rna_line(h2, base, threads):
    """Informational: spliced alignment with a device-resident splice-site DB (--known-splicesite-infile semantics) on
    RNA-like pairs: tools/sim_rna.py transcripts over the index's own sequence, 25 k distinct pairs x 8 copies."""
    import tempfile
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import sim_rna
    refs = sim_rna.load_fasta(base + ".fa")
    _, pairs, lines = sim_rna.sim(refs, 0, 25000, 7)
    reps = 8
    b1 = "".join(">r%dp%d/1\n%s\n" % (r, i, a) for r in range(reps) for i, (a, _) in enumerate(pairs)).encode()
    b2 = "".join(">r%dp%d/2\n%s\n" % (r, i, b) for r in range(reps) for i, (_, b) in enumerate(pairs)).encode()
    n_reads = 2 * reps * len(pairs)
    with tempfile.NamedTemporaryFile("w", suffix="_ss.txt", delete=False) as f:
        f.write("\n".join(lines) + "\n")
        ssf = f.name
    try:
        idx = h2.Index(base, no_spliced_alignment=0)
        nsites = idx.load_splicesites(ssf)
        idx.run_reads(data1=b1, data2=b2, collect=False, threads=threads)
        t0 = time.perf_counter()
        _, st = idx.run_reads(data1=b1, data2=b2, collect=False, threads=threads)
        dt = time.perf_counter() - t0
        idx.close()
    finally:
        os.remove(ssf)
    return {"reads": n_reads, "listed_splice_sites": nsites, "e2e_reads_per_s": n_reads / dt,
            "kernel_reads_per_s": n_reads / ((st["ms_align"] + st["ms_sam"]) / 1e3), "ms_align": st["ms_align"], "ms_sam": st["ms_sam"],
            "capacity_error_reads": st["n_err_reads"]}


def main():
    global INDEX, FASTA
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours")
    ap.add_argument("--index", default=INDEX, help="linear index (prefix of <index>.N.ht2 and <index>.fa); default: tests/golden/tiny")
    ap.add_argument("--pairs", type=int, default=10000000, help="pairs of the whole job (fixed as N grows)")
    ap.add_argument("--batch-reads", type=int, default=4000000, help="reads per device batch")
    ap.add_argument("--ref-sample-pairs", type=int, default=500000, help="pairs per step of the CPU reference (bounded sample)")
    ap.add_argument("--threads", type=int, default=0, help="host parser threads per rank (0 = cores / local ranks, at most 64)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-extras", action="store_true")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="after the timed steps, write a fixed sample of the last step's SAM records (rank 0) as DIR/<field>.npy")
    args = ap.parse_args()
    INDEX, FASTA = os.path.abspath(args.index), os.path.abspath(args.index) + ".fa"
    for f in (INDEX + ".1.ht2", FASTA):
        if not os.path.exists(f):
            raise SystemExit("bench.py: %s not found (--index %s)" % (f, args.index))
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if args.impl == "reference":
        reference_arm(args, rank)
        return 0

    import torch
    import hisat2_b200 as h2
    from hisat2_b200.parallel import broadcast_image, shard_range
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device; the alignment path has no CPU fallback")
    torch.cuda.set_device(local)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    # ---- index: parse on rank 0, NCCL-broadcast the packed image, adopt in place
    if world > 1:
        img = h2.Index.build_image(INDEX) if rank == 0 else None
        dev_img = broadcast_image(img, rank, device=torch.device("cuda", local))
        torch.cuda.synchronize()
        prefix = dev_img[:4096].cpu().numpy()
        idx = h2.Index(device_image=(dev_img.data_ptr(), dev_img.numel(), prefix), device=local)
    else:
        idx = h2.Index(INDEX, device=local)
    threads = args.threads or max(1, min(64, (os.cpu_count() or 1) // max(1, world)))
    # ---- this rank's shard of the fixed read set, as FASTA text in host memory
    lo, hi = shard_range(args.pairs, rank, world)
    d1, d2 = sim_fasta(lo, hi - lo)
    n_reads = 2 * (hi - lo)

    def barrier():
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()

    # ---- warm-up (also grows every pinned / device buffer to its final size)
    warm = max(args.warmup, 3)
    run_steps(idx, d1, d2, warm, args.batch_reads, threads)
    # ---- timed region: K steps, FASTA bytes in host memory -> SAM bytes in host memory
    sampler = ClockSampler(local)
    sam_sample = SamSample() if args.dump_outputs and rank == 0 else None
    barrier()
    sampler.start()
    wall, acc = run_steps(idx, d1, d2, args.steps, args.batch_reads, threads, last_sink=sam_sample)
    torch.cuda.synchronize()
    clocks = sampler.stop()
    barrier()
    kernel_ms = acc["ms_align"] + acc["ms_sam"]
    # ---- roofline inputs: algorithmic bytes / LF steps per read of the alignment kernel, counted in-kernel, from one
    #      structured-result batch of this shard (the same reads a pipeline batch holds)
    k = min(hi - lo, args.batch_reads // 2)
    sub = h2.ReadBatch.parse(data1=d1[:k * RECSZ], data2=d2[:k * RECSZ], threads=threads)
    res = idx.align(sub, resident_iters=2)
    alg_per_read = float(res.reads["alg_bytes"].astype(np.int64).sum()) / sub.n
    lf_per_read = float(res.reads["n_lf"].astype(np.int64).sum()) / sub.n
    aligned = float((res.reads["n_aln"].sum(axis=1) > 0).sum()) / len(res.reads)
    align_ms_batch = res.ms_kernel / 2
    res.close()
    # ---- informational: the LF-mapping kernel alone (seed search) on 200k reads
    lf_map = None
    if rank == 0:
        kk = min(100000, hi - lo)
        sb = h2.ReadBatch.parse(data1=d1[:kk * RECSZ], data2=d2[:kk * RECSZ], threads=threads)
        sb.paired = False
        best = None
        for _ in range(3):
            sr = idx.seed_search(sb, max_range=4)
            if best is None or sr.ms_kernel < best[0]:
                best = (sr.ms_kernel, sr.n_lf, sr.alg_bytes)
            sr.close()
        lf_map = {"kernel": "ht2_seed_kernel (count pass + fill pass)", "reads": sb.n, "ms": best[0], "lf_steps": int(best[1]),
                  "lf_per_s": best[1] / best[0] * 1e3, "achieved": best[2] / best[0] / 1e6, "unit": "GB/s",
                  "note": "algorithmic bytes of ONE pass over the time of BOTH passes; index is L2-resident; not part of value/e2e"}
    tk = torch.tensor([kernel_ms, wall * 1000.0, acc["ms_align"]], dtype=torch.float64, device="cuda")
    tot = torch.tensor([float(n_reads), float(acc["n_launches"]), float(acc["n_err_reads"]), float(acc["h2d_bytes"]), float(acc["d2h_bytes"]),
                        float(acc["sam_bytes"]), float(acc["n_batches"])], dtype=torch.float64, device="cuda")
    if dist is not None:
        dist.all_reduce(tk, op=dist.ReduceOp.MAX)
        dist.all_reduce(tot, op=dist.ReduceOp.SUM)
    kernel_ms, e2e_ms, align_ms = float(tk[0]), float(tk[1]), float(tk[2])
    dumped = dump_outputs(args.dump_outputs, sam_sample, idx.ref_names()) if sam_sample is not None else None
    idx.close()
    if rank != 0:
        if dist is not None:
            dist.destroy_process_group()
        return 0
    total_reads = float(tot[0])
    value = total_reads * args.steps / (kernel_ms / 1000.0)
    e2e_v = total_reads * args.steps / (e2e_ms / 1000.0)
    peaks = {}
    pk_path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(pk_path):
        peaks = json.load(open(pk_path))
    peak = float(peaks.get("hbm_gbs", 3350.0))
    peak_kind = "measured sustained copy bandwidth (MEASURED_PEAKS.json hbm_gbs)" if "hbm_gbs" in peaks else "H100 SXM data-sheet HBM3 bandwidth"
    # dominant kernel = the alignment kernel; one launch = one device batch
    per_launch_bytes = alg_per_read * sub.n
    achieved = per_launch_bytes / (align_ms_batch / 1e3) / 1e9
    traffic, traffic_note = None, "no ncu capture of the current kernel in profiles/traffic.json"
    tpath = os.path.join(ROOT, "profiles", "traffic.json")
    if os.path.exists(tpath):
        try:
            tj = json.load(open(tpath))
            from hisat2_b200.build import source_hash
            if tj.get("source_hash") == source_hash():
                traffic = tj.get("dram_bytes_per_launch")
                traffic_note = tj.get("note")
            else:
                traffic_note = "profiles/traffic.json was captured for other kernel sources (hash %s); not reported" % tj.get("source_hash")
        except Exception:
            pass
    line = {
        "metric": "reads_per_sec_aligned", "value": value, "unit": "reads/s", "n_gpus": world, "steps": args.steps,
        "warmup": warm, "ms_per_step": kernel_ms / args.steps, "higher_is_better": True, "scaling": "strong",
        "vs_baseline": None, "dtype": "u8/u32", "data": "synthetic",
        "config": workload_config(args.pairs),
        "run": {"reads_per_step_all_ranks": int(total_reads), "device_batch_reads": args.batch_reads, "host_parser_threads_per_rank": threads,
                "parallelism": "contiguous pair ranges x%d, index replicated (NCCL broadcast at load), no data-path collective; "
                               "SAM stays in rank order in host memory" % world,
                "sam_MB_per_step_per_rank": float(tot[5]) / world / args.steps / 1e6,
                "aligned_fraction": aligned, "lf_steps_per_read": lf_per_read, "capacity_error_reads": int(tot[2])},
        "e2e": {"value": e2e_v, "unit": "reads/s", "h2d_bytes_per_step": int(tot[3] / args.steps), "d2h_bytes_per_step": int(tot[4] / args.steps),
                "ms_per_step": e2e_ms / args.steps, "sam_bytes_per_step": int(tot[5] / args.steps),
                "what": "ht2gpu_run_reads: FASTA text in host memory -> SAM text in (pinned) host memory; record indexing, multi-threaded parsing, "
                        "H2D, alignment kernel, SAM kernels and D2H all inside the timed region (host wall clock, max over ranks)"},
        "kernels_ms_per_step": {"align": align_ms / args.steps, "align_plus_sam": kernel_ms / args.steps},
        "host_s_per_step_rank0": {k: acc[k] / args.steps for k in ("s_index", "s_parse", "s_submit", "s_wait", "s_sink", "s_total")},
        "lf_map": lf_map,
        "gpu_launches": int(tot[1]),
        "clocks": clocks,
        "gpu": gpu_info(local),
        "roofline": {"bound": "hbm", "kernel": "ht2_align_pool_kernel<8,4,false>", "achieved": achieved, "peak": peak, "unit": "GB/s",
                     "frac": achieved / peak, "traffic": traffic, "traffic_note": traffic_note, "peak_source": peak_kind,
                     "algorithmic_bytes_per_read": alg_per_read, "reads_per_launch": sub.n, "launch_ms": align_ms_batch,
                     "note": "algorithmic bytes = sides touched x 32 B (rank sides) + ftab/SA-sample entries + 2-bit reference bytes, counted in-kernel; "
                             "launch time = CUDA events around back-to-back launches on the launch stream"},
    }
    if dumped is not None:
        line["dump_outputs"] = {"dir": args.dump_outputs, "sam_records": dumped,
                                "note": "the last timed step ran a Python SAM sink that copies at most 2 MB per batch (16 MB in all) "
                                        "inside the timed region; a run without --dump-outputs uses no sink"}
    if dist is not None:
        dist.destroy_process_group()
    if world == 1 and not args.no_extras:
        ex = {}
        ke = min(hi - lo, 250000)
        s1, s2 = d1[:ke * RECSZ], d2[:ke * RECSZ]
        try:
            ex["configs1_SE_1M_reads"] = extra_line(h2, INDEX, d1[:min(hi - lo, 1000000) * RECSZ], None, min(hi - lo, 1000000), threads)
            ex["graph_index_%s_snp_PE" % os.path.basename(INDEX)] = extra_line(h2, INDEX + "_snp", s1, s2, 2 * ke, threads)
            ex["sensitive_PE (bowtie2_dp 1, score-min L,0,-0.5)"] = extra_line(h2, INDEX, s1, s2, 2 * ke, threads, bowtie2_dp=1, score_min_type=ord("L"),
                                                                              score_min_const=0.0, score_min_coeff=-0.5)
            ex["very_sensitive_PE (bowtie2_dp 2, -k 30, score-min L,0,-1)"] = extra_line(h2, INDEX, s1, s2, 2 * ke, threads, bowtie2_dp=2, khits=30,
                                                                                       score_min_type=ord("L"), score_min_const=0.0, score_min_coeff=-1.0)
            ex["spliced_no_temp_splicesite_PE"] = extra_line(h2, INDEX, s1, s2, 2 * ke, threads, no_spliced_alignment=0)
            ex["spliced_known_splicesites_RNA_like_PE"] = extra_rna_line(h2, INDEX, threads)
        except Exception as e:  # informational only
            ex["error"] = repr(e)
        line["extra"] = ex
    # ---- CPU baseline (rank 0, N=1 only): the unmodified reference on a bounded sample of the same read set
    if world == 1 and not args.no_cpu_baseline and os.path.exists(REFBIN):
        npairs = min(args.ref_sample_pairs, hi - lo)
        f1, f2 = reference_sample(npairs, "cpu")
        threads_ref, table = thread_table(f1, f2, 2 * npairs)
        os.remove(f1); os.remove(f2)
        line["cpu_baseline"] = {"value": float(table[str(threads_ref)]), "unit": "reads/s", "cores": threads_ref, "kind": "reference",
                                "sample": "first %d pairs (%d reads) of the workload, hisat2-align-s -p %d --reorder (fastest of the -p table measured on "
                                          "this full sample), wall clock incl. index load, FASTA parsing and SAM to /dev/null" % (npairs, 2 * npairs, threads_ref),
                                "threads_table_reads_per_s": table, "host_cores": os.cpu_count()}
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    sys.exit(main())
