"""The host read pipeline (ht2_pipeline.cpp: batch planning over read-file lists, gzip inflate, read files, errors) on
the CPU, against the fake device of tests/hostsim/ht2_pipesim.cpp, built plain, under AddressSanitizer +
UndefinedBehaviorSanitizer and under ThreadSanitizer.

The fake formats every batch from the pipeline's staging when the batch is waited for, one line per read (name,
sequence, qualities, seed), and gives each unit the outcome FNV-1a(name of its first read) & 7.  The expected text of a
run comes from the host-only calls of the same library: ht2gpu_parse_reads on each stream's files back to back (the
plain text of tools/multi_input_ref.py's corpus) and ht2gpu_route_reads of that text by the same outcomes.  A stream
with a unit at ordinal skip + upto ends the run, so the unpaired reads are read only when the pairs ran out first."""
import gzip
import os
import subprocess
import sys

import pytest

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tools"))
import multi_input_ref as mref  # noqa: E402

CASES = sorted(mref.CASES)
SRCS = [os.path.join(ROOT, "tests", "hostsim", "ht2_pipesim.cpp"),
        os.path.join(ROOT, "hisat2_b200", "csrc", "ht2_pipeline.cpp"), os.path.join(ROOT, "hisat2_b200", "csrc", "ht2_reads.cpp")]
VARIANTS = {"plain": ["-O2"],
            "asan": ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all"],
            "tsan": ["-O1", "-g", "-fsanitize=thread"]}
SAN_ENV = dict(os.environ, TSAN_OPTIONS="halt_on_error=1 exitcode=66", ASAN_OPTIONS="detect_leaks=1")
# (--batch, --slots, --gpus, -p): every value of each against the others on the plain build, a cover under sanitizers
CONFIGS = [(b, s, g, p) for b in (0, 7, 64) for s in (1, 4) for g in (1, 2) for p in (1, 8)]
SAN_CONFIGS = [(0, 1, 1, 1), (7, 4, 2, 8), (64, 1, 2, 8), (64, 4, 1, 1)]
OUTS = [("--un", "un"), ("--al", "al"), ("--un-conc", "un_conc.%"), ("--al-conc", "al_conc.%"), ("--al-conc-disc", "al_conc_disc.%")]
FILES = ["un", "al"] + [o + "." + m for o in ("un_conc", "al_conc", "al_conc_disc") for m in "12"]


@pytest.fixture(scope="module")
def pipesim(tmp_path_factory):
    d = tmp_path_factory.mktemp("pipesim")
    out = {}
    for v, flags in VARIANTS.items():
        out[v] = str(d / ("ht2_pipesim_" + v))
        subprocess.run(["g++", "-std=c++14", "-pthread"] + flags + ["-o", out[v]] + SRCS, check=True)
    return out


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    return mref.generate(str(tmp_path_factory.mktemp("pipe_corpus")))


def fnv1a(name):
    h = 2166136261
    for c in name:
        h = ((h ^ c) * 16777619) & 0xFFFFFFFF
    return h


def run(exe, args, cwd):
    r = subprocess.run([exe] + args, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=SAN_ENV, timeout=120)   # a hang fails
    assert b"Sanitizer" not in r.stderr and b"runtime error" not in r.stderr, r.stderr.decode()[-4000:]
    return r


def read_files(d):
    return {k: open(os.path.join(d, k), "rb").read() for k in FILES}


def out_args(d):
    return [a for o, n in OUTS for a in (o, os.path.join(d, n))]


def front(case):
    f = mref.CASES[case].get("front", {})
    return f.get("skip", 0), f.get("upto", 0)


def fmt(case):
    return mref.CASES[case]["fmt"]


def list_args(d, case):
    c = mref.CASES[case]
    p = lambda fs: ",".join(os.path.join(d, f[0]) for f in fs)
    return (["-1", p(c["m1"]), "-2", p(c["m2"])] if c["m1"] else []) + (["-U", p(c["u"])] if c["u"] else [])


def expect_stream(exe, d, tmp, case, names, paired):
    """(reads text, read files) of ht2gpu_parse_reads / ht2gpu_route_reads on the plain text of a stream's files."""
    skip, upto = front(case)
    paths = []
    for k, fs in enumerate(names):
        paths.append(os.path.join(tmp, "stream_%d_%d" % (paired, k)))
        with open(paths[-1], "wb") as o:
            for f in fs:
                o.write(open(os.path.join(d, "plain", f[0]), "rb").read())
    inp = ["-1", paths[0], "-2", paths[1]] if paired else ["-U", paths[0]]
    opts = [fmt(case), "-s", str(skip), "-u", str(upto)]
    text = os.path.join(tmp, "parsed_%d" % paired)
    subprocess.run([exe, "--parse"] + inp + opts + ["-S", text], check=True)
    reads = open(text, "rb").read()
    lines = reads.splitlines()[::2 if paired else 1]
    oc = os.path.join(tmp, "outcomes_%d" % paired)
    open(oc, "wb").write(bytes(fnv1a(l.split(b"\t")[0]) & 7 for l in lines))
    rd = os.path.join(tmp, "routed_%d" % paired)
    os.makedirs(rd)
    subprocess.run([exe, "--route"] + inp + opts + ["--outcomes", oc] + out_args(rd), check=True)
    return reads, read_files(rd), paths


_EXPECTED = {}


def expected(pipesim, d, tmp_path_factory, case):
    """Per case: reads text, read files, units per stream [(paired, units)], and the stream files back to back."""
    if case not in _EXPECTED:
        c = mref.CASES[case]
        tmp = str(tmp_path_factory.mktemp("expect_" + case))
        skip, upto = front(case)
        reads, files, streams, concat = b"", {k: b"" for k in FILES}, [], {}
        if c["m1"]:
            r, f, concat[1] = expect_stream(pipesim["plain"], d, tmp, case, [c["m1"], c["m2"]], True)
            reads += r
            files = {k: files[k] + f[k] for k in FILES}
            streams.append((1, r.count(b"\n") // 2))
        n_pairs = sum(f[3] - f[2] for f in c["m1"])
        if c["u"]:
            r, f, concat[0] = expect_stream(pipesim["plain"], d, tmp, case, [c["u"]], False)
            if not c["m1"] or not upto or n_pairs <= skip + upto:
                reads += r
                files = {k: files[k] + f[k] for k in FILES}
                streams.append((0, r.count(b"\n")))
        _EXPECTED[case] = reads, files, streams, concat
    return _EXPECTED[case]


def check_log(log, streams, cfg, first_plain):
    """Batches in order: no batch mixes pairs and unpaired reads, batch i on device i % gpus and slot (i / gpus) % slots,
    every unit once, and a first batch a quarter of a full one."""
    batch, slots, gpus, _ = cfg
    rows = [tuple(int(x) for x in l.split()) for l in log.splitlines()]
    for i, (dev, slot, _, _) in enumerate(rows):
        assert (dev, slot) == (i % gpus, (i // gpus) % slots), (i, rows[:i + 1])
    flags = [r[2] for r in rows]
    assert flags == sorted(flags, reverse=True)
    for paired, units in streams:
        assert sum(r[3] for r in rows if r[2] == paired) == units * (2 if paired else 1)
    if streams:
        paired, units = streams[0]
        per = ((batch or 4000000) + 1) // 2 if paired else batch or 4000000   # --batch counts reads
        quarter = per // 4 if per >= 8 else per
        first = rows[0][3] // (2 if paired else 1)
        assert first <= quarter
        if first_plain:
            assert first == min(quarter, units)


def first_files_plain(case):
    c = mref.CASES[case]
    fs = [c["m1"][0], c["m2"][0]] if c["m1"] else [c["u"][0]]
    return all(f[4] is None for f in fs)


def run_case(exe, d, tmp, case, cfg, extra=(), inputs=None):
    batch, slots, gpus, p = cfg
    skip, upto = front(case)
    os.makedirs(tmp, exist_ok=True)
    sam, log = os.path.join(tmp, "out.txt"), os.path.join(tmp, "log.txt")
    args = (inputs or list_args(d, case)) + [fmt(case), "-s", str(skip), "-u", str(upto), "--batch", str(batch),
                                             "--slots", str(slots), "--gpus", str(gpus), "-p", str(p), "-S", sam, "--log", log]
    r = run(exe, args + out_args(tmp) + list(extra), d)
    return r, open(sam, "rb").read(), open(log).read(), read_files(tmp)


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("case", CASES)
def test_lists_match_parse_and_route(pipesim, corpus, tmp_path_factory, tmp_path, variant, case):
    """ht2gpu_run_reads_files over every batch size, slot count, device count and thread count gives the reads and
    read files of the host-only calls."""
    reads, files, streams, _ = expected(pipesim, corpus, tmp_path_factory, case)
    gz = [f for k in ("m1", "m2", "u") for f in mref.CASES[case][k] if f[4]]
    cfgs = CONFIGS if variant == "plain" else SAN_CONFIGS
    for j, cfg in enumerate(cfgs):
        extra = [] if variant == "plain" else ["--sleep", str(j)]
        r, sam, log, got = run_case(pipesim[variant], corpus, str(tmp_path / str(j)), case, cfg, extra)
        assert r.returncode == 0, (cfg, r.stderr.decode()[-2000:])
        assert sam == reads, cfg
        assert got == files, cfg
        check_log(log, streams, cfg, first_files_plain(case))
        st = dict(kv.split(b"=") for kv in r.stdout.split())
        assert int(st[b"n_batches"]) == len(log.splitlines()) and int(st[b"n_reads"]) == reads.count(b"\n")
        if not front(case)[1]:   # every gzip file was read: its inflate is in the run's stats
            assert int(st[b"gz_out_bytes"]) == sum(os.path.getsize(os.path.join(corpus, "plain", f[0])) for f in gz)
            assert int(st[b"gz_in_bytes"]) == sum(os.path.getsize(os.path.join(corpus, f[0])) for f in gz)


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_single_input_entry_point(pipesim, corpus, tmp_path_factory, tmp_path, variant):
    """ht2gpu_run_reads_routed on one stream (a plain -1 file with a gzip -2 file, or one -U file) gives what
    ht2gpu_run_reads_files gives on the same reads."""
    for case in ("mixed_skip30_upto200", "se_fq_plain_gz_bgzf", "graph_alt_lanes"):
        reads, files, streams, concat = expected(pipesim, corpus, tmp_path_factory, case)
        paired = 1 if 1 in concat else 0
        paths = list(concat[paired])
        if paired:
            paths[1] += ".gz"
            open(paths[1], "wb").write(gzip.compress(open(concat[1][1], "rb").read(), 6, mtime=0))
        inputs = ["--routed"] + (["-1", paths[0], "-2", paths[1]] if paired else ["-U", paths[0]])
        n = streams[0][1] * (2 if paired else 1)
        for j, cfg in enumerate(CONFIGS[::5] if variant == "plain" else SAN_CONFIGS[1:3]):
            r, sam, log, got = run_case(pipesim[variant], corpus, str(tmp_path / ("%s_%d" % (case, j))), case, cfg, inputs=inputs)
            assert r.returncode == 0, (case, cfg, r.stderr.decode()[-2000:])
            assert sam.splitlines() == reads.splitlines()[:n], (case, cfg)
            for k in FILES:
                if (k.startswith(("un_conc", "al_conc")) if paired else k in ("un", "al")):
                    assert got[k] == files[k], (case, cfg, k)
                else:
                    assert got[k] == b""
            assert all(int(l.split()[2]) == paired for l in log.splitlines())


def assert_handles_idle(r, gpus):
    """After a run, failed or not: every handle has outcome recording off and no slot holding a batch."""
    st = dict(kv.split(b"=") for kv in r.stdout.split())
    for g in range(gpus):
        assert (st[b"outcomes_%d" % g], st[b"busy_%d" % g]) == (b"0", b"0"), (g, r.stdout)
    return st


def corrupt(src, dst):
    """A gzip file whose last member's CRC-32 is wrong: every byte inflates, the check fails."""
    b = bytearray(open(src, "rb").read())
    b[-8] ^= 0xFF
    open(dst, "wb").write(bytes(b))


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_errors(pipesim, corpus, tmp_path, variant):
    """Mate totals that differ, a missing file, a corrupt gzip file in a list and a failed wait end the run with their
    message, write nothing they must not, never hang, and leave every handle with outcome recording off and no batch in
    flight.  Every run routes reads (read files), so recording is on while it runs."""
    exe = pipesim[variant]
    cfgs = [(7, 4, 2, 8), (64, 1, 1, 1)]
    # -1 and -2 totals that differ: the reference's message (pat.cpp:270, 279); not an error when -u ends the run first
    d = os.path.join(corpus, "")
    for m1, m2, short in (("l1_1.fa,l2_1.fa.gz", "l2_2.fa,l2_2.fa", 2), ("l1_1.fa,l1_1.fa", "l1_2.fa.gz,l2_2.fa", 1)):
        inputs = ["-1", ",".join(d + x for x in m1.split(",")), "-2", ",".join(d + x for x in m2.split(","))]
        for j, cfg in enumerate(cfgs):
            r, _, _, _ = run_case(exe, corpus, str(tmp_path / ("mates%d_%d" % (short, j))), "pe_two_lanes", cfg, inputs=inputs)
            assert r.returncode == 1
            other = 3 - short
            assert b"fewer reads in file specified with -%d than in file specified with -%d" % (short, other) in r.stderr
            assert_handles_idle(r, cfg[2])
        r, sam, _, _ = run_case(exe, corpus, str(tmp_path / ("mates%d_u" % short)), "pe_two_lanes", cfgs[0],
                                inputs=inputs, extra=["-u", "300"])
        assert r.returncode == 0 and sam.count(b"\n") == 600
    # a missing file fails the run before anything is submitted
    for j, cfg in enumerate(cfgs):
        inputs = ["-U", d + "s1.fq," + d + "no_such_file.fq"]
        r, sam, log, got = run_case(exe, corpus, str(tmp_path / ("missing%d" % j)), "se_fq_plain_gz_bgzf", cfg, inputs=inputs)
        assert r.returncode == 1 and b"no_such_file.fq" in r.stderr
        assert_handles_idle(r, cfg[2])
        assert sam == b"" and log == "" and all(v == b"" for v in got.values())
    # a corrupt gzip file: the inflate's message; no record of it (or after it) is written, nothing at all when it is first
    bad = str(tmp_path / "bad.fq.gz")
    corrupt(d + "s2.fq.gz", bad)
    ok = str(tmp_path / "s1_parsed.txt")
    subprocess.run([pipesim["plain"], "--parse", "-q", "-U", d + "plain/s1.fq", "-S", ok], check=True)
    s1 = open(ok, "rb").read().splitlines(True)
    s1_text = open(d + "plain/s1.fq", "rb").read()
    msgs = set()
    for j, cfg in enumerate(cfgs):
        r, sam, _, got = run_case(exe, corpus, str(tmp_path / ("bad_mid%d" % j)), "se_fq_plain_gz_bgzf", cfg,
                                  inputs=["-U", ",".join([d + "s1.fq", bad, d + "s3.fq.bgz"])])
        assert r.returncode == 1 and b"gzip input: " in r.stderr
        assert_handles_idle(r, cfg[2])
        msgs.add(r.stderr.split(b"error: ")[-1])
        lines = sam.splitlines(True)
        assert lines == s1[:len(lines)]
        routed = got["un"] + got["al"]
        assert len(routed) <= len(s1_text) and all(rec in s1_text for rec in routed.split(b"\n@") if rec)
        for first in (["-U", bad + "," + d + "s1.fq"], ["-1", d + "p1a.fq," + d + "p1b.fq.gz", "-2", bad + "," + d + "p2b.fq"]):
            r, sam, _, got = run_case(exe, corpus, str(tmp_path / ("bad_first%d" % j)), "se_fq_plain_gz_bgzf", cfg, inputs=first)
            assert r.returncode == 1 and b"gzip input: " in r.stderr
            assert_handles_idle(r, cfg[2])
            msgs.add(r.stderr.split(b"error: ")[-1])
            assert sam == b"" and all(v == b"" for v in got.values())
    assert len(msgs) == 1, msgs
    # a failed wait: the device's message; the batches before it reached the sink, in order.  With 4 slots on each of 2
    # devices, the wait fails while later batches are in flight: they are drained before recording is turned off.
    reads = None
    for k in (0, 3):
        for j, cfg in enumerate(cfgs):
            r, sam, log, _ = run_case(exe, corpus, str(tmp_path / ("wait%d_%d" % (k, j))), "mixed_read_files_no_unal_new_summary",
                                      cfg, extra=["--fail-wait", str(k)])
            assert r.returncode == 1 and b"fake device: the wait of batch %d failed" % k in r.stderr
            st = assert_handles_idle(r, cfg[2])
            assert st[b"in_flight_at_fail"] == (b"1" if cfg[1] * cfg[2] > 1 else b"0"), (k, cfg)
            n = sum(int(l.split()[3]) for l in log.splitlines()[:k])
            if reads is None:
                full = run_case(pipesim["plain"], corpus, str(tmp_path / "wait_full"), "mixed_read_files_no_unal_new_summary", cfg)
                reads = full[1].splitlines(True)
            assert sam.splitlines(True) == reads[:n]
