"""The reference's spliced-alignment options: --pen-cansplice / --pen-noncansplice / --pen-conflictsplice (the splice
penalties), --pen-canintronlen / --pen-noncanintronlen (the intron-length penalty functions), --min-intronlen /
--max-intronlen, --dta / --dta-cufflinks (transcript assembly), --no-anchorstop, --tmo (known transcripts only) and
--avoid-pseudogene (unspliced alignments near listed sites rank as spliced ones) and --splicesite-db-only (accepted,
ignored).  tools/spliced_options_ref.py records the unmodified reference's SAM md5 per
case, its alignment summary and its argument errors in tests/golden/spliced_options_sets.json."""
import math
import os
import re
import subprocess
import sys

import pytest

from conftest import GOLDEN, ROOT

sys.path.insert(0, os.path.join(ROOT, "tools"))
import refsets  # noqa: E402
import spliced_options_ref as spo  # noqa: E402

REF = spo.load_expected()
CASES = sorted(spo.CASES)
INT_MIN = -2 ** 31
MAX_SPL_LEN = 0xfffff   # the longest intron a splice edit holds (HT2_MAX_SPL_LEN)
# cases whose output the reference itself does not change, against the case they equal
# (the new set has no junction pair of opposite sense that survives both penalties: spliced/edge_se's sense_ reads do)
SAME = {"db_only_so_ss": "default_so_ss", "can_type_only_so": "default_so", "dta_noncan_so": "dta_so",
        "pen_conflict0_so": "default_so",
        # --avoid-pseudogene needs a DB and spliced alignment; the repeat reads' site file alone changes nothing, and the
        # new set's unspliced reads all have one best locus
        "avoid_rep": "default_rep", "avoid_dna_se": "default_se_reads", "default_rep_ss": "default_rep",
        "avoid_so_ss": "default_so_ss"}


@pytest.fixture(scope="session")
def so_dir(tmp_path_factory):
    return spo.generate(str(tmp_path_factory.mktemp("splopt")))


def records(sam):
    return [l.split(b"\t") for l in sam.splitlines() if l and not l.startswith(b"@")]


def introns(cigar):
    return [int(n) for n in re.findall(rb"(\d+)N", cigar)]


def base_case(case):
    """The case a case's option is measured against: the recorded default run on the same input."""
    src = spo.CASES[case]["src"]
    base = [c for c in CASES if spo.CASES[c]["src"] == src and c.startswith("default")]
    assert len(base) == 1, case
    return base[0]


def check_shape(d, case, sam):
    """What each option visibly does to the records, so that a recorded md5 cannot stand for a case that tests nothing."""
    c = spo.CASES[case]
    o = c["opts"]
    recs = records(sam)
    assert recs
    aligned = [r for r in recs if not int(r[1]) & 4]
    for r in aligned:   # every intron is within the bounds of the case
        for n in introns(r[5]):
            assert o.get("min_intronlen", 20) <= n, (r[0], r[5])
            if o.get("no_spliced_alignment", 0) == 0 and "max_intronlen" in o:
                assert n <= o["max_intronlen"], (r[0], r[5])
    if o.get("dta") == 2:   # --dta-cufflinks: no spliced record without a sense
        spl = [r for r in aligned if introns(r[5])]
        assert all(any(t.startswith(b"XS:A:") for t in r[11:]) for r in spl)
    if o.get("tmo"):   # --tmo: every aligned record crosses listed sites only
        ss = spo.case_input(d, case)[5]
        if ss is None or o.get("no_spliced_alignment", 1) and c["src"][0] in ("se", "paired"):
            assert not aligned
        else:
            sites = set()
            for l in open(ss):
                f = l.split()
                sites.add((f[0], int(f[1]), int(f[2])))
            assert aligned
            for r in aligned:
                pos = int(r[3]) - 1
                ns = introns(r[5])
                assert ns
                for op_len, op in re.findall(rb"(\d+)([MIDNS])", r[5]):
                    if op in (b"M", b"D"):
                        pos += int(op_len)
                    elif op == b"N":
                        assert (r[2].decode(), pos - 1, pos + int(op_len)) in sites, (r[0], r[5])
                        pos += int(op_len)


def test_recorded_shapes():
    """Each option changes the reference's own output on its input, except where the reference shows it does not:
    --splicesite-db-only, a type-only function equal to the default, --dta with a non-canonical function (--dta
    overrides it) and --pen-conflictsplice 0 on a set without reads spliced in both senses."""
    m = REF["md5"]
    for case in CASES:
        if case in SAME:
            assert m[case] == m[SAME[case]], case
            continue
        b = base_case(case)
        if b != case:
            assert m[case] != m[b], case
    assert m["dta_cufflinks_so"] != m["dta_so"]
    assert m["tmo_so"] != m["tmo_so_ss"]
    assert all(REF["errors"][e][1] != 0 for e in spo.ERRORS)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the host build (tests/hostsim/ht2_sploptsim.cpp) and the intron-length penalty runs
# ---------------------------------------------------------------------------------------------------------------------
def _build(tmp_path_factory, name, flags):
    c = os.path.join(ROOT, "hisat2_b200", "csrc")
    exe = str(tmp_path_factory.mktemp(name) / "ht2_sploptsim")
    subprocess.run(["g++"] + flags + ["-std=c++14", "-o", exe, os.path.join(ROOT, "tests", "hostsim", "ht2_sploptsim.cpp"),
                                      os.path.join(c, "ht2_index.cpp"), os.path.join(c, "ht2_host.cpp"), "-lpthread"], check=True)
    return exe


@pytest.fixture(scope="session")
def sploptsim(tmp_path_factory):
    """TEST-ONLY host build of ht2_hostsim with the spliced-alignment options."""
    return _build(tmp_path_factory, "sploptsim", ["-O2"])


@pytest.fixture(scope="session")
def sploptsim_asan(tmp_path_factory):
    return _build(tmp_path_factory, "sploptsim_asan", ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined"])


SPL_KEYS = ("pen_cansplice", "pen_noncansplice", "pen_conflictsplice", "min_intronlen", "max_intronlen", "dta",
            "no_anchorstop", "tmo", "avoid_pseudogene")


def host_env(o):
    """HT2_OPTS / HT2_SPL_OPTS of a case's library options."""
    kv, so = [], []
    for k, v in sorted(o.items()):
        if k == "no_spliced_alignment":
            kv.append("spliced=%d" % (v == 0))
        elif k in SPL_KEYS:
            so.append("%s=%d" % (k, v))
        elif k in ("can_intronlen_type", "noncan_intronlen_type"):
            pre = k[:-5]
            so.append("%s=%s:%r:%r" % (pre.split("_")[0], v, o[pre + "_const"], o[pre + "_coeff"]))
        elif k == "score_min_type":
            kv.append("score_min=%s:%r:%r" % (chr(v), o["score_min_const"], o["score_min_coeff"]))
        elif k.endswith("_const") or k.endswith("_coeff"):
            continue
        else:
            kv.append("%s=%d" % (k, v))
    return ",".join(kv), ",".join(so)


def hostsim(exe, d, tmp_path, case):
    index, fs, _, _, opts, ss = spo.case_input(d, case)
    kv, so = host_env(opts)
    o = str(tmp_path / "o.sam")
    env = dict(os.environ, HT2_OPTS=kv, HT2_SPL_OPTS=so, ASAN_OPTIONS="detect_leaks=0")
    if ss:
        env["HT2_SS"] = ss
    r = subprocess.run([exe, os.path.join(GOLDEN, index), fs[0], o] + fs[1:], cwd=GOLDEN, stderr=subprocess.PIPE, env=env)
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    assert r.stderr.count(b"err=") <= len(spo.flagged(case))
    return open(o, "rb").read()


@pytest.mark.parametrize("case", CASES)
def test_host_build_matches_reference(sploptsim, so_dir, tmp_path, case):
    """Every case through the host build: the md5 of the reference's SAM (header without @PG) and the shape each
    option gives its records."""
    sam = hostsim(sploptsim, so_dir, tmp_path, case)
    assert refsets.sam_md5(sam, spo.flagged(case)) == REF["md5"][case]
    check_shape(so_dir, case, sam)


def primaries(sam):
    return {r[0]: (r[2], int(r[3])) for r in records(sam) if not int(r[1]) & (4 | 256)}


def test_avoid_pseudogene_prefers_the_copy_near_a_site(sploptsim, so_dir, tmp_path):
    """--avoid-pseudogene on reads of two-copy repeats: the primary alignment moves on some reads, and wherever it
    moves, the new locus has a listed site within 10 000 bases and the old one has none."""
    ss = spo.generate_rep(so_dir)
    sites = [l.split() for l in open(ss)]
    near = lambda chrom, pos: any(f[0] == chrom and (pos - 1 - 10000 <= int(f[1]) <= pos - 1 + 100 + 10000 or
                                                     pos - 1 - 10000 <= int(f[2]) <= pos - 1 + 100 + 10000) for f in sites)
    base = primaries(hostsim(sploptsim, so_dir, tmp_path, "default_rep_ss"))
    avoid = primaries(hostsim(sploptsim, so_dir, tmp_path, "avoid_rep_ss"))
    moved = [q for q in base if base[q] != avoid[q]]
    assert moved
    for q in moved:
        (c0, p0), (c1, p1) = base[q], avoid[q]
        assert near(c1.decode(), p1) and not near(c0.decode(), p0), q


@pytest.mark.parametrize("case", ["can_G2_so", "noncan_S_so", "dta_cufflinks_so_ss", "tmo_so_ss", "dta_dp2_so",
                                  "no_anchorstop_k1_so", "avoid_rep_ss"])
def test_host_build_under_sanitizers(sploptsim_asan, so_dir, tmp_path, case):
    """The same host build under ASan / UBSan on the new read set, the DP case included."""
    sam = hostsim(sploptsim_asan, so_dir, tmp_path, case)
    assert refsets.sam_md5(sam, spo.flagged(case)) == REF["md5"][case]


def intron_pen(t, c, l, x):
    """max(0, SimpleFunc::f<int>(x)) (simple_func.h:86-108, min -DBL_MAX, max DBL_MAX), converted as x86-64 converts:
    DBL_MAX gives INT_MAX, DBL_MIN and anything outside int's range INT_MIN, which the max makes 0."""
    dmax, dmin = 1.7976931348623157e308, 2.2250738585072014e-308
    smin = lambda a, b: b if b < a else a   # std::min / std::max, NaN included
    smax = lambda a, b: b if a < b else a
    X = {"C": 0.0, "L": float(x), "S": math.sqrt(x), "G": math.log(x)}[t]
    v = smax(-dmax, smin(dmax, c + l * X))
    if v == dmax:
        return 2 ** 31 - 1
    if v == dmin or not (-2 ** 31 <= v < 2 ** 31):
        return 0
    return max(0, int(v))


def runs(exe, t, c, l, upto):
    r = subprocess.run([exe, "--intron-pen", t, repr(c), repr(l), str(upto)], stdout=subprocess.PIPE)
    if r.returncode == 3:
        return None
    assert r.returncode == 0
    return [tuple(int(v) for v in line.split()) for line in r.stdout.decode().splitlines()]


@pytest.mark.parametrize("fn,upto", [(("G", -8.0, 1.0), 500000), (("G", -8.0, 2.0), 500000), (("L", 0.0, 0.01), 100000),
                                     (("S", -10.0, 0.5), MAX_SPL_LEN), (("C", 3.0, 1.0), 500000), (("G", -4.0, 1.0), MAX_SPL_LEN),
                                     (("L", -2.0, 0.001), 500000), (("G", -6.0, 1.0), 500000), (("S", -5.0, 0.3), 500000),
                                     (("L", 3e9, 1.0), 1000), (("C", 1.7976931348623157e308, 0.0), 1000),
                                     (("L", 0.0, 1e308), 1000)])
def test_intron_pen_runs(sploptsim, fn, upto):
    """The runs the host builds give max(0, f<int>(x)) for every intron length up to the covered maximum, each function
    of the cases and the default included, out-of-range values too."""
    rs = runs(sploptsim, *fn, upto)
    assert rs and rs[0] == (0, 0)
    starts = [s for s, _ in rs] + [upto + 1]
    for k, (s, p) in enumerate(rs[1:], 1):
        assert p == intron_pen(*fn, s) != intron_pen(*fn, s - 1) if s > 1 else True
    # every length, run by run (the value is constant inside a run)
    k = 0
    for x in range(1, upto + 1):
        while starts[k + 1] <= x:
            k += 1
        assert rs[k][1] == intron_pen(*fn, x), x


def test_default_intron_pen_breakpoints(sploptsim):
    """G,-8,1 over every length a splice edit holds: the breakpoints of the default penalty."""
    rs = runs(sploptsim, "G", -8.0, 1.0, MAX_SPL_LEN)
    assert rs == [(0, 0), (8104, 1), (22027, 2), (59875, 3), (162755, 4), (442414, 5)]


@pytest.mark.parametrize("fn,upto", [(("L", 0.0, 1.0), 500000), (("S", 0.0, 3.0), 500000), (("L", 0.0, 0.01), 500000)])
def test_steep_functions_are_refused(sploptsim, fn, upto):
    """A function with more values over the covered lengths than the device holds is refused by the host builder."""
    assert runs(sploptsim, *fn, upto) is None


def test_python_settings_are_checked(lib):
    from hisat2_b200 import api
    with pytest.raises(ValueError):
        api._options(lib, dict(dta="assembler"))
    o = api._options(lib, dict(dta="cufflinks", can_intronlen_type="S", can_intronlen_const=1.0, can_intronlen_coeff=0.5))
    assert (o.dta, o.can_intronlen_type, o.can_intronlen_const, o.can_intronlen_coeff) == (2, ord("S"), 1.0, 0.5)
    assert api._options(lib, dict(dta=True)).dta == 1
    d = api._options(lib, {})
    assert (d.pen_cansplice, d.pen_noncansplice, d.pen_conflictsplice, d.min_intronlen, d.max_intronlen) == (0, 12, 1000000, 20, 500000)
    assert (d.can_intronlen_type, d.noncan_intronlen_type, d.dta, d.no_anchorstop, d.tmo, d.avoid_pseudogene) == (0, 0, 0, 0, 0, 0)


@pytest.mark.parametrize("field,value", [("pen_cansplice", -1), ("pen_noncansplice", -1), ("pen_conflictsplice", -5),
                                         ("min_intronlen", 19), ("max_intronlen", 0), ("dta", 3),
                                         ("can_intronlen_type", ord("X")), ("noncan_intronlen_type", 1)])
def test_open_refuses_bad_values(lib, field, value):
    """ht2gpu_open refuses a negative penalty, an intron bound below 20, an unknown --dta mode or function type before
    it uses a device."""
    import ctypes as C
    from hisat2_b200 import api
    o = api.Options()
    lib.ht2gpu_default_options(C.byref(o))
    setattr(o, field, value)
    h = C.c_void_p()
    rc = lib.ht2gpu_open(os.path.join(GOLDEN, "tiny").encode(), C.byref(o), C.byref(h))
    msg = lib.ht2gpu_last_error(h).decode()
    lib.ht2gpu_close(h)
    assert rc == -1 and msg


def test_open_refuses_min_above_max(lib):
    import ctypes as C
    from hisat2_b200 import api
    o = api._options(lib, dict(min_intronlen=600, max_intronlen=500))
    h = C.c_void_p()
    rc = lib.ht2gpu_open(os.path.join(GOLDEN, "tiny").encode(), C.byref(o), C.byref(h))
    msg = lib.ht2gpu_last_error(h).decode()
    lib.ht2gpu_close(h)
    assert rc == -1 and "--min-intronlen" in msg


def cli(args, **kw):
    exe = os.path.join(ROOT, "hisat2_b200", "hisat2-b200")
    return subprocess.run([exe] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, cwd=GOLDEN, **kw)


@pytest.fixture(scope="module")
def cli_built(lib):
    from hisat2_b200 import build
    build.build_cli()


@pytest.mark.parametrize("err", sorted(spo.ERRORS))
def test_cli_argument_errors(cli_built, so_dir, tmp_path, err):
    """A bad spliced-alignment option: the reference's message and exit status, before any device is opened."""
    line, status = REF["errors"][err]
    r = cli(["-x", "tiny", "-f", "--no-temp-splicesite", "-U", os.path.join(so_dir, "reads_1.fa"), "-S", str(tmp_path / "o.sam")] +
            spo.ERRORS[err])
    assert r.returncode == status
    assert r.stderr.decode().splitlines()[0] == line


def test_cli_refuses_empty_function(cli_built, so_dir, tmp_path):
    """An empty function type, which the reference does not handle, is an error."""
    for v in ("", ",2"):
        r = cli(["-x", "tiny", "-f", "-U", os.path.join(so_dir, "reads_1.fa"), "-S", str(tmp_path / "o.sam"),
                 "--pen-canintronlen", v])
        assert r.returncode != 0 and "--pen-canintronlen" in r.stderr.decode()


# ---------------------------------------------------------------------------------------------------------------------
# GPU: ht2gpu_run_reads, ht2gpu_align_sam, the summary, the CLI and the seed search
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def h2(lib):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import hisat2_b200
    return hisat2_b200


def open_case(h2, d, case):
    index, fs, fmt, _, opts, ss = spo.case_input(d, case)
    idx = h2.Index(os.path.join(GOLDEN, index), **opts)
    if ss:
        idx.load_splicesites(ss)
    return idx, fs, fmt, opts


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_device_matches_reference(h2, so_dir, case):
    """Every case through ht2gpu_run_reads in one batch and in 64-read batches, the alignment summary of the run, and
    ht2gpu_align_sam against the host formatter."""
    idx, fs, fmt, opts = open_case(h2, so_dir, case)
    try:
        for batch_reads in (0, 64):
            idx.align_counts(reset=True)
            sam, st = idx.run_reads(path1=fs[0], path2=fs[1] if len(fs) == 2 else None, fastq=fmt == "-q", batch_reads=batch_reads)
            sam = idx.sam_header() + sam
            assert st["n_err_reads"] <= len(spo.flagged(case))
            assert refsets.sam_md5(sam, spo.flagged(case)) == REF["md5"][case], batch_reads
            summ = h2.format_align_summary(idx.align_counts())
            if not spo.flagged(case):
                assert summ == REF["summary"][case], batch_reads
        check_shape(so_dir, case, sam)
        batch = h2.ReadBatch.parse(path1=fs[0], path2=fs[1] if len(fs) == 2 else None, fastq=fmt == "-q")
        host = idx.format_sam(batch, idx.align(batch))
        assert idx.align_sam(batch) == host, "device SAM differs from the host formatter's"
    finally:
        idx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_cli_matches_reference(h2, so_dir, tmp_path, case):
    """hisat2-b200 with the reference's flags gives the reference's SAM and summary."""
    index, fs, fmt, flags, _, _ = spo.case_input(so_dir, case)
    reads = ["-1", fs[0], "-2", fs[1]] if len(fs) == 2 else ["-U", fs[0]]
    out = str(tmp_path / "o.sam")
    r = cli(["-x", index, fmt] + flags + reads + ["-S", out, "--batch", "512"])
    assert r.returncode == 0, r.stderr
    assert refsets.sam_md5(open(out, "rb").read(), spo.flagged(case)) == REF["md5"][case]
    if not spo.flagged(case):
        assert refsets.summary_text(r.stderr) == REF["summary"][case]


@pytest.mark.gpu
def test_open_refuses_steep_function(h2):
    """A function with more values over the covered intron lengths than the device holds is HT2GPU_ERR_UNSUPPORTED,
    naming the option; without spliced alignment no intron is scored and it is accepted."""
    with pytest.raises(h2.Ht2GpuError) as e:
        h2.Index(os.path.join(GOLDEN, "tiny"), no_spliced_alignment=0, can_intronlen_type="L", can_intronlen_const=0.0,
                 can_intronlen_coeff=1.0)
    assert "--pen-canintronlen" in str(e.value)
    h2.Index(os.path.join(GOLDEN, "tiny"), no_spliced_alignment=1, can_intronlen_type="L", can_intronlen_const=0.0,
             can_intronlen_coeff=1.0).close()
    h2.Index(os.path.join(GOLDEN, "tiny"), no_spliced_alignment=0, max_intronlen=1000, can_intronlen_type="L",
             can_intronlen_const=0.0, can_intronlen_coeff=1.0).close()


def host_seed_dump(exe, reads, no_spliced, spl_opts):
    env = dict(os.environ, HT2_SPL_OPTS=spl_opts)
    return subprocess.run([exe, "--seed-dump", "tiny", reads, no_spliced], cwd=GOLDEN, check=True, env=env,
                          stdout=subprocess.PIPE).stdout.decode().splitlines(True)


@pytest.mark.gpu
@pytest.mark.parametrize("no_spliced", [0, 1])
def test_seed_search_without_anchorstop(h2, sploptsim, so_dir, no_spliced):
    """ht2gpu_seed_search under no_anchorstop equals the host build's seed dump with the same setting, in both modes;
    no partial search stops at a unique anchor, and the chains differ from the default's."""
    reads = os.path.join(so_dir, "splopt_se.fa")
    batch = h2.ReadBatch.from_fasta(reads)
    res = {}
    for nas in (0, 1):
        idx = h2.Index(os.path.join(GOLDEN, "tiny"), no_spliced_alignment=no_spliced, no_anchorstop=nas)
        try:
            res[nas] = idx.seed_search(batch, max_range=4)
        finally:
            idx.close()
        assert res[nas].dump_lines(False) == host_seed_dump(sploptsim, reads, str(no_spliced), "no_anchorstop=%d" % nas), nas
    assert int(res[0].hits["anchor_stop"].sum()) > 0
    assert int(res[1].hits["anchor_stop"].sum()) == 0 and int((res[1].hits["hit_type"] == 3).sum()) == 0
    assert res[0].dump_lines(False) != res[1].dump_lines(False)


@pytest.mark.gpu
def test_multi_handle_runs_refuse_different_settings(h2, so_dir):
    """run_reads_multi refuses handles whose spliced-alignment options differ; peers take them from their source."""
    f = os.path.join(so_dir, "splopt_se.fa")
    opts = dict(no_spliced_alignment=0, dta=2, can_intronlen_type="G", can_intronlen_const=-8.0, can_intronlen_coeff=2.0)
    idx = h2.Index(os.path.join(GOLDEN, "tiny"), **opts)
    try:
        peer = idx.peer(0)
        try:
            sam, _ = idx.run_reads(path1=f, peers=(peer,), batch_reads=64)
            alone, _ = idx.run_reads(path1=f, batch_reads=64)
            assert sam == alone
        finally:
            peer.close()
        for other_opts in (dict(no_spliced_alignment=0, dta=2), dict(no_spliced_alignment=0, can_intronlen_type="G",
                                                                     can_intronlen_const=-8.0, can_intronlen_coeff=2.0),
                           dict(opts, tmo=1), dict(opts, max_intronlen=1000), dict(opts, pen_conflictsplice=0),
                           dict(opts, avoid_pseudogene=1)):
            other = h2.Index(os.path.join(GOLDEN, "tiny"), **other_opts)
            try:
                with pytest.raises(h2.Ht2GpuError):
                    idx.run_reads(path1=f, peers=(other,), batch_reads=64)
            finally:
                other.close()
    finally:
        idx.close()
