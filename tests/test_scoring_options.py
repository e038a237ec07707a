"""The reference's mate orientation, N ceiling, soft-clipping, quality encoding and match bonus options: --fr / --rf /
--ff (which mate faces which way in a concordant pair), --n-ceil (the most Ns a read may hold, and the N ceiling of the
--bowtie2-dp extension), --no-softclip (end-to-end alignments only), --solexa-quals / --int-quals (Solexa-64 and
integer FASTQ qualities) and --ma (warned about and ignored in end-to-end mode).  tools/scoring_options_ref.py records the unmodified reference's
SAM md5 per case, its alignment summary, its warnings and its argument errors in
tests/golden/scoring_options_sets.json."""
import math
import os
import subprocess
import sys

import pytest

from conftest import GOLDEN, ROOT

sys.path.insert(0, os.path.join(ROOT, "tools"))
import refsets  # noqa: E402
import scoring_options_ref as sor  # noqa: E402

REF = sor.load_expected()
CASES = sorted(sor.CASES)
HOST_CASES = [c for c in CASES if sor.CASES[c]["src"][0] != "golden"]   # the host build reads no Solexa / integer qualities
QUAL_CASES = [c for c in CASES if sor.CASES[c]["src"][0] == "golden"]
INT_MIN = -2 ** 31
F15 = sor.F15


@pytest.fixture(scope="session")
def so_dir(tmp_path_factory):
    return sor.generate(str(tmp_path_factory.mktemp("scoreopt")))


def concordant_counts(summary):
    """The paired section's concordant 0 / 1 / >1 lines of a classic summary."""
    return [l.strip().split(" ", 1)[0] for l in summary.splitlines() if "aligned concordantly" in l and "of these" not in l]


def records(sam):
    return [l.split(b"\t") for l in sam.splitlines() if l and not l.startswith(b"@")]


def check_shape(case, sam):
    """What each option visibly does to the records, so that a recorded md5 cannot stand for a case that tests nothing."""
    c = sor.CASES[case]
    recs = records(sam)
    assert recs
    o = c["opts"].get("pe_orient")
    if o and c["src"][0] != "se":
        conc = [r for r in recs if int(r[1]) & 2]
        if c["xform"] is None and o != "fr":
            assert not conc          # an FR library has no concordant pair under --rf / --ff
        else:
            assert conc
            for r in conc:           # a concordant mate's strand is the one --fr / --rf / --ff gives it
                rev = int(r[1]) & 16
                if o == "ff":
                    assert (int(r[1]) & 32 != 0) == (rev != 0)
                else:
                    assert (int(r[1]) & 32 != 0) != (rev != 0)
                if o == "rf" and int(r[8]) > 0:   # the leftmost mate of an RF pair is reverse-complemented
                    assert rev
                if o == "fr" and int(r[8]) > 0 and int(r[3]) < int(r[7]):
                    assert not rev
    if c["opts"].get("sp_max") == sor.INT_MAX:   # --no-softclip: end-to-end alignments only
        aligned = [r for r in recs if not int(r[1]) & 4]
        assert aligned and not any(b"S" in r[5] for r in aligned)
    if c["xform"] == "nrich":   # YF:Z:NS exactly on the reads with more Ns than the ceiling of their length
        o = c["opts"]
        fn = (chr(o["n_ceil_type"]) if isinstance(o["n_ceil_type"], int) else o["n_ceil_type"], o["n_ceil_const"], o["n_ceil_coeff"]) \
            if "n_ceil_type" in o else ("L", 0.0, F15)
        for r in recs:
            ceil = simple_func_int(*fn, len(r[9])) % 2 ** 32   # compared as size_t
            assert (b"YF:Z:NS" in r[11:]) == (r[9].count(b"N") > ceil), r[:2]
        assert any(b"YF:Z:NS" in r[11:] for r in recs) == (case != "nceil_big_se")


def test_recorded_shapes():
    """The reference's own output: an RF library under --rf pairs as the FR library under --fr does; an FR library has
    no concordant pair under --rf or --ff; --ma changes nothing but a warning; each N ceiling filters another set."""
    s, m = REF["summary"], REF["md5"]
    assert len(concordant_counts(s["fr_pe_reads"])) == 3
    assert concordant_counts(s["rf_pe_reads_rf"]) == concordant_counts(s["fr_pe_reads"])
    assert concordant_counts(s["rf_pe_hard20k_rf"]) == concordant_counts(s["fr_pe_hard20k"])
    for case in ("rf_pe_reads_fr", "ff_pe_reads_fr"):
        assert concordant_counts(s[case])[1:] == ["0", "0"]
    assert m["ma_se_reads"] == m["rf_se_reads"]
    assert REF["warnings"]["ma_se_reads"] == ["Warning: Match bonus always = 0 in --end-to-end mode; ignoring user setting"]
    assert not any(REF["warnings"][c] for c in CASES if c != "ma_se_reads")
    assert REF["warnings"]["ma_last_wins_se_reads"] == [] and m["ma_last_wins_se_reads"] == m["ma_se_reads"]
    assert m["sp_then_nosc_edge_se"] == m["nosc_edge_se"] != m["nosc_then_sp_edge_se"]
    assert m["qual_solexa_phred64"] == m["qual_solexa_se"] != m["qual_solexa_then_phred33"]
    assert m["qual_int_phred64"] == m["qual_int_se"]
    assert all(REF["qual_errors"][e] != 0 for e in sor.QUAL_ERRORS)
    f = REF["files"]
    assert f["rf_pe_reads_fr"]["al_conc/1"] == f["rf_pe_reads_fr"]["al_conc/2"] == "d41d8cd98f00b204e9800998ecf8427e"
    assert f["rf_pe_reads_rf"]["al_conc/1"] != "d41d8cd98f00b204e9800998ecf8427e"
    nc = [m[c] for c in CASES if c.startswith("nceil_") and c != "nceil_comma_se"]
    assert len(set(nc)) == len(nc)
    assert m["nceil_comma_se"] == m["nceil_zero_se"]


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the host build (tests/hostsim/ht2_scoreoptsim.cpp) and the N-ceiling table
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="session")
def scoreoptsim(tmp_path_factory):
    """TEST-ONLY host build of ht2_hostsim with the mate orientation and the N ceiling."""
    c = os.path.join(ROOT, "hisat2_b200", "csrc")
    exe = str(tmp_path_factory.mktemp("scoreoptsim") / "ht2_scoreoptsim")
    subprocess.run(["g++", "-O2", "-std=c++14", "-o", exe, os.path.join(ROOT, "tests", "hostsim", "ht2_scoreoptsim.cpp"),
                    os.path.join(c, "ht2_index.cpp"), os.path.join(c, "ht2_host.cpp"), "-lpthread"], check=True)
    return exe


def host_env(d, case):
    """HT2_OPTS / HT2_SCORE_OPTS of a case's library options and SAM settings."""
    o = sor.case_input(d, case)[4]
    kv, so = [], []
    for k, v in sorted(o.items()):
        if k == "no_spliced_alignment":
            kv.append("spliced=%d" % (v == 0))
        elif k == "pe_orient":
            so.append("pe_orient=%d" % {"fr": 0, "rf": 1, "ff": 2}[v])
        elif k in ("n_ceil_type", "score_min_type"):
            pre, t = k[:-5], chr(v) if isinstance(v, int) else v
            (so if pre == "n_ceil" else kv).append("%s=%s:%r:%r" % (pre, t, o[pre + "_const"], o[pre + "_coeff"]))
        elif k.endswith("_const") or k.endswith("_coeff"):
            continue
        else:
            kv.append("%s=%d" % (k, v))
    out = sor.CASES[case].get("out", {})
    if out.get("rna_strandness"):
        so.append("rna_strandness=%d" % {"F": 1, "R": 2, "FR": 3, "RF": 4}[out["rna_strandness"]])
    return ",".join(kv), ",".join(so)


def hostsim(exe, d, tmp_path, case):
    index, fs, _, _, _, ss = sor.case_input(d, case)
    kv, so = host_env(d, case)
    o = str(tmp_path / "o.sam")
    env = dict(os.environ, HT2_OPTS=kv, HT2_SCORE_OPTS=so, ASAN_OPTIONS="detect_leaks=0")
    if ss:
        env["HT2_SS"] = ss
    r = subprocess.run([exe, os.path.join(GOLDEN, index), fs[0], o] + fs[1:], cwd=GOLDEN, stderr=subprocess.PIPE, env=env)
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    assert r.stderr.count(b"err=") <= len(sor.flagged(case))
    return open(o, "rb").read()


@pytest.mark.parametrize("case", HOST_CASES)
def test_host_build_matches_reference(scoreoptsim, so_dir, tmp_path, case):
    """Every case through the host build: the md5 of the reference's SAM (header without @PG) and the shape each
    option gives its records."""
    sam = hostsim(scoreoptsim, so_dir, tmp_path, case)
    assert refsets.sam_md5(sam, sor.flagged(case)) == REF["md5"][case]
    check_shape(case, sam)


@pytest.fixture(scope="session")
def scoreoptsim_asan(tmp_path_factory):
    c = os.path.join(ROOT, "hisat2_b200", "csrc")
    exe = str(tmp_path_factory.mktemp("scoreoptsim_asan") / "ht2_scoreoptsim")
    subprocess.run(["g++", "-O1", "-g", "-std=c++14", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-o", exe,
                    os.path.join(ROOT, "tests", "hostsim", "ht2_scoreoptsim.cpp"), os.path.join(c, "ht2_index.cpp"),
                    os.path.join(c, "ht2_host.cpp"), "-lpthread"], check=True)
    return exe


@pytest.mark.parametrize("case", ["rf_pe_reads_rf", "ff_pe_reads_ff", "nceil_G_pe", "nceil_sensitive_pe", "nceil_dp2_se",
                                  "nosc_edge_se", "nosc_edge_se_dp"])
def test_host_build_under_sanitizers(scoreoptsim_asan, so_dir, tmp_path, case):
    """The same host build under ASan / UBSan on the small sets of each option, the DP cases included."""
    sam = hostsim(scoreoptsim_asan, so_dir, tmp_path, case)
    assert refsets.sam_md5(sam, sor.flagged(case)) == REF["md5"][case]


def simple_func_int(t, c, l, x):
    """SimpleFunc::f<int> (simple_func.h:86-108) with min 0 and max DBL_MAX, converted as x86-64 converts: DBL_MAX
    gives INT_MAX, any other value at or above 2^31 gives INT_MIN."""
    dmax = 1.7976931348623157e308
    smin = lambda a, b: b if b < a else a   # std::min / std::max, NaN included
    smax = lambda a, b: b if a < b else a
    X = {"C": 0.0, "L": float(x), "S": math.sqrt(x), "G": math.log(x) if x > 0 else -math.inf}[t]
    y = c + (l * X if not (l == 0 and math.isinf(X)) else math.nan)   # 0 * -inf is NaN in C
    v = smax(0.0, smin(dmax, y))
    if v == dmax:
        return 2 ** 31 - 1
    return INT_MIN if v >= 2 ** 31 else int(v)


@pytest.mark.parametrize("fn", [("L", 0.0, 0.15), ("C", 3.0, 0.0), ("S", 1.0, 1.5), ("G", -1.0, 2.5), ("G", 0.0, 0.0),
                                ("L", -5.0, 0.01), ("C", 1e10, 0.0), ("L", 0.0, 5e6), ("C", 1.7976931348623157e308, 0.0)])
def test_nceil_table(scoreoptsim, fn):
    """Ht2Params::nCeilTab equals SimpleFunc restated in Python at every read length, out-of-range values included."""
    t, c, l = fn
    out = subprocess.run([scoreoptsim, "--nceil-table", t, repr(c), repr(l)], check=True, stdout=subprocess.PIPE).stdout.decode()
    got = [int(line.split()[1]) for line in out.splitlines()]
    assert got == [simple_func_int(t, c, l, x) for x in range(len(got))]


def test_scpen_conversion(scoreoptsim):
    """ht2_scpen converts as x86-64 does in both builds: at --sp INT_MAX,INT_MAX (--no-softclip) the float is 2^31 and
    gives INT_MIN above quality 33, while sc(q <= 33) is scpMin itself; ordinary penalties are unchanged."""
    def pen(mx, mn):
        out = subprocess.run([scoreoptsim, "--scpen", str(mx), str(mn)], check=True, stdout=subprocess.PIPE).stdout.decode()
        return [int(l.split()[1]) for l in out.splitlines()]
    p = pen(sor.INT_MAX, sor.INT_MAX)
    assert p[:34] == [sor.INT_MAX] * 34 and p[34:] == [INT_MIN] * 47
    assert pen(2, 1) == [1] * 34 + [int((min(q - 33, 40) / 40.0) * 1 + 1) for q in range(34, 81)]
    assert pen(6, 2)[73] == 6 and pen(6, 2)[53] == 4


def expected_quals(path, reads):
    """The Phred+33 qualities the reference reads from a FASTQ file (pat.cpp:997-1090, qual.h:46-170), per record."""
    sol = lambda s: 0 if s < -10 else int(10 * math.log10(10 ** (min(s, 255) / 10.0) + 1) + 0.5)
    lines = open(path, "rb").read().split(b"\n")
    t5, t3 = reads.get("trim5", 0), reads.get("trim3", 0)
    out = []
    for i in range(3, len(lines), 4):
        n = max(0, len(lines[i - 2]) - t5 - t3)
        q = lines[i]
        if reads.get("int_quals"):
            toks = q.decode().split(" ")
            toks = toks[:1] + [t for t in toks[1:] if t] if q else []
            vals = [(sol(int(t or 0)) if reads.get("solexa_quals") else min(int(t or 0), 93)) + 33 for t in toks][t5:]
            vals = vals[:max(0, len(vals) - t3)][:n]
        elif reads.get("solexa_quals"):
            vals = [sol((c if c < 128 else c - 256) - 64) + 33 for c in q][t5:t5 + n]
        else:
            vals = list(q[t5:t5 + n])
        out.append(bytes(vals))
    return out


@pytest.mark.parametrize("case", QUAL_CASES)
def test_quality_parsing(lib, so_dir, case):
    """ht2gpu_parse_reads (the front end of ht2gpu_run_reads and the pipeline) reads Solexa and integer qualities as the
    reference does, and the per-read seeds follow the converted qualities."""
    from hisat2_b200 import ReadBatch
    _, fs, _, _, _, _ = sor.case_input(so_dir, case)
    reads = sor.CASES[case]["reads"]
    b = ReadBatch.parse(path1=fs[0], path2=fs[1] if len(fs) == 2 else None, fastq=True, lib=lib, **reads)
    want = [expected_quals(f, reads) for f in fs]
    want = [q for pair in zip(*want) for q in pair] if len(fs) == 2 else want[0]
    got = [bytes(b.qual[b.offs[i]:b.offs[i + 1]]) for i in range(len(b.offs) - 1)]
    assert got == want
    if reads.get("solexa_quals") and not reads.get("int_quals"):   # the same characters read as Phred+33
        plain = ReadBatch.parse(path1=fs[0], path2=fs[1] if len(fs) == 2 else None, fastq=True, lib=lib,
                                **{k: v for k, v in reads.items() if k in ("trim5", "trim3")})
        assert list(plain.seeds) != list(b.seeds)


@pytest.mark.parametrize("err", sorted(sor.QUAL_ERRORS))
def test_quality_errors(lib, so_dir, err):
    """Fewer or more integer values than bases (beyond one), a negative integer quality, a space among Solexa
    characters: the reference stops with an error, and so does the front end."""
    from hisat2_b200 import ReadBatch, Ht2GpuError
    kind, how, _ = sor.QUAL_ERRORS[err]
    f = sor.golden_fq(so_dir, kind, how)[0]
    kw = dict(int_quals=1) if how.startswith("int") else dict(solexa_quals=1)
    assert REF["qual_errors"][err] != 0
    with pytest.raises(Ht2GpuError):
        ReadBatch.parse(path1=f, fastq=True, lib=lib, **kw)


def test_python_settings_are_checked(lib):
    from hisat2_b200 import api
    with pytest.raises(ValueError):
        api._options(lib, dict(pe_orient="rr"))
    o = api._options(lib, dict(pe_orient="ff", n_ceil_type="S", n_ceil_const=1.0, n_ceil_coeff=0.5))
    assert (o.pe_orient, o.n_ceil_type, o.n_ceil_const, o.n_ceil_coeff) == (2, ord("S"), 1.0, 0.5)
    d = api._options(lib, {})
    assert (d.pe_orient, d.n_ceil_type) == (0, 0)


@pytest.mark.parametrize("field,value", [("pe_orient", 3), ("pe_orient", -1), ("n_ceil_type", ord("X"))])
def test_open_refuses_bad_values(lib, field, value):
    """ht2gpu_open refuses an unknown orientation or N-ceiling type before it uses a device."""
    import ctypes as C
    from hisat2_b200 import api
    o = api.Options()
    lib.ht2gpu_default_options(C.byref(o))
    setattr(o, field, value)
    h = C.c_void_p()
    rc = lib.ht2gpu_open(os.path.join(GOLDEN, "tiny").encode(), C.byref(o), C.byref(h))
    msg = lib.ht2gpu_last_error(h).decode()
    lib.ht2gpu_close(h)
    assert rc == -1 and field in msg


def cli(args, **kw):
    exe = os.path.join(ROOT, "hisat2_b200", "hisat2-b200")
    return subprocess.run([exe] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, cwd=GOLDEN, **kw)


@pytest.fixture(scope="module")
def cli_built(lib):
    from hisat2_b200 import build
    build.build_cli()


@pytest.mark.parametrize("err", sorted(sor.ERRORS))
def test_cli_argument_errors(cli_built, so_dir, tmp_path, err):
    """A bad --n-ceil: the reference's message and exit status, before any device is opened."""
    line, status = REF["errors"][err]
    if err == "ma_two_tokens":   # the reference numbers the setting within its whole policy string
        line = line.split(" setting ")[0]
    r = cli(["-x", "tiny", "-f", "--no-spliced-alignment", "-U", os.path.join(so_dir, "reads_1.fa"), "-S", str(tmp_path / "o.sam")] +
            sor.ERRORS[err])
    assert r.returncode == status
    assert r.stderr.decode().splitlines()[0].startswith(line)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: ht2gpu_run_reads, ht2gpu_align_sam, the summary and the CLI
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def h2(lib):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import hisat2_b200
    return hisat2_b200


def open_case(h2, d, case):
    index, fs, fmt, _, opts, ss = sor.case_input(d, case)
    idx = h2.Index(os.path.join(GOLDEN, index), **opts)
    if ss:
        idx.load_splicesites(ss)
    out = sor.CASES[case].get("out")
    if out:
        idx.set_sam_output(**out)
    return idx, fs, fmt, opts


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_device_matches_reference(h2, so_dir, case):
    """Every case through ht2gpu_run_reads in one batch and in 64-read batches, the alignment summary of the run, and
    ht2gpu_align_sam against the host formatter."""
    idx, fs, fmt, opts = open_case(h2, so_dir, case)
    reads = sor.CASES[case].get("reads", {})
    try:
        for batch_reads in (0, 64):
            idx.align_counts(reset=True)
            sam, st = idx.run_reads(path1=fs[0], path2=fs[1] if len(fs) == 2 else None, fastq=fmt == "-q", batch_reads=batch_reads,
                                    **reads)
            sam = idx.sam_header() + sam
            assert st["n_err_reads"] <= len(sor.flagged(case))
            assert refsets.sam_md5(sam, sor.flagged(case)) == REF["md5"][case], batch_reads
            summ = h2.format_align_summary(idx.align_counts(), discordant=not opts.get("no_discordant"), mixed=not opts.get("no_mixed"))
            if not sor.flagged(case):
                assert summ == REF["summary"][case], batch_reads
        check_shape(case, sam)
        batch = h2.ReadBatch.parse(path1=fs[0], path2=fs[1] if len(fs) == 2 else None, fastq=fmt == "-q", **reads)
        host = idx.format_sam(batch, idx.align(batch))
        assert idx.align_sam(batch) == host, "device SAM differs from the host formatter's"
    finally:
        idx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_cli_matches_reference(h2, so_dir, tmp_path, case):
    """hisat2-b200 with the reference's flags gives the reference's SAM, summary and warnings."""
    index, fs, fmt, flags, _, _ = sor.case_input(so_dir, case)
    reads = ["-1", fs[0], "-2", fs[1]] if len(fs) == 2 else ["-U", fs[0]]
    out = str(tmp_path / "o.sam")
    r = cli(["-x", index, fmt] + flags + reads + ["-S", out, "--batch", "512"])
    assert r.returncode == 0, r.stderr
    assert refsets.sam_md5(open(out, "rb").read(), sor.flagged(case)) == REF["md5"][case]
    err = r.stderr.decode()
    if not sor.flagged(case):
        assert refsets.summary_text(r.stderr) == REF["summary"][case]
    for w in REF["warnings"][case]:
        assert w in err.splitlines()
    assert ("Match bonus" in err) == bool(REF["warnings"][case])


@pytest.mark.gpu
@pytest.mark.parametrize("case", sor.READ_FILE_CASES)
def test_cli_read_files_follow_orientation(h2, so_dir, tmp_path, case):
    """--un-conc / --al-conc under --rf: the mates of the pairs that are (not) concordant in the RF sense, as the
    reference's wrapper writes them."""
    index, fs, fmt, flags, _, _ = sor.case_input(so_dir, case)
    un, al = str(tmp_path / "un.fa"), str(tmp_path / "al.fa")
    r = cli(["-x", index, fmt] + flags + ["-1", fs[0], "-2", fs[1], "-S", str(tmp_path / "o.sam"), "--quiet",
                                          "--un-conc", un, "--al-conc", al])
    assert r.returncode == 0, r.stderr
    import hashlib
    for k, want in REF["files"][case].items():
        kind, m = k.split("/")
        path = str(tmp_path / ("%s.%s.fa" % ("un" if kind == "un_conc" else "al", m)))
        assert hashlib.md5(open(path, "rb").read()).hexdigest() == want, k


@pytest.mark.gpu
def test_multi_handle_runs_refuse_different_settings(h2, so_dir):
    """run_reads_multi refuses handles whose orientation or N ceiling differ; peers take both from their source."""
    f1, f2 = sor.case_input(so_dir, "rf_pe_reads_rf")[1]
    idx = h2.Index(os.path.join(GOLDEN, "tiny"), pe_orient="rf", n_ceil_type="L", n_ceil_const=0.0, n_ceil_coeff=0.3)
    try:
        peer = idx.peer(0)
        try:
            sam, _ = idx.run_reads(path1=f1, path2=f2, peers=(peer,), batch_reads=64)
            alone, _ = idx.run_reads(path1=f1, path2=f2, batch_reads=64)
            assert sam == alone
        finally:
            peer.close()
        for other_opts in (dict(n_ceil_type="L", n_ceil_const=0.0, n_ceil_coeff=0.3), dict(pe_orient="rf")):
            other = h2.Index(os.path.join(GOLDEN, "tiny"), **other_opts)
            try:
                with pytest.raises(h2.Ht2GpuError):
                    idx.run_reads(path1=f1, path2=f2, peers=(other,), batch_reads=64)
            finally:
                other.close()
    finally:
        idx.close()
