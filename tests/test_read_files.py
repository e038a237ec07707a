"""--un, --al, --un-conc, --al-conc and --al-conc-disc against the unmodified reference: tools/readfiles_ref.py records
md5, size and record count of every read file the hisat2 wrapper writes (hisat2:546-650) in
tests/golden/read_files_sets.json.  Read files hold each record's original input text; which file a record goes to
follows the outcome byte the SAM counting pass stores per read or pair (ht2gpu_record_outcomes)."""
import bz2
import gzip
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

sys.path.insert(0, os.path.join(ROOT, "tools"))
import readfiles_ref  # noqa: E402

REF = readfiles_ref.load_expected()
CASES = sorted(readfiles_ref.CASES)
# the golden file names of each read file of the library ((output, mate) of api.READ_FILES)
GOLDEN_KEY = {("un", 0): "un", ("al", 0): "al"}
for _o in ("un_conc", "al_conc", "al_conc_disc"):
    for _m in (1, 2):
        GOLDEN_KEY[(_o, _m)] = "%s/%d" % (_o, _m)
CLI = os.path.join(ROOT, "hisat2_b200", "hisat2-b200")


@pytest.fixture(scope="session")
def data_dir(tmp_path_factory):
    return readfiles_ref.generate(str(tmp_path_factory.mktemp("readfiles")))


def summary(files):
    """{golden key: md5 / bytes / records} of {(output, mate): bytes}, with the record count taken from the input."""
    return {GOLDEN_KEY[k]: {"md5": hashlib.md5(v).hexdigest(), "bytes": len(v)} for k, v in files.items()}


def expect(case):
    return {k: {"md5": v["md5"], "bytes": v["bytes"]} for k, v in REF[case]["files"].items()}


def front_kw(case):
    return dict(readfiles_ref.CASES[case][3])


def test_golden_cases_cover_the_read_files():
    """Every output appears non-empty in some case, secondary records (-k 30 --secondary) and mixed / discordant pairs
    included, so that a recorded md5 cannot stand for a file that is always empty."""
    seen = set(k for c in CASES for k, v in REF[c]["files"].items() if v["records"])
    assert seen == set(GOLDEN_KEY.values())
    assert set(REF) == set(CASES)
    pe = REF["pe_hard20k"]["files"]
    assert pe["al_conc_disc/1"]["records"] > pe["al_conc/1"]["records"]           # mixed and discordant pairs
    assert REF["pe_hard20k_no_mixed"]["files"]["al_conc_disc/1"]["records"] < pe["al_conc_disc/1"]["records"]
    sec = REF["pe_sim10k_k30_secondary"]["files"]
    assert sec["al_conc/1"]["records"] + sec["un_conc/1"]["records"] == 10000      # one record per mate, not per alignment
    assert REF["se_reads_skip100_upto300"]["files"]["al"]["records"] + REF["se_reads_skip100_upto300"]["files"]["un"]["records"] == 300


def test_corpus_record_text_shapes(data_dir):
    """The corpus holds the shapes the read files must keep: blank lines (LF, CRLF) before the first FASTQ record,
    CRLF ends, '+name' lines, '%' and tabs in names, lower case, a record over 8 KiB, no final newline, and FASTA
    comment lines, an empty record and unnamed records."""
    fq = open(os.path.join(data_dir, "corpus.fq"), "rb").read()
    assert fq.startswith(b"\n\r\n@") and b"\r\n" in fq[3:] and not fq.endswith(b"\n")
    assert b"\n+q5" in fq and b"%20pct" in fq and b"\t" in fq and b"L" * 9000 in fq
    assert any(l.islower() for l in fq.split(b"\n")[3::4] if l)
    fa = open(os.path.join(data_dir, "corpus.fa"), "rb").read()
    assert fa.startswith(b"#") and b"\n; a semicolon" in fa and b">empty20\n>" in fa and b"\n>\n" in fa
    # the long record is cut at 8192 bytes, as the reference's parser keeps it
    assert REF["corpus_fq"]["files"]["al"]["bytes"] + REF["corpus_fq"]["files"]["un"]["bytes"] < len(fq)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the host build of the formatter's outcome bytes, and host-only routing
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="session")
def readsim(tmp_path_factory):
    """TEST-ONLY host builds of tests/hostsim/ht2_readsim.cpp, without and with the spliced-alignment pieces."""
    c = os.path.join(ROOT, "hisat2_b200", "csrc")
    out = []
    for name, defs in (("ht2_readsim", []), ("ht2_readsim_spliced", ["-DHT2_ENABLE_SPLICED"])):
        exe = str(tmp_path_factory.mktemp(name) / name)
        subprocess.run(["g++", "-O2", "-std=c++14"] + defs + ["-o", exe, os.path.join(ROOT, "tests", "hostsim", "ht2_readsim.cpp"),
                        os.path.join(c, "ht2_index.cpp"), os.path.join(c, "ht2_host.cpp"), "-lpthread"], check=True)
        out.append(exe)
    return tuple(out)


def fasta_slice(src, dst, r0, r1):
    recs = open(src, "rb").read().split(b">")[1:]
    open(dst, "wb").write(b"".join(b">" + r for r in recs[r0:r1]))
    return dst


# the host build reads plain FASTA / strict FASTQ and has no -5 / -3 / --phred64: these cases run on the device only
HOST_CASES = [c for c in CASES if not ({"trim5", "trim3", "phred64"} & set(front_kw(c))) and not c.startswith("corpus")]


def host_outcomes(bins, d, tmp_path, case):
    index, fs, fmt, _, opts = readfiles_ref.case_input(d, case)
    opts = dict(opts, **readfiles_ref.CASES[case][2])
    spliced = opts.pop("no_spliced_alignment", 1) == 0
    kv = (["spliced=1"] if spliced else []) + ["%s=%s" % x for x in sorted(opts.items())]
    fr = front_kw(case)
    if "skip" in fr:
        fs = [fasta_slice(f, str(tmp_path / ("slice%d.fa" % i)), fr["skip"], fr["skip"] + fr["upto"]) for i, f in enumerate(fs)]
    oc = str(tmp_path / "outcomes.bin")
    env = dict(os.environ, HT2_OPTS=",".join(kv), HT2_OUTCOMES=oc)
    r = subprocess.run([bins[1] if spliced else bins[0], index, fs[0], str(tmp_path / "o.sam")] + fs[1:], cwd=GOLDEN,
                       stderr=subprocess.PIPE, env=env)
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    return np.fromfile(oc, dtype=np.uint8)


@pytest.mark.parametrize("case", HOST_CASES)
def test_host_outcomes_route_to_reference_files(lib, readsim, data_dir, tmp_path, case):
    """Outcome bytes of the host build's counting pass + ht2gpu_route_reads reproduce every file of the wrapper."""
    from hisat2_b200 import route_reads
    out = host_outcomes(readsim, data_dir, tmp_path, case)
    _, fs, fmt, _, _ = readfiles_ref.case_input(data_dir, case)
    files = route_reads(out, path1=fs[0], path2=fs[1] if len(fs) == 2 else None, fastq=fmt == "-q", **front_kw(case))
    assert summary(files) == expect(case)


def test_route_reads_record_text_corpus(lib, data_dir):
    """Routing alone on the record-text corpus: with the reference's own outcomes (taken from its read files), the
    files come back byte for byte, the 8 KiB cut and the blank lines before the first FASTQ record included."""
    from hisat2_b200 import route_reads
    for case, fmt in (("corpus_fq", True), ("corpus_fa", False)):
        path = os.path.join(data_dir, readfiles_ref.CASES[case][0][1])
        n = REF[case]["files"]["al"]["records"] + REF[case]["files"]["un"]["records"]
        everything = route_reads(np.ones(n, np.uint8), path1=path, fastq=fmt, read_files=("al",))[("al", 0)]
        nothing = route_reads(np.zeros(n, np.uint8), path1=path, fastq=fmt, read_files=("al", "un"))
        assert nothing[("al", 0)] == b"" and nothing[("un", 0)] == everything
        if fmt:
            assert everything.startswith(b"\n\r\n@q0\r\n")
            assert b"L" * 9000 not in everything and b"_" + b"L" * 100 in everything


def test_route_reads_spans_and_mates(lib):
    """Pairs: mate 1 / mate 2 files, concordant vs not, al-conc-disc for any aligned mate; runs of consecutive records
    are one span."""
    from hisat2_b200 import route_reads, READ_FILES
    d1 = b"".join(b">r%d/1\nACGT\n" % i for i in range(4))
    d2 = b"".join(b">r%d/2\nTTTT\n" % i for i in range(4))
    out = np.array([7, 0, 3, 1], np.uint8)     # concordant, unaligned, discordant, mate 1 only
    f = route_reads(out, data1=d1, data2=d2, read_files=READ_FILES)
    rec = lambda d, i: d.split(b">")[1:][i] and b">" + d.split(b">")[1:][i]
    assert f[("al_conc", 1)] == rec(d1, 0) and f[("al_conc", 2)] == rec(d2, 0)
    assert f[("un_conc", 1)] == rec(d1, 1) + rec(d1, 2) + rec(d1, 3)
    assert f[("al_conc_disc", 2)] == rec(d2, 0) + rec(d2, 2) + rec(d2, 3)
    assert f[("un", 0)] == b"" and f[("al", 0)] == b""
    single = route_reads(np.array([1, 0], np.uint8), data1=b">a\nAC\n>b\nGT", read_files=READ_FILES)
    assert single[("al", 0)] == b">a\nAC\n" and single[("un", 0)] == b">b\nGT" and single[("un_conc", 1)] == b""


def test_route_reads_errors(lib):
    from hisat2_b200 import route_reads, Ht2GpuError
    with pytest.raises(Ht2GpuError, match="do not cover"):
        route_reads(np.zeros(3, np.uint8), data1=b">a\nAC\n>b\nGT\n")
    with pytest.raises(ValueError):
        route_reads(np.zeros(2, np.uint8), data1=b">a\nAC\n>b\nGT\n", read_files=("unaligned",))
    with pytest.raises(Ht2GpuError, match="could not open"):
        route_reads(np.zeros(0, np.uint8), path1="/nonexistent/reads.fa")


def run_cli(args, cwd):
    return subprocess.run([CLI] + args, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.PIPE)


def test_cli_names_and_unwritable_path_without_device(lib, tmp_path):
    """The wrapper's names, opened before anything else runs (so without a usable index or device the files exist,
    empty): a directory gives <opt>-seqs / <opt>-mate.1, '%' becomes 1 / 2, .1 / .2 goes before the last extension or
    is appended.  An unwritable path is an error with a message and a nonzero exit, and no compressor outlives it."""
    if not os.path.exists(CLI):
        from hisat2_b200 import build
        build.build_cli()
    (tmp_path / "d").mkdir()
    fa = tmp_path / "r.fa"
    fa.write_bytes(b">a\nACGT\n")
    r = run_cli(["-x", str(tmp_path / "missing"), "-f", "-U", str(fa), "--un", "d", "--un-conc", "d",
                 "--al-conc", "p%.fq", "--al-conc-disc-gz", "x.fq.gz", "--al-bz2", "b.bz2"], str(tmp_path))
    assert r.returncode != 0
    for f in ("d/un-seqs", "b.bz2", "d/un-conc-mate.1", "d/un-conc-mate.2", "p1.fq", "p2.fq", "x.fq.1.gz", "x.fq.2.gz"):
        assert (tmp_path / f).exists(), f
    assert gzip.decompress((tmp_path / "x.fq.1.gz").read_bytes()) == b"" and bz2.decompress((tmp_path / "b.bz2").read_bytes()) == b""
    r = run_cli(["-x", str(tmp_path / "missing"), "-f", "-U", str(fa), "--un-gz", str(tmp_path / "no" / "such" / "dir" / "u.gz")], str(tmp_path))
    assert r.returncode != 0 and b"could not open --un output file" in r.stderr


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def h2(lib):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import hisat2_b200
    return hisat2_b200


def open_case(h2, d, case, device=0):
    index, fs, fmt, _, opts = readfiles_ref.case_input(d, case)
    idx = h2.Index(os.path.join(GOLDEN, index), device=device, **dict(opts, **readfiles_ref.CASES[case][2]))
    return idx, fs, fmt


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_device_read_files_match_reference(h2, data_dir, case):
    """ht2gpu_run_reads_routed in batches of 128 reads (many batches, every slot): every file equals the wrapper's, the
    SAM equals the run without routing, and (where the host build runs the case) the device's outcome bytes equal the
    host build's."""
    idx, fs, fmt = open_case(h2, data_dir, case)
    kw = dict(path1=fs[0], path2=fs[1] if len(fs) == 2 else None, fastq=fmt == "-q", batch_reads=128, **front_kw(case))
    try:
        sam, st, files = idx.run_reads(read_files=h2.READ_FILES, **kw)
        plain, _ = idx.run_reads(**kw)
    finally:
        idx.close()
    assert st["n_batches"] >= 2 and st["n_err_reads"] == 0
    assert sam == plain
    assert summary(files) == expect(case)
    assert st["route_bytes"] == sum(len(v) for v in files.values())
    # the reference's SAM for the same input: a read file difference is then a routing difference
    assert readfiles_ref.refsets.sam_md5(sam_header(h2, data_dir, case) + sam) == REF[case]["sam_md5"]


def sam_header(h2, d, case):
    idx, _, _ = open_case(h2, d, case)
    try:
        return idx.sam_header()
    finally:
        idx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", HOST_CASES)
def test_device_outcomes_equal_host_build(h2, readsim, data_dir, tmp_path, case):
    """ht2gpu_align_sam with ht2gpu_record_outcomes: the device bytes equal the host build's, and route_reads of
    them gives the reference's files."""
    want = host_outcomes(readsim, data_dir, tmp_path, case)
    idx, fs, fmt = open_case(h2, data_dir, case)
    fr = front_kw(case)
    try:
        batch = h2.ReadBatch.parse(path1=fs[0], path2=fs[1] if len(fs) == 2 else None, fastq=fmt == "-q", **fr)
        idx.record_outcomes(True)
        idx.align_sam(batch)
        got = idx.unit_outcomes()
        idx.record_outcomes(False)
    finally:
        idx.close()
    assert np.array_equal(got, want)
    files = h2.route_reads(got, path1=fs[0], path2=fs[1] if len(fs) == 2 else None, fastq=fmt == "-q", **fr)
    assert summary(files) == expect(case)


@pytest.mark.gpu
def test_device_read_files_two_gpus(h2, data_dir):
    """--gpus 2: batches alternate between devices; the files are still the wrapper's."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one CUDA device")
    for case in ("pe_hard20k", "edge_fq"):
        idx, fs, fmt = open_case(h2, data_dir, case)
        other = idx.peer(1)
        try:
            _, _, files = idx.run_reads(path1=fs[0], path2=fs[1] if len(fs) == 2 else None, fastq=fmt == "-q", batch_reads=128,
                                        peers=(other,), read_files=h2.READ_FILES, **front_kw(case))
        finally:
            other.close()
            idx.close()
        assert summary(files) == expect(case)


def golden_bytes_md5(case, key):
    return REF[case]["files"][key]["md5"]


@pytest.mark.gpu
def test_cli_read_files(h2, data_dir, tmp_path):
    """The CLI: every option spelling, -gz / -bz2 (decompressed bytes compared), directory, '%' and extension names,
    with --no-unal and -S /dev/null."""
    md5 = lambda b: hashlib.md5(b).hexdigest()
    _, fs, _, _, _ = readfiles_ref.case_input(data_dir, "pe_hard20k")
    (tmp_path / "dir").mkdir()
    r = run_cli(["-x", os.path.join(GOLDEN, "tiny"), "-f", "--no-spliced-alignment", "-1", fs[0], "-2", fs[1], "--batch", "4096",
                 "--no-unal", "-S", "/dev/null", "--un-conc-gz", "uc%.fa.gz", "--al-conc-bz2", "ac.fa.bz2", "--al-conc-disc", "dir",
                 "--un", "un.fa", "--al-gz", "al.fa.gz"], str(tmp_path))
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    got = {"un_conc/1": gzip.decompress((tmp_path / "uc1.fa.gz").read_bytes()),
           "un_conc/2": gzip.decompress((tmp_path / "uc2.fa.gz").read_bytes()),
           "al_conc/1": bz2.decompress((tmp_path / "ac.fa.1.bz2").read_bytes()),   # .1 / .2 before the last extension
           "al_conc/2": bz2.decompress((tmp_path / "ac.fa.2.bz2").read_bytes()),
           "al_conc_disc/1": (tmp_path / "dir" / "al-conc-disc-mate.1").read_bytes(),
           "al_conc_disc/2": (tmp_path / "dir" / "al-conc-disc-mate.2").read_bytes()}
    for k, v in got.items():
        assert md5(v) == golden_bytes_md5("pe_hard20k", k), k
    assert (tmp_path / "un.fa").read_bytes() == b"" and gzip.decompress((tmp_path / "al.fa.gz").read_bytes()) == b""
    # unpaired FASTQ, the remaining spellings
    _, fs, _, _, _ = readfiles_ref.case_input(data_dir, "corpus_fq")
    r = run_cli(["-x", os.path.join(GOLDEN, "tiny"), "-q", "--no-spliced-alignment", "-U", fs[0], "-S", str(tmp_path / "o.sam"),
                 "--un-bz2", "u.bz2", "--al", "dir", "--un-conc", "never.fq", "--al-conc-gz", "never2.gz",
                 "--al-conc-disc-gz", "never3.gz", "--al-conc-disc-bz2", "never4.bz2"], str(tmp_path))
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    assert md5(bz2.decompress((tmp_path / "u.bz2").read_bytes())) == golden_bytes_md5("corpus_fq", "un")
    assert md5((tmp_path / "dir" / "al-seqs").read_bytes()) == golden_bytes_md5("corpus_fq", "al")
    assert (tmp_path / "never.1.fq").read_bytes() == b"" and (tmp_path / "never4.1.bz2").exists()
    # an unwritable path: a message and a nonzero exit before any alignment
    r = run_cli(["-x", os.path.join(GOLDEN, "tiny"), "-q", "--no-spliced-alignment", "-U", fs[0], "-S", "/dev/null",
                 "--al-conc", str(tmp_path / "missing" / "x.fq")], str(tmp_path))
    assert r.returncode != 0 and b"could not open --al-conc mate-1 output file" in r.stderr
