"""Read-file lists (-1 a1,a2 -2 b1,b2 -U u1,u2) against the unmodified reference: tools/multi_input_ref.py records the
SAM md5, the alignment summary and the read files of every case in tests/golden/multi_input_sets.json.  The -1 files
back to back and the -2 files back to back are one stream of pairs, the -U files one stream of unpaired reads aligned
after the pairs; read ids, -s and -u count per stream."""
import hashlib
import os
import subprocess
import sys

import pytest

from conftest import GOLDEN, ROOT

sys.path.insert(0, os.path.join(ROOT, "tools"))
import multi_input_ref as mref  # noqa: E402
import refsets  # noqa: E402

REF = mref.load_expected()
CASES = sorted(mref.CASES)
CLI = os.path.join(ROOT, "hisat2_b200", "hisat2-b200")
GOLDEN_KEY = {("un", 0): "un", ("al", 0): "al"}
for _o in ("un_conc", "al_conc", "al_conc_disc"):
    for _m in (1, 2):
        GOLDEN_KEY[(_o, _m)] = "%s/%d" % (_o, _m)


@pytest.fixture(scope="session")
def data_dir(tmp_path_factory):
    return mref.generate(str(tmp_path_factory.mktemp("multi_input")))


def run_cli(args, cwd):
    if not os.path.exists(CLI):
        from hisat2_b200 import build
        build.build_cli()
    return subprocess.run([CLI] + args, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.PIPE)


def bounds(files):
    """Record ordinals at which the files of a list end."""
    out, n = [], 0
    for f in files:
        n += f[3] - f[2]
        out.append(n)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_golden_cases_cover_the_streams():
    """The goldens cover what they claim: cases with both streams non-empty (the summary has paired and unpaired
    sections), a -u case that drops every unpaired read and one that cuts the unpaired stream, -1 and -2 files that end
    at different records, plain / gzip / BGZF in one list, and read files with records in every output kind."""
    both = [c for c in CASES if mref.CASES[c]["m1"] and mref.CASES[c]["u"]]
    assert len(both) >= 6
    for c in both:
        s = REF[c]["summary"]
        if c != "mixed_upto100":
            assert ("were paired" in s and "were unpaired" in s) or ("Total pairs" in s and "Total unpaired reads" in s), c
    # -u 100 < 150 pairs: no unpaired read; -u 250: 150 pairs and 250 unpaired reads
    assert "were unpaired" not in REF["mixed_upto100"]["summary"] and REF["mixed_upto100"]["summary"].startswith("100 reads")
    assert REF["mixed_upto250"]["summary"].startswith("400 reads")
    assert REF["mixed_skip40"]["summary"].startswith("470 reads")   # -s 40 skips 40 pairs and 40 unpaired reads
    for c in CASES:
        m1, m2 = mref.CASES[c]["m1"], mref.CASES[c]["m2"]
        if len(m1) > 1:
            assert bounds(m1)[:-1] != bounds(m2)[:-1] and bounds(m1)[-1] == bounds(m2)[-1], c
    comps = {f[4] for f in mref.CASES["se_fq_plain_gz_bgzf"]["u"]}
    assert comps == {None, "gz", "bgzf"}
    files = REF["mixed_read_files_no_unal_new_summary"]["files"]
    assert all(files[k]["records"] > 0 for k in ("un", "al", "un_conc/1", "al_conc/1", "al_conc_disc/1")), files


def test_cli_list_errors_without_device(tmp_path):
    """Errors found before any device is opened: -1 and -2 lists of different lengths, -1 without -2 (the reference's
    message, hisat2.cpp:1911-1913), and stdin named twice."""
    fa = tmp_path / "r.fa"
    fa.write_bytes(b">a\nACGTACGT\n")
    x = ["-x", str(tmp_path / "missing"), "-f"]
    r = run_cli(x + ["-1", "%s,%s" % (fa, fa), "-2", str(fa)], str(tmp_path))
    assert r.returncode == 1
    assert b"Error: 2 mate files/sequences were specified with -1, but 1\nmate files/sequences were specified with -2." in r.stderr
    r = run_cli(x + ["-U", str(fa), "-1", str(fa)], str(tmp_path))
    assert r.returncode == 1 and b"1 mate files/sequences were specified with -1, but 0" in r.stderr
    r = run_cli(x + ["-1", str(fa), "-1", str(fa), "-2", "%s,,%s" % (fa, fa)], str(tmp_path))   # repeated, empty names dropped
    assert r.returncode != 0 and b"mate files/sequences" not in r.stderr
    r = run_cli(x + ["-U", "-", "-1", "-", "-2", str(fa)], str(tmp_path))
    assert r.returncode == 1 and b"standard input ('-') can be read only once" in r.stderr


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def h2(lib):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import hisat2_b200
    return hisat2_b200


def open_case(h2, case, device=0):
    c = mref.CASES[case]
    idx = h2.Index(os.path.join(GOLDEN, c["index"]), device=device, **mref.lib_opts(case))
    if c.get("sam_output"):
        idx.set_sam_output(**c["sam_output"])
    return idx


def run_case(h2, idx, d, case, batch_reads, peers=()):
    """(SAM with header, summary text, read files or None) of the library entry point on a case."""
    c = mref.CASES[case]
    p = lambda fs: [os.path.join(d, f[0]) for f in fs]
    kw = dict(path1=p(c["m1"]), path2=p(c["m2"]), unpaired=p(c["u"]), fastq=c["fmt"] == "-q", batch_reads=batch_reads,
              peers=peers, **c.get("front", {}))
    idx.align_counts(peers=peers, reset=True)
    if c.get("read_files"):
        sam, st, files = idx.run_reads(read_files=h2.READ_FILES, **kw)
    else:
        (sam, st), files = idx.run_reads(**kw), None
    assert st["n_err_reads"] == 0
    summ = h2.format_align_summary(idx.align_counts(peers=peers), new_style=bool(c.get("new_summary")))
    return idx.sam_header() + sam, summ, st, files


def check(case, sam, summ, files):
    e = REF[case]
    assert refsets.sam_md5(sam) == e["sam_md5"]
    assert summ == e["summary"]
    if files is not None:
        got = {GOLDEN_KEY[k]: {"md5": hashlib.md5(v).hexdigest(), "bytes": len(v)} for k, v in files.items()}
        assert got == {k: {"md5": v["md5"], "bytes": v["bytes"]} for k, v in e["files"].items()}


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_library_lists_match_reference(h2, data_dir, case):
    """ht2gpu_run_reads_files in one large batch per stream and in batches of 64 reads (batches that cross file
    boundaries, a short last batch of pairs before the unpaired reads)."""
    idx = open_case(h2, case)
    try:
        for batch_reads in (0, 64):
            sam, summ, st, files = run_case(h2, idx, data_dir, case, batch_reads)
            check(case, sam, summ, files)
            if batch_reads:
                assert st["n_batches"] >= 3
    finally:
        idx.close()


@pytest.mark.gpu
def test_library_gunzip_stats_add_up(h2, data_dir):
    """The inflate stats of a run sum over its gzip and BGZF files."""
    c = mref.CASES["se_fq_plain_gz_bgzf"]
    idx = open_case(h2, "se_fq_plain_gz_bgzf")
    try:
        run_case(h2, idx, data_dir, "se_fq_plain_gz_bgzf", 64)
        g = idx.gunzip_stats()
    finally:
        idx.close()
    gz = [f for f in c["u"] if f[4]]
    assert g["in_bytes"] == sum(os.path.getsize(os.path.join(data_dir, f[0])) for f in gz)
    assert g["out_bytes"] == sum(os.path.getsize(os.path.join(data_dir, "plain", f[0])) for f in gz)
    assert g["members"] >= 3


@pytest.mark.gpu
def test_library_lists_two_gpus(h2, data_dir):
    """--gpus 2: batches alternate between the devices, across file and stream boundaries."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one CUDA device")
    for case in ("mixed_read_files_no_unal_new_summary", "pe_two_lanes"):
        idx = open_case(h2, case)
        other = idx.peer(1)
        try:
            sam, summ, _, files = run_case(h2, idx, data_dir, case, 64, peers=(other,))
        finally:
            other.close()
            idx.close()
        check(case, sam, summ, files)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_cli_lists_match_reference(h2, data_dir, tmp_path, case):
    """hisat2-b200 with the case's comma-separated lists (gzip files as they are), -U before or after -1 / -2."""
    c = mref.CASES[case]
    args = ["-x", os.path.join(GOLDEN, c["index"]), c["fmt"]] + mref.base_flags(case) + list(c.get("flags", [])) + \
        mref.reads_args(data_dir, case) + ["--batch", "100", "-S", str(tmp_path / "o.sam"), "--summary-file", str(tmp_path / "s.txt")]
    if c.get("read_files"):
        args += ["--un", "un.fq", "--al", "al.fq", "--un-conc", "uc%.fq", "--al-conc", "ac%.fq", "--al-conc-disc", "acd%.fq"]
    r = run_cli(args, str(tmp_path))
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    files = None
    if c.get("read_files"):
        names = {("un", 0): "un.fq", ("al", 0): "al.fq", ("un_conc", 1): "uc1.fq", ("un_conc", 2): "uc2.fq",
                 ("al_conc", 1): "ac1.fq", ("al_conc", 2): "ac2.fq", ("al_conc_disc", 1): "acd1.fq", ("al_conc_disc", 2): "acd2.fq"}
        files = {k: (tmp_path / v).read_bytes() for k, v in names.items()}
    check(case, (tmp_path / "o.sam").read_bytes(), (tmp_path / "s.txt").read_text(), files)
