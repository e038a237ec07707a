"""The reference's remaining SAM record options: --rna-strandness (XS:A of every aligned record), --remove-chrname /
--add-chrname (the handle's reference names in @SQ, RNAME, RNEXT and the splice-site files), --no-templatelen-adjustment
(TLEN of concordant pairs) and --sam-no-qname-trunc (the whole read name as QNAME).  tools/sam_record_ref.py records the
unmodified reference's SAM md5 per case, its --novel-splicesite-outfile text and its argument errors in
tests/golden/sam_record_sets.json."""
import os
import subprocess
import sys

import pytest

from conftest import GOLDEN, ROOT, sam_lines

sys.path.insert(0, os.path.join(ROOT, "tools"))
import refsets  # noqa: E402
import sam_record_ref as srr  # noqa: E402

REF = srr.load_expected()
REF_SETS = refsets.load_expected()
CASES = sorted(srr.CASES)
REFBIN = refsets.REFBIN


@pytest.fixture(scope="session")
def rec_dir(tmp_path_factory):
    return srr.generate(str(tmp_path_factory.mktemp("samrec")))


def records(sam):
    """The fields of every record (QNAMEs without tabs: the qname cases are checked apart, by qname_shape)."""
    return [l.split(b"\t") for l in sam.splitlines() if l and not l.startswith(b"@")]


def printed_names(path, paired):
    """The QNAMEs the reference prints for a FASTA / FASTQ file under --sam-no-qname-trunc: the whole name line, with
    a mate's trailing /1 or /2 left out, and the read ordinal for an unnamed read."""
    lines = open(path, "rb").read().split(b"\n")
    step = 4 if path.endswith(".fq") else 2
    out = []
    for i, l in enumerate(lines[0:len(lines) - 1:step]):
        n = l[1:] or str(i).encode()
        if paired and n[-2:] in (b"/1", b"/2"):
            n = n[:-2]
        out.append(n)
    return out


def qname_shape(case, sam, fs):
    """Default: every QNAME is cut at white space and at 255 characters.  --sam-no-qname-trunc: every read's whole
    name starts a record, and such names are longer than 255 characters or hold a space or a tab."""
    lines = [l for l in sam.splitlines() if l and not l.startswith(b"@")]
    names = printed_names(fs[0], len(fs) == 2)
    if srr.CASES[case].get("out", {}).get("no_qname_trunc"):
        assert all(any(l.startswith(n + b"\t") for l in lines) for n in set(names))
        assert any(len(n) > 255 for n in names) and any(b" " in n for n in names) and any(b"\t" in n for n in names)
    else:
        q = [l.split(b"\t")[0] for l in lines]
        assert all(len(x) <= 255 and b" " not in x for x in q) and any(len(x) == 255 for x in q)


def xs_expected(flag, strandness):
    """sam.h:938-963 restated: the XS:A of an aligned record from FLAG bits 16 (reverse), 64 / 128 (mate 1 / 2)."""
    mate1 = not flag & 128          # an unpaired read takes the mate-1 rule
    fw = not flag & 16
    if mate1:
        minus = strandness in ("R", "RF") if fw else strandness in ("F", "FR")
    else:
        minus = strandness == "FR" if fw else strandness == "RF"
    return b"-" if minus else b"+"


def check_shape(case, sam, fs, default_sam=None):
    """What each option visibly does, so that a recorded md5 cannot stand for a case that tests nothing."""
    c = srr.CASES[case]
    out = c.get("out", {})
    if c["src"][0] == "qname":
        qname_shape(case, sam, fs)
        return
    recs = records(sam)
    assert recs
    s = out.get("rna_strandness")
    if s:
        aligned = [r for r in recs if not int(r[1]) & 4]
        assert aligned
        for r in aligned:
            xs = [f for f in r[11:] if f.startswith(b"XS:A:")]
            assert xs == [b"XS:A:" + xs_expected(int(r[1]), s)], r[:2]
        assert not any(f.startswith(b"XS:A:") for r in recs if int(r[1]) & 4 for f in r[11:])
        assert {xs_expected(int(r[1]), s) for r in aligned} == {b"+", b"-"}
    if out.get("no_templatelen_adjustment") and default_sam is not None:
        d = records(default_sam)
        assert len(d) == len(recs)
        conc = [(a, b) for a, b in zip(recs, d) if int(a[1]) & 2]
        assert conc and any(a[8] != b[8] for a, b in conc)
        assert all(abs(int(a[8])) >= abs(int(b[8])) for a, b in conc)
    names = c.get("chr_names")
    if names:
        sq = [l.split(b"\t")[1][3:] for l in sam.splitlines() if l.startswith(b"@SQ")]
        want = {"remove": [b"A", b"B"], "add": [b"chrA", b"chrB"]}[names]
        assert sq == want
        assert {r[2] for r in recs} - {b"*"} <= set(want) and {r[2] for r in recs} & set(want)
        assert {r[6] for r in recs} - {b"*", b"="} <= set(want)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the host build of the same formatter (tests/hostsim/ht2_samoptsim.cpp)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="session")
def samoptsim(tmp_path_factory):
    """TEST-ONLY host build of ht2_hostsim with every SAM output setting and the reference-name table."""
    c = os.path.join(ROOT, "hisat2_b200", "csrc")
    exe = str(tmp_path_factory.mktemp("samoptsim") / "ht2_samoptsim")
    subprocess.run(["g++", "-O2", "-std=c++14", "-o", exe, os.path.join(ROOT, "tests", "hostsim", "ht2_samoptsim.cpp"),
                    os.path.join(c, "ht2_index.cpp"), os.path.join(c, "ht2_host.cpp"), "-lpthread"], check=True)
    return exe


def out_env(out, chr_names):
    so = ["chr_names=%d" % {None: 0, "remove": 1, "add": 2}[chr_names]]
    for k, v in sorted(out.items()):
        if k == "rg_id":
            so.append("rg_id=%s" % v)
        elif k == "rna_strandness":
            so.append("rna_strandness=%d" % {"F": 1, "R": 2, "FR": 3, "RF": 4}[v])
        else:
            so.append("%s=%d" % (k, int(v)))
    return ",".join(so)


def hostsim(exe, d, tmp_path, case, out=None):
    """(SAM, novel-splice-site text or None) of the host build on a case; out overrides the case's SAM settings."""
    index, fs, _, _, opts, ss = srr.case_input(d, case)
    opts = dict(opts)
    chr_names = opts.pop("chr_names", None)
    spliced = opts.pop("no_spliced_alignment", 1) == 0
    kv = (["spliced=1"] if spliced else []) + ["%s=%s" % x for x in sorted(opts.items())]
    o, novel = str(tmp_path / "o.sam"), str(tmp_path / "novel.txt")
    env = dict(os.environ, HT2_OPTS=",".join(kv), HT2_SAM_OUTPUT=out_env(srr.CASES[case].get("out", {}) if out is None else out, chr_names))
    if ss:
        env["HT2_SS"] = ss
    if srr.CASES[case].get("novel"):
        env["HT2_SS_OUT"] = novel
    r = subprocess.run([exe, index, fs[0], o] + fs[1:], cwd=GOLDEN, stderr=subprocess.PIPE, env=env)
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    assert r.stderr.count(b"err=") <= len(srr.flagged(case))   # a flagged read may fit without the known sites
    return open(o, "rb").read(), (open(novel).read() if srr.CASES[case].get("novel") else None)


@pytest.mark.parametrize("case", CASES)
def test_host_build_matches_reference(samoptsim, rec_dir, tmp_path, case):
    """Every case through the host build: the md5 of the reference's SAM (header without @PG), the reference's
    --novel-splicesite-outfile byte for byte, and the shape each option gives its records."""
    sam, novel = hostsim(samoptsim, rec_dir, tmp_path, case)
    assert refsets.sam_md5(sam, srr.flagged(case)) == REF["md5"][case]
    if case in REF["novel"]:
        assert novel == REF["novel"][case] and novel.startswith("A\t")
    default = None
    if srr.CASES[case].get("out", {}).get("no_templatelen_adjustment"):
        default, _ = hostsim(samoptsim, rec_dir, tmp_path, case, out=dict(srr.CASES[case]["out"], no_templatelen_adjustment=False))
    check_shape(case, sam, srr.case_input(rec_dir, case)[1], default)


def test_defaults_give_the_recorded_sam(samoptsim, rec_dir, tmp_path):
    """Zero settings print today's bytes: the default runs of the TLEN sets equal refsets' recorded md5."""
    for case, key in (("tlen_spliced_ss_sim_pe", "spliced/ss_sim_pe"), ("tlen_spliced_graph_ss_sim_pe", "spliced/graph_ss_sim_pe")):
        sam, _ = hostsim(samoptsim, rec_dir, tmp_path, case, out={})
        assert refsets.sam_md5(sam, srr.flagged(case)) == REF_SETS["md5"][key]


def test_recorded_cases_differ_from_the_defaults():
    """Each option changes the reference's output on its cases (same-input pairs with different md5s)."""
    m = REF["md5"]
    assert m["strand_F_se_reads"] != m["strand_R_se_reads"]
    assert m["strand_FR_pe_hard20k"] != m["strand_RF_pe_hard20k"]
    assert m["qname_pe_fa"] != m["qname_pe_fa_whole"] and m["qname_se_fa"] != m["qname_se_fa_whole"]
    assert m["tlen_spliced_ss_sim_pe"] != REF_SETS["md5"]["spliced/ss_sim_pe"]
    assert m["names_remove_ss_renamed"] != m["names_remove_ss_chr"]
    # the two indexes of the same sequence print the same names once both are renamed the same way
    assert m["names_remove_nochr_pe_reads"] == m["names_remove_pe_reads"]


def cli(args, **kw):
    exe = os.path.join(ROOT, "hisat2_b200", "hisat2-b200")
    return subprocess.run([exe] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, cwd=GOLDEN, **kw)


@pytest.fixture(scope="module")
def cli_built(lib):
    from hisat2_b200 import build
    build.build_cli()


@pytest.mark.parametrize("err", sorted(srr.ERRORS))
def test_cli_argument_errors(cli_built, rec_dir, tmp_path, err):
    """Both --remove-chrname and --add-chrname, or a --rna-strandness other than F, R, FR, RF: the reference's message
    and exit status, before any device is opened."""
    line, status = REF["errors"][err]
    r = cli(["-x", "tiny", "-f", "--no-spliced-alignment", "-U", os.path.join(rec_dir, "reads_1.fa"), "-S", str(tmp_path / "o.sam")] +
            srr.ERRORS[err])
    assert r.returncode == status
    assert r.stderr.decode().splitlines()[0] == line


def test_python_settings_are_checked(lib):
    from hisat2_b200 import api
    with pytest.raises(ValueError):
        api._options(lib, dict(chr_names="both"))
    assert api._options(lib, dict(chr_names="add")).chr_names == 2


@pytest.mark.parametrize("chr_names", [3, 7, -1])
def test_open_refuses_bad_chr_names(lib, chr_names):
    """ht2gpu_open refuses both rename flags (with the reference's message) and unknown values before it uses a device."""
    import ctypes as C
    from hisat2_b200 import api
    o = api.Options()
    lib.ht2gpu_default_options(C.byref(o))
    o.chr_names = chr_names
    h = C.c_void_p()
    rc = lib.ht2gpu_open(os.path.join(GOLDEN, "tiny").encode(), C.byref(o), C.byref(h))
    msg = lib.ht2gpu_last_error(h).decode()
    lib.ht2gpu_close(h)
    assert rc == -1
    assert (msg == REF["errors"]["both_chrname"][0][len("Error: "):]) == (chr_names == 3)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: ht2gpu_run_reads, ht2gpu_align_sam and the CLI
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def h2(lib):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import hisat2_b200
    return hisat2_b200


def open_case(h2, d, case):
    index, fs, fmt, _, opts, ss = srr.case_input(d, case)
    idx = h2.Index(os.path.join(GOLDEN, index), **opts)
    if ss:
        idx.load_splicesites(ss)
    out = dict(srr.CASES[case].get("out", {}))
    idx.set_sam_output(**out)
    return idx, fs, fmt


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_device_matches_reference(h2, rec_dir, tmp_path, case):
    """Every case through ht2gpu_run_reads in one batch per stream and in 64-read batches (many batches; long names
    re-run the SAM kernels), the --novel-splicesite-outfile, and ht2gpu_align_sam against the host formatter."""
    idx, fs, fmt = open_case(h2, rec_dir, case)
    try:
        novel = srr.CASES[case].get("novel")
        for batch_reads in (0, 64):
            if novel:
                idx.collect_splicesites(True)
            sam, st = idx.run_reads(path1=fs[0], path2=fs[1] if len(fs) == 2 else None, fastq=fmt == "-q", batch_reads=batch_reads)
            sam = idx.sam_header() + sam
            assert st["n_err_reads"] <= len(srr.flagged(case))
            assert refsets.sam_md5(sam, srr.flagged(case)) == REF["md5"][case], batch_reads
            if novel:
                p = str(tmp_path / "novel.txt")
                idx.write_novel_splicesites(p)
                idx.collect_splicesites(False)
                assert open(p).read() == REF["novel"][case]
        check_shape(case, sam, fs)
        batch = h2.ReadBatch.parse(path1=fs[0], path2=fs[1] if len(fs) == 2 else None, fastq=fmt == "-q")
        host = idx.format_sam(batch, idx.align(batch))
        assert idx.align_sam(batch) == host, "device SAM differs from the host formatter's"
    finally:
        idx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_cli_matches_reference(h2, rec_dir, tmp_path, case):
    """hisat2-b200 with the reference's flags gives the reference's SAM (and novel splice sites); the reference is
    re-run here when oracle/_ref is present."""
    index, fs, fmt, flags, _, _ = srr.case_input(rec_dir, case)
    reads = ["-1", fs[0], "-2", fs[1]] if len(fs) == 2 else ["-U", fs[0]]
    out, novel = str(tmp_path / "o.sam"), str(tmp_path / "novel.txt")
    extra = ["--novel-splicesite-outfile", novel] if srr.CASES[case].get("novel") else []
    r = cli(["-x", index, fmt] + flags + extra + reads + ["-S", out, "--quiet", "--batch", "512"])
    assert r.returncode == 0, r.stderr
    sam = open(out, "rb").read()
    assert refsets.sam_md5(sam, srr.flagged(case)) == REF["md5"][case]
    if extra:
        assert open(novel).read() == REF["novel"][case]
    if os.path.exists(REFBIN):
        ro, rn = str(tmp_path / "ref.sam"), str(tmp_path / "ref_novel.txt")
        subprocess.run([REFBIN, fmt, "-x", os.path.join(GOLDEN, index)] + flags + (["--novel-splicesite-outfile", rn] if extra else []) +
                       reads + ["-S", ro, "--reorder", "-p", "4"], check=True, stderr=subprocess.DEVNULL)
        keep = lambda t: [l for l in sam_lines(t) if l.split(b"\t")[0] not in [n.encode() for n in srr.flagged(case)]]
        assert keep(sam) == keep(open(ro, "rb").read())
        if extra:
            assert open(novel).read() == open(rn).read()


@pytest.mark.gpu
def test_multi_handle_runs_refuse_different_settings(h2, rec_dir):
    """run_reads_multi refuses handles whose new SAM settings or reference names differ; peers inherit both."""
    f = os.path.join(rec_dir, "reads_1.fa")
    idx = h2.Index(os.path.join(GOLDEN, "tiny"), chr_names="remove")
    try:
        on = dict(rna_strandness="RF", no_qname_trunc=True, no_templatelen_adjustment=True)
        idx.set_sam_output(**on)
        peer = idx.peer(0)
        try:
            sam, _ = idx.run_reads(path1=f, peers=(peer,), batch_reads=64)
            alone, _ = idx.run_reads(path1=f, batch_reads=64)
            assert sam == alone and b"\tXS:A:" in sam and b"\tA\t" in sam
            for k, off in (("rna_strandness", None), ("no_qname_trunc", False), ("no_templatelen_adjustment", False)):
                peer.set_sam_output(**dict(on, **{k: off}))
                with pytest.raises(h2.Ht2GpuError):
                    idx.run_reads(path1=f, peers=(peer,), batch_reads=64)
        finally:
            peer.close()
        other = h2.Index(os.path.join(GOLDEN, "tiny"))
        try:
            other.set_sam_output(**on)
            with pytest.raises(h2.Ht2GpuError):
                idx.run_reads(path1=f, peers=(other,), batch_reads=64)
        finally:
            other.close()
    finally:
        idx.close()


@pytest.mark.gpu
def test_whole_names_grow_the_sam_text(h2, tmp_path):
    """Reads of segments tiny.fa holds twice, named with 500-character names and a comment, under -k 30 --secondary and
    --sam-no-qname-trunc: two records per read print each whole name twice, more text than the first estimate, so the
    SAM kernels run again.  The device text equals the host formatter's and every QNAME is the whole name."""
    d = refsets.generate_repeats(str(tmp_path))
    recs = open(os.path.join(d, "rep_1.fa")).read().split(">")[1:]
    f = str(tmp_path / "long.fa")
    with open(f, "w") as o:
        for i, r in enumerate(recs):
            name, seq = r.split("\n", 1)
            o.write(">%s_%s %s\n%s" % (name, "x" * 500, "c%d\tz" % i, seq))
    idx = h2.Index(os.path.join(GOLDEN, "tiny"), khits=30, secondary=1)
    try:
        idx.set_sam_output(no_qname_trunc=True)
        batch = h2.ReadBatch.parse(path1=f)
        sam, st = idx.align_sam(batch, with_stats=True)
        assert st["n_launches"] > 4, st
        assert sam == idx.format_sam(batch, idx.align(batch))
        want = set(printed_names(f, False))
        lines = sam.splitlines()
        assert len(lines) >= 2 * len(want) and all(any(l.startswith(n + b"\t") for n in want) for l in lines[:50])
    finally:
        idx.close()
