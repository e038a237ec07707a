"""The alignment summary (ReportingMetrics + AlnSink::printAlSumm) and the SAM output options (--no-unal, --rg-id /
--rg, --omit-sec-seq, --no-hd / --no-sq) against the unmodified reference: tools/refsets.py --output records the
reference's summary text (classic and --new-summary) under summary/* and summary_new/*, and the md5 of its SAM under
the output options under output/*, in tests/golden/output_sets.json."""
import os
import re
import subprocess
import sys

import pytest

from conftest import GOLDEN, ROOT

sys.path.insert(0, os.path.join(ROOT, "tools"))
import refsets  # noqa: E402

REF = refsets.load_output_expected()
REF_SETS = refsets.load_expected()
SUMMARY_IDS = sorted(refsets.SUMMARY_CASES)
OUTPUT_IDS = sorted(refsets.OUTPUT_CASES)


@pytest.fixture(scope="session")
def out_dir(tmp_path_factory):
    return refsets.generate_output_sets(str(tmp_path_factory.mktemp("output")))


def summary_flags(lib_opts):
    """(discordant, mixed) sections of the classic summary: off under --no-discordant / --no-mixed."""
    return not lib_opts.get("no_discordant"), not lib_opts.get("no_mixed")


def fasta_slice(src, dst, r0, r1):
    """Records [r0, r1) of a FASTA file (what -s r0 -u r1-r0 aligns)."""
    recs = open(src, "rb").read().split(b">")[1:]
    open(dst, "wb").write(b"".join(b">" + r for r in recs[r0:r1]))
    return dst


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the host build of the same formatter (tests/hostsim) and the summary text on its own
# ---------------------------------------------------------------------------------------------------------------------
def hostsim(bins, d, tmp_path, src, lib_opts, out_opts=None, front=None, summary_new=False):
    """Run the host build (tests/hostsim/ht2_outsim.cpp) on an OUTPUT_CASES / SUMMARY_CASES input; returns
    (SAM bytes, summary text)."""
    index, fs, _, _, opts, ss = refsets.output_input(d, src)
    opts = dict(opts, **lib_opts)
    spliced = opts.pop("no_spliced_alignment", 1) == 0
    kv = (["spliced=1"] if spliced else []) + ["%s=%s" % x for x in sorted(opts.items())]
    so = []
    for k, v in sorted((out_opts or {}).items()):
        if k == "rg":
            so += ["rg=%s" % f for f in v]
        elif k == "rg_id":
            so.append("rg_id=%s" % v)
        else:
            so.append("%s=%d" % (k, int(v)))
    if front:
        fs = [fasta_slice(f, str(tmp_path / ("slice%d.fa" % i)), front["skip"], front["skip"] + front["upto"]) for i, f in enumerate(fs)]
    out, summ = str(tmp_path / "o.sam"), str(tmp_path / "summary.txt")
    env = dict(os.environ, HT2_OPTS=",".join(kv), HT2_SAM_OUTPUT=",".join(so), HT2_SUMMARY=summ,
               HT2_NEW_SUMMARY="1" if summary_new else "0")
    if ss:
        env["HT2_SS"] = ss
    r = subprocess.run([bins[1] if spliced else bins[0], index, fs[0], out] + fs[1:], cwd=GOLDEN, stderr=subprocess.PIPE, env=env)
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    assert b"err=" not in r.stderr
    return open(out, "rb").read(), open(summ).read()


@pytest.fixture(scope="session")
def bins(tmp_path_factory):
    """TEST-ONLY host builds of tests/hostsim/ht2_outsim.cpp (ht2_hostsim with the SAM output settings and the
    summary), without and with the spliced-alignment pieces."""
    c = os.path.join(ROOT, "hisat2_b200", "csrc")
    out = []
    for name, defs in (("ht2_outsim", []), ("ht2_outsim_spliced", ["-DHT2_ENABLE_SPLICED"])):
        exe = str(tmp_path_factory.mktemp(name) / name)
        subprocess.run(["g++", "-O2", "-std=c++14"] + defs + ["-o", exe, os.path.join(ROOT, "tests", "hostsim", "ht2_outsim.cpp"),
                        os.path.join(c, "ht2_index.cpp"), os.path.join(c, "ht2_host.cpp"), "-lpthread"], check=True)
        out.append(exe)
    return tuple(out)


@pytest.mark.parametrize("case", SUMMARY_IDS)
def test_host_build_summary_matches_reference(bins, out_dir, tmp_path, case):
    """The ReportingMetrics tally of the formatter's counting pass, printed like AlnSink::printAlSumm, equals the
    reference's summary in both formats (small and large sets, SE / PE, graph index, spliced mode, edge reads with
    empty and N-filtered reads, --no-mixed / --no-discordant, -k 1, -s / -u, --sensitive, repeats under -k 30)."""
    src, _, lib_opts, front = refsets.SUMMARY_CASES[case]
    _, classic = hostsim(bins, out_dir, tmp_path, src, lib_opts, front=front)
    assert classic == REF["summary"]["summary/" + case]
    _, new = hostsim(bins, out_dir, tmp_path, src, lib_opts, front=front, summary_new=True)
    assert new == REF["summary"]["summary_new/" + case]


@pytest.mark.parametrize("case", OUTPUT_IDS)
def test_host_build_output_options_match_reference(bins, out_dir, tmp_path, case):
    """--no-unal, --rg-id / --rg (header and RG:Z:), --omit-sec-seq and --no-sq through the host build: the md5 of the
    reference's SAM (header without @PG)."""
    src, _, lib_opts, out_opts = refsets.OUTPUT_CASES[case]
    sam, _ = hostsim(bins, out_dir, tmp_path, src, lib_opts, out_opts)
    assert refsets.sam_md5(sam) == REF["md5"]["output/" + case]
    check_output_shape(sam, out_opts, lib_opts)


def check_output_shape(sam, out_opts, lib_opts):
    """What each option visibly does, so that a recorded md5 cannot stand for a case that exercises nothing."""
    lines = [l for l in sam.splitlines() if l]
    recs = [l.split(b"\t") for l in lines if not l.startswith(b"@")]
    flags = [int(r[1]) for r in recs]
    rg_id = out_opts.get("rg_id")
    if out_opts.get("no_unal"):
        assert all(f & 4 == 0 for f in flags)
        if any(f & 1 for f in flags) and not lib_opts.get("no_mixed"):   # pairs: a mate whose mate did not align keeps its record
            assert any(f & 8 for f in flags)
    if out_opts.get("omit_sec_seq"):
        sec = [r for r in recs if int(r[1]) & 256]
        assert sec and all(r[9] == b"*" and r[10] == b"*" for r in sec)
        assert all(r[9] != b"*" for r in recs if not int(r[1]) & 256)
    if rg_id:
        rg = [l for l in lines if l.startswith(b"@RG")]
        assert rg == [b"\t".join([b"@RG", b"ID:" + rg_id.encode()] + [f.encode() for f in out_opts.get("rg", ())])]
        assert all(b"RG:Z:" + rg_id.encode() in r for r in recs)
    else:
        assert not any(l.startswith(b"@RG") for l in lines) and not any(b"RG:Z:" in l for l in lines)
    assert any(l.startswith(b"@SQ") for l in lines) == (not out_opts.get("no_sq"))


def counts(**kw):
    from hisat2_b200 import api
    d = {k: 0 for k in api.ALIGN_COUNTS}
    d.update(kw)
    return d


def test_format_align_summary_zero_reads(lib):
    from hisat2_b200 import format_align_summary
    assert format_align_summary(counts()) == "0 reads\n0.00% overall alignment rate\n"
    assert format_align_summary(counts(), new_style=True) == (
        "HISAT2 summary stats:\n\tTotal reads: 0\n\t\tAligned 0 time: 0 (0.00%)\n\t\tAligned 1 time: 0 (0.00%)\n"
        "\t\tAligned >1 times: 0 (0.00%)\n\tOverall alignment rate: 0.00%\n")


def test_format_align_summary_unpaired(lib):
    from hisat2_b200 import format_align_summary
    c = counts(nread=3, nunpaired=3, nunp_0=1, nunp_uni1=1, nunp_uni2=1)
    assert format_align_summary(c) == (
        "3 reads; of these:\n"
        "  3 (100.00%) were unpaired; of these:\n"
        "    1 (33.33%) aligned 0 times\n"
        "    1 (33.33%) aligned exactly 1 time\n"
        "    1 (33.33%) aligned >1 times\n"
        "66.67% overall alignment rate\n")
    assert format_align_summary(c, new_style=True) == (
        "HISAT2 summary stats:\n\tTotal reads: 3\n\t\tAligned 0 time: 1 (33.33%)\n\t\tAligned 1 time: 1 (33.33%)\n"
        "\t\tAligned >1 times: 1 (33.33%)\n\tOverall alignment rate: 66.67%\n")


def test_format_align_summary_paired_sections(lib):
    from hisat2_b200 import format_align_summary
    # 8 pairs: 3 concordant once, 1 concordant more than once, 1 discordant, 3 neither: mates 2 unaligned, 3 once, 1 more
    c = counts(nread=8, npaired=8, nconcord_0=4, nconcord_uni1=3, nconcord_uni2=1, ndiscord=1,
               nunp_0_0=2, nunp_0_uni1=3, nunp_0_uni2=1)
    head = ("8 reads; of these:\n"
            "  8 (100.00%) were paired; of these:\n"
            "    4 (50.00%) aligned concordantly 0 times\n"
            "    3 (37.50%) aligned concordantly exactly 1 time\n"
            "    1 (12.50%) aligned concordantly >1 times\n")
    disc = ("    ----\n"
            "    4 pairs aligned concordantly 0 times; of these:\n"
            "      1 (25.00%) aligned discordantly 1 time\n")
    mixed = ("    ----\n"
             "    3 pairs aligned 0 times concordantly or discordantly; of these:\n"
             "      6 mates make up the pairs; of these:\n"
             "        2 (33.33%) aligned 0 times\n"
             "        3 (50.00%) aligned exactly 1 time\n"
             "        1 (16.67%) aligned >1 times\n")
    tail = "87.50% overall alignment rate\n"   # (4 * 2 + 1 * 2 + 4) / 16
    assert format_align_summary(c) == head + disc + mixed + tail
    assert format_align_summary(c, discordant=False) == head + mixed + tail
    assert format_align_summary(c, mixed=False) == head + disc + tail
    assert format_align_summary(c, discordant=False, mixed=False) == head + tail
    assert format_align_summary(c, new_style=True) == (
        "HISAT2 summary stats:\n\tTotal pairs: 8\n"
        "\t\tAligned concordantly or discordantly 0 time: 3 (37.50%)\n"
        "\t\tAligned concordantly 1 time: 3 (37.50%)\n"
        "\t\tAligned concordantly >1 times: 1 (12.50%)\n"
        "\t\tAligned discordantly 1 time: 1 (12.50%)\n"
        "\tTotal unpaired reads: 6\n"
        "\t\tAligned 0 time: 2 (33.33%)\n\t\tAligned 1 time: 3 (50.00%)\n\t\tAligned >1 times: 1 (16.67%)\n"
        "\tOverall alignment rate: 87.50%\n")


def test_format_align_summary_new_style_zero_denominator(lib):
    """--new-summary with every pair aligned concordantly: the unpaired-mate section divides by 0 and prints 0.00%."""
    from hisat2_b200 import format_align_summary
    c = counts(nread=2, npaired=2, nconcord_uni1=2)
    assert format_align_summary(c, new_style=True) == (
        "HISAT2 summary stats:\n\tTotal pairs: 2\n"
        "\t\tAligned concordantly or discordantly 0 time: 0 (0.00%)\n"
        "\t\tAligned concordantly 1 time: 2 (100.00%)\n"
        "\t\tAligned concordantly >1 times: 0 (0.00%)\n"
        "\t\tAligned discordantly 1 time: 0 (0.00%)\n"
        "\tTotal unpaired reads: 0\n"
        "\t\tAligned 0 time: 0 (0.00%)\n\t\tAligned 1 time: 0 (0.00%)\n\t\tAligned >1 times: 0 (0.00%)\n"
        "\tOverall alignment rate: 100.00%\n")


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the tally of the device SAM kernels, the output settings there, and the CLI
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def h2(lib):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import hisat2_b200
    return hisat2_b200


def open_case(h2, d, src, lib_opts):
    index, fs, fmt, _, opts, ss = refsets.output_input(d, src)
    idx = h2.Index(os.path.join(GOLDEN, index), **dict(opts, **lib_opts))
    if ss:
        idx.load_splicesites(ss)
    return idx, fs, fmt


@pytest.mark.gpu
@pytest.mark.parametrize("case", SUMMARY_IDS)
def test_device_counts_give_reference_summary(h2, out_dir, case):
    """A fresh handle runs the set through ht2gpu_run_reads in batches of 128 reads (counts summed over many batches
    and all three slots); the summary of its counts equals the reference's in both formats."""
    src, _, lib_opts, front = refsets.SUMMARY_CASES[case]
    idx, fs, fmt = open_case(h2, out_dir, src, lib_opts)
    try:
        _, st = idx.run_reads(path1=fs[0], path2=fs[1] if len(fs) == 2 else None, fastq=fmt == "-q", batch_reads=128,
                              collect=False, **front)
        assert st["n_batches"] >= 4 and st["n_err_reads"] == 0
        c = idx.align_counts()
    finally:
        idx.close()
    disc, mixed = summary_flags(lib_opts)
    assert c["nread"] == st["n_units"]
    assert h2.format_align_summary(c, discordant=disc, mixed=mixed) == REF["summary"]["summary/" + case]
    assert h2.format_align_summary(c, new_style=True, discordant=disc, mixed=mixed) == REF["summary"]["summary_new/" + case]


@pytest.mark.gpu
@pytest.mark.parametrize("case", OUTPUT_IDS)
def test_device_output_options_match_reference(h2, out_dir, case):
    """Each output case through ht2gpu_run_reads (md5 of the reference's SAM) and through ht2gpu_align_sam (device
    text == the host formatter's)."""
    src, _, lib_opts, out_opts = refsets.OUTPUT_CASES[case]
    idx, fs, fmt = open_case(h2, out_dir, src, lib_opts)
    try:
        idx.set_sam_output(**out_opts)
        sam, _ = idx.run_reads(path1=fs[0], path2=fs[1] if len(fs) == 2 else None, fastq=fmt == "-q", batch_reads=4096)
        sam = idx.sam_header() + sam
        assert refsets.sam_md5(sam) == REF["md5"]["output/" + case]
        check_output_shape(sam, out_opts, lib_opts)
        batch = h2.ReadBatch.parse(path1=fs[0], path2=fs[1] if len(fs) == 2 else None, fastq=fmt == "-q")
        host = idx.format_sam(batch, idx.align(batch))
        assert idx.align_sam(batch) == host, "device SAM differs from the host formatter's"
    finally:
        idx.close()


@pytest.mark.gpu
def test_sam_rerun_does_not_count_a_batch_twice(h2, out_dir):
    """Reads of segments tiny.fa holds twice, -k 30 --secondary: two records per read, more text than the first
    estimate, so ht2gpu_wait_sam runs the SAM kernels again.  The counts of that batch are still the reference's."""
    case = "rep_k30_secondary"
    src, _, lib_opts, _ = refsets.SUMMARY_CASES[case]
    idx, fs, _ = open_case(h2, out_dir, src, lib_opts)
    try:
        batch = h2.ReadBatch.parse(path1=fs[0])
        _, st = idx.align_sam(batch, with_stats=True)
        assert st["n_launches"] > 4, st
        c = idx.align_counts(reset=True)
        assert idx.align_counts() == counts()
    finally:
        idx.close()
    assert h2.format_align_summary(c) == REF["summary"]["summary/" + case]


@pytest.mark.gpu
def test_sam_output_settings_follow_the_handle(h2, out_dir):
    """Defaults leave the SAM unchanged; peer() carries the settings; run_reads_multi refuses handles that differ."""
    import torch
    idx = h2.Index(os.path.join(GOLDEN, "tiny"))
    try:
        batch = h2.ReadBatch.from_fasta(os.path.join(GOLDEN, "tiny_se.fa"))
        plain_hdr, plain = idx.sam_header(), idx.align_sam(batch)
        idx.set_sam_output(rg_id="x", no_sq=True)
        assert idx.sam_header() == b"@HD\tVN:1.0\tSO:unsorted\n@RG\tID:x\n"
        assert idx.align_sam(batch).count(b"\tRG:Z:x") == plain.count(b"\n")
        idx.set_sam_output()
        assert (idx.sam_header(), idx.align_sam(batch)) == (plain_hdr, plain)
        if torch.cuda.device_count() > 1:
            idx.set_sam_output(no_unal=True)
            peer = idx.peer(1)
            try:
                f = os.path.join(GOLDEN, "tiny_se.fa")
                sam, _ = idx.run_reads(path1=f, peers=(peer,), batch_reads=64)
                assert b"\t4\t*\t" not in sam
                peer.set_sam_output()
                with pytest.raises(h2.Ht2GpuError):
                    idx.run_reads(path1=f, peers=(peer,), batch_reads=64)
            finally:
                peer.close()
    finally:
        idx.close()


def cli(args, **kw):
    exe = os.path.join(ROOT, "hisat2_b200", "hisat2-b200")
    return subprocess.run([exe] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, cwd=GOLDEN, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("gpus", [1, 2])
def test_cli_summary_and_output_options(h2, out_dir, tmp_path, gpus):
    """hisat2-b200 prints the reference's summary at the end of stderr (summed over --gpus devices), writes the
    --new-summary text to --summary-file, prints neither under --quiet, and honours --no-hd and --rg-id / --rg."""
    import torch
    if gpus > torch.cuda.device_count():
        pytest.skip("needs %d devices" % gpus)
    case = "pe_hard20k"
    src = refsets.SUMMARY_CASES[case][0]
    _, fs, _, _, _, _ = refsets.output_input(out_dir, src)
    base = ["-x", "tiny", "-f", "--no-spliced-alignment", "-1", fs[0], "-2", fs[1], "--batch", "4096", "--gpus", str(gpus)]
    out, summ = str(tmp_path / "o.sam"), str(tmp_path / "summary.txt")
    r = cli(base + ["-S", out])
    assert r.returncode == 0, r.stderr
    assert r.stderr.decode().endswith(REF["summary"]["summary/" + case])
    assert refsets.sam_md5(open(out, "rb").read()) == REF_SETS["md5"]["paired/hard20k"]
    r = cli(base + ["-S", out, "--new-summary", "--summary-file", summ])
    assert r.returncode == 0 and r.stderr.decode().endswith(REF["summary"]["summary_new/" + case])
    assert open(summ).read() == REF["summary"]["summary_new/" + case]
    os.remove(summ)
    r = cli(base + ["-S", out, "--quiet", "--summary-file", summ])
    assert r.returncode == 0 and r.stderr == b"" and not os.path.exists(summ)
    r = cli(base + ["-S", out, "--no-hd", "--rg-id", "g1", "--rg", "SM:s1", "--quiet"])
    sam = open(out, "rb").read()
    assert r.returncode == 0 and sam and not sam.startswith(b"@")
    assert sam.count(b"\tRG:Z:g1") == sam.count(b"\n")
    # the reference's output/* case through the CLI: --rg-id with two --rg fields on the graph index
    src, flags, _, out_opts = refsets.OUTPUT_CASES["rg_graph_pe_alt20k"]
    _, gfs, _, _, _, _ = refsets.output_input(out_dir, src)
    r = cli(["-x", "tiny_snp", "-f", "--no-spliced-alignment", "-1", gfs[0], "-2", gfs[1], "--gpus", str(gpus), "-S", out, "--quiet"] + flags)
    assert r.returncode == 0, r.stderr
    assert refsets.sam_md5(open(out, "rb").read()) == REF["md5"]["output/rg_graph_pe_alt20k"]
    assert re.search(rb"^@RG\tID:g1\tSM:s1\tPL:ILLUMINA$", open(out, "rb").read(), re.M)
