"""Alignment against splice-site / exon graph indexes (hisat2-build --ss / --exon: the `_tran` and `_snp_tran` indexes
RNA-seq users align against).  tools/tran_index_ref.py records the unmodified reference's SAM md5 (header without @PG)
and alignment summary per case in tests/golden/tran_index_sets.json; the indexes are tests/golden/tiny_tran and
tiny_snp_tran (tools/tran_index_ref.py fixtures)."""
import ctypes as C
import os
import struct
import subprocess
import sys

import pytest

from conftest import GOLDEN, ROOT

sys.path.insert(0, os.path.join(ROOT, "tools"))
import refsets  # noqa: E402
import tran_index_ref as tir  # noqa: E402

REF = tir.load_expected()
CASES = sorted(tir.CASES)
ALT_SNP_INS, ALT_SNP_DEL, ALT_SPLICESITE, ALT_EXON = 2, 3, 5, 6


def spliced_records(sam):
    return sum(1 for l in sam.splitlines() if l and not l.startswith(b"@") and b"N" in l.split(b"\t")[5])


def test_recorded_cases_differ():
    """Each mode changes the reference's output on its input, so that no recorded md5 stands for a case that tests
    nothing: --tmo, --avoid-pseudogene (the exon table), --dta, -k 20 --secondary, the extra site file and
    --no-spliced-alignment each differ from the default run."""
    m = REF["md5"]
    for index in tir.INDEXES:
        for src in ("se", "pe"):
            base = m["%s_%s_default" % (index, src)]
            for mode in tir.MODES:
                if mode != "default":
                    assert m["%s_%s_%s" % (index, src, mode)] != base, (index, src, mode)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the image builder, the ALT table's order and the host build
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="session")
def seedsim(tmp_path_factory):
    """The library's image builder through a small host program: prints the header's counts and the ALT table."""
    c = os.path.join(ROOT, "hisat2_b200", "csrc")
    d = tmp_path_factory.mktemp("tranimg")
    src = d / "img.cpp"
    src.write_text(r'''
#include <stdio.h>
#include "ht2_index.h"
int main(int argc, char** argv) {
    std::string err;
    Ht2Image* img = ht2_image_load(argv[1], err);
    if (!img) { fprintf(stderr, "%s\n", err.c_str()); return 1; }
    const Ht2ImageHeader* H = img->header();
    printf("%u %u %u %u %u\n", H->global.linearFM, H->nAlts, H->nSpliceSites, H->nExons, H->altsUnsupported);
    const Ht2Alt* a = (const Ht2Alt*)(img->blob.data() + H->o_alts);
    const char* names = (const char*)(img->blob.data() + H->o_altNames);
    const uint32_t* no = (const uint32_t*)(img->blob.data() + H->o_altNameOffs);
    for (uint32_t i = 0; i < H->nAlts; i++) printf("%u %u %u %llu %s\n", a[i].pos, a[i].type, a[i].len, (unsigned long long)a[i].seq, names + no[i]);
    return 0;
}
''')
    exe = str(d / "img")
    subprocess.run(["g++", "-O1", "-std=c++14", "-I", c, "-o", exe, str(src), os.path.join(c, "ht2_index.cpp")], check=True)
    return exe


def image_alts(exe, index):
    out = subprocess.run([exe, os.path.join(GOLDEN, index)], check=True, stdout=subprocess.PIPE).stdout.decode().splitlines()
    head = [int(x) for x in out[0].split()]
    alts = [(int(p), int(t), int(l), int(s), n) for p, t, l, s, n in (x.split() for x in out[1:])]
    return head, alts


def read_alts(index):
    """The .7.ht2 records and .8.ht2 names of an index, as the reference reads them (gfm.h:714-771)."""
    b7 = open(os.path.join(GOLDEN, index + ".7.ht2"), "rb").read()
    n = struct.unpack_from("<I", b7, 4)[0]
    recs = [struct.unpack_from("<IIIQ", b7, 8 + 20 * i) for i in range(n)]
    names = open(os.path.join(GOLDEN, index + ".8.ht2"), "rb").read()[8:].split()
    return [(p, t, l, s) for p, t, l, s in recs], [x.decode() for x in names[:n]]


def reference_order(index):
    """The reference loader's table: every splice site gets a reversed copy (left and right swapped, named "ssr"), every
    deletion one at its last base (the low byte of seq set), then a stable sort by ALT::operator< (alt.h:89-103)."""
    import functools
    recs, names = read_alts(index)
    alts = [(p, t, l, s, names[i]) for i, (p, t, l, s) in enumerate(recs)]
    for p, t, l, s, nm in list(alts):
        if t == ALT_SPLICESITE:
            alts.append((l, t, p, s, "ssr"))
        elif t == ALT_SNP_DEL:
            alts.append((p + l - 1, t, l, (s & ~0xff) | 1, nm))

    def less(x, y):
        if x[0] != y[0]:
            return x[0] < y[0]
        if x[1] != y[1]:
            if x[1] == 0 or y[1] == 0:
                return x[1] == 0
            if x[1] == ALT_SNP_INS:
                return True
            if y[1] == ALT_SNP_INS:
                return False
            return x[1] < y[1]
        if x[2] != y[2]:
            return x[2] < y[2]
        return x[3] < y[3]
    return sorted(alts, key=functools.cmp_to_key(lambda x, y: -1 if less(x, y) else (1 if less(y, x) else 0)))


@pytest.mark.parametrize("index", tir.INDEXES)
def test_image_loads_tran_index(seedsim, index):
    """Both fixtures load as graph indexes with their splice-site and exon counts and no refusal flag, and the ALT
    table holds the reversed splice-site copies in the reference loader's order."""
    (linear, nalts, nss, nex, unsupported), alts = image_alts(seedsim, index)
    recs, _ = read_alts(index)
    assert linear == 0 and unsupported == 0
    assert nss == sum(1 for r in recs if r[1] == ALT_SPLICESITE) > 0
    assert nex == sum(1 for r in recs if r[1] == ALT_EXON) > 0
    assert alts == reference_order(index)
    assert nalts == len(alts) == len(recs) + nss + sum(1 for r in recs if r[1] == ALT_SNP_DEL)


def _build(tmp_path_factory, name, flags):
    c = os.path.join(ROOT, "hisat2_b200", "csrc")
    exe = str(tmp_path_factory.mktemp(name) / "ht2_transim")
    subprocess.run(["g++"] + flags + ["-std=c++14", "-o", exe, os.path.join(ROOT, "tests", "hostsim", "ht2_transim.cpp"),
                                      os.path.join(c, "ht2_index.cpp"), os.path.join(c, "ht2_host.cpp"), "-lpthread"], check=True)
    return exe


@pytest.fixture(scope="session")
def transim(tmp_path_factory):
    """TEST-ONLY host build of the aligner for splice-site / exon indexes (tests/hostsim/ht2_transim.cpp)."""
    return _build(tmp_path_factory, "transim", ["-O2"])


def host_env(opts):
    kv = ["spliced=%d" % (opts["no_spliced_alignment"] == 0)]
    so = []
    for k, v in sorted(opts.items()):
        if k in ("tmo", "avoid_pseudogene", "dta"):
            so.append("%s=%d" % (k, v))
        elif k in ("khits", "secondary"):
            kv.append("%s=%d" % (k, v))
    return ",".join(kv), ",".join(so)


@pytest.mark.parametrize("case", CASES)
def test_host_build_matches_reference(transim, tmp_path, case):
    """Every case through the host build: the reference's SAM md5, with no read flagged."""
    index, fs, _, opts, ss = tir.case_input(case)
    kv, so = host_env(opts)
    o = str(tmp_path / "o.sam")
    env = dict(os.environ, HT2_OPTS=kv, HT2_SPL_OPTS=so)
    env.pop("HT2_SS", None)
    if ss:
        env["HT2_SS"] = ss
    r = subprocess.run([transim, os.path.join(GOLDEN, index), fs[0], o] + fs[1:], cwd=GOLDEN, stderr=subprocess.PIPE, env=env)
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    assert b"errors=0" in r.stderr, r.stderr.decode()[-2000:]
    sam = open(o, "rb").read()
    assert refsets.sam_md5(sam) == REF["md5"][case]
    if tir.CASES[case][2] == "nospl":
        assert spliced_records(sam) == 0
    elif tir.CASES[case][1] != "dna_pe":
        assert spliced_records(sam) > 0


@pytest.mark.skipif(not os.path.exists(refsets.REFBIN), reason="oracle/_ref not built")
@pytest.mark.parametrize("case", CASES)
def test_reference_reproduces_recorded(tmp_path, case):
    """The reference driver still gives the recorded md5 and summary."""
    sam, err = tir.reference_run(case, str(tmp_path / "ref.sam"))
    assert refsets.sam_md5(sam) == REF["md5"][case]
    assert refsets.summary_text(err.encode()) == REF["summary"][case]


# ---------------------------------------------------------------------------------------------------------------------
# GPU: ht2gpu_run_reads, the CLI, the index's splice-site DB and replicas
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def h2():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import hisat2_b200
    return hisat2_b200


def open_case(h2, case):
    index, fs, _, opts, ss = tir.case_input(case)
    idx = h2.Index(os.path.join(GOLDEN, index), **opts)
    if ss:
        idx.load_splicesites(ss)
    return idx, fs


def run(idx, fs, **kw):
    sam, st = idx.run_reads(path1=fs[0], path2=fs[1] if len(fs) == 2 else None, **kw)
    return idx.sam_header() + sam, st


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_device_matches_reference(h2, case):
    """Every case through ht2gpu_run_reads in one batch and in 64-read batches: the reference's SAM md5 and alignment
    summary, with no read flagged."""
    idx, fs = open_case(h2, case)
    try:
        for batch_reads in (0, 64):
            idx.align_counts(reset=True)
            sam, st = run(idx, fs, batch_reads=batch_reads)
            assert st["n_err_reads"] == 0, batch_reads
            assert refsets.sam_md5(sam) == REF["md5"][case], batch_reads
            assert h2.format_align_summary(idx.align_counts()) == REF["summary"][case], batch_reads
    finally:
        idx.close()


def cli(args, **kw):
    exe = os.path.join(ROOT, "hisat2_b200", "hisat2-b200")
    return subprocess.run([exe] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, cwd=GOLDEN, **kw)


@pytest.fixture(scope="module")
def cli_built(h2):
    from hisat2_b200 import build
    build.build_cli()


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_cli_matches_reference(cli_built, tmp_path, case):
    """hisat2-b200 -x <_tran index> with the reference's flags gives the reference's SAM and summary."""
    index, fs, flags, _, _ = tir.case_input(case)
    reads = ["-1", fs[0], "-2", fs[1]] if len(fs) == 2 else ["-U", fs[0]]
    out = str(tmp_path / "o.sam")
    r = cli(["-x", index, "-f"] + flags + reads + ["-S", out, "--batch", "512"])
    assert r.returncode == 0, r.stderr
    assert refsets.sam_md5(open(out, "rb").read()) == REF["md5"][case]
    assert refsets.summary_text(r.stderr) == REF["summary"][case]


@pytest.mark.gpu
def test_index_db_is_restored_and_collecting_is_refused(h2, cli_built, tmp_path):
    """load_splicesites(None, None) on a _tran handle goes back to the index's own sites (the SAM is unchanged);
    collecting novel sites is refused there, through the library and the CLI, naming the index as the reason."""
    case = "tiny_tran_pe_default"
    idx, fs = open_case(h2, case)
    try:
        assert idx.load_splicesites(None, None) > 0
        sam, st = run(idx, fs)
        assert st["n_err_reads"] == 0 and refsets.sam_md5(sam) == REF["md5"][case]
        with pytest.raises(h2.Ht2GpuError) as e:
            idx.collect_splicesites(True)
        assert "splice sites / exons" in str(e.value)
    finally:
        idx.close()
    r = cli(["-x", "tiny_tran", "-f", "--no-temp-splicesite", "-U", fs[0], "-S", str(tmp_path / "o.sam"),
             "--novel-splicesite-outfile", str(tmp_path / "novel.txt")])
    assert r.returncode != 0 and b"splice sites / exons" in r.stderr


def check_replica(h2, case, device):
    idx, fs = open_case(h2, case)
    try:
        one, _ = run(idx, fs, batch_reads=64)
        assert refsets.sam_md5(one) == REF["md5"][case]
        p = idx.peer(device)
        try:
            alone, st = run(p, fs, batch_reads=64)
            assert st["n_err_reads"] == 0 and alone == one
            two, st = run(idx, fs, batch_reads=64, peers=[p])
            assert st["n_err_reads"] == 0 and two == one
        finally:
            p.close()
    finally:
        idx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["tiny_snp_tran_pe_default", "tiny_snp_tran_pe_known"])
def test_replica_has_the_index_db(h2, case):
    """A peer handle on the same device, alone and with the original through ht2gpu_run_reads_multi, gives the single
    handle's SAM: replicas build the same splice-site DB from the index image (plus the files loaded on the original)."""
    check_replica(h2, case, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["tiny_snp_tran_pe_default", "tiny_snp_tran_pe_known"])
def test_replica_on_another_device_has_the_index_db(h2, case):
    """The same with the replica on a second device."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    check_replica(h2, case, 1)
