"""GPU parity tests: every case goes through the C ABI (ctypes) on cuda:0 and is
compared with (a) the committed golden output of the unmodified reference,
(b) the reference binary run on the same box (oracle/_ref), (c) size-independent
properties at full batch sizes."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, REFDIR, ROOT, sam_lines

pytestmark = pytest.mark.gpu

DATA = os.path.join(REFDIR, "data")
REFBIN = os.path.join(REFDIR, "hisat2-align-s")
sys.path.insert(0, os.path.join(ROOT, "tools"))
import refsets  # noqa: E402

# md5 of the unmodified reference's SAM for every read set of tools/refsets.py (+ the reads it flags, where a case can)
REF_SETS = refsets.load_expected()


@pytest.fixture(scope="module")
def h2(lib):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import hisat2_b200
    return hisat2_b200


# Index handles are per test: the device workspace lives as long as a handle of the process does (~50 GB on an
# H100), and tests that run the command line front end start a second process that needs its own.
@pytest.fixture
def tiny(h2):
    idx = h2.Index(os.path.join(GOLDEN, "tiny"))
    yield idx
    idx.close()


@pytest.fixture(scope="session")
def sets(tmp_path_factory):
    """The read sets of tools/refsets.py, generated from the committed tiny fixtures."""
    return refsets.generate(str(tmp_path_factory.mktemp("sets")))


def set_files(sets, name):
    return os.path.join(sets, name + "_1.fa"), os.path.join(sets, name + "_2.fa")


def n_batches(units, batch_reads, paired=False):
    """Batches ht2gpu_run_reads cuts `units` reads (pairs) into: the first batch is a quarter of the others."""
    per = batch_reads if batch_reads else 4000000
    if paired:
        per = (per + 1) // 2
    first = per // 4 if per >= 8 else per
    return 1 if units <= first else 1 + -(-(units - first) // per)


def gpu_sam(idx, batch):
    """Header + SAM records of a batch.  The records are formatted ON THE DEVICE (ht2gpu_align_sam: the alignment
    kernel followed by the SAM kernels, csrc/ht2_sam.h) and must equal, byte for byte, what the host formatter
    makes of the structured results of ht2gpu_align_batch -- every parity test therefore checks both paths."""
    res = idx.align(batch)
    assert int((res.reads["err"] != 0).sum()) == 0
    assert res.n_launches >= 1
    host = idx.format_sam(batch, res)
    dev, st = idx.align_sam(batch, with_stats=True)
    assert st["n_launches"] >= 4 and st["n_err_reads"] == 0
    assert dev == host, "device SAM differs from the host formatter's"
    return idx.sam_header() + dev, res


def test_tiny_se_matches_golden_reference_sam(h2, tiny):
    batch = h2.ReadBatch.from_fasta(os.path.join(GOLDEN, "tiny_se.fa"))
    sam, res = gpu_sam(tiny, batch)
    assert sam_lines(sam) == sam_lines(open(os.path.join(GOLDEN, "tiny_se.sam"), "rb").read())
    # every CIGAR class of the fixture is exercised: M, I, D, S and unaligned
    txt = sam.decode()
    for op in ("I", "D", "S"):
        assert any(op in l.split("\t")[5] for l in txt.splitlines() if not l.startswith("@"))


def test_tiny_pe_matches_golden_reference_sam(h2, tiny):
    """Paired-end (--fr, -I 0 -X 1000): concordant, rescued, unpaired and unaligned mates."""
    batch = h2.ReadBatch.from_fasta(os.path.join(GOLDEN, "tiny_pe_1.fa"), path2=os.path.join(GOLDEN, "tiny_pe_2.fa"))
    assert batch.paired and batch.n == 600
    sam, res = gpu_sam(tiny, batch)
    assert sam_lines(sam) == sam_lines(open(os.path.join(GOLDEN, "tiny_pe.sam"), "rb").read())
    flags = set(int(l.split(b"\t")[1]) for l in sam_lines(sam) if not l.startswith(b"@"))
    assert {99, 147, 83, 163}.issubset(flags) and (73 in flags or 89 in flags) and 77 in flags


@pytest.mark.parametrize("name", ["sim10k", "hard20k", "len36", "len150", "len500"])
def test_chr22_paired_matches_reference_binary_run_here(h2, tiny, sets, name):
    """BASELINE configs[2]-shaped input (2x101 bp pairs; also short, long, ragged, with indels and Ns) simulated from the
    tiny fixture: SAM identical to the reference's (md5 of its output, tests/golden/ref_sets.json)."""
    f1, f2 = set_files(sets, name)
    batch = h2.ReadBatch.from_fasta(f1, path2=f2)
    sam, res = gpu_sam(tiny, batch)
    assert refsets.sam_md5(sam) == REF_SETS["md5"]["paired/" + name]


def test_in_kernel_seed_search_matches_oracle(h2, tiny, oracle_bin):
    """LF-step counts and alignments imply the same search as oracle/ht2_oracle.c:
    the first partial search of every strand recorded by the oracle must be
    consistent with what the kernel reported (aligned reads have an anchor whose
    resolved coordinate the oracle also finds)."""
    batch = h2.ReadBatch.from_fasta(os.path.join(GOLDEN, "tiny_se.fa"))
    res = tiny.align(batch)
    out = subprocess.run([oracle_bin, "dump", "tiny", "tiny_se.fa", "1"], cwd=GOLDEN, check=True,
                         stdout=subprocess.PIPE).stdout.decode().splitlines()
    coords = {}
    for l in out:
        f = l.split()
        if f[0] == "C":
            coords.setdefault(int(f[1]), set()).add((int(f[6]), int(f[7])))  # (tidx, toff) of a seed
    checked = 0
    for i in range(250):  # clean reads: full-length exact alignments
        rr = res.reads[i]
        if rr["n_aln"][0] == 0:
            continue
        al = res.alns[rr["aln_off"]]
        if al["n_edits"] != 0 or i not in coords:
            continue
        # an exact 101M alignment at toff must contain every oracle seed hit of the same reference
        ok = any(t == al["tidx"] and al["toff"] <= o < al["toff"] + 101 for (t, o) in coords[i])
        assert ok, (i, al, coords[i])
        checked += 1
    assert checked > 150


def test_fastq_qualities_match_golden_reference_sam(h2, tiny):
    """FASTQ reads with low-quality stretches (quality-aware penalties), SE and PE."""
    b = h2.ReadBatch.from_fastq(os.path.join(GOLDEN, "tiny_se.fq"))
    sam, _ = gpu_sam(tiny, b)
    assert sam_lines(sam) == sam_lines(open(os.path.join(GOLDEN, "tiny_se_fq.sam"), "rb").read())
    b = h2.ReadBatch.from_fastq(os.path.join(GOLDEN, "tiny_pe_1.fq"), path2=os.path.join(GOLDEN, "tiny_pe_2.fq"))
    sam, _ = gpu_sam(tiny, b)
    assert sam_lines(sam) == sam_lines(open(os.path.join(GOLDEN, "tiny_pe_fq.sam"), "rb").read())


def test_command_line_front_end_matches_golden(tmp_path):
    """`hisat2-b200` (host C++ over the C ABI) with the reference's own flags: -x/-U/-1/-2/-S/-q/-f,
    --no-spliced-alignment; SAM equals the reference's golden output (the @PG line differs by design)."""
    cli = os.path.join(ROOT, "hisat2_b200", "hisat2-b200")
    if not os.path.exists(cli):
        pytest.skip("CLI not built (python -m hisat2_b200.build)")
    for index, args, gold in (("tiny", ["-q", "-U", "tiny_se.fq"], "tiny_se_fq.sam"), ("tiny", ["-f", "-U", "tiny_se.fa"], "tiny_se.sam"),
                              ("tiny", ["-q", "-1", "tiny_pe_1.fq", "-2", "tiny_pe_2.fq"], "tiny_pe_fq.sam"),
                              ("tiny_snp", ["-f", "-1", "tiny_alt_1.fa", "-2", "tiny_alt_2.fa"], "tiny_snp_alt_pe.sam")):   # graph index
        out = str(tmp_path / "cli.sam")
        subprocess.run([cli, "--no-spliced-alignment", "-x", index] + args + ["-S", out, "-p", "4"], cwd=GOLDEN, check=True,
                       stderr=subprocess.DEVNULL)
        assert sam_lines(open(out, "rb").read()) == sam_lines(open(os.path.join(GOLDEN, gold), "rb").read()), args
    # the reference's default (spliced, temporary splice sites) runs as --no-temp-splicesite, with a warning
    out = str(tmp_path / "spl.sam")
    r = subprocess.run([cli, "-x", "tiny", "-f", "-U", "tiny_rna.fa", "-S", out], cwd=GOLDEN, stderr=subprocess.PIPE)
    assert r.returncode == 0 and b"no-temp-splicesite" in r.stderr
    assert sam_lines(open(out, "rb").read()) == sam_lines(open(os.path.join(GOLDEN, "tiny_spliced_rna.sam"), "rb").read())
    # options the build does not know are refused with a non-zero exit code
    r = subprocess.run([cli, "-x", "tiny", "-q", "-U", "tiny_se.fq", "--local", "-S", str(tmp_path / "x.sam")], cwd=GOLDEN,
                       stderr=subprocess.PIPE)
    assert r.returncode != 0 and b"not supported" in r.stderr


def test_pipeline_reads_in_sam_out_matches_golden(h2, tiny):
    """ht2gpu_run_reads: FASTA / FASTQ (paths and bytes in host memory) -> SAM through the overlapped pipeline
    (multi-threaded parser, three device slots, SAM formatted on the device).  Small batches force many
    batches per run, i.e. slot reuse and ordered hand-over."""
    g = lambda n: os.path.join(GOLDEN, n)
    want = sam_lines(open(g("tiny_se.sam"), "rb").read())
    hdr = tiny.sam_header()
    for batch_reads in (0, 64, 7):
        sam, st = tiny.run_reads(path1=g("tiny_se.fa"), batch_reads=batch_reads)
        assert sam_lines(hdr + sam) == want, batch_reads
        assert st["n_reads"] == 700 and st["n_err_reads"] == 0 and st["sam_bytes"] == len(sam)
        assert st["n_batches"] == n_batches(700, batch_reads)
    sam, st = tiny.run_reads(data1=open(g("tiny_se.fq"), "rb").read(), fastq=True, batch_reads=100, threads=3)
    assert sam_lines(hdr + sam) == sam_lines(open(g("tiny_se_fq.sam"), "rb").read())
    sam, st = tiny.run_reads(path1=g("tiny_pe_1.fq"), path2=g("tiny_pe_2.fq"), fastq=True, batch_reads=90)
    assert sam_lines(hdr + sam) == sam_lines(open(g("tiny_pe_fq.sam"), "rb").read())
    assert st["n_units"] * 2 == st["n_reads"]
    sam, st = tiny.run_reads(data1=open(g("tiny_pe_1.fa"), "rb").read(), data2=open(g("tiny_pe_2.fa"), "rb").read(), batch_reads=128)
    assert sam_lines(hdr + sam) == sam_lines(open(g("tiny_pe.sam"), "rb").read())
    # -s / -u select a record range (hisat2.cpp:1959-1964, 3319)
    sam, st = tiny.run_reads(path1=g("tiny_se.fa"), skip=100, upto=50)
    recs = [l for l in want if not l.startswith(b"@")]
    names = []
    for l in recs:
        if not names or names[-1] != l.split(b"\t")[0]:
            names.append(l.split(b"\t")[0])
    keep = set(names[100:150])
    assert sam.splitlines() == [l for l in recs if l.split(b"\t")[0] in keep]
    # mismatching mate files are an error, not a truncation
    with pytest.raises(h2.Ht2GpuError):
        tiny.run_reads(path1=g("tiny_pe_1.fa"), path2=g("tiny_se.fa"))


def test_pipeline_and_cli_match_reference_binary_at_scale(h2, tiny, sets, tmp_path):
    """200k pairs through ht2gpu_run_reads (50k-read batches: nine batches over three slots) and through the hisat2-b200
    command line: both identical to the reference's SAM."""
    f1, f2 = set_files(sets, "sim200k")
    want = REF_SETS["md5"]["paired/sim200k"]
    sam, st = tiny.run_reads(path1=f1, path2=f2, batch_reads=50000)
    assert st["n_batches"] == n_batches(200000, 50000, paired=True) and st["n_err_reads"] == 0
    assert refsets.sam_md5(tiny.sam_header() + sam) == want
    tiny.close()                    # the CLI below is a second process on the device
    cli = os.path.join(ROOT, "hisat2_b200", "hisat2-b200")
    out2 = str(tmp_path / "cli.sam")
    subprocess.run([cli, "--no-spliced-alignment", "-f", "-x", os.path.join(GOLDEN, "tiny"), "-1", f1, "-2", f2, "-S", out2, "--batch", "120000"],
                   check=True, stderr=subprocess.DEVNULL)
    assert refsets.sam_md5(open(out2, "rb").read()) == want


def _option_cases():
    import json
    return json.load(open(os.path.join(GOLDEN, "option_matrix.json")))


@pytest.mark.parametrize("case", range(23))
def test_option_matrix_matches_reference(h2, case, tmp_path):
    """Same option names and meaning as the reference's command line (-k, --mp, --np, --rdg, --rfg, --sp,
    --ignore-quals, --nofw/--norc, --secondary, --no-mixed, --no-discordant, -I/-X, --score-min, --bowtie2-dp,
    --gbar and the --sensitive / --very-sensitive presets; linear and graph index): md5 of the SAM equals
    the committed md5 of the unmodified reference's output, and the reference is re-run on this box when
    oracle/_ref is present."""
    import hashlib
    c = _option_cases()[case]
    opts = {k: (float(v) if k in ("score_min_const", "score_min_coeff") else int(v))
            for k, v in (kv.split("=") for kv in c["options"].split(","))}
    idx = h2.Index(os.path.join(GOLDEN, c["index"]), **opts)
    files = [os.path.join(GOLDEN, f) for f in c["reads"]]
    reader = h2.ReadBatch.from_fastq if c["format"] == "-q" else h2.ReadBatch.from_fasta
    if c["paired"]:
        batch = reader(files[0], path2=files[1])
        inp = ["-1", files[0], "-2", files[1]]
    else:
        batch = reader(files[0])
        inp = ["-U", files[0]]
    sam, _ = gpu_sam(idx, batch)
    assert hashlib.md5(b"\n".join(sam_lines(sam)) + b"\n").hexdigest() == c["md5"]
    if os.path.exists(REFBIN):
        out = str(tmp_path / "ref.sam")
        subprocess.run([REFBIN, "--no-spliced-alignment", c["format"], "-x", os.path.join(GOLDEN, c["index"])] + c["flags"] + inp + ["-S", out],
                       check=True, stderr=subprocess.DEVNULL)
        assert sam_lines(sam) == sam_lines(open(out, "rb").read())
    idx.close()


KEEP = set(list(range(0, 100)) + list(range(250, 350)) + list(range(500, 600)))


@pytest.mark.parametrize("idx,name", [("tiny", "tiny_dump.txt"), ("tiny_snp", "tiny_snp_dump.txt")])
def test_seed_search_kernel_matches_reference_dump(h2, idx, name):
    """ht2gpu_seed_search (ht2_seed_kernel) == the unmodified reference's partialSearch chains, node
    ranges, in-edge lists and getOffset / joinedToTextOff results, on the linear and the GRAPH fixture."""
    index = h2.Index(os.path.join(GOLDEN, idx))
    assert index.is_graph() == (idx == "tiny_snp")
    batch = h2.ReadBatch.from_fasta(os.path.join(GOLDEN, "tiny_se.fa"))
    res = index.seed_search(batch, max_range=4)
    got = [l for l in res.dump_lines(index.is_graph()) if int(l.split()[1]) in KEEP]
    want = open(os.path.join(GOLDEN, name)).readlines()
    assert got == want
    assert res.n_lf > 0 and res.alg_bytes > 0 and res.err == 0
    index.close()


def test_graph_index_alignment_matches_golden_reference_sam(h2):
    """GRAPH (SNP) index end to end on the GPU (pool kernel with the ALT-aware aligner): SE, PE, FASTQ and
    reads carrying ALT alleles; byte-identical SAM incl. Zs:Z tags."""
    index = h2.Index(os.path.join(GOLDEN, "tiny_snp"))
    for args, gold in ((("tiny_se.fa",), "tiny_snp_se.sam"), (("tiny_pe_1.fa", "tiny_pe_2.fa"), "tiny_snp_pe.sam"),
                       (("tiny_se.fq",), "tiny_snp_se_fq.sam"), (("tiny_alt_1.fa",), "tiny_snp_alt_se.sam"),
                       (("tiny_alt_1.fa", "tiny_alt_2.fa"), "tiny_snp_alt_pe.sam")):
        rd = h2.ReadBatch.from_fastq if args[0].endswith(".fq") else h2.ReadBatch.from_fasta
        batch = rd(os.path.join(GOLDEN, args[0]), path2=os.path.join(GOLDEN, args[1]) if len(args) > 1 else None)
        sam, _ = gpu_sam(index, batch)
        assert sam_lines(sam) == sam_lines(open(os.path.join(GOLDEN, gold), "rb").read()), gold
    index.close()


@pytest.mark.parametrize("name,paired", [("reads", False), ("hard20k", False), ("alt20k", False), ("sim200k", False), ("sim10k", True),
                                         ("alt20k", True), ("hard20k", True)])
def test_bundled_graph_index_matches_reference_binary_run_here(h2, sets, name, paired):
    """The graph (SNP) index tiny_snp (BASELINE configs[0]-shaped): SAM identical to the reference's, incl. 20k reads /
    pairs that carry ALT alleles."""
    f1, f2 = set_files(sets, name)
    index = h2.Index(os.path.join(GOLDEN, "tiny_snp"))
    batch = h2.ReadBatch.from_fasta(f1, path2=f2 if paired else None)
    sam, _ = gpu_sam(index, batch)
    assert refsets.sam_md5(sam) == REF_SETS["md5"]["graph_%s/%s" % ("pe" if paired else "se", name)]
    index.close()


def test_warp_wide_dp_fill_equals_lane_fill_cell_by_cell(h2):
    """ht2_sw.h: the DP rounds of the pool kernel fill the score planes with a whole warp per problem (64 rows per
    vector, lazy-F across lanes by shuffle).  On 3000 random problems (20..256 rows, random penalties, gap
    barriers, N's, indels) every H, E and F cell, every last-row score and the best score must equal the lane
    fill's, which the host self-test pins to a plain scalar statement of the recurrences (test_cpu.py)."""
    from hisat2_b200 import api
    r = api.sw_selftest(3000, seed=5)
    assert r["problems"] == 3000 and r["cells"] > 3000 * 20 * 60 and r["valid"] > 300
    assert r["mismatches"] == 0


@pytest.mark.parametrize("case", range(len(refsets.DP_CASES)))
def test_dynamic_programming_extension_matches_reference_binary_run_here(h2, sets, case):
    """--bowtie2-dp / --sensitive / --very-sensitive (SURVEY a30: the SwAligner seed extension): SAM identical to
    the reference's wherever no read hit a fixed device capacity (such reads are flagged, must be rare, and are
    exactly the ones recorded with the expected output)."""
    index, name, paired, flags, opts = refsets.DP_CASES[case]
    f1, f2 = set_files(sets, name)
    idx = h2.Index(os.path.join(GOLDEN, index), **opts)
    batch = h2.ReadBatch.from_fasta(f1, path2=f2 if paired else None)
    res = idx.align(batch)
    errs = np.nonzero(res.reads["err"])[0]
    assert len(errs) <= 0.002 * len(res.reads["err"])
    bad = sorted(set(batch.names[int(u) * (2 if paired else 1)].split(b"/")[0].decode() for u in errs))
    assert bad == REF_SETS["flagged"].get("dp/%d" % case, [])
    sam = idx.sam_header() + idx.format_sam(batch, res)
    assert refsets.sam_md5(sam, bad) == REF_SETS["md5"]["dp/%d" % case]
    idx.close()


def test_spliced_alignment_when_compiled_in(h2, tmp_path):
    """Spliced mode (== hisat2 --no-temp-splicesite: empty splice-site DB, reads independent), compiled into the
    default library (a build with HT2_NO_SPLICED=1 refuses it loudly, with no CPU or approximate path): the
    committed golden SAM of the reference on the RNA-like fixture (340 spliced alignments) and the DNA
    fixtures, and, when oracle/_ref is on the box, the reference run in place on 20k chr22 pairs."""
    try:
        idx = h2.Index(os.path.join(GOLDEN, "tiny"), no_spliced_alignment=0)
    except h2.Ht2GpuError as e:
        assert "spliced" in str(e)
        pytest.skip("library built with HT2_NO_SPLICED=1: spliced mode is refused loudly")
    for args, gold, rd in ((("tiny_rna.fa",), "tiny_spliced_rna.sam", h2.ReadBatch.from_fasta), (("tiny_se.fa",), "tiny_spliced_se.sam", h2.ReadBatch.from_fasta),
                           (("tiny_pe_1.fq", "tiny_pe_2.fq"), "tiny_spliced_pe_fq.sam", h2.ReadBatch.from_fastq)):
        batch = rd(os.path.join(GOLDEN, args[0]), path2=os.path.join(GOLDEN, args[1]) if len(args) > 1 else None)
        sam, _ = gpu_sam(idx, batch)
        assert sam_lines(sam) == sam_lines(open(os.path.join(GOLDEN, gold), "rb").read()), gold
    idx.close()
    base = os.path.join(DATA, "22_20-21M")
    f1, f2 = os.path.join(DATA, "hard20k_1.fa"), os.path.join(DATA, "hard20k_2.fa")
    if os.path.exists(REFBIN) and os.path.exists(base + ".1.ht2") and os.path.exists(f1):
        idx = h2.Index(base, no_spliced_alignment=0)
        batch = h2.ReadBatch.from_fasta(f1, path2=f2)
        sam, _ = gpu_sam(idx, batch)
        out = str(tmp_path / "ref.sam")
        subprocess.run([REFBIN, "--no-temp-splicesite", "-f", "-x", base, "-1", f1, "-2", f2, "-S", out, "-p", str(min(16, os.cpu_count() or 1)), "--reorder"],
                       check=True, stderr=subprocess.DEVNULL)
        assert sam_lines(sam) == sam_lines(open(out, "rb").read())
        idx.close()


def test_populated_splice_site_db_matches_reference(h2, tmp_path):
    """SURVEY 8f.3, the read-only part: --known-splicesite-infile / --novel-splicesite-infile with --no-temp-splicesite.
    The DB lives in HBM (ht2gpu_load_splicesites); the pool kernel runs the three `if(!ssdb.empty())` branches of
    hybridSearch_recur and the SAM kernel adjusts the template length of concordant pairs.  Golden SAM of the
    unmodified reference on the tiny fixtures (linear + graph index, -k 20 --secondary, two site files), the command
    line front end, and -- when oracle/_ref is on the box -- 20 k reads + 10 k pairs simulated over the chr22 example
    region with 34 k site lines, against the reference run in place."""
    g = lambda n: os.path.join(GOLDEN, n)
    for index, known, novel, opts, args, gold in (
            ("tiny", "tiny_ss_rna_ss.txt", None, {}, ("tiny_ss_rna.fa",), "tiny_ss_rna_se.sam"),
            ("tiny", "tiny_ss_rna_ss.txt", None, {}, ("tiny_ss_rna_1.fa", "tiny_ss_rna_2.fa"), "tiny_ss_rna_pe.sam"),
            ("tiny_snp", "tiny_ss_rna_ss.txt", None, {}, ("tiny_ss_rna_1.fa", "tiny_ss_rna_2.fa"), "tiny_snp_ss_rna_pe.sam"),
            ("tiny", "tiny_ss_rna_ss.txt", None, dict(khits=20, secondary=1), ("tiny_ss_rna.fa",), "tiny_ss_rna_se_k20_secondary.sam"),
            ("tiny", "tiny_ss_known.txt", "tiny_ss_novel.txt", {}, ("tiny_ss_rna_1.fa", "tiny_ss_rna_2.fa"), "tiny_ss_rna_pe_known_novel.sam")):
        idx = h2.Index(g(index), no_spliced_alignment=0, **opts)
        n = idx.load_splicesites(g(known), g(novel) if novel else None)
        assert n > 250
        batch = h2.ReadBatch.from_fasta(g(args[0]), path2=g(args[1]) if len(args) > 1 else None)
        sam, _ = gpu_sam(idx, batch)           # device SAM == host formatter is asserted inside
        assert sam_lines(sam) == sam_lines(open(g(gold), "rb").read()), gold
        if index == "tiny" and not opts and len(args) == 1:
            assert idx.load_splicesites(None, None) == 0          # unloading restores the empty-DB behaviour
            sam0, _ = gpu_sam(idx, batch)
            assert sam_lines(sam0) != sam_lines(sam)
        idx.close()
    cli = os.path.join(ROOT, "hisat2_b200", "hisat2-b200")
    if os.path.exists(cli):
        out = str(tmp_path / "cli.sam")
        subprocess.run([cli, "--no-temp-splicesite", "--known-splicesite-infile", "tiny_ss_rna_ss.txt", "-x", "tiny", "-f", "-1", "tiny_ss_rna_1.fa",
                        "-2", "tiny_ss_rna_2.fa", "-S", out], cwd=GOLDEN, check=True, stderr=subprocess.DEVNULL)
        assert sam_lines(open(out, "rb").read()) == sam_lines(open(g("tiny_ss_rna_pe.sam"), "rb").read())
        r = subprocess.run([cli, "--known-splicesite-infile", "/nonexistent/ss.txt", "-x", "tiny", "-f", "-U", "tiny_ss_rna.fa", "-S", out], cwd=GOLDEN,
                           stderr=subprocess.PIPE)
        assert r.returncode != 0 and b"cannot open" in r.stderr
    # --novel-splicesite-outfile (first pass of the two-pass use): junctions collected by the SAM kernel == the reference's file
    idx = h2.Index(g("tiny"), no_spliced_alignment=0)
    idx.collect_splicesites(True)
    sam, st = idx.run_reads(path1=g("tiny_ss_rna_1.fa"), path2=g("tiny_ss_rna_2.fa"), fastq=False, batch_reads=128)   # several batches
    novel = str(tmp_path / "novel.txt")
    assert idx.write_novel_splicesites(novel) == 89
    assert open(novel).read() == open(g("tiny_ss_rna_pe_novel_out.txt")).read()
    with pytest.raises(h2.Ht2GpuError):
        idx.load_splicesites(g("tiny_ss_rna_ss.txt"))            # a DB while collecting: order dependent in the reference, refused
    idx.close()
    if os.path.exists(cli):
        out = str(tmp_path / "cli2.sam")
        subprocess.run([cli, "--no-temp-splicesite", "--novel-splicesite-outfile", novel, "-x", "tiny", "-f", "-U", "tiny_rna.fa", "-S", out], cwd=GOLDEN,
                       check=True, stderr=subprocess.DEVNULL)
        assert open(novel).read() == open(g("tiny_rna_novel_out.txt")).read()
        assert sam_lines(open(out, "rb").read()) == sam_lines(open(g("tiny_spliced_rna.sam"), "rb").read())
    base = os.path.join(DATA, "22_20-21M")
    if os.path.exists(REFBIN) and os.path.exists(base + ".1.ht2") and os.path.exists(base + ".fa"):
        sys.path.insert(0, os.path.join(ROOT, "tools"))
        import sim_rna
        se, pairs, lines = sim_rna.sim(sim_rna.load_fasta(base + ".fa"), 20000, 10000, 5)
        pre = str(tmp_path / "c")
        sim_rna.write(pre, se, pairs, lines)
        idx = h2.Index(base, no_spliced_alignment=0)
        assert idx.load_splicesites(pre + "_ss.txt") > 20000
        for paired in (False, True):
            batch = h2.ReadBatch.from_fasta(pre + ("_1.fa" if paired else ".fa"), path2=pre + "_2.fa" if paired else None)
            sam, _ = gpu_sam(idx, batch)
            out = str(tmp_path / "ref.sam")
            subprocess.run([REFBIN, "--no-temp-splicesite", "--known-splicesite-infile", pre + "_ss.txt", "-f", "-x", base] +
                           (["-1", pre + "_1.fa", "-2", pre + "_2.fa"] if paired else ["-U", pre + ".fa"]) +
                           ["-S", out, "-p", str(min(16, os.cpu_count() or 1)), "--reorder"], check=True, stderr=subprocess.DEVNULL)
            want = sam_lines(open(out, "rb").read())
            assert sam_lines(sam) == want
            assert sum(1 for l in want if not l.startswith(b"@") and b"N" in l.split(b"\t")[5]) > (3000 if paired else 8000)
        idx.close()
        # two-pass: pass one writes the novel sites (== the reference's outfile), pass two uses them (== the reference again)
        idx = h2.Index(base, no_spliced_alignment=0)
        idx.collect_splicesites(True)
        idx.run_reads(path1=pre + "_1.fa", path2=pre + "_2.fa", fastq=False, collect=False)
        novel, refnovel = str(tmp_path / "n.txt"), str(tmp_path / "rn.txt")
        assert idx.write_novel_splicesites(novel) > 2000
        subprocess.run([REFBIN, "--no-temp-splicesite", "--novel-splicesite-outfile", refnovel, "-f", "-x", base, "-1", pre + "_1.fa", "-2", pre + "_2.fa",
                        "-S", "/dev/null", "-p", "4"], check=True, stderr=subprocess.DEVNULL)
        assert open(novel).read() == open(refnovel).read()
        idx.collect_splicesites(False)
        assert idx.load_splicesites(None, novel) > 2000
        batch = h2.ReadBatch.from_fasta(pre + "_1.fa", path2=pre + "_2.fa")
        sam, _ = gpu_sam(idx, batch)
        out = str(tmp_path / "ref2.sam")
        subprocess.run([REFBIN, "--no-temp-splicesite", "--novel-splicesite-infile", refnovel, "-f", "-x", base, "-1", pre + "_1.fa", "-2", pre + "_2.fa",
                        "-S", out, "-p", str(min(16, os.cpu_count() or 1)), "--reorder"], check=True, stderr=subprocess.DEVNULL)
        assert sam_lines(sam) == sam_lines(open(out, "rb").read())
        idx.close()


def test_seed_search_bundled_graph_index_matches_oracle(h2, sets, oracle_bin):
    """The graph fixture tiny_snp: every H/G/C record of 20k hard reads equals the pinned oracle's."""
    base = os.path.join(GOLDEN, "tiny_snp")
    fa = set_files(sets, "hard20k")[0]
    index = h2.Index(base)
    assert index.is_graph()
    batch = h2.ReadBatch.from_fasta(fa)
    res = index.seed_search(batch, max_range=4)
    want = subprocess.run([oracle_bin, "dump", base, fa, "1"], check=True, stdout=subprocess.PIPE).stdout.decode().splitlines(True)
    assert res.dump_lines(True) == want
    index.close()


def test_batch_composition_invariance_and_determinism(h2, tiny):
    """Reads are independent units: any split of the batch gives the same records."""
    batch = h2.ReadBatch.from_fasta(os.path.join(GOLDEN, "tiny_se.fa"))
    full, _ = gpu_sam(tiny, batch)
    again, _ = gpu_sam(tiny, batch)
    assert full == again
    k = 333
    offs = batch.offs
    a = h2.ReadBatch(batch.seq[:int(offs[k])], offs[:k + 1], batch.seeds[:k], batch.names[:k])
    b = h2.ReadBatch(batch.seq[int(offs[k]):], offs[k:] - offs[k], batch.seeds[k:], batch.names[k:])
    sa, _ = gpu_sam(tiny, a)
    sb, _ = gpu_sam(tiny, b)
    hdr = tiny.sam_header()
    assert full == hdr + sa[len(hdr):] + sb[len(hdr):]


def test_edge_cases(h2, tiny):
    """empty batch, reads shorter than the ftab, all-N read, 1-base read, max-length (1 024-base) read."""
    lib = h2.load_library()
    empty = h2.ReadBatch(np.zeros(0, np.uint8), np.zeros(1, np.uint64), np.zeros(0, np.uint32), [])
    r = tiny.align(empty)
    assert len(r.reads) == 0 and len(r.alns) == 0
    rng = np.random.default_rng(5)
    seqs = [np.array([0, 1, 2], np.uint8), np.full(60, 4, np.uint8), np.array([2], np.uint8),
            rng.integers(0, 4, 1024).astype(np.uint8), rng.integers(0, 4, 7).astype(np.uint8)]
    names = [b"short3", b"allN", b"one", b"len1024", b"short7"]
    offs = np.cumsum([0] + [len(s) for s in seqs]).astype(np.uint64)
    seeds = np.array([lib.ht2gpu_read_seed(np.ascontiguousarray(s).ctypes.data, None, len(s), n, 0)
                      for s, n in zip(seqs, names)], dtype=np.uint32)
    b = h2.ReadBatch(np.concatenate(seqs), offs, seeds, names)
    res = tiny.align(b)
    assert int((res.reads["err"] != 0).sum()) == 0
    sam = tiny.format_sam(b, res).decode().splitlines()
    assert len(sam) == 5
    assert all(l.split("\t")[1] == "4" for l in sam)           # nothing aligns
    assert "YF:Z:NS" in sam[1] and "YF:Z:LN" in sam[2]           # N filter / length filter (hisat2.cpp:3417-3440)
    # over-long read: reported as a capacity error, never silently truncated
    long_ = h2.ReadBatch(rng.integers(0, 4, 1100).astype(np.uint8), np.array([0, 1100], np.uint64), np.array([1], np.uint32), [b"len1100"])
    res = tiny.align(long_)                      # the call succeeds; the read is flagged and counted
    assert res.reads["err"][0] != 0 and res.n_err_reads == 1
    sam, st = tiny.align_sam(long_, with_stats=True)
    assert st["n_err_reads"] == 1


def test_slot_buffers_have_their_own_capacities(h2, tmp_path):
    """ADVICE r1 (medium): a handle that first sees a big FASTA batch (no qualities), then a small FASTQ batch, then a
    medium FASTQ batch must not write the third batch's qualities past the buffer sized for the second: every slot
    buffer tracks its own capacity.  The SAM of each batch must equal the golden output whatever came before (a
    quality overflow corrupts neighbouring buffers, i.e. the records of the batch)."""
    g = lambda n: os.path.join(GOLDEN, n)
    idx = h2.Index(g("tiny"))
    big = h2.ReadBatch.from_fasta(g("tiny_se.fa"))                      # 700 reads, qual == NULL
    fq = h2.ReadBatch.from_fastq(g("tiny_se.fq"))
    gold_fq = sam_lines(open(g("tiny_se_fq.sam"), "rb").read())
    nsq = sum(1 for l in gold_fq if l.startswith(b"@"))
    def sub(b, lo, hi):
        o = b.offs
        return h2.ReadBatch(b.seq[int(o[lo]):int(o[hi])], (o[lo:hi + 1] - o[lo]).astype(np.uint64), b.seeds[lo:hi], b.names[lo:hi],
                            qual=None if b.qual is None else b.qual[int(o[lo]):int(o[hi])])
    body = lambda sam: [l for l in sam_lines(sam) if not l.startswith(b"@")]
    want = [l for l in gold_fq[nsq:]]
    per_read = {}
    for l in want:
        per_read.setdefault(l.split(b"\t")[0], []).append(l)
    expect = lambda b: [l for n in b.names for l in per_read[n.split(b" ")[0]]]
    assert body(idx.align_sam(big)) == body(open(g("tiny_se.sam"), "rb").read())
    assert fq.n >= 300 and big.offs[-1] > 2 * fq.offs[300]
    small, medium = sub(fq, 0, 40), sub(fq, 40, 300)
    assert body(idx.align_sam(small)) == expect(small)
    assert body(idx.align_sam(medium)) == expect(medium)
    assert body(idx.align_sam(fq)) == want
    idx.close()


@pytest.mark.parametrize("name", ["reads", "hard20k", "sim200k", "len36", "len150", "len250", "len500", "len1000"])
def test_chr22_matches_reference_binary_run_here(h2, tiny, sets, name):
    """BASELINE configs[0]/[1]-shaped single-end inputs: SAM identical to the reference's."""
    batch = h2.ReadBatch.from_fasta(set_files(sets, name)[0])
    sam, res = gpu_sam(tiny, batch)
    assert refsets.sam_md5(sam) == REF_SETS["md5"]["se/" + name]


@pytest.mark.skipif(not (os.path.exists(REFBIN) and os.path.exists(os.path.join(DATA, "22_20-21M.1.ht2"))),
                    reason="oracle/_ref and its staged data (oracle/make_data.sh) not built")
@pytest.mark.parametrize("index,name,paired", [("22_20-21M", "sim10k", True), ("22_20-21M", "hard20k", True), ("22_20-21M", "len500", False),
                                               ("22_20-21M_snp", "alt20k", True), ("22_20-21M_snp", "reads", False)])
def test_example_region_indexes_match_reference_binary_run_here(h2, index, name, paired, tmp_path):
    """Where oracle/_ref and its staged data are present: the 1 Mbp 22_20-21M example region (many local indexes; the
    bundled graph index with 3,689 SNPs / indels) against the reference binary run on the same machine."""
    base = os.path.join(DATA, index)
    f1, f2 = os.path.join(DATA, name + "_1.fa"), os.path.join(DATA, name + "_2.fa")
    idx = h2.Index(base)
    batch = h2.ReadBatch.from_fasta(f1, path2=f2 if paired else None)
    sam, _ = gpu_sam(idx, batch)
    idx.close()
    out = str(tmp_path / "ref.sam")
    subprocess.run([REFBIN, "--no-spliced-alignment", "-f", "-x", base] + (["-1", f1, "-2", f2] if paired else ["-U", f1]) +
                   ["-S", out, "-p", str(min(16, os.cpu_count() or 1)), "--reorder"], check=True, stderr=subprocess.DEVNULL)
    assert sam_lines(sam) == sam_lines(open(out, "rb").read())


@pytest.mark.parametrize("name", ["len250", "len1000"])
def test_long_pairs_capacity_errors_are_flagged_never_silent(h2, tiny, sets, name):
    """2x250 bp and 2x1000 bp pairs with indels and Ns.  Capacities are compile-time (1 024 bases, 128 edits per
    trial alignment, 48 nested extensions): a pair that needs more is flagged (err != 0, counted in n_err_reads), the
    call succeeds, and every OTHER pair is identical to the reference.  2x250 flags nothing."""
    f1, f2 = set_files(sets, name)
    batch = h2.ReadBatch.from_fasta(f1, path2=f2)
    res = tiny.align(batch)
    bad = set(np.flatnonzero(res.reads["err"] != 0).tolist())
    assert len(bad) == res.n_err_reads and len(bad) <= (0 if name == "len250" else 150)
    badnames = sorted(set(batch.names[2 * u].split(b"/")[0].decode() for u in bad))
    assert badnames == REF_SETS["flagged"].get("long/" + name, [])
    sam = tiny.sam_header() + tiny.format_sam(batch, res)
    assert refsets.sam_md5(sam, badnames) == REF_SETS["md5"]["long/" + name]


def test_full_size_byte_parity_1M_reads_and_500k_pairs(h2, tiny):
    """BASELINE configs[1] size (1M x 101 bp SE) and the configs[2] shape (500k pairs 2x101): the bench workload's own
    generator, FASTA bytes through ht2gpu_run_reads, identical to the reference's SAM; plus determinism of a second pass."""
    sys.path.insert(0, ROOT)
    import bench
    d1, d2 = bench.sim_fasta(0, 1000000)
    hdr = tiny.sam_header()
    sam, st = tiny.run_reads(data1=d1)
    assert st["n_reads"] == 1000000 and st["n_err_reads"] == 0
    assert refsets.sam_md5(hdr + sam) == REF_SETS["md5"]["full/se1M"]
    assert sam.count(b"\tYT:Z:UU") >= 1000000 and sam.count(b"\n") >= 1000000
    sam2, _ = tiny.run_reads(data1=d1, batch_reads=300000)
    assert sam2 == sam                      # batch composition does not change a byte
    del sam, sam2
    k = 500000
    sam, st = tiny.run_reads(data1=d1[:k * bench.RECSZ], data2=d2[:k * bench.RECSZ])
    assert st["n_units"] == k and st["n_err_reads"] == 0
    assert refsets.sam_md5(hdr + sam) == REF_SETS["md5"]["full/pe500k"]


def test_two_devices_one_process_equal_one_device(h2, sets, tmp_path):
    """hisat2-b200 --gpus 2 / ht2gpu_run_reads_multi: batches round-robin over two devices of one process (index
    replicated device to device), output in input order -- byte-identical to the single-device run."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    base = os.path.join(GOLDEN, "tiny")
    f1, f2 = set_files(sets, "sim200k")
    a = h2.Index(base, device=0)
    one, _ = a.run_reads(path1=f1, path2=f2, batch_reads=40000)
    b = a.peer(1)
    two, st = a.run_reads(path1=f1, path2=f2, batch_reads=40000, peers=[b])
    assert st["n_batches"] == n_batches(200000, 40000, paired=True) and two == one
    b.close(); a.close()
    cli = os.path.join(ROOT, "hisat2_b200", "hisat2-b200")
    out = str(tmp_path / "cli2.sam")
    subprocess.run([cli, "--no-spliced-alignment", "-f", "-x", base, "-1", f1, "-2", f2, "-S", out, "--batch", "40000", "--gpus", "2"], check=True,
                   stderr=subprocess.DEVNULL)
    body = open(out, "rb").read()
    assert body[body.index(b"\n@PG") + 1:].split(b"\n", 1)[1] == one


def test_torchrun_two_ranks_concatenate_to_the_single_rank_output(h2, sets, tmp_path):
    """The bench's N-rank layout on hardware: two torchrun ranks (NCCL broadcast of the index image, contiguous pair
    ranges) each write their shard's SAM; the rank-order concatenation equals the one-GPU output byte for byte."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    f1, f2 = set_files(sets, "sim200k")
    script = str(tmp_path / "rank.py")
    open(script, "w").write("""
import os, sys
sys.path.insert(0, %r)
import numpy as np, torch, torch.distributed as dist
import hisat2_b200 as h2
from hisat2_b200.parallel import broadcast_image, shard_range
rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
img = h2.Index.build_image(%r) if rank == 0 else None
dev = broadcast_image(img, rank, device=torch.device("cuda", local))
torch.cuda.synchronize()
idx = h2.Index(device_image=(dev.data_ptr(), dev.numel(), dev[:4096].cpu().numpy()), device=local)
lo, hi = shard_range(200000, rank, world)
sam, st = idx.run_reads(path1=%r, path2=%r, skip=lo, upto=hi - lo, batch_reads=60000)
open(os.path.join(%r, "part%%d.sam" %% rank), "wb").write(sam)
dist.barrier(); dist.destroy_process_group()
""" % (ROOT, os.path.join(GOLDEN, "tiny"), f1, f2, str(tmp_path)))
    subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                    "--master-port", "29517", script], check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    a = h2.Index(os.path.join(GOLDEN, "tiny"), device=0)
    one, _ = a.run_reads(path1=f1, path2=f2)
    a.close()
    assert open(str(tmp_path / "part0.sam"), "rb").read() + open(str(tmp_path / "part1.sam"), "rb").read() == one
