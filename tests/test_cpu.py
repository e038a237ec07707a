"""CPU-side tests (no GPU): oracle vs golden vectors, host logic, C ABI."""
import hashlib
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, sam_lines

sys.path.insert(0, os.path.join(ROOT, "tools"))
import refsets  # noqa: E402

REF_SETS = refsets.load_expected()
KEEP = set(list(range(0, 100)) + list(range(250, 350)) + list(range(500, 600)))


@pytest.fixture(scope="session")
def spliced_dir(tmp_path_factory):
    return refsets.generate_spliced(str(tmp_path_factory.mktemp("spliced")))


def test_oracle_matches_reference_dump(oracle_bin):
    """oracle/ht2_oracle.c == golden vectors dumped from the unmodified
    reference's partialSearch/getOffset/joinedToTextOff (tests/golden/make_golden.py)."""
    for idx, mode, name in (("tiny", "1", "tiny_dump.txt"), ("tiny", "0", "tiny_dump_spliced.txt"),
                            ("tiny_snp", "1", "tiny_snp_dump.txt")):   # tiny_snp = GRAPH index (SNPs, indels)
        out = subprocess.run([oracle_bin, "dump", idx, "tiny_se.fa", mode], cwd=GOLDEN, check=True,
                             stdout=subprocess.PIPE).stdout.decode().splitlines(True)
        got = [l for l in out if int(l.split()[1]) in KEEP]
        want = open(os.path.join(GOLDEN, name)).readlines()
        assert len(want) > 1000
        assert got == want


def test_host_state_machine_matches_golden_sam(hostsim_bin, tmp_path):
    """Host build of ht2_core.h + the host SAM back end reproduce the reference's
    SAM byte for byte on the tiny fixture (two references, N gap, indels, Ns,
    ragged lengths, unalignable reads)."""
    out = str(tmp_path / "se.sam")
    subprocess.run([hostsim_bin, "tiny", "tiny_se.fa", out], cwd=GOLDEN, check=True, stderr=subprocess.DEVNULL)
    assert sam_lines(open(out, "rb").read()) == sam_lines(open(os.path.join(GOLDEN, "tiny_se.sam"), "rb").read())


def test_host_state_machine_matches_golden_sam_paired(hostsim_bin, tmp_path):
    """Paired-end: concordant pairs, mate rescue (alignMate), unpaired mates, unaligned mates."""
    out = str(tmp_path / "pe.sam")
    subprocess.run([hostsim_bin, "tiny", "tiny_pe_1.fa", out, "tiny_pe_2.fa"], cwd=GOLDEN, check=True, stderr=subprocess.DEVNULL)
    assert sam_lines(open(out, "rb").read()) == sam_lines(open(os.path.join(GOLDEN, "tiny_pe.sam"), "rb").read())


def test_host_seed_search_matches_reference_dump(hostsim_bin):
    """Host build of the product's seed-search headers (ht2_seed.h, ht2_graph.h: mapGLF / mapGLF1 /
    rank_M / select_F / getInEdgeCount / getOffset over the packed image) == the unmodified
    reference's partialSearch + getOffset dump, on the linear AND the graph (SNP) fixture."""
    for idx, mode, name in (("tiny", "1", "tiny_dump.txt"), ("tiny", "0", "tiny_dump_spliced.txt"),
                            ("tiny_snp", "1", "tiny_snp_dump.txt")):
        out = subprocess.run([hostsim_bin, "--seed-dump", idx, "tiny_se.fa", mode], cwd=GOLDEN, check=True,
                             stdout=subprocess.PIPE).stdout.decode().splitlines(True)
        got = [l for l in out if int(l.split()[1]) in KEEP]
        want = open(os.path.join(GOLDEN, name)).readlines()
        assert got == want, (idx, mode)
    graph = open(os.path.join(GOLDEN, "tiny_snp_dump.txt")).read()
    assert graph.count("\nG ") > 3000 and any(l.split()[6] != "0" for l in graph.splitlines() if l.startswith("G "))


def test_host_state_machine_fastq_qualities(hostsim_bin, tmp_path):
    """FASTQ input with low-quality stretches: quality-aware mismatch and soft-clip penalties
    (Scoring::mm / COST_MODEL_QUAL, scoring.h:117-128), SE and PE, byte-identical SAM."""
    for args, gold in ((["tiny_se.fq"], "tiny_se_fq.sam"), (["tiny_pe_1.fq", "tiny_pe_2.fq"], "tiny_pe_fq.sam")):
        out = str(tmp_path / gold)
        cmd = [hostsim_bin, "tiny", args[0], out] + args[1:]
        subprocess.run(cmd, cwd=GOLDEN, check=True, stderr=subprocess.DEVNULL)
        assert sam_lines(open(out, "rb").read()) == sam_lines(open(os.path.join(GOLDEN, gold), "rb").read())


def test_host_graph_index_alignment_matches_golden_reference_sam(hostsim_bin, tmp_path):
    """GRAPH (SNP) index end to end: graph searches with in-edge lists, the group walk, adjustWithALT and the
    ALT-aware extension (SNP / deletion / insertion ALTs), Zs:Z tags.  SE, PE, FASTQ, and reads that carry ALT
    alleles (129 of 400 alignments go through ALTs): byte-identical SAM with the unmodified reference."""
    for args, gold in ((["tiny_se.fa"], "tiny_snp_se.sam"), (["tiny_pe_1.fa", "tiny_pe_2.fa"], "tiny_snp_pe.sam"),
                       (["tiny_se.fq"], "tiny_snp_se_fq.sam"), (["tiny_alt_1.fa"], "tiny_snp_alt_se.sam"),
                       (["tiny_alt_1.fa", "tiny_alt_2.fa"], "tiny_snp_alt_pe.sam")):
        out = str(tmp_path / gold)
        subprocess.run([hostsim_bin, "tiny_snp", args[0], out] + args[1:], cwd=GOLDEN, check=True, stderr=subprocess.DEVNULL)
        want = open(os.path.join(GOLDEN, gold), "rb").read()
        assert sam_lines(open(out, "rb").read()) == sam_lines(want)
    assert open(os.path.join(GOLDEN, "tiny_snp_alt_se.sam")).read().count("Zs:Z:") > 100


def test_host_state_machine_option_matrix(hostsim_bin, tmp_path):
    """Every option of the reference's command line that reaches the path (-k, --mp, --np, --rdg, --rfg,
    --sp, --ignore-quals, --nofw/--norc, --secondary, --no-mixed, --no-discordant, -I/-X, --score-min,
    --bowtie2-dp, --gbar, --sensitive, --very-sensitive) against the md5 of the unmodified reference's SAM
    for the same flags (tests/golden/option_matrix.json), on the linear and the graph index."""
    import hashlib, json
    cases = json.load(open(os.path.join(GOLDEN, "option_matrix.json")))
    assert len(cases) >= 23
    assert sum("bowtie2_dp" in c["options"] for c in cases) >= 7
    for c in cases:
        out = str(tmp_path / "o.sam")
        args = [c["reads"][0], out] + c["reads"][1:]
        r = subprocess.run([hostsim_bin, c["index"]] + args, cwd=GOLDEN, check=True, stderr=subprocess.PIPE,
                           env=dict(os.environ, HT2_OPTS=c["options"]))
        assert b"err=" not in r.stderr, c
        got = hashlib.md5(b"\n".join(sam_lines(open(out, "rb").read())) + b"\n").hexdigest()
        assert got == c["md5"], c


def test_batch_sam_back_end_matches_golden_and_is_thread_invariant(hostsim_bin, tmp_path):
    """ht2_format_batch -- the body of ht2gpu_format_sam: C-ABI result batch -> SAM on host threads --
    fed with the host state machine's results: golden SAM on the tiny fixtures, and the same text for 1
    and 7 threads on a batch large enough (> 4096 units) to be split."""
    env = dict(os.environ, HT2_VIA_BATCH="1")
    for idx, args, gold in (("tiny", ["tiny_pe_1.fa", "tiny_pe_2.fa"], "tiny_pe.sam"),
                            ("tiny_snp", ["tiny_alt_1.fa", "tiny_alt_2.fa"], "tiny_snp_alt_pe.sam"),
                            ("tiny", ["tiny_se.fq"], "tiny_se_fq.sam")):
        out = str(tmp_path / "o.sam")
        subprocess.run([hostsim_bin, idx, args[0], out] + args[1:], cwd=GOLDEN, check=True, stderr=subprocess.DEVNULL, env=env)
        assert sam_lines(open(out, "rb").read()) == sam_lines(open(os.path.join(GOLDEN, gold), "rb").read()), gold
    big = str(tmp_path / "big.fa")
    recs = open(os.path.join(GOLDEN, "tiny_se.fa")).read().split(">")[1:]
    with open(big, "w") as f:
        for rep in range(7):
            for r in recs:
                name, rest = r.split("\n", 1)
                f.write(">%s_%d\n%s" % (name, rep, rest))
    outs = []
    for threads, via in (("1", "1"), ("7", "1"), ("1", None)):
        out = str(tmp_path / ("big_%s_%s.sam" % (threads, via)))
        e = dict(os.environ, HT2_THREADS=threads)
        if via:
            e["HT2_VIA_BATCH"] = via
        subprocess.run([hostsim_bin, "tiny", big, out], cwd=GOLDEN, check=True, stderr=subprocess.DEVNULL, env=e)
        outs.append(open(out, "rb").read())
    assert outs[0] == outs[1] == outs[2] and outs[0].count(b"\n") > 4900


def test_spliced_alignment_host_build_matches_golden_reference_sam(hostsim_spliced_bin, tmp_path):
    """Spliced alignment (the reference's default mode, run with --no-temp-splicesite so that the splice-site
    DB stays empty and reads are independent): the host build with the spliced pieces enabled -- splice
    edits, the spliced branch of combineWith (motif classes, intron-length rules, probability model),
    calculateScore for splice edits, N / XS:A / fragment lengths in SAM -- against golden SAM of the
    unmodified reference: 400 RNA-like reads over one or two introns (340 spliced alignments), the DNA
    fixtures SE / PE FASTQ, and ALT-allele pairs on the graph index.  The CUDA library compiles the same
    pieces into its kernels (tests/test_gpu.py and tests/test_geometry_edges.py run them on the device)."""
    env = dict(os.environ, HT2_OPTS="spliced=1")
    for idx, args, gold in (("tiny", ["tiny_rna.fa"], "tiny_spliced_rna.sam"), ("tiny", ["tiny_se.fa"], "tiny_spliced_se.sam"),
                            ("tiny", ["tiny_pe_1.fq", "tiny_pe_2.fq"], "tiny_spliced_pe_fq.sam"),
                            ("tiny_snp", ["tiny_alt_1.fa", "tiny_alt_2.fa"], "tiny_snp_spliced_alt_pe.sam")):
        out = str(tmp_path / "o.sam")
        r = subprocess.run([hostsim_spliced_bin, idx, args[0], out] + args[1:], cwd=GOLDEN, check=True, stderr=subprocess.PIPE, env=env)
        assert b"err=" not in r.stderr, gold
        assert sam_lines(open(out, "rb").read()) == sam_lines(open(os.path.join(GOLDEN, gold), "rb").read()), gold
    # the same through the C ABI's result structures (splice edits packed into ht2gpu_edit_t) and ht2_format_batch
    out = str(tmp_path / "ob.sam")
    subprocess.run([hostsim_spliced_bin, "tiny", "tiny_rna.fa", out], cwd=GOLDEN, check=True, stderr=subprocess.DEVNULL,
                   env=dict(env, HT2_VIA_BATCH="1"))
    assert sam_lines(open(out, "rb").read()) == sam_lines(open(os.path.join(GOLDEN, "tiny_spliced_rna.sam"), "rb").read())
    rna = open(os.path.join(GOLDEN, "tiny_spliced_rna.sam")).read().splitlines()
    assert sum(1 for l in rna if not l.startswith("@") and "N" in l.split("\t")[5]) >= 300
    assert any("XS:A:+" in l for l in rna) and any("XS:A:-" in l for l in rna)
    # and the same build without spliced mode still reproduces the --no-spliced-alignment goldens
    out = str(tmp_path / "o2.sam")
    subprocess.run([hostsim_spliced_bin, "tiny", "tiny_pe_1.fa", out, "tiny_pe_2.fa"], cwd=GOLDEN, check=True, stderr=subprocess.DEVNULL)
    assert sam_lines(open(out, "rb").read()) == sam_lines(open(os.path.join(GOLDEN, "tiny_pe.sam"), "rb").read())


def test_populated_splice_site_db_host_build_matches_golden_reference_sam(hostsim_spliced_bin, tmp_path):
    """--known-splicesite-infile / --novel-splicesite-infile with --no-temp-splicesite (SURVEY 8f.3): the three
    `if(!ssdb.empty())` branches of hybridSearch_recur (spliced_aligner.h:409-668, 685-811, 1365-1494), combineWith
    pinned to a listed site, known-site scoring, and the template-length adjustment of concordant pairs
    (aligner_result.h:1631-1690) -- host build of the same sources against golden SAM of the unmodified reference:
    600 RNA-like reads (many with 1-11 bases beyond a junction), 300 pairs with mates in different exons, on the
    linear and the graph index, with -k 20 --secondary, and with the sites split over the two files."""
    env = dict(os.environ, HT2_OPTS="spliced=1")
    for idx, ss, opts, args, gold in (
            ("tiny", "tiny_ss_rna_ss.txt", "", ["tiny_ss_rna.fa"], "tiny_ss_rna_se.sam"),
            ("tiny", "tiny_ss_rna_ss.txt", "", ["tiny_ss_rna_1.fa", "tiny_ss_rna_2.fa"], "tiny_ss_rna_pe.sam"),
            ("tiny_snp", "tiny_ss_rna_ss.txt", "", ["tiny_ss_rna_1.fa", "tiny_ss_rna_2.fa"], "tiny_snp_ss_rna_pe.sam"),
            ("tiny", "tiny_ss_rna_ss.txt", ",khits=20,secondary=1", ["tiny_ss_rna.fa"], "tiny_ss_rna_se_k20_secondary.sam"),
            ("tiny", "tiny_ss_known.txt,tiny_ss_novel.txt", "", ["tiny_ss_rna_1.fa", "tiny_ss_rna_2.fa"], "tiny_ss_rna_pe_known_novel.sam")):
        out = str(tmp_path / "o.sam")
        e = dict(env, HT2_SS=ss, HT2_OPTS=env["HT2_OPTS"] + opts)
        r = subprocess.run([hostsim_spliced_bin, idx, args[0], out] + args[1:], cwd=GOLDEN, check=True, stderr=subprocess.PIPE, env=e)
        assert b"errors=0" in r.stderr, gold
        assert sam_lines(open(out, "rb").read()) == sam_lines(open(os.path.join(GOLDEN, gold), "rb").read()), gold
    # the DB matters: without it the same reads align differently (so the test above is not vacuous)
    out = str(tmp_path / "o2.sam")
    subprocess.run([hostsim_spliced_bin, "tiny", "tiny_ss_rna.fa", out], cwd=GOLDEN, check=True, stderr=subprocess.DEVNULL, env=env)
    a, b = sam_lines(open(out, "rb").read()), sam_lines(open(os.path.join(GOLDEN, "tiny_ss_rna_se.sam"), "rb").read())
    assert sum(1 for x, y in zip(a, b) if x != y) > 200
    gold = open(os.path.join(GOLDEN, "tiny_ss_rna_se.sam")).read().splitlines()
    assert sum(1 for l in gold if not l.startswith("@") and "N" in l.split("\t")[5]) >= 350
    # --novel-splicesite-outfile: the junctions of the printed alignments, collected by the formatter and filtered like
    # SpliceSiteDB::print (read-count cutoffs, near-duplicate suppression) == the reference's file
    for args, gold in ((["tiny_ss_rna_1.fa", "tiny_ss_rna_2.fa"], "tiny_ss_rna_pe_novel_out.txt"), (["tiny_rna.fa"], "tiny_rna_novel_out.txt")):
        out, ss = str(tmp_path / "o3.sam"), str(tmp_path / "novel.txt")
        subprocess.run([hostsim_spliced_bin, "tiny", args[0], out] + args[1:], cwd=GOLDEN, check=True, stderr=subprocess.DEVNULL, env=dict(env, HT2_SS_OUT=ss))
        assert open(ss).read() == open(os.path.join(GOLDEN, gold)).read(), gold
    # read-count cutoffs: tiny_rna.fa plus a renamed copy of its first 200 reads -> 70 % of the sites have one read, the
    # cutoff becomes 2 and single-read sites survive only with edit distance 0 (275 sites, 223 written by the reference)
    dup = str(tmp_path / "dup.fa")
    lines = open(os.path.join(GOLDEN, "tiny_rna.fa")).read().splitlines(True)
    open(dup, "w").write("".join(lines) + "".join(l.replace(">t", ">dup", 1) if l.startswith(">") else l for l in lines[:400]))
    ss = str(tmp_path / "novel_dup.txt")
    subprocess.run([hostsim_spliced_bin, "tiny", dup, str(tmp_path / "o4.sam")], cwd=GOLDEN, check=True, stderr=subprocess.DEVNULL, env=dict(env, HT2_SS_OUT=ss))
    got = open(ss).read()
    assert got == open(os.path.join(GOLDEN, "tiny_rna_dup_novel_out.txt")).read() and got.count("\n") == 223
    # a malformed site file is an error, not a silent skip
    bad = str(tmp_path / "bad_ss.txt")
    open(bad, "w").write("chrA\t100\n")
    r = subprocess.run([hostsim_spliced_bin, "tiny", "tiny_rna.fa", str(tmp_path / "o5.sam")], cwd=GOLDEN, stderr=subprocess.PIPE, env=dict(env, HT2_SS=bad))
    assert r.returncode != 0 and b"truncated splice-site record" in r.stderr


@pytest.mark.parametrize("case", sorted(refsets.SPLICED_CASES))
def test_spliced_corpus_host_build_matches_reference(hostsim_spliced_bin, spliced_dir, tmp_path, case):
    """The spliced corpus (tools/splicereads.py: every motif, anchors of 1-30 bases, intron lengths at every rule
    boundary, several junctions per read, sequence ends and the N gap) and its simulated bulk through the host build
    of the spliced aligner: the md5 of the reference's SAM (--no-temp-splicesite) for every spliced/* case, and of its
    --novel-splicesite-outfile where recorded.  The reads the library flags for a device capacity are the recorded
    ones (the host build has the device's capacities) and are left out of the md5, as on the GPU."""
    index, _, _, _, opts, _ = refsets.SPLICED_CASES[case]
    fs, ss = refsets.spliced_files(spliced_dir, case)
    out, novel = str(tmp_path / "o.sam"), str(tmp_path / "novel.txt")
    env = dict(os.environ, HT2_OPTS=",".join(["spliced=1"] + ["%s=%s" % kv for kv in sorted(opts.items())]))
    if ss:
        env["HT2_SS"] = ss
    if case in refsets.SPLICED_NOVEL:
        env["HT2_SS_OUT"] = novel
    r = subprocess.run([hostsim_spliced_bin, index, fs[0], out] + fs[1:], cwd=GOLDEN, check=True, stderr=subprocess.PIPE, env=env)
    key = "spliced/" + case
    bad = sorted(set(re.findall(r"(?:read|pair) \d+ \(([^)/]*)[^)]*\): err=", r.stderr.decode())))
    assert bad == REF_SETS["flagged"].get(key, [])
    sam = open(out, "rb").read()
    assert refsets.sam_md5(sam, bad) == REF_SETS["md5"][key]
    assert sum(1 for l in sam_lines(sam) if not l.startswith(b"@") and b"N" in l.split(b"\t")[5]) > 250
    if case in refsets.SPLICED_NOVEL:
        assert hashlib.md5(open(novel, "rb").read()).hexdigest() == REF_SETS["md5"]["spliced_novel/" + case]


def test_spliced_corpus_is_deterministic(tmp_path):
    """tools/splicereads.py writes the same bytes for the same seed, and the recorded md5s belong to those bytes."""
    import splicereads
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    splicereads.generate(os.path.join(GOLDEN, "tiny.fa"), a, refsets.SPLICE_SEED)
    splicereads.generate(os.path.join(GOLDEN, "tiny.fa"), b, refsets.SPLICE_SEED)
    for suffix in ("_se.fa", "_q.fq", "_pe_1.fa", "_pe_2.fa", "_ss.txt", "_sim.fa", "_sim_1.fa", "_sim_2.fa", "_sim_ss.txt"):
        assert open(a + suffix, "rb").read() == open(b + suffix, "rb").read(), suffix
    names = [l[1:].split("_")[0] for l in open(a + "_se.fa").read().split() if l.startswith(">")]
    assert 1800 < len(names) < 4000
    assert {"motif", "anchor", "len", "multi", "sense", "redge", "gap", "join"} <= set(names)


def test_striped_dp_fill_and_backtrace_against_plain_scalar_dp(hostsim_bin):
    """The --bowtie2-dp kernel on its own (ht2_sw.h: striped s16x2 fill with the DPX-style max(a+b,c) steps +
    plane-derived backtrace) against an independent scalar statement of the recurrences: 400 random problems
    (read lengths 20-255, random penalties / gap barriers / qualities / Ns): every last-row score equal, and
    the returned edits turn the read into the reference window at exactly the optimal score."""
    r = subprocess.run([hostsim_bin, "--sw-selftest", "400", "3"], check=True, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    out = r.stdout.decode()
    assert "400 problems" in out and " 0 failures" in out, out + r.stderr.decode()
    assert int(out.split(" backtraces")[0].split()[-1]) > 200


def test_read_front_end_matches_python_restatement(lib, tmp_path):
    """csrc/ht2_reads.cpp (multi-threaded record index + batch parser behind ht2gpu_parse_reads / ht2gpu_run_reads)
    against the independent Python restatement of FastaPatternSource / FastqPatternSource in api.py: bases,
    qualities, offsets, names (default names, /1 /2 fixing) and per-read seeds, single- and multi-threaded,
    CRLF, missing final newline, blank lines between FASTQ records, -5/-3, --phred64, -s/-u."""
    from hisat2_b200 import api
    RB = api.ReadBatch

    def same(a, b):
        assert a.n == b.n and a.paired == b.paired
        assert np.array_equal(a.offs, b.offs) and np.array_equal(a.seq, b.seq) and np.array_equal(a.seeds, b.seeds)
        assert a.names == b.names
        assert (a.qual is None) == (b.qual is None)
        if a.qual is not None:
            assert np.array_equal(a.qual, b.qual)
    g = lambda n: os.path.join(GOLDEN, n)
    same(RB.parse(g("tiny_se.fa")), RB.from_fasta(g("tiny_se.fa")))
    same(RB.parse(g("tiny_pe_1.fa"), g("tiny_pe_2.fa")), RB.from_fasta(g("tiny_pe_1.fa"), path2=g("tiny_pe_2.fa")))
    same(RB.parse(g("tiny_se.fq"), fastq=True), RB.from_fastq(g("tiny_se.fq")))
    same(RB.parse(g("tiny_pe_1.fq"), g("tiny_pe_2.fq"), fastq=True), RB.from_fastq(g("tiny_pe_1.fq"), path2=g("tiny_pe_2.fq")))
    same(RB.parse(data1=open(g("tiny_se.fq"), "rb").read(), fastq=True, threads=5), RB.from_fastq(g("tiny_se.fq")))
    # a file large enough to be indexed and parsed by several threads (> 1 MiB, > 2048 records)
    rng = np.random.default_rng(11)
    big = str(tmp_path / "big.fa")
    with open(big, "wb") as f:
        for i in range(9000):
            L = int(rng.integers(1, 250))
            sq = rng.choice(np.frombuffer(b"ACGTNacgtnRY-", dtype=np.uint8), L).tobytes()
            if i % 3 == 0 and L > 80:
                sq = sq[:70] + b"\r\n" + sq[70:]          # multi-line record, CRLF
            f.write(b">" + (b"" if i % 1000 == 7 else b"r%d some text/%d" % (i, i % 3)) + b"\n" + sq + (b"\n" if i < 8999 else b""))
    same(RB.parse(big, threads=1), RB.from_fasta(big))
    same(RB.parse(big, threads=7), RB.from_fasta(big))
    same(RB.parse(big, big, threads=6), RB.from_fasta(big, path2=big))
    fq = str(tmp_path / "big.fq")
    fq_blank = str(tmp_path / "blank.fq")
    with open(fq, "wb") as f, open(fq_blank, "wb") as fb:
        for i in range(12000):
            L = int(rng.integers(1, 200))
            sq = rng.choice(np.frombuffer(b"ACGTN.", dtype=np.uint8), L, p=[.24, .24, .24, .24, .02, .02]).tobytes()
            ql = rng.integers(33, 74, L).astype(np.uint8).tobytes()      # '@' (64) occurs at line starts too
            rec = b"@q%d\n" % i + sq + b"\n+\n" + ql + b"\n"
            f.write(rec)
            fb.write(rec + (b"\n" if i % 5 == 0 else b""))
    same(RB.parse(fq, fastq=True, threads=1), RB.from_fastq(fq))
    same(RB.parse(fq, fastq=True, threads=8), RB.from_fastq(fq))
    same(RB.parse(fq_blank, fastq=True, threads=8), RB.from_fastq(fq))           # falls back to the sequential record scan
    # -s / -u, -5 / -3, --phred64
    a, b = RB.parse(fq, fastq=True, skip=100, upto=50, threads=4), RB.from_fastq(fq)
    assert a.n == 50 and a.names == b.names[100:150]
    t = RB.parse(g("tiny_se.fq"), fastq=True, trim5=3, trim3=5)
    full = RB.from_fastq(g("tiny_se.fq"))
    for i in (0, 1, 17, full.n - 1):
        lo, hi = int(full.offs[i]), int(full.offs[i + 1])
        keep = slice(lo + 3, max(lo + 3, hi - 5)) if hi - lo > 3 else slice(lo, lo)
        assert np.array_equal(t.seq[int(t.offs[i]):int(t.offs[i + 1])], full.seq[keep])
        assert np.array_equal(t.qual[int(t.offs[i]):int(t.offs[i + 1])], full.qual[keep])
    p64 = str(tmp_path / "p64.fq")
    src = open(g("tiny_se.fq"), "rb").read().split(b"\n")
    with open(p64, "wb") as f:
        for i in range(0, len(src) - 1, 4):
            f.write(b"\n".join([src[i], src[i + 1], src[i + 2], bytes(c + 31 for c in src[i + 3])]) + b"\n")
    same(RB.parse(p64, fastq=True, phred64=1), full)
    with pytest.raises(api.Ht2GpuError):
        RB.parse(g("tiny_se.fa"), fastq=True)
    with pytest.raises(api.Ht2GpuError):
        RB.parse(g("tiny_pe_1.fa"), g("tiny_se.fa"))


def test_ht2_h_clients_link_unchanged(lib, tmp_path):
    """libht2gpu.so exports the hisat2lib API (hisat2lib/ht2.h:67-150) under the reference's names and struct
    layouts: a C client built from the declarations of the reference's ht2.h, written out here, links to this
    library and reads the reference names of the tiny fixture."""
    src = str(tmp_path / "client.c")
    decls = """
#include <stdint.h>
typedef int ht2_error_t; typedef void* ht2_handle_t;
struct ht2_options { int offRate, useMm, useShmem, mmSweep, noRefNames, noSplicedAlignment, gVerbose, startVerbose, sanityCheck, useHaplotype; };
typedef struct ht2_options ht2_option_t;
struct ht2_index_getrefnames_result { int count; char* names[0]; };
ht2_handle_t ht2_init(const char*, ht2_option_t*); void ht2_close(ht2_handle_t); ht2_error_t ht2_init_options(ht2_option_t*);
const char* ht2_index_getrefnamebyid(ht2_handle_t, uint32_t);
ht2_error_t ht2_index_getrefnames(ht2_handle_t, struct ht2_index_getrefnames_result**);
"""
    open(src, "w").write(decls + """
#include <stdio.h>
#include <stdlib.h>
int main(int argc, char** argv) {
    ht2_option_t o;
    if (ht2_init_options(&o) != 0 || o.offRate != -1 || o.noSplicedAlignment != 0) return 2;
    ht2_handle_t h = ht2_init(argv[1], &o);
    if (!h) return 3;
    struct ht2_index_getrefnames_result* r = NULL;
    if (ht2_index_getrefnames(h, &r) != 0) return 4;
    printf("%d\\n", r->count);
    for (int i = 0; i < r->count; i++) printf("%s|%s\\n", r->names[i], ht2_index_getrefnamebyid(h, (uint32_t)i));
    printf("%s\\n", ht2_index_getrefnamebyid(h, (uint32_t)r->count) ? "extra" : "null");
    free(r);
    ht2_close(h);
    return 0;
}
""")
    exe = str(tmp_path / "client")
    libdir = os.path.join(ROOT, "hisat2_b200")
    subprocess.run(["gcc", "-std=gnu99", "-o", exe, src, "-L", libdir, "-l:libht2gpu.so", "-Wl,-rpath," + libdir], check=True)
    out = subprocess.run([exe, os.path.join(GOLDEN, "tiny")], check=True, stdout=subprocess.PIPE).stdout.decode().splitlines()
    from hisat2_b200 import api
    names = [l.split("\t")[1][3:] for l in open(os.path.join(GOLDEN, "tiny_se.sam")).read().splitlines() if l.startswith("@SQ")]
    assert int(out[0]) == len(names) and out[-1] == "null"
    for tok, nm in zip(out[1:-1], names):
        a, b = tok.split("|")
        assert a == b and a.split()[0] == nm


def test_abi_exports_every_declared_symbol(lib):
    hdr = open(os.path.join(ROOT, "include", "ht2gpu.h")).read()
    declared = sorted(set(re.findall(r"\b(ht2gpu_[a-z_]+)\s*\(", hdr)))
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(lib, name), name
    from hisat2_b200 import api
    assert sorted(api.EXPORTS) == declared


def test_image_build_is_host_only_and_consistent(lib):
    from hisat2_b200 import api
    img = api.Index.build_image(os.path.join(GOLDEN, "tiny"))
    assert img[:4].tobytes() == b"HT2B"
    hdr = np.frombuffer(img[:16].tobytes(), dtype="<u4")
    assert hdr[1] == 6  # image version
    total = int(np.frombuffer(img[8:16].tobytes(), dtype="<u8")[0])
    assert total == img.nbytes and total % 128 == 0
    # global geometry (Ht2Gfm at offset 16): len, gbwtLen, numNodes, eftabLen, linearFM, sideSz, sideGbwtSz, sideGbwtLen
    g = np.frombuffer(img[16:16 + 32].tobytes(), dtype="<u4")
    raw = np.fromfile(os.path.join(GOLDEN, "tiny.1.ht2"), dtype="<u4", count=11)
    assert g[0] == raw[2] and g[1] == raw[3]
    # linear indexes are re-laid as 32-byte rank sides of 64 rows (ht2_image.h)
    assert g[4] == 1 and g[5] == 32 and g[6] == 16 and g[7] == 64
    # the rank sides must restate the .ht2 file: same BW string, occ = fchr + running counts without '$'
    gbwt_len = int(g[1])
    geom = np.frombuffer(img[16:16 + 136].tobytes(), dtype="<u4")
    fchr, z0 = geom[18:23], int(geom[27])
    o_gfm = int(np.frombuffer(img[16 + 112:16 + 120].tobytes(), dtype="<u8")[0])
    f = open(os.path.join(GOLDEN, "tiny.1.ht2"), "rb").read()
    npat = int(np.frombuffer(f[44:48], "<u4")[0])
    pos = 48 + 4 * npat
    nfrag = int(np.frombuffer(f[pos:pos + 4], "<u4")[0])
    pos += 4 + 12 * nfrag
    nsides_old = (gbwt_len // 4 + 1 + 47) // 48
    old = np.frombuffer(f[pos:pos + 64 * nsides_old], np.uint8).reshape(-1, 64)
    bw_old = ((old[:, :48, None] >> np.array([0, 2, 4, 6])) & 3).reshape(-1)[:gbwt_len]
    nsides = (gbwt_len >> 6) + 1
    new = np.frombuffer(img[o_gfm:o_gfm + 32 * nsides].tobytes(), np.uint8).reshape(-1, 32)
    bw_new = ((new[:, :16, None] >> np.array([0, 2, 4, 6])) & 3).reshape(-1)[:gbwt_len]
    assert (bw_old == bw_new).all()
    occ = new[:, 16:].copy().view("<u4")
    onehot = (bw_new[:, None] == np.arange(4)).astype(np.int64)
    onehot[z0] = 0
    cum = np.vstack([np.zeros((1, 4), np.int64), np.cumsum(onehot, axis=0)])
    want = cum[np.minimum(np.arange(nsides) * 64, gbwt_len)] + fchr[:4].astype(np.int64)
    assert (occ.astype(np.int64) == want).all()
    # graph (SNP) fixture: 64-byte graph rank sides; M_occ / F_loc restate rank1(M) / select1(F)
    gimg = api.Index.build_image(os.path.join(GOLDEN, "tiny_snp"))
    gg = np.frombuffer(gimg[16:16 + 136].tobytes(), dtype="<u4")
    assert gg[4] == 0 and gg[5] == 64 and gg[7] == 64 and gg[1] > gg[2] > gg[0]      # rows > nodes > bases
    o = int(np.frombuffer(gimg[16 + 112:16 + 120].tobytes(), dtype="<u8")[0])
    ns = (int(gg[1]) >> 6) + 1
    sides = np.frombuffer(gimg[o:o + 64 * ns].tobytes(), np.uint8).reshape(-1, 64)
    fbits = np.unpackbits(sides[:, 16:24], axis=1, bitorder="little").reshape(-1)[:int(gg[1])]
    mbits = np.unpackbits(sides[:, 24:32], axis=1, bitorder="little").reshape(-1)[:int(gg[1])]
    assert int(fbits.sum()) == int(gg[2])                                              # one F bit per node
    tr = sides[:, 32:56].copy().view("<u4")
    mocc = np.concatenate([[0], np.cumsum(mbits, dtype=np.int64)]).astype(np.int64)[np.minimum(np.arange(ns) * 64, int(gg[1]))]
    assert (tr[:, 4] == mocc).all()
    fpos = np.flatnonzero(fbits)
    ok = mocc > 0
    assert (tr[ok, 5] == fpos[mocc[ok] - 1]).all()
    with pytest.raises(api.Ht2GpuError):
        api.Index.build_image(os.path.join(GOLDEN, "does_not_exist"))


def test_open_fails_loudly_without_cuda(lib):
    """No CPU fallback: without a usable device open() must fail."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from hisat2_b200 import api
    with pytest.raises(api.Ht2GpuError) as e:
        api.Index(os.path.join(GOLDEN, "tiny"))
    assert "CUDA" in str(e.value)


def test_read_seed_matches_reference_formula(lib):
    """genRandSeed (pat.h:55-91) known answer computed by hand from the formula."""
    seq = np.array([0, 1, 2, 3, 4, 0], dtype=np.uint8)
    name = b"r7/1"
    want = ((0 + 101) * 59 * 61 * 67 * 71 * 73 * 79 * 83) & 0xffffffff
    for i, p in enumerate(seq):
        want ^= (int(p) << ((i & 15) << 1)) & 0xffffffff
    for i in range(len(seq)):
        want ^= (ord("I") << ((i & 3) << 3)) & 0xffffffff
    for i, ch in enumerate(name):
        if ch == ord("/"):
            break
        want ^= (ch << ((i & 3) << 3)) & 0xffffffff
    got = lib.ht2gpu_read_seed(seq.ctypes.data, None, len(seq), name, 0)
    assert got == want


def test_fasta_parser_and_simulator_are_deterministic(lib):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import simreads
    from hisat2_b200 import api
    _, seq = simreads.load_fasta_codes(os.path.join(GOLDEN, "tiny.fa"))
    a1, a2 = simreads.simulate(seq, 50, seed=3)
    b1, b2 = simreads.simulate(seq, 50, seed=3)
    assert (a1 == b1).all() and (a2 == b2).all() and a1.shape == (50, 101)
    batch = api.ReadBatch.from_fasta(os.path.join(GOLDEN, "tiny_se.fa"))
    assert batch.n == 700 and batch.offs[-1] == len(batch.seq) and batch.seq.max() <= 4
    assert batch.names[0] == b"s0"


def test_shard_ranges_cover_input_in_order():
    from hisat2_b200.parallel import shard_range
    for n in (0, 1, 7, 8, 1000003):
        for w in (1, 2, 3, 8):
            pos = 0
            for r in range(w):
                lo, hi = shard_range(n, r, w)
                assert lo == pos and hi >= lo
                pos = hi
            assert pos == n


def _gloo_worker(rank, world, port, tmpdir):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from hisat2_b200 import api
    from hisat2_b200.parallel import broadcast_image, gather_bytes, shard_range
    img = api.Index.build_image(os.path.join(GOLDEN, "tiny")) if rank == 0 else None
    t = broadcast_image(img, rank)
    ref = api.Index.build_image(os.path.join(GOLDEN, "tiny"))
    assert t.numpy().tobytes() == ref.tobytes()
    lines = open(os.path.join(GOLDEN, "tiny_se.sam"), "rb").read().splitlines(True)
    recs = [l for l in lines if not l.startswith(b"@")]
    lo, hi = shard_range(len(recs), rank, world)
    chunks = gather_bytes(b"".join(recs[lo:hi]), rank, world)
    if rank == 0:
        assert b"".join(chunks) == b"".join(recs)
        open(os.path.join(tmpdir, "ok"), "w").write("ok")
    dist.destroy_process_group()


def test_two_rank_gloo_broadcast_and_ordered_gather(lib, tmp_path):
    """world_size-2 CPU run of the multi-GPU plumbing: image broadcast + rank-ordered gather."""
    import torch.multiprocessing as mp
    port = 29500 + (os.getpid() % 2000)
    mp.spawn(_gloo_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    assert os.path.exists(os.path.join(str(tmp_path), "ok"))
