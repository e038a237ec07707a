"""The edge-read corpus (tools/edgereads.py) and the spliced corpus (tools/splicereads.py) under every launch geometry
of the alignment kernel, and a plain restatement of the alignment score, splices included.

The pool kernel has four linear-index instantiations (8 warps x 4 read slots, the DNA-only 8 x 2 that a default handle
falls back to when the device lacks room for the 4-slot workspace, 4 x 8, and any of them with several blocks per SM).
Every one must write the reference's SAM, so every case runs under each and asserts which kernel ran
(Index.geometry()).  score_record() recomputes AS:i, XM, XO, XG, NM, YS:i and the --score-min test from each record's
CIGAR, MD:Z, SEQ and QUAL with exact integers (numpy.float32 where the reference computes in float), and the splice
penalties from the reference sequence at each intron; it is pinned to the reference by the committed golden SAMs (CPU)
and applied to every GPU run."""
import glob
import math
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, sam_lines

sys.path.insert(0, os.path.join(ROOT, "tools"))
import edgereads  # noqa: E402
import refsets  # noqa: E402

REF_SETS = refsets.load_expected()

# ---------------------------------------------------------------------------------------------------------------------
# score_record: the reference's end-to-end scoring (Scoring::mm / n / sc / readGap / refGap, SimpleFunc::f) restated
# ---------------------------------------------------------------------------------------------------------------------
# Splice motifs by the intron's first and last two reference bases (hi_aligner.h: GT-AG and its reverse complement
# CT-AC are canonical; GC-AG, AT-AC and their reverse complements CT-GC, GT-AT are semi-canonical; anything else is
# non-canonical and has no sense).  '+' / '-' is the transcript strand of XS:A.
MOTIFS = {("GT", "AG"): ("can", "+"), ("CT", "AC"): ("can", "-"), ("GC", "AG"): ("semi", "+"), ("AT", "AC"): ("semi", "+"),
          ("CT", "GC"): ("semi", "-"), ("GT", "AT"): ("semi", "-")}


def intron_pen(n):
    """--pen-canintronlen / --pen-noncanintronlen G,-8,1: max(0, (int)(-8 + ln(n))) in double."""
    return max(0, int(-8.0 + math.log(n)))


# can_pen / noncan_pen: --pen-cansplice 0 / --pen-noncansplice 12 (semi-canonical motifs pay the non-canonical one)
DEFAULT_SCORING = dict(mp_max=6, mp_min=2, sp_max=2, sp_min=1, np=1, rdg_const=5, rdg_linear=3, rfg_const=5, rfg_linear=3,
                       ignore_quals=0, score_min=None, can_pen=0, noncan_pen=12, intron_pen=intron_pen, motifs=MOTIFS)
MIN_INTRON_LEN = 20          # --min-intronlen: a shorter reference skip is a deletion
MIN_ANCHOR = 7               # minAnchorLen (canonical) / minAnchorLenNoncan (semi- and non-canonical)
MIN_ANCHOR_NONCAN = 14
F32 = np.float32


def mm_penalty(o, q):
    """Quality-aware mismatch penalty for Phred quality q: MN + floor((MX - MN) * min(q, 40) / 40), in float."""
    if o["ignore_quals"]:
        return o["mp_max"]
    frac = F32(min(max(q, 0), 40)) / F32(40.0)
    return o["mp_min"] + int(frac * F32(o["mp_max"] - o["mp_min"]))


def sc_penalty(o, q):
    """Soft-clip penalty for Phred quality q: MN + (MX - MN) * min(q, 40) / 40, truncated, in float."""
    if q <= 0:
        return o["sp_min"]
    return int((F32(min(q, 40)) / F32(40.0)) * F32(o["sp_max"] - o["sp_min"]) + F32(o["sp_min"]))


def min_score(o, n):
    """--score-min at read length n: SimpleFunc::f in double, truncated, <= 0 end to end.  score_min is None (the default
    L,0,-0.2f) or (type, const, coeff).  Double, not exact rationals: L,-0.6,-0.15 at 36 is -6 exactly but
    -5.999999999999999 in double, and the reference accepts AS -5 there and not -6."""
    return edgereads.minsc((None, 0, 0) if o["score_min"] is None else o["score_min"], n)


def parse_tags(fields):
    return {f[:2]: f[5:] for f in fields[11:]}


def parse_md(md):
    """MD:Z -> list of ('=', n) / ('X', refbase) / ('^', refbases)."""
    out, i = [], 0
    while i < len(md):
        if md[i].isdigit():
            j = i
            while j < len(md) and md[j].isdigit():
                j += 1
            if int(md[i:j]):
                out.append(("=", int(md[i:j])))
            i = j
        elif md[i] == "^":
            j = i + 1
            while j < len(md) and md[j].isalpha():
                j += 1
            out.append(("^", md[i + 1:j]))
            i = j
        else:
            out.append(("X", md[i]))
            i += 1
    return out


def parse_cigar(c):
    out, n = [], ""
    for ch in c:
        if ch.isdigit():
            n += ch
        else:
            out.append((ch, int(n)))
            n = ""
    return out


def known_alt_positions(zs):
    """Zs:Z (graph indexes): read offsets (from the first aligned base; each entry counts from the base after the
    previous SNP) of SNP / indel ALTs the alignment goes through; those edits cost nothing and are not counted in
    XM / XO / XG / NM."""
    pos, at = set(), 0
    for ent in zs.split(","):
        off, typ, _ = ent.split("|")
        at += int(off)
        pos.add((at, typ))
        at += typ == "S"
    return pos


_TINY = []


def tiny_contigs():
    """{name: bases} of tests/golden/tiny.fa, the sequence of both committed indexes (tiny, tiny_snp)."""
    if not _TINY:
        _TINY.append({k: v.decode() for k, v in edgereads.load_contigs(os.path.join(GOLDEN, "tiny.fa")).items()})
    return _TINY[0]


def load_sites(*paths):
    """{(chrom, last exon base, first base after the intron)} of splice-site files (0-based, the files' convention)."""
    out = set()
    for p in paths:
        for l in open(p):
            t = l.split()
            if len(t) >= 3:
                out.add((t[0], int(t[1]), int(t[2])))
    return out


def record_introns(f, o=DEFAULT_SCORING, ref=None, sites=frozenset()):
    """The N operations of a split SAM record as dicts: length, motif class ('can', 'semi' or None), sense ('+', '-' or
    None), whether the site list holds it, and the aligned bases (M) left and right of it in the read."""
    ref = tiny_contigs() if ref is None else ref
    chrom, rp = f[2], int(f[3]) - 1
    cig = parse_cigar(f[5])
    out = []
    for k, (op, n) in enumerate(cig):
        if op == "N":
            motif = (ref[chrom][rp:rp + 2], ref[chrom][rp + n - 2:rp + n])
            cls, sense = o["motifs"].get(motif, (None, None))
            out.append(dict(len=n, cls=cls, sense=sense, known=(chrom, rp - 1, rp + n) in sites,
                            left=sum(m for c, m in cig[:k] if c == "M"), right=sum(m for c, m in cig[k + 1:] if c == "M")))
        if op in "MDN":
            rp += n
    return out


def splice_penalty(introns, o=DEFAULT_SCORING):
    """What the introns of one alignment cost (an intron of the site list costs nothing)."""
    return sum(o["intron_pen"](i["len"]) + (o["can_pen"] if i["cls"] == "can" else o["noncan_pen"])
               for i in introns if not i["known"])


def score_record(line, o=DEFAULT_SCORING, ref=None, sites=frozenset()):
    """Recompute (AS, XM, XO, XG, NM) of an aligned SAM record from CIGAR, MD:Z, SEQ and QUAL, or None if unaligned.
    Phred qualities are SAM's (+33).  AS:i is read from the record only where reference Ns leave a choice: it must then
    be the computed penalty plus 0..(number of reference Ns) N penalties.  A spliced record (N in its CIGAR) is scored
    as the same record without its Ns, minus splice_penalty() of its introns: their motifs come from `ref` (tiny.fa by
    default), and those in `sites` are free, or else all of them are charged."""
    f = line.split("\t")
    if int(f[1]) & 4:
        return None
    tags = parse_tags(f)
    cig = parse_cigar(f[5])
    spl = alt_spl = 0
    if any(op == "N" for op, _ in cig):
        introns = record_introns(f, o, ref, sites)
        spl = splice_penalty(introns, o)
        # a listed intron costs nothing if the search path that found the alignment consulted the site list; the
        # reference charges some listed introns as unlisted ones (secondary alignments, alignments through a graph ALT)
        alt_spl = splice_penalty([dict(i, known=False) for i in introns], o)
    cig = [c for c in cig if c[0] != "N"]
    seq, qual = f[9], [ord(c) - 33 for c in f[10]]
    md = parse_md(tags["MD"])
    alts = known_alt_positions(tags["Zs"]) if "Zs" in tags else set()
    pen = xm = xo = xg = nm = ref_n = 0
    rd = 0           # offset in SEQ
    al = 0           # offset from the first aligned (not soft-clipped) base
    mi = 0           # MD element
    left = 0         # bases left in the current MD match run

    def md_next():
        nonlocal mi, left
        while left == 0:
            kind, v = md[mi]
            mi += 1
            if kind == "=":
                left = v
            else:
                return kind, v
        left -= 1
        return "=", None

    for op, n in cig:
        if op == "S":
            # the reference charges the qualities of the first n bases of QUAL, whichever end is clipped
            # (hi_aligner.h:3872-3878)
            pen += sum(sc_penalty(o, q) for q in qual[:n])
            rd += n
        elif op == "M":
            for _ in range(n):
                kind, refc = md_next()
                if kind == "X" and (al, "S") not in alts:
                    nm += 1
                    xm += 1
                    if seq[rd] == "N":
                        pen += o["np"]
                    elif refc == "N":
                        # a reference N (a base overhanging into a gap or off a sequence end): the reference charges it
                        # the N penalty or nothing, depending on the search path that found the alignment
                        ref_n += 1
                    else:
                        pen += mm_penalty(o, qual[rd])
                rd += 1
                al += 1
        elif op == "I":
            if (al, "I") not in alts:
                pen += o["rdg_const"] + o["rdg_linear"] * n
                xo += 1; xg += n; nm += n
            rd += n
            al += n
        elif op == "D":
            kind, refs = md[mi]
            mi += 1
            assert kind == "^" and len(refs) == n, line
            if (al, "D") not in alts:
                pen += o["rfg_const"] + o["rfg_linear"] * n
                xo += 1; xg += n; nm += n
        else:
            raise AssertionError("CIGAR op %s: %s" % (op, line))
    assert rd == len(seq) and left == 0 and mi == len(md), line
    if alt_spl != spl and int(tags["AS"]) == -(pen + alt_spl):
        spl = alt_spl
    pen += spl
    if ref_n:
        as_ = int(tags["AS"])
        if -pen - ref_n * o["np"] <= as_ <= -pen and (pen + as_) % o["np"] == 0:
            pen = -as_
    return -pen, xm, xo, xg, nm


def max_intron_len(cls, anchor):
    """The longest unknown intron an alignment may have when its shorter anchor is `anchor` bases and it has no other
    edit (MaxIntronLen): 2^clamp(2a - 4, 13, 30) canonical, 2^min(2a - 10, 30) otherwise; 0 below the minimum anchor."""
    if cls == "can":
        return 1 << min(max(2 * anchor - 4, 13), 30) if anchor >= MIN_ANCHOR else 0
    return 1 << min(2 * max(anchor, 5) - 10, 30) if anchor >= MIN_ANCHOR_NONCAN else 0


def check_splices(f, tags, o=DEFAULT_SCORING, ref=None, sites=frozenset()):
    """The splice rules a split record must satisfy beyond its score: every N is an intron of at least --min-intronlen
    bases; XS:A never contradicts the sense of an intron's motif, is absent when two canonical introns' senses
    disagree, and is the sense of the motifs when every intron is canonical and they agree; an unknown intron of a
    record with no other edit respects MaxIntronLen of its shorter anchor.  (XS:A is the direction the aligner recorded
    with the splice, not a function of the final CIGAR: the reference gives some non-canonical introns the sense '-'
    and some semi-canonical introns none, so only canonical introns pin it.)"""
    introns = record_introns(f, o, ref, sites)
    line = "\t".join(f)
    assert all(i["len"] >= MIN_INTRON_LEN for i in introns), line
    senses = set(i["sense"] for i in introns) - {None}
    xs = tags.get("XS")
    if len(set(i["sense"] for i in introns if i["cls"] == "can")) > 1:
        assert xs is None, line
    if senses:
        assert xs in (None,) + tuple(senses), line
        if all(i["cls"] == "can" for i in introns) and len(senses) == 1:
            assert xs == senses.pop(), line
    cig = parse_cigar(f[5])
    if len(introns) == 1 and not introns[0]["known"] and int(tags["NM"]) == 0 and all(op in "MN" for op, _ in cig):
        i = introns[0]
        assert i["len"] <= max_intron_len(i["cls"], min(i["left"], i["right"])), line
    return introns


def check_records(sam, o=DEFAULT_SCORING, ref=None, sites=frozenset(), stats=None):
    """score_record against every aligned record, spliced ones with check_splices as well; YS:i against the mate's AS:i.
    Returns the number of records checked; `stats`, a dict, collects the spliced records checked ('spliced') and the
    lengths of their introns ('intron_lens')."""
    recs = [l for l in (sam.decode() if isinstance(sam, bytes) else sam).splitlines() if l and not l.startswith("@")]
    primary_as = {}
    for l in recs:
        f = l.split("\t")
        if not int(f[1]) & 0x904 and "AS" in parse_tags(f):
            primary_as[(f[0], int(f[1]) & 0xC0)] = int(parse_tags(f)["AS"])
    n = 0
    for l in recs:
        f = l.split("\t")
        flag = int(f[1])
        tags = parse_tags(f)
        if flag & 1 and not flag & 0x108 and "YS" in tags:
            mate = primary_as.get((f[0], (flag & 0xC0) ^ 0xC0))
            assert mate is not None and int(tags["YS"]) == mate, l
        if flag & 4:
            continue
        got = score_record(l, o, ref, sites)
        want = tuple(int(tags[k]) for k in ("AS", "XM", "XO", "XG", "NM"))
        assert got == want, "%s\nrecomputed AS/XM/XO/XG/NM %s" % (l, got)
        assert got[0] >= min_score(o, len(f[9])), l
        if "N" in f[5]:
            introns = check_splices(f, tags, o, ref, sites)
            if stats is not None:
                stats["spliced"] = stats.get("spliced", 0) + 1
                stats.setdefault("intron_lens", set()).update(i["len"] for i in introns)
        n += 1
    return n


def golden_sites(path):
    """The splice-site list a golden SAM was made with (empty for the runs without --known-splicesite-infile)."""
    name = os.path.basename(path)
    if name == "tiny_ss_rna_pe_known_novel.sam":
        return load_sites(os.path.join(GOLDEN, "tiny_ss_known.txt"), os.path.join(GOLDEN, "tiny_ss_novel.txt"))
    if "_ss_rna_" in name:
        return load_sites(os.path.join(GOLDEN, "tiny_ss_rna_ss.txt"))
    return frozenset()


def test_score_restatement_matches_every_golden_sam():
    """Every aligned record of every committed golden SAM of the reference (default scoring; FASTA and FASTQ, SE and PE,
    linear and graph indexes, spliced mode with and without a splice-site list, the edge corpora): AS:i, XM, XO, XG, NM
    and YS:i equal score_record's, AS >= minsc(len), and spliced records keep the splice rules of check_splices.  The
    spliced edge corpus holds introns on both sides of the first two intron-length penalty steps."""
    total, files, stats = 0, 0, {}
    for path in sorted(glob.glob(os.path.join(GOLDEN, "*.sam"))):
        total += check_records(open(path, "rb").read(), sites=golden_sites(path), stats=stats)
        files += 1
    assert files >= 20 and total > 9000 and stats["spliced"] > 1500
    assert {8103, 8104, 22026, 22027} <= stats["intron_lens"]


def test_score_restatement_detects_changed_penalties():
    """The restatement is not vacuous: clamping the quality at 41, rounding the soft-clip penalty, or a one-off
    --score-min each disagree with the reference somewhere in the golden SAMs or at the edge lengths."""
    assert [mm_penalty(dict(DEFAULT_SCORING, mp_max=42, mp_min=2), q) for q in (0, 1, 16, 27, 40, 41, 93)] == [2, 3, 18, 29, 42, 42, 42]
    assert [sc_penalty(DEFAULT_SCORING, q) for q in (0, 1, 19, 20, 39, 40, 41, 93)] == [1, 1, 1, 1, 1, 2, 2, 2]
    assert [min_score(dict(DEFAULT_SCORING, score_min=("L", -0.6, -0.15)), n) for n in (36, 96)] == [-5, -14]
    assert int(np.float32(-0.6 - 0.15 * 36)) == -6          # what a float table would hold
    assert min_score(DEFAULT_SCORING, 100) == -20 and min_score(DEFAULT_SCORING, 101) == -20
    line = open(os.path.join(GOLDEN, "tiny_se_fq.sam")).read().splitlines()
    clipped = [l for l in line if not l.startswith("@") and "S" in l.split("\t")[5] and not int(l.split("\t")[1]) & 4]
    assert clipped
    off = dict(DEFAULT_SCORING, sp_max=3)
    assert any(score_record(l, off) != score_record(l) for l in clipped)
    # the splice terms: the first intron-length step at 8105 instead of 8104, --pen-noncansplice 11, or the two
    # semi-canonical classes' senses swapped each disagree with a golden spliced record
    assert [intron_pen(n) for n in (8103, 8104, 22026, 22027)] == [0, 1, 1, 2]
    swapped = {m: (c, {"+": "-", "-": "+"}[s] if c == "semi" else s) for m, (c, s) in MOTIFS.items()}
    for o in (dict(DEFAULT_SCORING, intron_pen=lambda n: intron_pen(n - 1)), dict(DEFAULT_SCORING, noncan_pen=11),
              dict(DEFAULT_SCORING, motifs=swapped)):
        assert any(golden_disagrees(path, o) for path in sorted(glob.glob(os.path.join(GOLDEN, "*.sam"))))


def golden_disagrees(path, o):
    try:
        check_records(open(path, "rb").read(), o, sites=golden_sites(path))
    except AssertionError:
        return True
    return False


# ---------------------------------------------------------------------------------------------------------------------
# GPU: every case under every geometry
# ---------------------------------------------------------------------------------------------------------------------
# name -> (options, (warps per block, slots per lane, blocks per SM) expected from Index.geometry())
GEOMETRIES = {
    "8x4": (dict(slots_per_lane=4), (8, 4, 1)),
    "8x2": (dict(slots_per_lane=2), (8, 2, 1)),
    "4x8": (dict(threads_per_block=128, slots_per_lane=8), (4, 8, 1)),
    "8x2_bpsm2": (dict(blocks_per_sm=2, slots_per_lane=2), (8, 2, 2)),
}
WORK_BYTES = 368256          # sizeof(Ht2Work): the workspace of one read slot
DP_BYTES = 520632            # sizeof(Ht2SwScratch) + 4 * HT2_SW_POOL_WORDS: --bowtie2-dp scratch of one launched thread
RESERVE = 10 << 30           # HT2_MEM_RESERVE


def pool_bytes(geom, dp, n_sm):
    warps, k, bpsm = geom
    threads = n_sm * bpsm * warps * 32
    return threads * k * WORK_BYTES + (threads * DP_BYTES if dp else 0)


def free_bytes():
    import torch
    return torch.cuda.mem_get_info(0)[0]


def n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def open_geometry(h2, index, gname, **opts):
    """Open `index` with geometry gname, or skip when the device has no room for its workspace (a shared card)."""
    gopts, want = GEOMETRIES[gname]
    need = pool_bytes(want, bool(opts.get("bowtie2_dp")), n_sm()) + RESERVE
    free = free_bytes()
    if need > free:
        pytest.skip("geometry %s needs %.1f GB of device memory, %.1f GB free" % (gname, need / 1e9, free / 1e9))
    idx = h2.Index(os.path.join(GOLDEN, index), **dict(opts, **gopts))
    assert idx.geometry() == want          # graph indexes: always 8 x 4, the only geometry they are run with here
    return idx


@pytest.fixture(scope="module")
def h2(lib):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import hisat2_b200
    return hisat2_b200


@pytest.fixture(scope="session")
def edge_dir(tmp_path_factory):
    return refsets.generate_edge(str(tmp_path_factory.mktemp("edge")))


@pytest.fixture(scope="session")
def sets(tmp_path_factory):
    return refsets.generate(str(tmp_path_factory.mktemp("sets")), ["hard20k", "len150", "alt20k"])


def scoring_of(opts):
    o = dict(DEFAULT_SCORING)
    for k in ("mp_max", "mp_min", "sp_max", "sp_min", "np", "rdg_const", "rdg_linear", "rfg_const", "rfg_linear", "ignore_quals"):
        if k in opts:
            o[k] = opts[k]
    if "score_min_type" in opts:
        o["score_min"] = (chr(opts["score_min_type"]), opts["score_min_const"], opts["score_min_coeff"])
    return o


def run_case(idx, batch, paired, opts, sites=frozenset()):
    """Align; device SAM == host formatter's for every read no capacity flagged; the restatement holds on every record
    (`sites`: the splice sites loaded into the handle).  Returns (header + host SAM, sorted flagged read names)."""
    res = idx.align(batch)
    errs = np.nonzero(res.reads["err"])[0]
    bad = sorted(set(batch.names[int(u) * (2 if paired else 1)].split(b"/")[0].decode() for u in errs))
    host = idx.format_sam(batch, res)
    dev, st = idx.align_sam(batch, with_stats=True)
    assert st["n_err_reads"] == len(errs)
    keep = lambda s: [l for l in s.splitlines() if l.split(b"\t")[0].decode() not in bad]
    assert keep(dev) == keep(host), "device SAM differs from the host formatter's"
    check_records(b"\n".join(keep(host)), scoring_of(opts), sites=sites)
    return idx.sam_header() + host, bad


def edge_batch(h2, d, case):
    _, _, fmt, _, _, front = refsets.EDGE_CASES[case]
    fs = refsets.edge_files(d, case)
    return h2.ReadBatch.parse(path1=fs[0], path2=fs[1] if len(fs) == 2 else None, fastq=fmt == "-q", **front), len(fs) == 2


# Graph-index cases run last (test_graph_index_cases_match_reference), after the linear edge, simulated and spliced
# cases: opening a graph index raises the context's per-thread stack limit for its recursive aligner, which takes
# ~11 GB of device memory for the rest of the process, and the 8 x 4 workspace with its --bowtie2-dp scratch only fits
# an 80 GB card before that.
EDGE_IDS = sorted(c for c in refsets.EDGE_CASES if refsets.EDGE_CASES[c][0] != "tiny_snp")


@pytest.mark.gpu
@pytest.mark.parametrize("case", EDGE_IDS)
@pytest.mark.parametrize("geometry", list(GEOMETRIES))
def test_edge_corpus_matches_reference_under_every_geometry(h2, edge_dir, geometry, case):
    """Sequence ends, the N gap, the chrA|chrB join, the N ceiling, IUPAC input, lengths 1..1024, the whole quality
    range (Phred+33 and +64, -5 / -3 trimming, --mp 42,2) and --score-min boundaries, with and without --bowtie2-dp 2:
    SAM equal to the reference's (md5 without the reads flagged for a device capacity, which are exactly the recorded
    ones) under each kernel geometry."""
    check_edge_case(h2, edge_dir, geometry, case)


def check_edge_case(h2, edge_dir, geometry, case):
    index, _, _, _, opts, _ = refsets.EDGE_CASES[case]
    idx = open_geometry(h2, index, geometry, **opts)
    try:
        batch, paired = edge_batch(h2, edge_dir, case)
        sam, bad = run_case(idx, batch, paired, opts)
    finally:
        idx.close()
    key = "edge/" + case
    assert bad == REF_SETS["flagged"].get(key, [])
    assert refsets.sam_md5(sam, bad) == REF_SETS["md5"][key]
    if case == "se":
        got = [l for l in sam_lines(sam)]
        want = sam_lines(open(os.path.join(GOLDEN, "edge_se.sam"), "rb").read())
        first = next((i for i, (a, b) in enumerate(zip(got, want)) if a != b), None)
        assert first is None and len(got) == len(want), (got[first], want[first]) if first is not None else len(got)


SIM_CASES = [("se/hard20k", "tiny", "hard20k", False, {}), ("paired/hard20k", "tiny", "hard20k", True, {})] + [
    ("dp/%d" % i, c[0], c[1], c[2], c[4]) for i, c in enumerate(refsets.DP_CASES)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c[0] for c in SIM_CASES if c[1] != "tiny_snp"])
@pytest.mark.parametrize("geometry", list(GEOMETRIES))
def test_simulated_sets_match_reference_under_every_geometry(h2, sets, geometry, case):
    """hard20k SE / PE and the --bowtie2-dp / preset cases of tools/refsets.py under each kernel geometry."""
    check_sim_case(h2, sets, geometry, case)


def check_sim_case(h2, sets, geometry, case):
    key, index, name, paired, opts = [c for c in SIM_CASES if c[0] == case][0]
    f1, f2 = os.path.join(sets, name + "_1.fa"), os.path.join(sets, name + "_2.fa")
    idx = open_geometry(h2, index, geometry, **opts)
    try:
        batch = h2.ReadBatch.from_fasta(f1, path2=f2 if paired else None)
        sam, bad = run_case(idx, batch, paired, opts)
    finally:
        idx.close()
    assert bad == REF_SETS["flagged"].get(key, [])
    assert refsets.sam_md5(sam, bad) == REF_SETS["md5"][key]


@pytest.fixture(scope="session")
def spliced_dir(tmp_path_factory):
    return refsets.generate_spliced(str(tmp_path_factory.mktemp("spliced")))


SPLICED_IDS = sorted(c for c in refsets.SPLICED_CASES if refsets.SPLICED_CASES[c][0] != "tiny_snp")


@pytest.mark.gpu
@pytest.mark.parametrize("case", SPLICED_IDS)
@pytest.mark.parametrize("geometry", list(GEOMETRIES))
def test_spliced_corpus_matches_reference_under_every_geometry(h2, spliced_dir, geometry, case):
    """Spliced mode (the reference's --no-temp-splicesite) on the spliced corpus (every motif, anchors of 1-30 bases
    with and without an edit, intron lengths at every rule boundary, 2-4 junctions per read, sequence ends, the N gap,
    pairs across junctions) and its simulated bulk, with and without a splice-site list and with --bowtie2-dp 2:
    SAM equal to the reference's under each kernel geometry, the splice score and rules of check_records on every
    record, and the --novel-splicesite-outfile equal to the reference's."""
    check_spliced_case(h2, spliced_dir, geometry, case)


def check_spliced_case(h2, d, geometry, case):
    index, _, fmt, _, opts, _ = refsets.SPLICED_CASES[case]
    fs, ss = refsets.spliced_files(d, case)
    idx = open_geometry(h2, index, geometry, no_spliced_alignment=0, **opts)
    try:
        sites = frozenset()
        if ss:
            assert idx.load_splicesites(ss) > 200
            sites = load_sites(ss)
        batch = h2.ReadBatch.parse(path1=fs[0], path2=fs[1] if len(fs) == 2 else None, fastq=fmt == "-q")
        sam, bad = run_case(idx, batch, len(fs) == 2, opts, sites)
        novel = None
        if case in refsets.SPLICED_NOVEL:
            # the junctions of the printed alignments, collected by the SAM kernel over several batches
            idx.collect_splicesites(True)
            idx.run_reads(path1=fs[0], path2=fs[1] if len(fs) == 2 else None, fastq=fmt == "-q", batch_reads=4096, collect=False)
            path = os.path.join(d, "novel_%s_%s.txt" % (case, geometry))
            assert idx.write_novel_splicesites(path) > 100
            novel = open(path, "rb").read()
    finally:
        idx.close()
    key = "spliced/" + case
    assert bad == REF_SETS["flagged"].get(key, [])
    assert refsets.sam_md5(sam, bad) == REF_SETS["md5"][key]
    assert sum(1 for l in sam_lines(sam) if not l.startswith(b"@") and b"N" in l.split(b"\t")[5]) > 250
    if novel is not None:
        import hashlib
        assert hashlib.md5(novel).hexdigest() == REF_SETS["md5"]["spliced_novel/" + case]
    if case == "edge_se":
        got = [l.rstrip(b"\n") for l in refsets.spliced_golden_lines(sam)]
        want = sam_lines(open(os.path.join(GOLDEN, "edge_spliced_se.sam"), "rb").read())
        first = next((i for i, (a, b) in enumerate(zip(got, want)) if a != b), None)
        assert first is None and len(got) == len(want), (got[first], want[first]) if first is not None else len(got)


@pytest.mark.gpu
def test_default_handle_follows_free_memory(h2, edge_dir):
    """A default handle runs 8 x 4 where the 4-slot workspace, its DP scratch and the reserve fit in free memory, and the
    DNA-only 8 x 2 kernel where they do not; either way the SAM is the reference's."""
    margin = 1 << 30
    need = pool_bytes((8, 4, 1), False, n_sm()) + RESERVE
    free = free_bytes()
    if abs(free - need) < margin:
        pytest.skip("free device memory (%.1f GB) is within 1 GB of the 4-slot threshold" % (free / 1e9))
    idx = h2.Index(os.path.join(GOLDEN, "tiny"))
    try:
        assert idx.geometry() == ((8, 4, 1) if free > need else (8, 2, 1))
        batch, _ = edge_batch(h2, edge_dir, "se")
        sam, bad = run_case(idx, batch, False, {})
    finally:
        idx.close()
    assert refsets.sam_md5(sam, bad) == REF_SETS["md5"]["edge/se"]


@pytest.mark.gpu
def test_default_handle_joins_an_existing_two_slot_pool(h2, edge_dir):
    """While the process holds the 2-slot workspace, a default handle shares it (8 x 2) instead of allocating the 4-slot
    one, and writes the same SAM."""
    need = pool_bytes((8, 2, 1), False, n_sm()) + RESERVE
    if need > free_bytes():
        pytest.skip("no room for the 2-slot workspace")
    half = h2.Index(os.path.join(GOLDEN, "tiny"), slots_per_lane=2)
    try:
        assert half.geometry() == (8, 2, 1)
        batch, _ = edge_batch(h2, edge_dir, "se")
        a, bad_a = run_case(half, batch, False, {})
        idx = h2.Index(os.path.join(GOLDEN, "tiny"))
        try:
            assert idx.geometry() == (8, 2, 1)
            b, bad_b = run_case(idx, batch, False, {})
        finally:
            idx.close()
    finally:
        half.close()
    assert a == b and bad_a == bad_b
    assert refsets.sam_md5(a, bad_a) == REF_SETS["md5"]["edge/se"]


@pytest.mark.gpu
@pytest.mark.parametrize("first,second", [("4x8", "8x4"), ("8x4", "8x2_bpsm2")])
def test_dp_scratch_covers_every_grid_sharing_a_pool(h2, edge_dir, first, second):
    """4 x 8 and 8 x 4 (and 8 x 4 and 8 x 2 with two blocks per SM) have the same number of read slots, so their handles
    share one workspace pool, but the second launches twice the threads of the first.  The --bowtie2-dp scratch is per
    launched thread: it must grow for the second handle, and both handles must then write the reference's SAM, in
    either order of use."""
    g1, g2 = GEOMETRIES[first][1], GEOMETRIES[second][1]
    assert g1[0] * g1[1] * g1[2] == g2[0] * g2[1] * g2[2]
    threads = max(g1[0] * g1[2], g2[0] * g2[2]) * 32 * n_sm()
    need = pool_bytes(g1, False, n_sm()) + threads * DP_BYTES + RESERVE
    free = free_bytes()
    if need > free:
        pytest.skip("the shared pool with the larger DP scratch needs %.1f GB, %.1f GB free" % (need / 1e9, free / 1e9))
    opts = dict(bowtie2_dp=2)
    batch, _ = edge_batch(h2, edge_dir, "se_dp")
    a = open_geometry(h2, "tiny", first, **opts)
    try:
        sa, bad_a = run_case(a, batch, False, opts)
        b = h2.Index(os.path.join(GOLDEN, "tiny"), **dict(opts, **GEOMETRIES[second][0]))
        try:
            assert b.geometry() == g2
            sb, bad_b = run_case(b, batch, False, opts)
            sa2, _ = run_case(a, batch, False, opts)
        finally:
            b.close()
    finally:
        a.close()
    want = REF_SETS["md5"]["edge/se_dp"]
    assert sa == sb == sa2 and bad_a == bad_b == REF_SETS["flagged"].get("edge/se_dp", [])
    assert refsets.sam_md5(sb, bad_b) == want


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["edge/" + c for c in sorted(refsets.EDGE_CASES) if refsets.EDGE_CASES[c][0] == "tiny_snp"] +
                         [c[0] for c in SIM_CASES if c[1] == "tiny_snp"] +
                         ["spliced/" + c for c in sorted(refsets.SPLICED_CASES) if refsets.SPLICED_CASES[c][0] == "tiny_snp"])
def test_graph_index_cases_match_reference(h2, edge_dir, sets, spliced_dir, case):
    """The graph-index (tiny_snp) cases, spliced ones included: graph indexes have one geometry, 8 x 4 (asserted by
    open_geometry)."""
    if case.startswith("edge/"):
        check_edge_case(h2, edge_dir, "8x4", case[5:])
    elif case.startswith("spliced/"):
        check_spliced_case(h2, spliced_dir, "8x4", case[8:])
    else:
        check_sim_case(h2, sets, "8x4", case)
