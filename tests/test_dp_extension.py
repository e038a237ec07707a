"""The --bowtie2-dp seed extension (csrc/ht2_sw.h) job by job.

tools/swjobs.py generates DP extension jobs on the tiny index at the shapes and edges where the kernel could go
wrong (read lengths around the warp fill's 32-row blocks and the 256-row maximum, rectangles trimmed at contig
ends or crossing the N gap, indels next to the gap barrier, repeats that make cells tie, N counts at nceil, minsc
at the u8 / i16 switch and the -15000 refusal, anchors off the read's diagonal, edit lists over capacity).
tests/golden/sw_extend_ref.txt holds the reference's answer for every job (oracle/ref_sw: SwAligner on the
unmodified reference): found, offset, score, best cell, the edit list the reference chose among equal-scoring
ones, and the next draw of its RandomSource.

Checked against it: a plain int64 restatement of the extension written from the reference's recurrences (CPU),
the host build of the shared code (tests/hostsim --sw-extend, CPU) and the device, with the warp fill of the pool
kernel's DP round and with the lane fill (GPU)."""
import collections
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, REFDIR, ROOT

sys.path.insert(0, os.path.join(ROOT, "tools"))
import swjobs  # noqa: E402

GOLDEN_FILE = os.path.join(GOLDEN, "sw_extend_ref.txt")
REF_SW = os.path.join(REFDIR, "ref_sw")
ERR_EDITS, ERR_SW = 1, 4096
MAX_EDITS, SW_MAX_EDITS, SW_MAX_ROWS = 128, 160, 256
INT64_MIN = -(1 << 63)
FIELDS = ("id", "found", "offset", "score", "best", "rnd", "edits")
NEG = -(1 << 40)


# ------------------------------------------------------------------------------------------------------------------
# the corpus and the reference's answers
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def jobs():
    return swjobs.generate()


def parse_result(line):
    f = line.split(" ")
    assert len(f) == 7, line
    edits = [] if f[6] == "-" else [tuple(e.split(":")) for e in f[6].split(",")]
    return {"line": f, "found": f[1] == "1", "offset": None if f[2] == "-" else int(f[2]),
            "score": None if f[3] == "-" else int(f[3]), "best": None if f[4] == "-" else int(f[4]),
            "rnd": int(f[5]), "edits": [(int(p), int(t), c, q) for p, t, c, q in edits]}


@pytest.fixture(scope="module")
def golden():
    lines = open(GOLDEN_FILE).read().splitlines()
    return lines[0].split(), [parse_result(l) for l in lines[1:]]


def runs_dp(job):
    return job["len"] < len(job["read"])


def expected_err(job, g):
    """The error bit the device must set: reads longer than its 256-row planes and minsc below -15000 are refused
    (HT2_ERR_SW); an alignment of more than HT2_MAX_EDITS edits does not fit a hit (HT2_ERR_EDITS)."""
    if not runs_dp(job):
        return 0
    if len(job["read"]) > SW_MAX_ROWS or job["minsc"] < -15000:
        return ERR_SW
    if g["found"] and len(g["edits"]) > MAX_EDITS:
        return ERR_EDITS
    return 0


def overran_ok(job, g, err):
    """A candidate that is rejected after its backtrace ran past the HT2_SW_MAX_EDITS edits the backtrace holds is
    flagged too: allowed only where the reference reports nothing."""
    return err == ERR_EDITS and expected_err(job, g) == 0 and not g["found"]


def expected_fields(job, g):
    """The golden line as the device reports it: the reference's best is its best last-row score even below minsc;
    the device keeps only a best that reaches minsc."""
    f = list(g["line"])
    if g["best"] is not None and g["best"] < job["minsc"]:
        f[4] = "-"
    return f


# ------------------------------------------------------------------------------------------------------------------
# the restatement: plain int64, from the reference's recurrences (dp_framer.cpp frameSeedExtensionRect,
# aligner_swsse_ee_*.cpp end-to-end fill, Scoring penalties), no saturation and no floor
# ------------------------------------------------------------------------------------------------------------------
CONTIGS = [s for _, s in swjobs.load_fasta()]
CODE = {"A": 0, "C": 1, "G": 2, "T": 3}


def frame(job):
    """frameSeedExtensionRect(refoff, rdlen, reflen, 10, 10, 0, 10) with trimToRef = false -> (refl, refr, triml)."""
    rdlen, reflen = len(job["read"]), len(CONTIGS[job["tidx"]])
    off = job["toff"] - job["rdoff"] if job["toff"] > job["rdoff"] else 0
    maxgap = 10
    refl, refr = off - 2 * maxgap, off + rdlen - 1 + 2 * maxgap
    maxns = 0
    trimr = refr - (reflen + maxns - 1) if refr >= reflen + maxns else 0
    triml = -refl - maxns if refl < -maxns else 0
    return refl + triml, refr - trimr, triml


def window(job, refl, refr):
    s = CONTIGS[job["tidx"]]
    return "".join(s[p] if 0 <= p < len(s) else "N" for p in range(refl, refr + 1))


def aligned(job):
    """The read as it is aligned (reverse complement on the reverse strand) and its qualities in that order."""
    q = [ord(c) - 33 for c in job["qual"]]
    return (job["read"], q) if job["fw"] else (swjobs.revcomp(job["read"]), q[::-1])


def restate_best(job):
    """Best last-row score of the end-to-end Gotoh fill, int64, gap moves in the barrier rows = -inf."""
    sc = swjobs.scoring(job["opt"])
    refl, refr, _ = frame(job)
    rf = window(job, refl, refr)
    rd, q = aligned(job)
    n, m = len(rd), len(rf)
    rdo, rde = sc["rdg_const"] + sc["rdg_linear"], sc["rdg_linear"]
    rfo, rfe = sc["rfg_const"] + sc["rfg_linear"], sc["rfg_linear"]
    gb = sc["gbar"]
    rfc = np.array([CODE.get(c, 4) for c in rf], dtype=np.int64)
    k = np.arange(m, dtype=np.int64)
    Hp = np.full(m, NEG, dtype=np.int64)
    Fp = np.full(m, NEG, dtype=np.int64)
    for i in range(n):
        c = CODE.get(rd[i], 4)
        pen = np.where((rfc > 3) | (c > 3), sc["np"], np.where(rfc == c, 0, swjobs.mmpen(sc, q[i]))).astype(np.int64)
        if i == 0:
            D = -pen                                           # row 0: any column may start the alignment
        else:
            D = np.concatenate(([NEG], Hp[:-1])) - pen         # column 0 has no diagonal
        barrier = i < gb or n - 1 - i < gb
        if barrier or i == 0:
            F = np.full(m, NEG, dtype=np.int64)
        else:
            F = np.maximum(Fp - rfe, Hp - rfo)
        G = np.maximum(np.maximum(D, F), NEG)
        if barrier:
            E = np.full(m, NEG, dtype=np.int64)
        else:
            # E[j] = max over k < j of G[k] - rdo - (j - k - 1) * rde (opening from an E cell never beats extending it)
            acc = np.maximum.accumulate(G + k * rde)
            E = np.concatenate(([NEG], acc[:-1] - rdo - (k[1:] - 1) * rde))
        H = np.maximum(np.maximum(G, E), NEG)
        Hp, Fp = H, np.maximum(F, NEG)
    return int(Hp.max())


def edit_score(job, g):
    """The score of the golden edit list recomputed against the window, checking every base it claims."""
    sc = swjobs.scoring(job["opt"])
    rdo, rde = sc["rdg_const"] + sc["rdg_linear"], sc["rdg_linear"]
    rfo, rfe = sc["rfg_const"] + sc["rfg_linear"], sc["rfg_linear"]
    rd, q = aligned(job)
    s = CONTIGS[job["tidx"]]
    ref = lambda p: s[p] if 0 <= p < len(s) else "N"  # noqa: E731
    eds = g["edits"]
    rp, k, score, prev = g["offset"], 0, 0, None
    for i in range(len(rd)):
        while k < len(eds) and eds[k][1] == 1 and eds[k][0] == i:          # reference bases skipped before row i
            assert eds[k][2] == ref(rp) and eds[k][3] == "-", (eds[k], ref(rp))
            score -= rde if prev == ("rdgap", i) else rdo
            prev = ("rdgap", i); rp += 1; k += 1
        if k < len(eds) and eds[k][1] == 2 and eds[k][0] == i:             # read base i against no reference base
            assert eds[k][2] == "-" and eds[k][3] == rd[i], eds[k]
            score -= rfe if prev == ("rfgap", i - 1) else rfo
            prev = ("rfgap", i); k += 1
            continue
        if k < len(eds) and eds[k][1] == 3 and eds[k][0] == i:
            assert eds[k][2] == ref(rp) and eds[k][3] == rd[i] and (rd[i] != ref(rp) or rd[i] == "N"), (eds[k], ref(rp), rd[i])
            score -= sc["np"] if "N" in (rd[i], ref(rp)) else swjobs.mmpen(sc, q[i])
            k += 1
        else:
            assert rd[i] == ref(rp) and rd[i] != "N", (i, rd[i], ref(rp))
        prev = None
        rp += 1
    assert k == len(eds)
    return score


@pytest.fixture(scope="module")
def restated(jobs):
    return [restate_best(j) if runs_dp(j) else None for j in jobs]


def derived_classes(jobs, golden_rows, restated):
    """Classes that follow from the answers: minsc at the optimum and one above it, a first candidate that failed
    while a later one was reported, edit lists over the two capacities."""
    c = collections.Counter()
    for j, g, b in zip(jobs, golden_rows, restated):
        if b is None:
            continue
        if j["minsc"] == b:
            c["minsc_eq_best"] += 1
        if j["minsc"] == b + 1:
            c["minsc_best_plus_1"] += 1
        if b >= j["minsc"] and (not g["found"] or g["score"] < b):
            c["first_candidate_failed"] += 1
            if g["found"]:
                c["later_candidate_reported"] += 1
        if g["found"] and len(g["edits"]) > MAX_EDITS:
            c["edits_over_128"] += 1
        if g["found"] and len(g["edits"]) > SW_MAX_EDITS:
            c["edits_over_160"] += 1
        if g["found"] and j["fw"] == 0 and g["edits"]:
            c["reverse_strand_edits"] += 1
    return c


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------
def test_job_generator_reproduces_the_golden_job_stream(jobs, golden):
    header, rows = golden
    assert header[0] == "sha1" and header[1] == swjobs.stream_sha1(jobs), "tools/swjobs.py no longer generates the jobs of the golden file"
    assert int(header[3]) == len(jobs) == len(rows)
    assert [int(r["line"][0]) for r in rows] == [j["id"] for j in jobs]
    assert len({j["opt"] for j in jobs}) == len(swjobs.OPTION_SETS)


def test_job_classes_are_all_present(jobs, golden, restated, capsys):
    tags = collections.Counter(t for j in jobs for t in j["tags"])
    derived = derived_classes(jobs, golden[1], restated)
    lengths = collections.Counter(len(j["read"]) for j in jobs)
    quals = {ord(c) - 33 for j in jobs for c in j["qual"]}
    with capsys.disabled():
        print("\n%d DP extension jobs; classes: %s" % (len(jobs), " ".join("%s=%d" % kv for kv in sorted(tags.items()))))
        print("derived classes: %s" % " ".join("%s=%d" % kv for kv in sorted(derived.items())))
    for t, n in swjobs.CLASS_MIN.items():
        assert tags[t] >= n, (t, tags[t], n)
    for L in swjobs.LENGTHS + swjobs.TOO_LONG:
        assert lengths[L] >= 2, L
    assert quals == set(range(94))
    assert derived["minsc_eq_best"] >= 15 and derived["minsc_best_plus_1"] >= 15
    assert derived["later_candidate_reported"] >= 20 and derived["first_candidate_failed"] >= 40
    assert derived["edits_over_128"] >= 15 and derived["edits_over_160"] >= 8
    assert derived["reverse_strand_edits"] >= 200
    per_set = collections.Counter(j["opt"] for j in jobs)
    assert min(per_set.values()) >= 120


def test_restatement_agrees_with_the_reference_on_every_job(jobs, golden, restated):
    """best: the reference's best cell equals the int64 restatement's wherever it reaches minsc (below minsc the
    reference's 8-bit fill may saturate); the reported edit list scores what the reference says it scores, against
    the window, and that score lies between minsc and best."""
    bad = []
    for j, g, b in zip(jobs, golden[1], restated):
        if b is None:
            assert g["found"] and g["offset"] is None, j["id"]
            continue
        try:
            if b >= j["minsc"]:
                assert g["best"] == b, ("best", g["best"], b)
            else:
                assert g["best"] is None or g["best"] < j["minsc"], ("best below minsc", g["best"], b)
                assert not g["found"]
            if g["found"]:
                s = edit_score(j, g)
                assert s == g["score"], ("edit list score", s, g["score"])
                assert j["minsc"] <= g["score"] <= b, ("score range", j["minsc"], g["score"], b)
        except AssertionError as e:
            bad.append("job %d %s: %s" % (j["id"], ",".join(j["tags"]), e))
    assert not bad, "\n".join(bad[:20])


def test_host_build_matches_the_reference_on_every_job(hostsim_bin, jobs, tmp_path):
    """tests/hostsim --sw-extend: swExtendAnchor (swPrepare + swFill + swFinish, the shared HT2_HD code) on the CPU."""
    p = str(tmp_path / "jobs.txt")
    swjobs.write_jobs(jobs, p)
    r = subprocess.run([hostsim_bin, "--sw-extend", os.path.join(GOLDEN, "tiny"), p, GOLDEN_FILE], stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE)
    err = r.stderr.decode()
    assert r.returncode == 0, err[-4000:]
    assert "%d jobs" % len(jobs) in err and " 0 mismatches" in err, err[-2000:]
    out = r.stdout.decode().splitlines()
    assert len(out) == len(jobs)
    flagged = collections.Counter(int(l.rsplit(" ", 1)[1]) for l in out)
    assert flagged[ERR_SW] >= 20 and flagged[ERR_EDITS] >= 15, flagged


@pytest.mark.skipif(not os.path.exists(REF_SW), reason="oracle/_ref/ref_sw is built only where the reference sources are")
def test_reference_driver_reproduces_the_golden_file(jobs, golden):
    assert swjobs.run_reference(jobs, REF_SW) == [" ".join(g["line"]) for g in golden[1]]


# ------------------------------------------------------------------------------------------------------------------
# GPU: ht2gpu_sw_extend, warp fill (the pool kernel's DP round) and lane fill
# ------------------------------------------------------------------------------------------------------------------
def device_fields(j, r, edits):
    dp = runs_dp(j)
    f = [str(j["id"]), "1" if r["found"] else "0"]
    f += [str(int(r["toff"])), str(int(r["score"]))] if r["found"] and dp else ["-", "-"]
    f.append(str(int(r["best"])) if dp and int(r["best"]) != INT64_MIN else "-")
    f.append(str(int(r["rnd_next"])))
    if r["found"] and dp and len(edits):
        f.append(",".join("%d:%d:%s:%s" % (e["pos"], e["type"], chr(e["chr"]), chr(e["qchr"])) for e in edits))
    else:
        f.append("-")
    return f


def _mixed_order(js):
    """A fixed permutation, so that warps hold jobs that fill next to ones that return early or are refused."""
    return sorted(js, key=lambda j: (j["id"] * 2654435761) & 0xffffffff)


@pytest.fixture(scope="module")
def h2(lib):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import hisat2_b200
    return hisat2_b200


@pytest.mark.gpu
@pytest.mark.parametrize("fill", ["warp", "lane"])
@pytest.mark.parametrize("opt", range(len(swjobs.OPTION_SETS)), ids=[n for n, _ in swjobs.OPTION_SETS])
def test_device_extension_matches_the_reference_job_by_job(h2, jobs, golden, restated, opt, fill):
    import torch
    sel = _mixed_order([j for j in jobs if j["opt"] == opt])
    from hisat2_b200 import api
    need = len(sel) * (1 << 20) + (1 << 30)              # Ht2Work + DP scratch + planes per job, with room to spare
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip("the harness needs %.1f GB of device memory, %.1f GB free" % (need / 1e9, free / 1e9))
    idx = h2.Index(os.path.join(GOLDEN, "tiny"), **swjobs.OPTION_SETS[opt][1])
    try:
        res, edits = idx.sw_extend(sel, warp_fill=(fill == "warp"))
    finally:
        idx.close()
    rows = golden[1]
    bad, flagged, overran = [], collections.Counter(), 0
    for k, j in enumerate(sel):
        g, r, b = rows[j["id"]], res[k], restated[j["id"]]
        err = int(r["err"])
        want = expected_err(j, g)
        where = "job %d (%s, %s strand, %d bases)" % (j["id"], ",".join(j["tags"]), "fw" if j["fw"] else "rc", len(j["read"]))
        if err != want:
            if overran_ok(j, g, err):
                overran += 1
                continue
            bad.append("%s: error bits %d, expected %d" % (where, err, want))
            continue
        if err:
            flagged[err] += 1
            continue
        mine, exp = device_fields(j, r, edits[k]), expected_fields(j, g)
        if mine != exp:
            i = next(i for i in range(len(FIELDS)) if mine[i] != exp[i])
            bad.append("%s: %s differs: device %s, reference %s" % (where, FIELDS[i], mine[i][:120], exp[i][:120]))
            continue
        # the best last-row cell against the restatement: the best where it reaches minsc, "none" otherwise
        if runs_dp(j):
            want_best = b if b >= j["minsc"] else INT64_MIN
            if int(r["best"]) != want_best:
                bad.append("%s: best %d, restatement %d (minsc %d)" % (where, int(r["best"]), b, j["minsc"]))
    assert not bad, "%d of %d jobs differ:\n%s" % (len(bad), len(sel), "\n".join(bad[:25]))
    assert overran <= len(sel) // 20
