"""The SAM counting pass stores each unit's records as a plan and the writing pass prints one record per thread; a batch
whose plan does not fit the overflow arena is printed one unit per thread instead (HT2GPU_SAM_PLAN_ARENA sets the
arena's capacity, -1 disables the plan).  Both writing passes must give the same SAM bytes, alignment summary and
per-unit outcome bytes.  (The host formatter, which prints each planned record as it is planned, is checked against
the golden SAMs by test_cpu.py.)"""
import os
import sys

import pytest

from conftest import GOLDEN, ROOT, sam_lines

sys.path.insert(0, os.path.join(ROOT, "tools"))
import refsets  # noqa: E402

pytestmark = pytest.mark.gpu

g = lambda n: os.path.join(GOLDEN, n)


@pytest.fixture(scope="module")
def h2(lib):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import hisat2_b200
    return hisat2_b200


@pytest.fixture(scope="module")
def sets(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("plan_sets"))
    refsets.generate(d, ["len500"])
    refsets.generate_repeats(d)
    return d


def run(h2, arena, batch, opts, out=None):
    """SAM text, stats, summary and outcome bytes of one align_sam on a fresh handle with the given arena capacity."""
    old = os.environ.get("HT2GPU_SAM_PLAN_ARENA")
    if arena is None:
        os.environ.pop("HT2GPU_SAM_PLAN_ARENA", None)
    else:
        os.environ["HT2GPU_SAM_PLAN_ARENA"] = str(arena)
    try:
        idx = h2.Index(g("tiny"), **opts.get("index", {}))
        try:
            if opts.get("sam_output"):
                idx.set_sam_output(**opts["sam_output"])
            if out:
                idx.collect_splicesites(True)
            idx.record_outcomes(True)
            sam, st = idx.align_sam(batch, with_stats=True)
            n_sites = idx.write_novel_splicesites(out) if out else None
            return sam, st, idx.align_counts(), idx.unit_outcomes().tobytes(), n_sites
        finally:
            idx.close()
    finally:
        if old is None:
            os.environ.pop("HT2GPU_SAM_PLAN_ARENA", None)
        else:
            os.environ["HT2GPU_SAM_PLAN_ARENA"] = old


def planned_equals_fallback(h2, batch, opts, tmp_path=None):
    a_out = str(tmp_path / "planned.txt") if tmp_path is not None else None
    b_out = str(tmp_path / "fallback.txt") if tmp_path is not None else None
    sam_a, st_a, cnt_a, oc_a, ns_a = run(h2, None, batch, opts, a_out)
    sam_b, st_b, cnt_b, oc_b, ns_b = run(h2, -1, batch, opts, b_out)
    assert st_a["sam_unplanned"] == 0 and st_b["sam_unplanned"] == 1
    assert st_a["n_err_reads"] == st_b["n_err_reads"] == 0
    assert sam_a == sam_b
    assert cnt_a == cnt_b
    assert oc_a == oc_b and len(oc_a) == st_a["n_units"]
    if a_out:
        assert ns_a == ns_b
        assert open(a_out).read() == open(b_out).read()
    return sam_a, st_a, a_out


def test_golden_pairs(h2):
    batch = h2.ReadBatch.from_fasta(g("tiny_pe_1.fa"), path2=g("tiny_pe_2.fa"))
    sam, _, _ = planned_equals_fallback(h2, batch, {})
    assert sam_lines(sam) == [l for l in sam_lines(open(g("tiny_pe.sam"), "rb").read()) if not l.startswith(b"@")]


def test_unstaged_blocks_2x500(h2, sets):
    batch = h2.ReadBatch.from_fasta(os.path.join(sets, "len500_1.fa"), path2=os.path.join(sets, "len500_2.fa"))
    planned_equals_fallback(h2, batch, {})


def test_k30_secondary_text_rerun(h2, sets):
    """-k 30 --secondary on reads of segments tiny.fa holds twice: more text than the first estimate, so the writing pass
    runs again after the buffer grows (from the kept plan)."""
    batch = h2.ReadBatch.from_fasta(os.path.join(sets, "rep_1.fa"))
    sam, st, _ = planned_equals_fallback(h2, batch, {"index": {"khits": 30, "secondary": 1}})
    assert st["n_launches"] > 5
    assert len(sam.splitlines()) == 2 * batch.n


@pytest.mark.parametrize("sam_output", [{"no_unal": True}, {"omit_sec_seq": True}, {"rna_strandness": "RF"}])
def test_sam_output_options(h2, sam_output):
    batch = h2.ReadBatch.from_fasta(g("tiny_pe_1.fa"), path2=g("tiny_pe_2.fa"))
    planned_equals_fallback(h2, batch, {"sam_output": sam_output, "index": {"khits": 10, "secondary": 1}})


def test_spliced_novel_splicesite_outfile(h2, tmp_path):
    batch = h2.ReadBatch.from_fasta(g("tiny_ss_rna_1.fa"), path2=g("tiny_ss_rna_2.fa"))
    _, _, out = planned_equals_fallback(h2, batch, {"index": {"no_spliced_alignment": 0}}, tmp_path=tmp_path)
    assert open(out).read() == open(g("tiny_ss_rna_pe_novel_out.txt")).read()
