"""The SAM writing pass stages a block's text in shared memory and copies it out with 16-byte stores; a block whose
text does not fit the staging buffer formats straight into global memory.  Both paths, and batches whose unit count
is not a multiple of the SAM kernels' block size (128 units), must give the host formatter's bytes and the
reference's SAM."""
import os
import sys

import pytest

from conftest import GOLDEN, ROOT

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(ROOT, "tools"))
import refsets  # noqa: E402

REF_SETS = refsets.load_expected()
SAM_TPB = 128                  # units per block of the SAM kernels (ht2_gpu.cu, HT2_SAM_TPB)
MAX_STAGE = 227 * 1024         # the most dynamic shared memory one block can have on sm_90: a block with more text never stages


@pytest.fixture(scope="module")
def h2(lib):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import hisat2_b200
    return hisat2_b200


@pytest.fixture(scope="module")
def sets(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("staging_sets"))
    refsets.generate(d, ["sim10k", "len150", "len500"])
    refsets.generate_repeats(d)
    return d


@pytest.fixture
def tiny(h2):
    idx = h2.Index(os.path.join(GOLDEN, "tiny"))
    yield idx
    idx.close()


def block_bytes(sam):
    """Bytes of SAM text per 128-unit block: a unit's records are consecutive and share the read (pair) name."""
    units, last = [], None
    for rec in sam.splitlines(True):
        name = rec.split(b"\t", 1)[0]
        if name != last:
            units.append(0)
            last = name
        units[-1] += len(rec)
    return [sum(units[i:i + SAM_TPB]) for i in range(0, len(units), SAM_TPB)], len(units)


def device_equals_host(idx, batch):
    host = idx.format_sam(batch, idx.align(batch))
    dev, st = idx.align_sam(batch, with_stats=True)
    assert st["n_err_reads"] == 0
    assert dev == host, "device SAM differs from the host formatter's"
    return dev


def first_records(src, dst, n):
    """The first n FASTA records of src (name line + sequence lines) into dst."""
    out, k = [], 0
    for line in open(src):
        if line.startswith(">"):
            k += 1
            if k > n:
                break
        out.append(line)
    with open(dst, "w") as f:
        f.writelines(out)
    return dst


@pytest.mark.parametrize("name", ["len500", "len150", "sim10k"])
def test_staged_and_direct_blocks_match_reference(h2, tiny, sets, name):
    """2x500-base pairs: every block's text is larger than any staging buffer (all blocks write straight to global
    memory).  2x150: blocks near the staging size (some staged, some not).  2x101: every block staged.  The sets hold
    3000, 20000 and 10000 pairs: the last block is partly empty."""
    f1, f2 = os.path.join(sets, name + "_1.fa"), os.path.join(sets, name + "_2.fa")
    batch = h2.ReadBatch.from_fasta(f1, path2=f2)
    assert batch.n // 2 % SAM_TPB != 0
    dev = device_equals_host(tiny, batch)
    assert refsets.sam_md5(tiny.sam_header() + dev) == REF_SETS["md5"]["paired/" + name]
    blocks, units = block_bytes(dev)
    assert units == batch.n // 2
    if name == "len500":
        assert min(blocks[:-1]) > MAX_STAGE


@pytest.mark.parametrize("n", [1, 127, 129, 1000])
def test_batch_sizes_off_the_block_size(h2, tiny, sets, tmp_path, n):
    """Batches of 1, 127, 129 and 1000 pairs of 2x101 (staged) and of 2x500 (direct): the same bytes as the host."""
    for name in ("sim10k", "len500"):
        f1 = first_records(os.path.join(sets, name + "_1.fa"), str(tmp_path / (name + "_1.fa")), n)
        f2 = first_records(os.path.join(sets, name + "_2.fa"), str(tmp_path / (name + "_2.fa")), n)
        batch = h2.ReadBatch.from_fasta(f1, path2=f2)
        assert batch.n == 2 * n
        dev = device_equals_host(tiny, batch)
        assert block_bytes(dev)[1] == n


def test_multimapping_records_k30_secondary(h2, sets):
    """Reads of the segments tiny.fa holds twice under -k 30 --secondary: two records per read, more text than the first
    estimate of the output buffer, so the SAM kernels run again after it grows; device text == host text."""
    idx = h2.Index(os.path.join(GOLDEN, "tiny"), khits=30, secondary=1)
    try:
        batch = h2.ReadBatch.from_fasta(os.path.join(sets, "rep_1.fa"))
        dev, st = idx.align_sam(batch, with_stats=True)
        assert st["n_launches"] > 4 and st["n_err_reads"] == 0
        assert dev == idx.format_sam(batch, idx.align(batch)), "device SAM differs from the host formatter's"
        assert len(dev.splitlines()) == 2 * batch.n
    finally:
        idx.close()
