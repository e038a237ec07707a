"""The handle's slot runtime through the C ABI: calls that change what a batch in flight reads are refused until the
batch is waited for, and a submit that fails leaves its slot free for the next batch."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import GOLDEN, sam_lines

ERR_ARG, ERR_CUDA = -1, -3
SITES = os.path.join(GOLDEN, "tiny_ss_rna_ss.txt")


@pytest.fixture(scope="module")
def h2(lib):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import hisat2_b200
    return hisat2_b200


def submit(lib, idx, slot, batch):
    """ht2gpu_submit_sam of batch on slot; returns (rc, what must stay alive until the wait)."""
    cb = batch.c_struct()
    blob, offs = batch.names_offsets()
    return lib.ht2gpu_submit_sam(idx._h, slot, C.byref(cb), blob, offs.ctypes.data, len(blob)), (cb, blob, offs)


def wait(h2, lib, idx, slot):
    r = h2.api.CSamResult()
    rc = lib.ht2gpu_wait_sam(idx._h, slot, C.byref(r))
    assert rc == 0, lib.ht2gpu_last_error(idx._h)
    return C.string_at(r.sam, r.sam_len) if r.sam_len else b""


def golden():
    return sam_lines(open(os.path.join(GOLDEN, "tiny_se.sam"), "rb").read())


@pytest.mark.gpu
def test_slot_calls_refused_while_a_batch_is_in_flight(h2):
    lib = h2.api.load_library()
    idx = h2.Index(os.path.join(GOLDEN, "tiny"), device=0)
    batch = h2.ReadBatch.from_fasta(os.path.join(GOLDEN, "tiny_se.fa"))
    rc, keep = submit(lib, idx, 1, batch)
    assert rc == 0, lib.ht2gpu_last_error(idx._h)
    cfg = h2.api.CSamOutput()
    cfg.no_unal = 1
    cfg.rg_id = b"g1"
    n = C.c_uint32(7)
    assert lib.ht2gpu_set_sam_output(idx._h, C.byref(cfg)) == ERR_ARG
    assert lib.ht2gpu_record_outcomes(idx._h, 1) == ERR_ARG
    assert lib.ht2gpu_load_splicesites(idx._h, SITES.encode(), None, C.byref(n)) == ERR_ARG
    assert b"in flight" in lib.ht2gpu_last_error(idx._h) and n.value == 7
    # nothing changed: the batch (and the header) print as without the calls, and no outcomes were recorded
    assert sam_lines(idx.sam_header() + wait(h2, lib, idx, 1)) == golden()
    p, nu = C.c_void_p(), C.c_uint32()
    assert lib.ht2gpu_unit_outcomes(idx._h, 1, C.byref(p), C.byref(nu)) == ERR_ARG
    del keep
    assert lib.ht2gpu_set_sam_output(idx._h, C.byref(cfg)) == 0
    assert lib.ht2gpu_record_outcomes(idx._h, 1) == 0
    assert lib.ht2gpu_load_splicesites(idx._h, SITES.encode(), None, C.byref(n)) == 0 and n.value > 0
    idx.close()


@pytest.mark.gpu
def test_failed_submit_frees_its_slot(h2):
    """Two reads whose offsets claim 2^40 bases: the upload's allocation fails (an ordinary out-of-memory error, before
    any copy).  The slot takes the next batch."""
    lib = h2.api.load_library()
    idx = h2.Index(os.path.join(GOLDEN, "tiny"), device=0)
    bad = h2.ReadBatch(np.zeros(8, np.uint8), np.array([0, 4, 1 << 40], np.uint64), np.zeros(2, np.uint32), [b"r1", b"r2"])
    rc, _ = submit(lib, idx, 1, bad)
    assert rc == ERR_CUDA and b"out of memory" in lib.ht2gpu_last_error(idx._h)
    batch = h2.ReadBatch.from_fasta(os.path.join(GOLDEN, "tiny_se.fa"))
    rc, keep = submit(lib, idx, 1, batch)
    assert rc == 0, lib.ht2gpu_last_error(idx._h)
    assert sam_lines(idx.sam_header() + wait(h2, lib, idx, 1)) == golden()
    assert lib.ht2gpu_record_outcomes(idx._h, 1) == 0
    del keep
    idx.close()
