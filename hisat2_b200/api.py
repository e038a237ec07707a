"""ctypes bindings for include/ht2gpu.h plus small batching helpers.

This is the reference-side binding a maintainer would add (INTEGRATION.md):
plain pointers and sizes cross the boundary, no torch types.  The product path
is the CUDA library; if it is missing or no CUDA device is usable the calls
raise -- there is no CPU fallback.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIBPATH = os.path.join(_HERE, "libht2gpu.so")
_lib = None


class Ht2GpuError(RuntimeError):
    pass


class Options(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "device", "no_spliced_alignment", "khits", "max_seeds", "secondary", "mp_max", "mp_min",
        "sp_max", "sp_min", "np", "rdg_const", "rdg_linear", "rfg_const", "rfg_linear",
        "ignore_quals", "nofw", "norc", "min_frag", "max_frag", "no_mixed", "no_discordant")] + [
        ("seed", C.c_uint32), ("threads_per_block", C.c_int32), ("blocks_per_sm", C.c_int32), ("slots_per_lane", C.c_int32), ("warp_per_read", C.c_int32),
        ("bowtie2_dp", C.c_int32), ("gbar", C.c_int32), ("score_min_type", C.c_int32),
        ("score_min_const", C.c_double), ("score_min_coeff", C.c_double)]


class CReadBatch(C.Structure):
    _fields_ = [("n_reads", C.c_uint32), ("paired", C.c_int32), ("seq", C.c_void_p), ("qual", C.c_void_p),
                ("offs", C.c_void_p), ("seeds", C.c_void_p)]


EDIT_DTYPE = np.dtype([("pos", "<u4"), ("chr", "u1"), ("qchr", "u1"), ("type", "u1"), ("pad", "u1"), ("snp_id", "<u4")])
SW_MAX_EDITS = 128   # HT2GPU_SW_MAX_EDITS
SW_JOB_DTYPE = np.dtype([("fw", "<u4"), ("tidx", "<u4"), ("toff", "<u4"), ("rdoff", "<u4"), ("len", "<u4"), ("seed", "<u4"),
                         ("minsc", "<i8"), ("read_off", "<u8"), ("read_len", "<u4"), ("pad", "<u4")])
SW_RESULT_DTYPE = np.dtype([("found", "<u4"), ("err", "<u4"), ("toff", "<u4"), ("n_edits", "<u4"), ("score", "<i8"),
                            ("best", "<i8"), ("rnd_next", "<u4"), ("pad", "<u4")])
ALN_DTYPE = np.dtype([("tidx", "<u4"), ("toff", "<u4"), ("score", "<i4"), ("fw", "u1"), ("mate", "u1"),
                      ("n_edits", "<u2"), ("trim5", "<u2"), ("trim3", "<u2"), ("ref_extent", "<u4"), ("edit_off", "<u4")])
READ_DTYPE = np.dtype([("aln_off", "<u4"), ("n_aln", "<u2", (2,)), ("pair_off", "<u4"), ("n_pairs", "<u4"),
                       ("rng_state", "<u4"), ("err", "<u4"), ("n_lf", "<u4"), ("alg_bytes", "<u4"), ("filt", "<u4")])


class CResultBatch(C.Structure):
    _fields_ = [("n_reads", C.c_uint32), ("reads", C.c_void_p), ("n_alns", C.c_uint32), ("alns", C.c_void_p),
                ("n_edits", C.c_uint32), ("edits", C.c_void_p), ("n_pairs", C.c_uint32), ("pairs", C.c_void_p),
                ("ms_h2d", C.c_float), ("ms_kernel", C.c_float), ("ms_d2h", C.c_float),
                ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64), ("n_launches", C.c_uint32), ("n_err_reads", C.c_uint32),
                ("priv", C.c_void_p)]


class CSamResult(C.Structure):
    _fields_ = [("sam", C.c_void_p), ("sam_len", C.c_size_t), ("n_units", C.c_uint32), ("n_alns", C.c_uint32),
                ("n_err_reads", C.c_uint32), ("n_launches", C.c_uint32),
                ("ms_h2d", C.c_float), ("ms_align", C.c_float), ("ms_sam", C.c_float), ("ms_d2h", C.c_float),
                ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64)]


class CReadsInput(C.Structure):
    _fields_ = [("path1", C.c_char_p), ("path2", C.c_char_p), ("data1", C.c_void_p), ("len1", C.c_size_t),
                ("data2", C.c_void_p), ("len2", C.c_size_t), ("format", C.c_int32), ("trim5", C.c_int32), ("trim3", C.c_int32),
                ("phred64", C.c_int32), ("seed", C.c_uint32), ("skip", C.c_uint64), ("upto", C.c_uint64),
                ("batch_reads", C.c_uint32), ("threads", C.c_int32)]


class CRunStats(C.Structure):
    _fields_ = [("n_reads", C.c_uint64), ("n_units", C.c_uint64), ("sam_bytes", C.c_uint64), ("n_err_reads", C.c_uint64),
                ("n_batches", C.c_uint64), ("s_index", C.c_double), ("s_parse", C.c_double), ("s_total", C.c_double),
                ("s_submit", C.c_double), ("s_wait", C.c_double), ("s_sink", C.c_double),
                ("ms_h2d", C.c_float), ("ms_align", C.c_float), ("ms_sam", C.c_float), ("ms_d2h", C.c_float),
                ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64), ("n_launches", C.c_uint32), ("pad", C.c_uint32)]


class CParsedReads(C.Structure):
    _fields_ = [("batch", CReadBatch), ("names", C.c_void_p), ("name_offs", C.c_void_p), ("names_bytes", C.c_size_t), ("priv", C.c_void_p)]


SINK_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t)

# The read files of --un, --al, --un-conc, --al-conc and --al-conc-disc, in the order of HT2GPU_READS_* (ht2gpu.h)
READ_FILES = ("un", "al", "un_conc", "al_conc", "al_conc_disc")
READS_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t)


class CReadRoutes(C.Structure):
    _fields_ = [("mask", C.c_uint32), ("write", READS_FN), ("ctx", C.c_void_p), ("n_spans", C.c_uint64), ("bytes", C.c_uint64),
                ("s_route", C.c_double)]


def _read_routes(read_files):
    """(CReadRoutes, {(output, mate): [chunks]}) collecting the spans of the outputs in read_files.  mate is 0 for
    un / al and 1 / 2 for the -conc outputs."""
    unknown = set(read_files) - set(READ_FILES)
    if unknown:
        raise ValueError("unknown read files %s (choose from %s)" % (sorted(unknown), READ_FILES))
    chunks = {}
    for w in read_files:
        for m in ((0,) if READ_FILES.index(w) < 2 else (1, 2)):
            chunks[(w, m)] = []

    def _write(ctx, which, mate, ptr, n):
        chunks[(READ_FILES[which], mate)].append(C.string_at(ptr, n))
        return 0
    rt = CReadRoutes()
    rt.mask = sum(1 << READ_FILES.index(w) for w in read_files)
    rt.write = READS_FN(_write)
    return rt, chunks


def _reads_input(path1=None, path2=None, data1=None, data2=None, fastq=False, **kw):
    """(CReadsInput, buffers to keep alive) for FASTA / FASTQ files or bytes in host memory."""
    ri = CReadsInput()
    keep = []
    if path1 is not None:
        ri.path1 = os.fsencode(path1)
    if path2 is not None:
        ri.path2 = os.fsencode(path2)
    for name, d in (("1", data1), ("2", data2)):
        if d is not None:
            buf = np.frombuffer(d, dtype=np.uint8)
            keep.append(buf)
            setattr(ri, "data" + name, buf.ctypes.data)
            setattr(ri, "len" + name, buf.nbytes)
    ri.format = 1 if fastq else 0
    for k, v in kw.items():
        setattr(ri, k, v)
    return ri, keep


def route_reads(outcomes, path1=None, path2=None, data1=None, data2=None, fastq=False, read_files=READ_FILES, **kw):
    """ht2gpu_route_reads, host only: the records of an input (after skip / upto) written to the read files by their
    units' outcome bytes (HT2GPU_OUTCOME_*, e.g. Index.unit_outcomes).  Returns {(output, mate): bytes}."""
    lib = load_library()
    ri, keep = _reads_input(path1, path2, data1, data2, fastq, **kw)
    out = np.ascontiguousarray(outcomes, dtype=np.uint8)
    rt, chunks = _read_routes(read_files)
    err = C.create_string_buffer(512)
    rc = lib.ht2gpu_route_reads(C.byref(ri), out.ctypes.data, len(out), C.byref(rt), err, 512)
    if rc != 0:
        raise Ht2GpuError("ht2gpu_route_reads rc=%d: %s" % (rc, err.value.decode()))
    return {k: b"".join(v) for k, v in chunks.items()}


class CSamOutput(C.Structure):
    _fields_ = [("no_unal", C.c_int32), ("omit_sec_seq", C.c_int32), ("no_sq", C.c_int32), ("rg_id", C.c_char_p),
                ("rg", C.POINTER(C.c_char_p)), ("n_rg", C.c_int32)]


# ReportingMetrics of ht2gpu_align_counts_t, in its field order
ALIGN_COUNTS = ("nread", "npaired", "nunpaired", "nconcord_0", "nconcord_uni1", "nconcord_uni2", "ndiscord",
                "nunp_0_0", "nunp_0_uni1", "nunp_0_uni2", "nunp_0", "nunp_uni1", "nunp_uni2")


class CAlignCounts(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ALIGN_COUNTS]


EXPORTS = [
    "ht2gpu_default_options", "ht2gpu_open", "ht2gpu_open_image", "ht2gpu_open_device_image", "ht2gpu_build_image",
    "ht2gpu_free_image", "ht2gpu_image_data", "ht2gpu_image_bytes", "ht2gpu_device_image", "ht2gpu_align_batch",
    "ht2gpu_align_resident", "ht2gpu_free_results", "ht2gpu_format_sam", "ht2gpu_sam_header", "ht2gpu_free_text",
    "ht2gpu_num_refs", "ht2gpu_ref_name", "ht2gpu_ref_len", "ht2gpu_read_seed", "ht2gpu_last_error", "ht2gpu_close",
    "ht2gpu_seed_search", "ht2gpu_free_seed_results", "ht2gpu_index_is_graph",
    "ht2gpu_sam_slots", "ht2gpu_submit_sam", "ht2gpu_wait_sam", "ht2gpu_align_sam", "ht2gpu_run_reads",
    "ht2gpu_host_alloc", "ht2gpu_host_free", "ht2gpu_set_error", "ht2gpu_parse_reads", "ht2gpu_free_parsed",
    "ht2gpu_ctx_get", "ht2gpu_ctx_set", "ht2gpu_run_reads_multi", "ht2gpu_open_peer", "ht2gpu_sw_selftest", "ht2gpu_load_splicesites", "ht2gpu_collect_splicesites",
    "ht2gpu_write_novel_splicesites", "ht2gpu_launch_geometry", "ht2gpu_set_sam_output", "ht2gpu_align_counts",
    "ht2gpu_format_align_summary", "ht2gpu_sw_extend", "ht2gpu_record_outcomes", "ht2gpu_unit_outcomes",
    "ht2gpu_run_reads_routed", "ht2gpu_route_reads",
]


class CSeedResult(C.Structure):
    _fields_ = [("n_reads", C.c_uint32), ("first_hit", C.c_void_p), ("n_hits", C.c_uint32), ("hits", C.c_void_p),
                ("n_iedges", C.c_uint32), ("iedges", C.c_void_p), ("n_coords", C.c_uint32), ("coords", C.c_void_p),
                ("n_lf", C.c_uint64), ("alg_bytes", C.c_uint64), ("ms_kernel", C.c_float), ("err", C.c_uint32),
                ("priv", C.c_void_p)]


SEED_HIT_DTYPE = np.dtype([("read", "<u4"), ("fw", "u1"), ("hit_type", "u1"), ("pseudogene_stop", "u1"), ("anchor_stop", "u1"),
                           ("bwoff", "<u4"), ("len", "<u4"), ("top", "<u4"), ("bot", "<u4"), ("node_top", "<u4"),
                           ("node_bot", "<u4"), ("n_iedges", "<u4"), ("iedge_off", "<u4"), ("n_coords", "<u4"),
                           ("coord_off", "<u4")])
SEED_COORD_DTYPE = np.dtype([("row", "<u4"), ("joined_off", "<u4"), ("tidx", "<u4"), ("toff", "<u4")])


def load_library(path=None):
    """dlopen the CUDA library; raises if it has not been built."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or os.environ.get("HT2GPU_LIB") or _LIBPATH
    if not os.path.exists(p):
        raise Ht2GpuError("%s not found: run `python -m hisat2_b200.build` (no CPU fallback exists)" % p)
    lib = C.CDLL(p)
    lib.ht2gpu_default_options.argtypes = [C.POINTER(Options)]
    lib.ht2gpu_open.argtypes = [C.c_char_p, C.POINTER(Options), C.POINTER(C.c_void_p)]
    lib.ht2gpu_open_image.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(Options), C.POINTER(C.c_void_p)]
    lib.ht2gpu_open_device_image.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(Options), C.POINTER(C.c_void_p)]
    lib.ht2gpu_build_image.argtypes = [C.c_char_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_char_p, C.c_size_t]
    lib.ht2gpu_free_image.argtypes = [C.c_void_p]
    lib.ht2gpu_image_data.argtypes = [C.c_void_p]; lib.ht2gpu_image_data.restype = C.c_void_p
    lib.ht2gpu_image_bytes.argtypes = [C.c_void_p]; lib.ht2gpu_image_bytes.restype = C.c_size_t
    lib.ht2gpu_device_image.argtypes = [C.c_void_p]; lib.ht2gpu_device_image.restype = C.c_void_p
    lib.ht2gpu_align_batch.argtypes = [C.c_void_p, C.POINTER(CReadBatch), C.POINTER(CResultBatch)]
    lib.ht2gpu_align_resident.argtypes = [C.c_void_p, C.POINTER(CReadBatch), C.c_int, C.POINTER(CResultBatch)]
    lib.ht2gpu_free_results.argtypes = [C.POINTER(CResultBatch)]
    lib.ht2gpu_format_sam.argtypes = [C.c_void_p, C.POINTER(CReadBatch), C.c_char_p, C.POINTER(CResultBatch),
                                      C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
    lib.ht2gpu_sam_header.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
    lib.ht2gpu_free_text.argtypes = [C.c_void_p]
    lib.ht2gpu_num_refs.argtypes = [C.c_void_p]; lib.ht2gpu_num_refs.restype = C.c_uint32
    lib.ht2gpu_ref_name.argtypes = [C.c_void_p, C.c_uint32]; lib.ht2gpu_ref_name.restype = C.c_char_p
    lib.ht2gpu_ref_len.argtypes = [C.c_void_p, C.c_uint32]; lib.ht2gpu_ref_len.restype = C.c_uint32
    lib.ht2gpu_read_seed.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_char_p, C.c_uint32]
    lib.ht2gpu_read_seed.restype = C.c_uint32
    lib.ht2gpu_last_error.argtypes = [C.c_void_p]; lib.ht2gpu_last_error.restype = C.c_char_p
    lib.ht2gpu_close.argtypes = [C.c_void_p]
    lib.ht2gpu_seed_search.argtypes = [C.c_void_p, C.POINTER(CReadBatch), C.c_uint32, C.POINTER(CSeedResult)]
    lib.ht2gpu_free_seed_results.argtypes = [C.POINTER(CSeedResult)]
    lib.ht2gpu_index_is_graph.argtypes = [C.c_void_p]
    lib.ht2gpu_sam_slots.argtypes = [C.c_void_p]
    lib.ht2gpu_submit_sam.argtypes = [C.c_void_p, C.c_int, C.POINTER(CReadBatch), C.c_void_p, C.c_void_p, C.c_size_t]
    lib.ht2gpu_wait_sam.argtypes = [C.c_void_p, C.c_int, C.POINTER(CSamResult)]
    lib.ht2gpu_align_sam.argtypes = [C.c_void_p, C.POINTER(CReadBatch), C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(CSamResult)]
    lib.ht2gpu_run_reads.argtypes = [C.c_void_p, C.POINTER(CReadsInput), SINK_FN, C.c_void_p, C.POINTER(CRunStats)]
    lib.ht2gpu_run_reads_multi.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.POINTER(CReadsInput), SINK_FN, C.c_void_p, C.POINTER(CRunStats)]
    lib.ht2gpu_run_reads_routed.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.POINTER(CReadsInput), SINK_FN, C.c_void_p,
                                            C.POINTER(CReadRoutes), C.POINTER(CRunStats)]
    lib.ht2gpu_route_reads.argtypes = [C.POINTER(CReadsInput), C.c_void_p, C.c_uint64, C.POINTER(CReadRoutes), C.c_char_p, C.c_size_t]
    lib.ht2gpu_record_outcomes.argtypes = [C.c_void_p, C.c_int]
    lib.ht2gpu_unit_outcomes.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_uint32)]
    lib.ht2gpu_open_peer.argtypes = [C.c_void_p, C.POINTER(Options), C.POINTER(C.c_void_p)]
    lib.ht2gpu_host_alloc.argtypes = [C.c_size_t]; lib.ht2gpu_host_alloc.restype = C.c_void_p
    lib.ht2gpu_host_free.argtypes = [C.c_void_p]
    lib.ht2gpu_set_error.argtypes = [C.c_void_p, C.c_char_p]
    lib.ht2gpu_parse_reads.argtypes = [C.POINTER(CReadsInput), C.POINTER(CParsedReads), C.c_char_p, C.c_size_t]
    lib.ht2gpu_free_parsed.argtypes = [C.POINTER(CParsedReads)]
    lib.ht2gpu_sw_selftest.argtypes = [C.c_int, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint64)]
    lib.ht2gpu_sw_extend.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    lib.ht2gpu_load_splicesites.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.POINTER(C.c_uint32)]
    lib.ht2gpu_collect_splicesites.argtypes = [C.c_void_p, C.c_int]
    lib.ht2gpu_write_novel_splicesites.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_char_p, C.POINTER(C.c_uint64)]
    lib.ht2gpu_launch_geometry.argtypes = [C.c_void_p, C.POINTER(C.c_int32)]
    lib.ht2gpu_set_sam_output.argtypes = [C.c_void_p, C.POINTER(CSamOutput)]
    lib.ht2gpu_align_counts.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.POINTER(CAlignCounts)]
    lib.ht2gpu_format_align_summary.argtypes = [C.POINTER(CAlignCounts), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p),
                                                C.POINTER(C.c_size_t)]
    if path is None:
        _lib = lib
    return lib


def sw_selftest(n=2000, seed=1, device=0):
    """ht2gpu_sw_selftest: warp-wide DP fill vs lane fill on n random problems -> dict(mismatches, problems, cells, valid)."""
    out = (C.c_uint64 * 4)()
    rc = load_library().ht2gpu_sw_selftest(device, n, seed, out)
    if rc != 0:
        raise Ht2GpuError("ht2gpu_sw_selftest failed (%d)" % rc)
    return {"mismatches": int(out[0]), "problems": int(out[1]), "cells": int(out[2]), "valid": int(out[3])}


def format_align_summary(counts, new_style=False, discordant=True, mixed=True):
    """ht2gpu_format_align_summary: the alignment summary hisat2 prints at the end of a run (AlnSink::printAlSumm),
    from a dict of ALIGN_COUNTS (Index.align_counts).  discordant / mixed = False under --no-discordant / --no-mixed.
    Host only."""
    lib = load_library()
    c = CAlignCounts(*[int(counts.get(k, 0)) for k in ALIGN_COUNTS])
    p, n = C.c_void_p(), C.c_size_t()
    rc = lib.ht2gpu_format_align_summary(C.byref(c), int(bool(new_style)), int(bool(discordant)), int(bool(mixed)), C.byref(p), C.byref(n))
    if rc != 0:
        raise Ht2GpuError("ht2gpu_format_align_summary rc=%d" % rc)
    s = C.string_at(p.value, n.value).decode()
    lib.ht2gpu_free_text(p)
    return s


_ASC2DNA = np.zeros(256, dtype=np.uint8)
_DNACAT = np.zeros(256, dtype=np.uint8)
for _ch in b"ACGTacgt":
    _DNACAT[_ch] = 1
for _ch in b"BDHKMNRSVWXYbdhkmnrsvwxy":
    _DNACAT[_ch] = 2
_DNACAT[ord("-")] = 3
for _ch, _v in ((b"Cc", 1), (b"Gg", 2), (b"Tt", 3), (b"Nn", 4)):
    for _c in _ch:
        _ASC2DNA[_c] = _v


class ReadBatch(object):
    """Structure-of-arrays read batch in host memory (see ht2gpu_read_batch_t).

    seq: uint8 codes 0..4 concatenated; offs: uint64 (n+1); seeds: uint32 (n);
    qual: uint8 ASCII or None (FASTA: all 'I'); names: list of bytes.
    """

    def __init__(self, seq, offs, seeds, names, qual=None, paired=False):
        self.seq = np.ascontiguousarray(seq, dtype=np.uint8)
        self.offs = np.ascontiguousarray(offs, dtype=np.uint64)
        self.seeds = np.ascontiguousarray(seeds, dtype=np.uint32)
        self.qual = None if qual is None else np.ascontiguousarray(qual, dtype=np.uint8)
        self.names = names
        self.paired = bool(paired)
        self.n = len(self.offs) - 1

    def c_struct(self):
        b = CReadBatch()
        b.n_reads = self.n
        b.paired = 1 if self.paired else 0
        b.seq = self.seq.ctypes.data
        b.qual = None if self.qual is None else self.qual.ctypes.data
        b.offs = self.offs.ctypes.data
        b.seeds = self.seeds.ctypes.data
        return b

    def names_blob(self):
        return b"\0".join(self.names) + b"\0"

    def names_offsets(self):
        """(blob, uint32 offsets[n+1]) in the layout ht2gpu_submit_sam takes."""
        lens = np.fromiter((len(x) + 1 for x in self.names), dtype=np.int64, count=len(self.names))
        offs = np.zeros(len(self.names) + 1, dtype=np.uint32)
        np.cumsum(lens, out=offs[1:])
        return self.names_blob(), offs

    @staticmethod
    def parse(path1=None, path2=None, data1=None, data2=None, fastq=False, lib=None, **kw):
        """The library's own multi-threaded front end (ht2gpu_parse_reads, csrc/ht2_reads.cpp): the whole input
        as one batch.  Host only."""
        lib = lib or load_library()
        ri = CReadsInput()
        keep = []
        if path1 is not None:
            ri.path1 = os.fsencode(path1)
        if path2 is not None:
            ri.path2 = os.fsencode(path2)
        for name, d in (("1", data1), ("2", data2)):
            if d is not None:
                buf = np.frombuffer(d, dtype=np.uint8)
                keep.append(buf)
                setattr(ri, "data" + name, buf.ctypes.data)
                setattr(ri, "len" + name, buf.nbytes)
        ri.format = 1 if fastq else 0
        for k, v in kw.items():
            setattr(ri, k, v)
        pr = CParsedReads()
        err = C.create_string_buffer(512)
        rc = lib.ht2gpu_parse_reads(C.byref(ri), C.byref(pr), err, 512)
        if rc != 0:
            raise Ht2GpuError("ht2gpu_parse_reads rc=%d: %s" % (rc, err.value.decode()))
        n = pr.batch.n_reads
        v = AlignResult._view
        offs = v(pr.batch.offs, n + 1, np.dtype("<u8")).copy()
        nb = int(offs[n]) if n else 0
        seq = v(pr.batch.seq, nb, np.dtype("u1")).copy()
        qual = v(pr.batch.qual, nb, np.dtype("u1")).copy() if pr.batch.qual else None
        seeds = v(pr.batch.seeds, n, np.dtype("<u4")).copy()
        blob = C.string_at(pr.names, pr.names_bytes) if pr.names_bytes else b""
        names = blob.split(b"\0")[:-1] if blob else []
        paired = bool(pr.batch.paired)
        lib.ht2gpu_free_parsed(C.byref(pr))
        return ReadBatch(seq, offs, seeds, names, qual, paired=paired)

    @staticmethod
    def from_fastq(path, lib=None, global_seed=0, path2=None):
        """Parse 4-line Phred+33 FASTQ like FastqPatternSource::parse (pat.cpp:1030-1290)."""
        lib = lib or load_library()

        def parse(p):
            names, seqs, quals = [], [], []
            with open(p, "rb") as f:
                lines = [l.rstrip(b"\r\n") for l in f]
            lines = [l for l in lines if l != b""]
            if len(lines) % 4:
                raise Ht2GpuError("%s: not a 4-line FASTQ file" % p)
            for i in range(0, len(lines), 4):
                if not lines[i].startswith(b"@") or not lines[i + 2].startswith(b"+"):
                    raise Ht2GpuError("%s: malformed FASTQ record %d" % (p, i // 4))
                sq = lines[i + 1].replace(b".", b"N")
                if len(lines[i + 3]) != len(sq):
                    raise Ht2GpuError("%s: quality / base count mismatch in record %d" % (p, i // 4))
                names.append(lines[i][1:] or str(i // 4).encode()); seqs.append(sq); quals.append(lines[i + 3])
            return names, seqs, quals

        names, seqs, quals = parse(path)
        if path2 is not None:
            n2, s2, q2 = parse(path2)
            if len(n2) != len(names):
                raise Ht2GpuError("mate files differ in read count")
            inames, iseqs, iquals = [], [], []
            for a, b, q, c, d, e in zip(names, seqs, quals, n2, s2, q2):
                inames += [a if a.endswith(b"/1") else a + b"/1", c if c.endswith(b"/2") else c + b"/2"]
                iseqs += [b, d]; iquals += [q, e]
            names, seqs, quals = inames, iseqs, iquals
        codes, offs = [], [0]
        for s in seqs:
            codes.append(_ASC2DNA[np.frombuffer(s, dtype=np.uint8)])
            offs.append(offs[-1] + len(s))
        seq = np.concatenate(codes) if codes else np.zeros(0, np.uint8)
        qual = np.frombuffer(b"".join(quals), dtype=np.uint8).copy() if quals else np.zeros(0, np.uint8)
        seeds = np.zeros(len(names), dtype=np.uint32)
        for i, nm in enumerate(names):
            c = np.ascontiguousarray(codes[i])
            q = np.ascontiguousarray(qual[offs[i]:offs[i + 1]])
            seeds[i] = lib.ht2gpu_read_seed(c.ctypes.data, q.ctypes.data, len(c), nm, global_seed)
        return ReadBatch(seq, offs, seeds, names, qual, paired=path2 is not None)

    @staticmethod
    def from_fasta(path, lib=None, global_seed=0, path2=None):
        """Parse FASTA like FastaPatternSource::read (pat.cpp:725-849)."""
        lib = lib or load_library()

        def parse(p):
            names, seqs = [], []
            name, chunks, cnt = None, [], 0
            with open(p, "rb") as f:
                for line in f:
                    if line.startswith(b">"):
                        if name is not None:
                            seqs.append(b"".join(chunks)); names.append(name)
                        name = line[1:].rstrip(b"\r\n") or str(cnt).encode()
                        cnt += 1
                        chunks = []
                    elif line[:1] in (b"#", b";"):
                        continue
                    else:
                        chunks.append(line.rstrip(b"\r\n"))
                if name is not None:
                    seqs.append(b"".join(chunks)); names.append(name)
            return names, seqs      # empty records stay: the reference reports them unaligned with YF:Z:LN

        names, seqs = parse(path)
        if path2 is not None:
            n2, s2 = parse(path2)
            if len(n2) != len(names):
                raise Ht2GpuError("mate files differ in read count")
            # the reference appends /1 and /2 to mate names (pat.cpp fixName)
            inames, iseqs = [], []
            for a, b, c, d in zip(names, seqs, n2, s2):
                inames += [a if a.endswith(b"/1") else a + b"/1", c if c.endswith(b"/2") else c + b"/2"]
                iseqs += [b, d]
            names, seqs = inames, iseqs
        codes, offs = [], [0]
        for s in seqs:
            a = np.frombuffer(s, dtype=np.uint8)
            a = a[_DNACAT[a] > 0]
            codes.append(_ASC2DNA[a])
            offs.append(offs[-1] + len(a))
        seq = np.concatenate(codes) if codes else np.zeros(0, np.uint8)
        seeds = np.zeros(len(names), dtype=np.uint32)
        for i, nm in enumerate(names):
            c = np.ascontiguousarray(codes[i])
            seeds[i] = lib.ht2gpu_read_seed(c.ctypes.data, None, len(c), nm, global_seed)
        return ReadBatch(seq, offs, seeds, names, None, paired=path2 is not None)


class AlignResult(object):
    """Owns one ht2gpu_result_batch_t; exposes zero-copy numpy views."""

    def __init__(self, lib, cres):
        self._lib = lib
        self._c = cres
        self.reads = self._view(cres.reads, cres.n_reads, READ_DTYPE)
        self.alns = self._view(cres.alns, cres.n_alns, ALN_DTYPE)
        self.edits = self._view(cres.edits, cres.n_edits, EDIT_DTYPE)
        self.pairs = self._view(cres.pairs, cres.n_pairs * 2, np.dtype("<u2")).reshape(-1, 2)
        self.ms_h2d, self.ms_kernel, self.ms_d2h = cres.ms_h2d, cres.ms_kernel, cres.ms_d2h
        self.h2d_bytes, self.d2h_bytes, self.n_launches = cres.h2d_bytes, cres.d2h_bytes, cres.n_launches
        self.n_err_reads = cres.n_err_reads

    @staticmethod
    def _view(ptr, n, dt):
        if not ptr or n == 0:
            return np.zeros(0, dtype=dt)
        buf = (C.c_uint8 * (n * dt.itemsize)).from_address(ptr)
        return np.frombuffer(buf, dtype=dt, count=n)

    def close(self):
        if self._c is not None:
            self._lib.ht2gpu_free_results(C.byref(self._c))
            self._c = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class SeedResult(object):
    """Owns one ht2gpu_seed_result_t (seed search on its own; linear and graph indexes)."""

    def __init__(self, lib, c):
        self._lib = lib
        self._c = c
        v = AlignResult._view
        self.first_hit = v(c.first_hit, c.n_reads + 1, np.dtype("<u4"))
        self.hits = v(c.hits, c.n_hits, SEED_HIT_DTYPE)
        self.iedges = v(c.iedges, c.n_iedges * 2, np.dtype("<u2")).reshape(-1, 2)
        self.coords = v(c.coords, c.n_coords, SEED_COORD_DTYPE)
        self.n_lf, self.alg_bytes, self.ms_kernel, self.err = c.n_lf, c.alg_bytes, c.ms_kernel, c.err

    def dump_lines(self, graph):
        """The record format of oracle/ref_dump.cpp (H / G / C lines), for parity tests."""
        out = []
        hits, co, ie = self.hits, self.coords, self.iedges
        order = np.zeros(len(hits), dtype=np.int64)
        for r in range(len(self.first_hit) - 1):
            lo, hi = int(self.first_hit[r]), int(self.first_hit[r + 1])
            k = {1: 0, 0: 0}
            for i in range(lo, hi):
                f = int(hits["fw"][i]); order[i] = k[f]; k[f] += 1
        for i in range(len(hits)):
            h = hits[i]
            out.append("H %d %d %d %d %d %d %d %d %d\n" % (h["read"], h["fw"], h["bwoff"], h["len"], h["top"], h["bot"], h["hit_type"],
                                                           h["pseudogene_stop"], h["anchor_stop"]))
            blank = int(h["top"]) == 0xffffffff
            if graph and not blank:
                e = ie[int(h["iedge_off"]):int(h["iedge_off"]) + int(h["n_iedges"])]
                out.append("G %d %d %d %d %d %d%s\n" % (h["read"], h["fw"], order[i], h["node_top"], h["node_bot"], h["n_iedges"],
                                                         "".join(" %d:%d" % (a, b) for a, b in e)))
            for c in co[int(h["coord_off"]):int(h["coord_off"]) + int(h["n_coords"])]:
                out.append("C %d %d %d %d %d %d %d\n" % (h["read"], h["fw"], order[i], c["row"], c["joined_off"], c["tidx"], c["toff"]))
        return out

    def close(self):
        if self._c is not None:
            self._lib.ht2gpu_free_seed_results(C.byref(self._c))
            self._c = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Index(object):
    """Device-resident HISAT2 index + alignment entry points."""

    def __init__(self, base=None, image=None, device_image=None, device=0, **opts):
        self._lib = load_library()
        self._opts = dict(opts)
        o = Options()
        self._lib.ht2gpu_default_options(C.byref(o))
        o.device = device
        for k, v in opts.items():
            setattr(o, k, v)
        self._h = C.c_void_p()
        if base is not None:
            rc = self._lib.ht2gpu_open(os.fsencode(base), C.byref(o), C.byref(self._h))
        elif image is not None:
            img = np.ascontiguousarray(image, dtype=np.uint8)
            rc = self._lib.ht2gpu_open_image(img.ctypes.data, img.nbytes, C.byref(o), C.byref(self._h))
        else:
            ptr, nbytes, prefix = device_image
            prefix = np.ascontiguousarray(prefix, dtype=np.uint8)
            self._keep = prefix
            rc = self._lib.ht2gpu_open_device_image(ptr, nbytes, prefix.ctypes.data, prefix.nbytes, C.byref(o), C.byref(self._h))
        if rc != 0:
            msg = self._lib.ht2gpu_last_error(self._h).decode() if self._h else "open failed"
            self.close()
            raise Ht2GpuError("ht2gpu_open rc=%d: %s" % (rc, msg))

    @staticmethod
    def build_image(base):
        """Parse the .ht2 files into the packed image (host only; no GPU needed)."""
        lib = load_library()
        p, n = C.c_void_p(), C.c_size_t()
        err = C.create_string_buffer(512)
        rc = lib.ht2gpu_build_image(os.fsencode(base), C.byref(p), C.byref(n), err, 512)
        if rc != 0:
            raise Ht2GpuError("ht2gpu_build_image rc=%d: %s" % (rc, err.value.decode()))
        arr = np.frombuffer((C.c_uint8 * n.value).from_address(p.value), dtype=np.uint8).copy()
        lib.ht2gpu_free_image(p)
        return arr

    def image(self):
        n = self._lib.ht2gpu_image_bytes(self._h)
        p = self._lib.ht2gpu_image_data(self._h)
        return np.frombuffer((C.c_uint8 * n).from_address(p), dtype=np.uint8)

    def _check(self, rc, what, allow_capacity=False):
        if rc != 0 and not (allow_capacity and rc == -4):
            raise Ht2GpuError("%s rc=%d: %s" % (what, rc, self._lib.ht2gpu_last_error(self._h).decode()))

    def align(self, batch, resident_iters=0, allow_capacity=False):
        cb = batch.c_struct()
        cr = CResultBatch()
        if resident_iters > 0:
            rc = self._lib.ht2gpu_align_resident(self._h, C.byref(cb), resident_iters, C.byref(cr))
        else:
            rc = self._lib.ht2gpu_align_batch(self._h, C.byref(cb), C.byref(cr))
        res = AlignResult(self._lib, cr)
        self._check(rc, "ht2gpu_align", allow_capacity)
        return res

    def align_sam(self, batch, with_stats=False):
        """ht2gpu_align_sam: align + SAM records formatted ON THE DEVICE for one batch (no header)."""
        cb = batch.c_struct()
        blob, offs = batch.names_offsets()
        cr = CSamResult()
        self._check(self._lib.ht2gpu_align_sam(self._h, C.byref(cb), blob, offs.ctypes.data, len(blob), C.byref(cr)), "ht2gpu_align_sam")
        s = C.string_at(cr.sam, cr.sam_len) if cr.sam_len else b""
        if with_stats:
            return s, {k: getattr(cr, k) for k, _ in CSamResult._fields_ if k != "sam"}
        return s

    def record_outcomes(self, enable=True):
        """ht2gpu_record_outcomes: the SAM counting pass stores each unit's outcome byte (for unit_outcomes)."""
        self._check(self._lib.ht2gpu_record_outcomes(self._h, 1 if enable else 0), "ht2gpu_record_outcomes")

    def unit_outcomes(self, slot=0):
        """ht2gpu_unit_outcomes: a copy of the outcome bytes (HT2GPU_OUTCOME_AL1 | AL2 | CONC per read or pair) of the
        slot's last batch; align_sam uses slot 0.  Needs record_outcomes() before that batch."""
        p, n = C.c_void_p(), C.c_uint32()
        self._check(self._lib.ht2gpu_unit_outcomes(self._h, slot, C.byref(p), C.byref(n)), "ht2gpu_unit_outcomes")
        return np.frombuffer(C.string_at(p.value, n.value), dtype=np.uint8).copy() if n.value else np.zeros(0, np.uint8)

    def load_splicesites(self, known=None, novel=None):
        """ht2gpu_load_splicesites: --known-splicesite-infile / --novel-splicesite-infile; returns the number of sites kept."""
        n = C.c_uint32(0)
        self._check(self._lib.ht2gpu_load_splicesites(self._h, known.encode() if known else None, novel.encode() if novel else None, C.byref(n)),
                    "ht2gpu_load_splicesites")
        self._ss = (known, novel) if (known or novel) else None      # replicas made by peer() afterwards load the same files
        return int(n.value)

    def collect_splicesites(self, enable=True):
        """ht2gpu_collect_splicesites: record the junctions of printed alignments (--novel-splicesite-outfile)."""
        self._check(self._lib.ht2gpu_collect_splicesites(self._h, 1 if enable else 0), "ht2gpu_collect_splicesites")

    def write_novel_splicesites(self, path, peers=()):
        """ht2gpu_write_novel_splicesites over this handle (+ peers); returns the number of sites written."""
        hs = (C.c_void_p * (1 + len(peers)))(self._h, *[p._h for p in peers])
        n = C.c_uint64(0)
        self._check(self._lib.ht2gpu_write_novel_splicesites(hs, 1 + len(peers), path.encode(), C.byref(n)), "ht2gpu_write_novel_splicesites")
        return int(n.value)

    def set_sam_output(self, no_unal=False, omit_sec_seq=False, no_sq=False, rg_id=None, rg=()):
        """ht2gpu_set_sam_output: --no-unal, --omit-sec-seq, --no-sq, --rg-id and the extra --rg fields of the @RG
        line (printed only with an rg_id).  Applies to the batches that follow and to sam_header()."""
        rg = [r.encode() if isinstance(r, str) else bytes(r) for r in rg]
        arr = (C.c_char_p * max(1, len(rg)))(*rg)
        cfg = CSamOutput(int(bool(no_unal)), int(bool(omit_sec_seq)), int(bool(no_sq)),
                         (rg_id.encode() if isinstance(rg_id, str) else rg_id) if rg_id else None, arr, len(rg))
        self._check(self._lib.ht2gpu_set_sam_output(self._h, C.byref(cfg)), "ht2gpu_set_sam_output")
        self._sam_output = dict(no_unal=no_unal, omit_sec_seq=omit_sec_seq, no_sq=no_sq, rg_id=rg_id, rg=tuple(rg))

    def align_counts(self, peers=(), reset=False):
        """ht2gpu_align_counts: the per-read outcome counts (ReportingMetrics) of every batch formatted on the device
        through this handle (+ peers) since open or the last reset, as a dict of ALIGN_COUNTS."""
        hs = (C.c_void_p * (1 + len(peers)))(self._h, *[p._h for p in peers])
        c = CAlignCounts()
        self._check(self._lib.ht2gpu_align_counts(hs, 1 + len(peers), int(bool(reset)), C.byref(c)), "ht2gpu_align_counts")
        return {k: int(getattr(c, k)) for k in ALIGN_COUNTS}

    def peer(self, device):
        """ht2gpu_open_peer: a replica of this index on another device of this process (device-to-device copy)."""
        o = Options()
        self._lib.ht2gpu_default_options(C.byref(o))
        for k, v in self._opts.items():
            setattr(o, k, v)
        o.device = device
        other = Index.__new__(Index)
        other._lib = self._lib
        other._opts = dict(self._opts)
        other._h = C.c_void_p()
        rc = self._lib.ht2gpu_open_peer(self._h, C.byref(o), C.byref(other._h))
        if rc != 0:
            msg = self._lib.ht2gpu_last_error(other._h).decode() if other._h else "open failed"
            other.close()
            raise Ht2GpuError("ht2gpu_open_peer rc=%d: %s" % (rc, msg))
        if getattr(self, "_ss", None):
            other.load_splicesites(*self._ss)
        if getattr(self, "_sam_output", None):
            other.set_sam_output(**self._sam_output)
        return other

    def run_reads(self, path1=None, path2=None, data1=None, data2=None, fastq=False, collect=True, peers=(), sink=None,
                  read_files=(), **kw):
        """ht2gpu_run_reads(_multi): FASTA/FASTQ (files or bytes in host memory) -> SAM records through the overlapped
        pipeline, on this index's device and on the devices of `peers`.  Returns (sam bytes or None, stats dict).
        `sink(ptr, n)`, if given, sees the SAM text of every batch in read order while it is valid (pinned host memory).
        With read_files (names of READ_FILES) the records are also routed (ht2gpu_run_reads_routed) and the call returns
        (sam, stats, {(output, mate): bytes}); stats then also holds route_spans, route_bytes and s_route."""
        ri, keep = _reads_input(path1, path2, data1, data2, fastq, **kw)
        chunks = []
        total = [0]

        def _sink(ctx, ptr, n):
            if collect:
                chunks.append(C.string_at(ptr, n))
            if sink is not None:
                sink(ptr, n)
            total[0] += n
            return 0
        cb = SINK_FN(_sink) if (collect or sink is not None) else SINK_FN()     # NULL sink: the text still lands in pinned host memory
        st = CRunStats()
        hs = (C.c_void_p * (1 + len(peers)))(self._h, *[p._h for p in peers])
        if read_files:
            rt, files = _read_routes(read_files)
            self._check(self._lib.ht2gpu_run_reads_routed(hs, len(hs), C.byref(ri), cb, None, C.byref(rt), C.byref(st)), "ht2gpu_run_reads_routed")
        else:
            self._check(self._lib.ht2gpu_run_reads_multi(hs, len(hs), C.byref(ri), cb, None, C.byref(st)), "ht2gpu_run_reads")
        stats = {k: getattr(st, k) for k, _ in CRunStats._fields_ if k != "pad"}
        if not read_files:
            return (b"".join(chunks) if collect else None), stats
        stats.update(route_spans=rt.n_spans, route_bytes=rt.bytes, s_route=rt.s_route)
        return (b"".join(chunks) if collect else None), stats, {k: b"".join(v) for k, v in files.items()}

    def is_graph(self):
        return bool(self._lib.ht2gpu_index_is_graph(self._h))

    def geometry(self):
        """ht2gpu_launch_geometry: (warps per block, read slots per lane, blocks per SM) of the alignment kernel."""
        out = (C.c_int32 * 3)()
        self._check(self._lib.ht2gpu_launch_geometry(self._h, out), "ht2gpu_launch_geometry")
        return tuple(int(v) for v in out)

    def sw_extend(self, jobs, warp_fill=True):
        """ht2gpu_sw_extend: the --bowtie2-dp seed extension on its own, one job per lane, with this handle's options.
        jobs: dicts with fw, tidx, toff, rdoff, len, minsc, seed, read (str of ACGTN) and qual (Phred+33 str).
        warp_fill: the pool kernel's DP round (True) or the lane fill.  Returns (SW_RESULT_DTYPE array, list of
        edit arrays in the reference's convention)."""
        n = len(jobs)
        cj = np.zeros(n, dtype=SW_JOB_DTYPE)
        seqs, quals, off = [], [], 0
        for i, j in enumerate(jobs):
            rd, qu = j["read"].encode(), j["qual"].encode()
            cj[i] = (j["fw"], j["tidx"], j["toff"], j["rdoff"], j["len"], j["seed"], j["minsc"], off, len(rd), 0)
            seqs.append(_ASC2DNA[np.frombuffer(rd, dtype=np.uint8)]); quals.append(np.frombuffer(qu, dtype=np.uint8))
            off += len(rd)
        seq = np.ascontiguousarray(np.concatenate(seqs) if seqs else np.zeros(1, np.uint8), dtype=np.uint8)
        qual = np.ascontiguousarray(np.concatenate(quals) if quals else np.zeros(1, np.uint8), dtype=np.uint8)
        res = np.zeros(n, dtype=SW_RESULT_DTYPE)
        ed = np.zeros(n * SW_MAX_EDITS, dtype=EDIT_DTYPE)
        self._check(self._lib.ht2gpu_sw_extend(self._h, n, cj.ctypes.data, seq.ctypes.data, qual.ctypes.data, 1 if warp_fill else 0,
                                               res.ctypes.data, ed.ctypes.data), "ht2gpu_sw_extend")
        edits = [ed[i * SW_MAX_EDITS:i * SW_MAX_EDITS + min(int(res["n_edits"][i]), SW_MAX_EDITS)] for i in range(n)]
        return res, edits

    def seed_search(self, batch, max_range=4):
        """ht2gpu_seed_search: partial-search chains + coordinates of small ranges."""
        cb = batch.c_struct()
        cr = CSeedResult()
        rc = self._lib.ht2gpu_seed_search(self._h, C.byref(cb), max_range, C.byref(cr))
        res = SeedResult(self._lib, cr)
        self._check(rc, "ht2gpu_seed_search")
        return res

    def sam_header(self):
        p, n = C.c_void_p(), C.c_size_t()
        self._check(self._lib.ht2gpu_sam_header(self._h, C.byref(p), C.byref(n)), "ht2gpu_sam_header")
        s = C.string_at(p.value, n.value)
        self._lib.ht2gpu_free_text(p)
        return s

    def format_sam(self, batch, res):
        cb = batch.c_struct()
        p, n = C.c_void_p(), C.c_size_t()
        names = batch.names_blob()
        self._check(self._lib.ht2gpu_format_sam(self._h, C.byref(cb), names, C.byref(res._c), C.byref(p), C.byref(n)),
                    "ht2gpu_format_sam")
        s = C.string_at(p.value, n.value)
        self._lib.ht2gpu_free_text(p)
        return s

    def ref_names(self):
        return [self._lib.ht2gpu_ref_name(self._h, i).decode() for i in range(self._lib.ht2gpu_num_refs(self._h))]

    def close(self):
        if getattr(self, "_h", None):
            self._lib.ht2gpu_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
