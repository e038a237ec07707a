"""gzip input inflated on the device (hisat2_b200/csrc/ht2_inflate.h, ht2_inflate.cu, ht2gpu_gunzip).

CPU: the host build of the same decoder source (tests/hostsim/ht2_gunzipsim.cpp, under AddressSanitizer and
UndefinedBehaviorSanitizer) against Python's zlib, byte for byte, on a corpus generated from a seed: levels, strategies,
flush points, multi-member / BGZF / optional header fields, tiny sizes, chunk multiples +-1, distance-32768 and 258-byte
matches across chunk boundaries, random payloads at hundreds of chunks; and a corrupt corpus that must fail every time.

GPU: ht2gpu_gunzip on the same corpus, the window cap, and the read pipeline (CLI and Index.run_reads) on gzip versions
of the golden inputs and of a simulated million pairs, whose SAM must equal that of the plain input.
"""
import gzip
import os
import random
import struct
import subprocess
import sys
import zlib

import pytest

from conftest import GOLDEN, ROOT, sam_lines

CLI = os.path.join(ROOT, "hisat2_b200", "hisat2-b200")
SMALL_CHUNK = 1024


# ---------------------------------------------------------------------------------------------------------------------
# corpus
# ---------------------------------------------------------------------------------------------------------------------
def deflate_raw(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, flushes=()):
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 8, strategy)
    out, at = [], 0
    for pos, mode in flushes:
        out.append(c.compress(data[at:pos]))
        out.append(c.flush(mode))
        at = pos
    out.append(c.compress(data[at:]))
    out.append(c.flush())
    return b"".join(out)


def member(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, flushes=(), extra=None, name=None, comment=None, hcrc=False):
    flg = (4 if extra is not None else 0) | (8 if name else 0) | (16 if comment else 0) | (2 if hcrc else 0)
    h = bytes([0x1F, 0x8B, 8, flg]) + struct.pack("<I", 0) + bytes([0, 255])
    if extra is not None:
        h += struct.pack("<H", len(extra)) + extra
    if name:
        h += name + b"\0"
    if comment:
        h += comment + b"\0"
    if hcrc:
        h += struct.pack("<H", zlib.crc32(h) & 0xFFFF)
    return h + deflate_raw(data, level, strategy, flushes) + struct.pack("<II", zlib.crc32(data), len(data) & 0xFFFFFFFF)


def bgzf(data, level=6, block=65280):
    out = []
    for i in range(0, len(data), block):
        part = data[i:i + block]
        raw = deflate_raw(part, level)
        extra = b"BC" + struct.pack("<HH", 2, 0)   # BSIZE filled below
        m = member(part, level, extra=extra)
        bsize = len(m) - 1
        m = m[:12] + b"BC" + struct.pack("<HH", 2, bsize) + m[18:]
        assert len(raw) + 26 == len(m)
        out.append(m)
    out.append(member(b"", level, extra=b"BC" + struct.pack("<HH", 2, 27)))   # the BGZF end-of-file member
    return b"".join(out)


def fastq_text(n, seed, rdlen=101):
    rnd = random.Random(seed)
    recs = []
    for i in range(n):
        seq = "".join(rnd.choice("ACGT") for _ in range(rdlen))
        qual = "".join(rnd.choice("FFFF:,F#") for _ in range(rdlen))
        recs.append("@r%d/1\n%s\n+\n%s\n" % (i, seq, qual))
    return "".join(recs).encode()


def corpus(seed=7):
    """{name: gzip bytes}, all generated here."""
    rnd = random.Random(seed)
    fq = fastq_text(3000, seed)
    binary = bytes(rnd.getrandbits(8) for _ in range(600000))
    block = bytes(rnd.getrandbits(8) for _ in range(32768))
    far = block * 4 + fq[:20000] + block          # matches at distance exactly 32768 and far back across chunks
    runs = b"".join(bytes([rnd.randrange(256)]) * rnd.randrange(200, 2000) for _ in range(400))   # 258-byte matches
    c = {}
    for lv in (0, 1, 6, 9):
        c["fq_l%d" % lv] = member(fq, lv)
    for st in ("Z_FILTERED", "Z_HUFFMAN_ONLY", "Z_RLE", "Z_FIXED"):
        c["fq_" + st] = member(fq, 6, getattr(zlib, st))
    c["sync_flush"] = member(fq, 6, flushes=[(i, zlib.Z_SYNC_FLUSH) for i in range(1000, len(fq), 7777)])
    c["full_flush"] = member(fq, 6, flushes=[(i, zlib.Z_FULL_FLUSH) for i in range(5000, len(fq), 33333)])
    c["multi_empty"] = member(b"") + member(fq[:100000], 1) + member(b"") + member(b"") + member(fq[100000:], 9) + member(b"")
    c["bgzf"] = bgzf(fq + binary[:100000])
    c["header_fields"] = (member(fq[:50000], 6, name=b"reads_1.fq", comment=b"a comment", hcrc=True)
                          + member(fq[50000:], 6, extra=b"XY\x03\x00abc", name=b"n", hcrc=True))
    c["size0"] = member(b"")
    c["size1"] = member(b"A")
    c["dist32768"] = member(far, 9)
    c["len258"] = member(runs, 9)
    c["random_l6"] = member(binary, 6)
    c["random_huffman"] = member(binary, 6, zlib.Z_HUFFMAN_ONLY)
    c["trailing_zeros"] = member(fq[:30000]) + b"\0" * 100
    return c


def chunk_sizes(name, data):
    """Default, small, and chunk multiples +-1 of the compressed size."""
    L = len(data)
    sizes = [0, SMALL_CHUNK]
    if name in ("fq_l6", "bgzf"):
        sizes += [L, L - 1, L + 1, (L - 1) // 2, (L + 1) // 2, (L + 1) // 3]
    return sorted(set(s for s in sizes if s >= 0))


def corrupt_corpus(seed=11):
    """[(name, bytes)]: every one is rejected by Python's gzip module."""
    rnd = random.Random(seed)
    fq = fastq_text(1500, seed)
    good = member(fq, 6)
    out = [("truncated_%d" % k, good[:k]) for k in (1, 2, 5, 10, 11, 100, len(good) // 2, len(good) - 8, len(good) - 4, len(good) - 1)]
    for i in range(40):
        pos = rnd.randrange(10, len(good))
        bad = bytearray(good)
        bad[pos] ^= 1 << rnd.randrange(8)
        out.append(("flip_%d_%d" % (i, pos), bytes(bad)))
    raw = deflate_raw(fq, 6)
    crc, isz = zlib.crc32(fq), len(fq)
    hdr = bytes([0x1F, 0x8B, 8, 0, 0, 0, 0, 0, 0, 255])
    out.append(("bad_crc", hdr + raw + struct.pack("<II", crc ^ 1, isz)))
    out.append(("bad_isize", hdr + raw + struct.pack("<II", crc, isz + 1)))
    out.append(("btype3", hdr + bytes([0x07, 0, 0]) + struct.pack("<II", 0, 0)))
    # a fixed block whose first symbol is a match of length 3 at distance 1: before the member's start
    out.append(("dist_before_start", hdr + bytes([0x03, 0x02, 0x00]) + struct.pack("<II", 0, 0)))
    # the same in a second member, after a complete first one
    out.append(("dist_before_member", member(b"abc") + hdr + bytes([0x03, 0x02, 0x00]) + struct.pack("<II", 0, 0)))
    out.append(("trailing_garbage", good + b"garbage"))
    out.append(("reserved_flags", bytes([0x1F, 0x8B, 8, 0x20]) + good[4:]))
    out.append(("bad_hcrc", member(fq[:1000], hcrc=True, name=b"x")[:13] + b"\xff\xff" + member(fq[:1000], hcrc=True, name=b"x")[15:]))
    out.append(("stored_nlen", hdr + bytes([0x01, 5, 0, 5, 0]) + b"hello" + struct.pack("<II", zlib.crc32(b"hello"), 5)))
    out.append(("not_gzip", b"\x1f\x8c" + good[2:]))
    keep = []
    for name, data in out:
        try:
            gzip.decompress(data)
        except Exception:
            keep.append((name, data))
    assert len(keep) > 40
    return keep


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the host build of the decoder
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gunzipsim(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("gunzipsim") / "ht2_gunzipsim")
    subprocess.run(["g++", "-O1", "-g", "-std=c++14", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-o", exe,
                    os.path.join(ROOT, "tests", "hostsim", "ht2_gunzipsim.cpp")], check=True)
    return exe


def host_gunzip(exe, tmp_path, data, chunk):
    src, dst = str(tmp_path / "in.gz"), str(tmp_path / "out")
    open(src, "wb").write(data)
    if os.path.exists(dst):
        os.unlink(dst)
    r = subprocess.run([exe, src, dst, str(chunk)], stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    if r.returncode != 0:
        assert r.returncode == 1, r.stderr.decode()     # 1 = a gzip error; a sanitizer report exits otherwise
        assert b"Sanitizer" not in r.stderr and b"runtime error" not in r.stderr, r.stderr.decode()
        return None, r.stderr.decode()
    stats = dict(kv.split("=") for kv in r.stdout.decode().split())
    return open(dst, "rb").read(), {k: int(v) for k, v in stats.items()}


CORPUS = corpus()


@pytest.mark.parametrize("name", sorted(CORPUS))
def test_host_inflate_equals_zlib(gunzipsim, tmp_path, name):
    data = CORPUS[name]
    want = gzip.decompress(data)
    for chunk in chunk_sizes(name, data):
        got, st = host_gunzip(gunzipsim, tmp_path, data, chunk)
        assert got == want, (name, chunk, st)
        assert st["out_bytes"] == len(want)
        members = data.count(b"\x1f\x8b\x08")
        assert 1 <= st["members"] <= members


def test_host_inflate_merges_where_expected(gunzipsim, tmp_path):
    # Z_FIXED: no block start can be found, every chunk is decoded by its predecessor
    _, st = host_gunzip(gunzipsim, tmp_path, CORPUS["fq_Z_FIXED"], SMALL_CHUNK)
    assert st["confirmed"] == 0 and st["merged_no_candidate"] >= len(CORPUS["fq_Z_FIXED"]) // SMALL_CHUNK - 2
    # random payloads at hundreds of chunks: false starts are found and merged
    _, st = host_gunzip(gunzipsim, tmp_path, CORPUS["random_l6"], SMALL_CHUNK)
    assert st["merged_false_positive"] > 0 and st["confirmed"] > 0
    assert len(CORPUS["random_l6"]) // SMALL_CHUNK > 300
    # an ordinary level-6 FASTQ stream: most chunks start speculatively and are confirmed
    _, st = host_gunzip(gunzipsim, tmp_path, CORPUS["fq_l6"], 4096)
    assert st["confirmed"] >= st["blocks"] // 2 and st["windows"] == 1
    # windows: with small chunks the input runs through several, the decoder state carried across
    big = member(fastq_text(12000, 3), 6)
    got, st = host_gunzip(gunzipsim, tmp_path, big, 512)
    assert st["windows"] > 1 and got == gzip.decompress(big)


def test_host_inflate_large_chunks_keep_every_chunk(gunzipsim, tmp_path):
    """Chunks of 1-4 MB: the chunk count per window shrinks so that each chunk's output fits its slice of the symbol
    buffer; no window is cut short by a full chunk (which would decode the rest of it again)."""
    big = member(fastq_text(4000, 9) * 60, 6)     # 52 MB of FASTQ, more than one 32 MB window of input at 4 MB chunks
    want = gzip.decompress(big)
    for chunk in (1 << 20, 4 << 20):
        got, st = host_gunzip(gunzipsim, tmp_path, big, chunk)
        assert got == want
        assert st["windows_cut"] == 0 and st["confirmed"] > 0, (chunk, st)


@pytest.mark.parametrize("name,data", corrupt_corpus(), ids=[n for n, _ in corrupt_corpus()])
def test_host_inflate_rejects_corrupt_input(gunzipsim, tmp_path, name, data):
    for chunk in (0, 64, SMALL_CHUNK):
        got, msg = host_gunzip(gunzipsim, tmp_path, data, chunk)
        assert got is None and msg.startswith("gunzip: "), (name, chunk)


def test_host_only_calls_refuse_compressed_input(lib, tmp_path):
    import numpy as np
    from hisat2_b200 import api
    gz = member(open(os.path.join(GOLDEN, "tiny_se.fa"), "rb").read())
    with pytest.raises(api.Ht2GpuError, match="ht2gpu_gunzip"):
        api.route_reads(np.zeros(0, np.uint8), data1=gz, read_files=())
    with pytest.raises(api.Ht2GpuError, match="bzip2"):
        api.route_reads(np.zeros(0, np.uint8), data1=b"BZh91AY&SY", read_files=())
    # ht2gpu_parse_reads
    import ctypes as C
    ri, keep = api._reads_input(data1=gz)
    out = api.CParsedReads()
    err = C.create_string_buffer(512)
    assert lib.ht2gpu_parse_reads(C.byref(ri), C.byref(out), err, 512) == -1
    assert b"ht2gpu_gunzip" in err.value


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def h2(lib):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import hisat2_b200
    return hisat2_b200


@pytest.mark.gpu
def test_device_inflate_equals_zlib(h2):
    for name in sorted(CORPUS):
        data = CORPUS[name]
        want = gzip.decompress(data)
        for chunk in chunk_sizes(name, data):
            got, st = h2.gunzip(data, chunk_bytes=chunk)
            assert got == want, (name, chunk, st)
            assert st["out_bytes"] == len(want) and st["in_bytes"] == len(data)
    _, st = h2.gunzip(CORPUS["fq_Z_FIXED"], chunk_bytes=SMALL_CHUNK)
    assert st["chunks_confirmed"] == 0 and st["chunks_merged_no_candidate"] > 0
    _, st = h2.gunzip(CORPUS["random_l6"], chunk_bytes=SMALL_CHUNK)
    assert st["chunks_merged_false_positive"] > 0


@pytest.mark.gpu
def test_device_inflate_rejects_corrupt_input(h2):
    for name, data in corrupt_corpus():
        for chunk in (0, 64):
            with pytest.raises(h2.Ht2GpuError, match="ht2gpu_gunzip rc=-6"):
                h2.gunzip(data, chunk_bytes=chunk)


@pytest.mark.gpu
def test_device_inflate_memory_is_capped(h2, tmp_path):
    text = fastq_text(4000, 5) * 40                 # 34 MB of FASTQ
    data = member(text, 6)
    path = str(tmp_path / "big.fq.gz")
    open(path, "wb").write(data)
    for chunk in (0, 4096):
        got, st = h2.gunzip(path, chunk_bytes=chunk)
        assert got == text
        assert st["windows"] > 1, st
        assert st["peak_device_bytes"] <= 256 << 20, st     # every device buffer of the call is allocated up front
        assert st["windows_cut"] == 0, st


def gz_variants(data):
    """One member, several members, BGZF-style, at levels 1 and 9."""
    out = {}
    for lv in (1, 9):
        out["one_l%d" % lv] = member(data, lv)
        cut = [0, len(data) // 3, len(data) // 2, len(data)]
        out["multi_l%d" % lv] = b"".join(member(data[a:b], lv) for a, b in zip(cut, cut[1:]))
        out["bgzf_l%d" % lv] = bgzf(data, lv, block=4096)
    return out


GOLDEN_CASES = [
    ("tiny", ["-q"], ("tiny_se.fq",), "tiny_se_fq.sam", {}),
    ("tiny", ["-q"], ("tiny_pe_1.fq", "tiny_pe_2.fq"), "tiny_pe_fq.sam", {}),
    ("tiny", ["-f"], ("tiny_pe_1.fa", "tiny_pe_2.fa"), "tiny_pe.sam", {}),
    ("tiny_snp", ["-f"], ("tiny_alt_1.fa", "tiny_alt_2.fa"), "tiny_snp_alt_pe.sam", {}),
    ("tiny", ["-f", "--no-temp-splicesite", "--known-splicesite-infile", "tiny_ss_rna_ss.txt"], ("tiny_ss_rna_1.fa", "tiny_ss_rna_2.fa"),
     "tiny_ss_rna_pe.sam", {"spliced": True}),
]


@pytest.mark.gpu
def test_golden_inputs_gzip_cli_and_run_reads(h2, tmp_path):
    g = lambda n: os.path.join(GOLDEN, n)
    for index, args, files, gold, kw in GOLDEN_CASES:
        want = sam_lines(open(g(gold), "rb").read())
        want_recs = [l for l in want if not l.startswith(b"@")]
        variants = [gz_variants(open(g(f), "rb").read()) for f in files]
        fastq = "-q" in args
        idx = h2.Index(g(index), no_spliced_alignment=0 if kw.get("spliced") else 1)
        if kw.get("spliced"):
            idx.load_splicesites(g("tiny_ss_rna_ss.txt"))
        for v in variants[0]:
            data = [vs[v] for vs in variants]
            sam, _ = idx.run_reads(data1=data[0], data2=data[1] if len(data) > 1 else None, fastq=fastq)
            assert [l for l in sam_lines(sam) if not l.startswith(b"@")] == want_recs, (gold, v)
            paths = []
            for f, d in zip(files, data):
                p = str(tmp_path / (f + "." + v))                 # no .gz suffix: detection is by content
                open(p, "wb").write(d)
                paths.append(p)
            sam, _ = idx.run_reads(path1=paths[0], path2=paths[1] if len(paths) > 1 else None, fastq=fastq)
            assert [l for l in sam_lines(sam) if not l.startswith(b"@")] == want_recs, (gold, v, "path")
            st = idx.gunzip_stats()
            assert st["out_bytes"] == sum(len(open(g(f), "rb").read()) for f in files)
        idx.close()
        for v in ("one_l9", "multi_l1", "bgzf_l9"):
            paths = []
            for f, vs in zip(files, variants):
                p = str(tmp_path / (f + ".gz"))
                open(p, "wb").write(vs[v])
                paths.append(p)
            reads = ["-U", paths[0]] if len(paths) == 1 else ["-1", paths[0], "-2", paths[1]]
            spl = [] if kw.get("spliced") else ["--no-spliced-alignment"]
            out = str(tmp_path / "cli.sam")
            subprocess.run([CLI] + spl + ["-x", index] + args + reads + ["-S", out], cwd=GOLDEN, check=True, stderr=subprocess.DEVNULL)
            assert sam_lines(open(out, "rb").read()) == want, (gold, v, "cli")


@pytest.mark.gpu
def test_run_reads_corrupt_gzip_sinks_nothing(h2):
    """The reads of a gzip input are parsed and aligned while it is inflated, but no SAM reaches the sink before every
    member is verified: a CRC-32 error in the last trailer of a multi-batch input yields an error and no records."""
    text = b"".join(sim_fastq(200000))[:200000 * 217]
    bad = bytearray(member(text, 6))
    bad[-8] ^= 1
    idx = h2.Index(os.path.join(GOLDEN, "tiny"))
    seen = []
    with pytest.raises(h2.Ht2GpuError, match="CRC-32"):
        idx.run_reads(data1=bytes(bad), fastq=True, batch_reads=20000, sink=lambda p, n: seen.append(n))
    assert seen == []
    sam, _ = idx.run_reads(data1=member(text, 6), fastq=True, batch_reads=20000)
    plain, _ = idx.run_reads(data1=text, fastq=True, batch_reads=20000)
    assert sam == plain and len(sam) > 0
    idx.close()


@pytest.mark.gpu
def test_cli_corrupt_gzip_fails_without_records(h2, tmp_path):
    fq = open(os.path.join(GOLDEN, "tiny_se.fq"), "rb").read()
    bad = bytearray(member(fq, 6))
    bad[-6] ^= 0x10                                   # CRC-32 / ISIZE mismatch
    p = str(tmp_path / "bad.fq.gz")
    open(p, "wb").write(bytes(bad))
    out = str(tmp_path / "o.sam")
    r = subprocess.run([CLI, "--no-spliced-alignment", "-x", "tiny", "-q", "-U", p, "-S", out], cwd=GOLDEN, stderr=subprocess.PIPE)
    assert r.returncode != 0 and b"gzip" in r.stderr
    assert not [l for l in open(out, "rb").read().splitlines() if not l.startswith(b"@")] if os.path.exists(out) else True
    r = subprocess.run([CLI, "--no-spliced-alignment", "-x", "tiny", "-q", "-U", "-", "-S", out], cwd=GOLDEN, input=b"BZh91AY&SY",
                       stderr=subprocess.PIPE)
    assert r.returncode != 0 and b"bzip2" in r.stderr


def sim_fastq(pairs, seed=1):
    """Simulated 2x101 pairs from the tiny fixture (tools/simreads_fast.c) as FASTQ text with varied qualities."""
    import numpy as np
    sys.path.insert(0, ROOT)
    import bench
    a, b = bench.sim_fasta(0, pairs, seed=seed)
    rng = np.random.default_rng(seed)
    out = []
    for buf in (a, b):
        r = np.asarray(buf).reshape(pairs, bench.RECSZ)
        q = np.empty((pairs, 217), np.uint8)
        q[:, 0] = ord("@")
        q[:, 1:113] = r[:, 1:113]                      # name, bases and their newlines
        q[:, 113:115] = np.frombuffer(b"+\n", np.uint8)
        q[:, 115:216] = np.frombuffer(b"FFFF:F,F#:FFFFFF", np.uint8)[rng.integers(0, 16, (pairs, 101))]
        q[:, 216] = ord("\n")
        out.append(q.tobytes())
    return out


@pytest.mark.gpu
def test_million_pairs_gzip_equals_plain(h2, tmp_path):
    pairs = 1000000
    f1, f2 = sim_fastq(pairs)
    plain, gz = [], []
    for i, txt in enumerate((f1, f2)):
        p = str(tmp_path / ("r_%d.fq" % (i + 1)))
        open(p, "wb").write(txt)
        plain.append(p)
        open(p + ".gz", "wb").write(zlib.compress(txt, 6, wbits=31))
        gz.append(p + ".gz")
    base = ["--no-spliced-alignment", "-x", "tiny", "-q", "-p", "8"]

    def run(reads, extra=(), stdin=None, tag="x"):
        out = str(tmp_path / ("%s.sam" % tag))
        r = subprocess.run([CLI] + base + list(extra) + reads + ["-S", out], cwd=GOLDEN, stdin=stdin, stderr=subprocess.PIPE)
        assert r.returncode == 0, r.stderr.decode()[-2000:]
        return open(out, "rb").read()

    for extra in ([], ["-s", "1234", "-u", "300000", "-5", "3", "-3", "7"]):
        a = run(["-1", plain[0], "-2", plain[1]], extra, tag="plain")
        b = run(["-1", gz[0], "-2", gz[1]], extra, tag="gz")
        assert sam_lines(a) == sam_lines(b), extra
    a = run(["-U", plain[0]], tag="plain_se")
    with open(gz[0], "rb") as fin:
        b = run(["-U", "-"], stdin=fin, tag="gz_stdin")
    assert sam_lines(a) == sam_lines(b)
    # read files: the decompressed record text, equal to what the plain input gives
    outs = {}
    for kind, reads in (("plain", plain), ("gz", gz)):
        d = tmp_path / kind
        d.mkdir()
        run(["-1", reads[0], "-2", reads[1]], ["--un-conc-gz", str(d / "un_%.fq.gz"), "--al-conc", str(d / "al_%.fq")], tag=kind + "_rf")
        outs[kind] = [gzip.decompress(open(str(d / ("un_%d.fq.gz" % m)), "rb").read()) for m in (1, 2)] + \
                     [open(str(d / ("al_%d.fq" % m)), "rb").read() for m in (1, 2)]
    assert outs["plain"] == outs["gz"] and sum(len(x) for x in outs["plain"]) > 0
    import torch
    if torch.cuda.device_count() >= 2:
        a = run(["-1", plain[0], "-2", plain[1]], ["--gpus", "2"], tag="plain2")
        b = run(["-1", gz[0], "-2", gz[1]], ["--gpus", "2"], tag="gz2")
        assert sam_lines(a) == sam_lines(b)
