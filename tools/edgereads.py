#!/usr/bin/env python3
"""Seeded edge-read corpus over tests/golden/tiny.fa: the reads the simulated sets never produce.

tools/simreads.py samples N-free fragments inside the first sequence, so its reads never touch chrB, the N gap of
chrB, the chrA|chrB boundary of the joined text, or a sequence end, and FASTA gives every base quality 'I'.  This
generator writes reads at exactly those places, every read name starting with its category:

  end_*   reads overhanging the start / end of chrA and chrB by 1..30 bases, both strands
  gap_*   reads abutting, overlapping (1..20 bases) and spanning the 137-base N gap of chrB
  join_*  the last k bases of chrA followed by the first 101-k bases of chrB
  nce_*   floor(0.15 len) Ns and one more (the N ceiling), Ns on the first / last base, IUPAC and lower-case input
  len_*   lengths 1, 2, around the ftab width and minK, 255..257 (the DP extension's limit), 1023, 1024
  near_*  reads within a fragment of every end, gap side and the join, with substitutions, indels and Ns
  q_*     (FASTQ) every quality character from '!' to '~'; mismatches on Q0/Q1, Q16-Q27 and Q41+ bases and at the
          read ends, where soft clipping competes with the mismatch penalty
  sc_*    (one file per --score-min function) mismatches and Ns placed so that the intended alignment scores
          exactly minsc(len), minsc + 1 or minsc - 1, at lengths where the function is at or next to an integer

  python tools/edgereads.py tests/golden/tiny.fa OUT [--seed 11]

writes OUT_se.fa (the placed single-end reads), OUT_near.fa (near_*), OUT_pe_1.fa / OUT_pe_2.fa, OUT_q.fq, OUT_q64.fq (the same reads, Phred+64) and OUT_sc<i>.fa for
every entry of SCORE_MIN.  Deterministic for a given (reference, seed).  numpy only."""
import argparse
import math

import numpy as np

COMP = bytes.maketrans(b"ACGTNacgtn", b"TGCANtgcan")
GAP_LEN = 137

# --score-min functions of the score-boundary files: (type, const, coeff, read lengths).  The lengths put
# C + L * f(len) on an integer (L,0,-0.6 at multiples of 5, S at squares) or just beside one: at 36 and 96,
# L,-0.6,-0.15 is 1e-15 above -6 and -15, where rounding the value to float before truncation gives the next integer.
# None is the library's and the reference's default, L,0,-0.2 with the coefficient -0.2f.
SCORE_MIN = [
    (None, 0.0, 0.0, (20, 50, 100, 101)),
    ("L", 0.0, -0.6, (20, 25, 50, 100, 150)),
    ("L", -0.6, -0.15, (36, 96, 100)),
    ("C", -18.0, 0.0, (60, 101)),
    ("S", -1.0, -2.3, (37, 100, 245)),
    ("G", 2.0, -7.1, (39, 120, 243)),
    ("L", 0.0, -0.35, (180, 340)),
]


def score_min_flag(sm):
    """--score-min argument of a SCORE_MIN entry (None for the default)."""
    t, c, l = sm[:3]
    return None if t is None else "%s,%r,%r" % (t, c, l)


def minsc(sm, n):
    """The reference's minimum score for a read of length n under SCORE_MIN entry sm (SimpleFunc::f, in double)."""
    t, c, l = sm[:3]
    if t is None:
        t, c, l = "L", float(np.float32(0.0)), float(np.float32(-0.2))
    x = {"C": 0.0, "L": float(n), "S": math.sqrt(n), "G": math.log(n) if n > 0 else -math.inf}[t]
    return min(0, int(c + l * x))


def load_contigs(path):
    """{name: ASCII upper-case bytes} of every sequence of a FASTA file, in file order."""
    out, name, chunks = {}, None, []
    with open(path, "rb") as f:
        for line in f:
            if line.startswith(b">"):
                if name is not None:
                    out[name] = b"".join(chunks)
                name, chunks = line[1:].split()[0].decode(), []
            else:
                chunks.append(line.strip().upper())
    if name is not None:
        out[name] = b"".join(chunks)
    return out


class Gen(object):
    def __init__(self, contigs, seed):
        self.c = contigs
        self.rng = np.random.default_rng(seed)
        b = self.c["chrB"]
        self.gap = b.index(b"N" * GAP_LEN)

    def rand(self, n):
        return bytes(self.rng.choice(np.frombuffer(b"ACGT", np.uint8), n)) if n > 0 else b""

    def sub(self, s, rate):
        b = bytearray(s)
        for i in np.nonzero(self.rng.random(len(b)) < rate)[0]:
            b[int(i)] = b"ACGT"[(b"ACGT".index(b[int(i)]) + int(self.rng.integers(1, 4))) & 3] if b[int(i)] in b"ACGT" else b[int(i)]
        return bytes(b)

    def mutate_at(self, s, pos, ch=None):
        b = bytearray(s)
        for p in pos:
            b[p] = ord(ch) if ch else b"ACGT"[(b"ACGT".index(b[p]) + 1 + int(self.rng.integers(0, 3))) & 3]
        return bytes(b)

    def strand(self, s, rc):
        return s.translate(COMP)[::-1] if rc else s

    def unique_locus(self, n):
        """A chrA window of length n away from the ends (chrA is a random sequence: windows of >= 20 bases are unique)."""
        a = self.c["chrA"]
        p = int(self.rng.integers(2000, len(a) - n - 2000))
        return a[p:p + n]


def single_end(g):
    out = []
    A, B = g.c["chrA"], g.c["chrB"]
    # sequence ends
    for chrom, s in (("A", A), ("B", B)):
        for k in range(1, 31):
            for rc in (0, 1):
                for rep in range(3):
                    r = g.rand(k) + s[:101 - k]
                    out.append(("end_%s_start_%d_%d_%d" % (chrom, k, rc, rep), g.strand(r, rc)))
                    r = s[len(s) - (101 - k):] + g.rand(k)
                    out.append(("end_%s_end_%d_%d_%d" % (chrom, k, rc, rep), g.strand(r, rc)))
        for rc in (0, 1):
            out.append(("end_%s_start_0_%d" % (chrom, rc), g.strand(s[:101], rc)))
            out.append(("end_%s_end_0_%d" % (chrom, rc), g.strand(s[-101:], rc)))
    # the N gap of chrB: abutting, overlapping by j (random bases where the reference has Ns, or the Ns themselves), spanning
    lo, hi = g.gap, g.gap + GAP_LEN
    for rc in (0, 1):
        out.append(("gap_abut_left_%d" % rc, g.strand(B[lo - 101:lo], rc)))
        out.append(("gap_abut_right_%d" % rc, g.strand(B[hi:hi + 101], rc)))
        for j in range(1, 21):
            out.append(("gap_left_%d_%d" % (j, rc), g.strand(B[lo - 101 + j:lo] + g.rand(j), rc)))
            out.append(("gap_right_%d_%d" % (j, rc), g.strand(g.rand(j) + B[hi:hi + 101 - j], rc)))
            out.append(("gap_leftN_%d_%d" % (j, rc), g.strand(B[lo - 101 + j:lo + j], rc)))
            out.append(("gap_rightN_%d_%d" % (j, rc), g.strand(B[hi - j:hi + 101 - j], rc)))
        for flank in (10, 40, 100):
            out.append(("gap_span_%d_%d" % (flank, rc), g.strand(B[lo - flank:lo] + g.rand(GAP_LEN) + B[hi:hi + flank], rc)))
            out.append(("gap_spanN_%d_%d" % (flank, rc), g.strand(B[lo - flank:hi + flank], rc)))
    # the chrA|chrB boundary of the joined text
    for k in (1, 2, 5, 10, 15, 20, 30, 40, 50, 60, 70, 80, 86, 91, 96, 99, 100):
        for rc in (0, 1):
            out.append(("join_%d_%d" % (k, rc), g.strand(A[len(A) - k:] + B[:101 - k], rc)))
    # the N ceiling floor(0.15 len) (0.15f in float) and one more; Ns on the first / last base; IUPAC, lower case
    for n in (20, 40, 60, 100, 101, 33, 87):
        ceil_ = int(0.15000000596046448 * n)
        for extra in (0, 1):
            for rep in range(4):
                s = g.unique_locus(n)
                pos = sorted(int(p) for p in g.rng.choice(n, ceil_ + extra, replace=False))
                out.append(("nce_%d_%d_%d" % (n, ceil_ + extra, rep), g.strand(g.mutate_at(s, pos, "N"), rep & 1)))
        for rep in range(2):
            s = g.unique_locus(n)
            out.append(("nce_first_%d_%d" % (n, rep), g.strand(g.mutate_at(s, [0], "N"), rep)))
            out.append(("nce_last_%d_%d" % (n, rep), g.strand(g.mutate_at(s, [n - 1], "N"), rep)))
            out.append(("nce_both_%d_%d" % (n, rep), g.strand(g.mutate_at(s, [0, n - 1], "N"), rep)))
    for rep in range(20):
        s = bytearray(g.unique_locus(101))
        for p in g.rng.choice(101, 3, replace=False):
            s[int(p)] = int(g.rng.choice(list(b"RYKMSWBDHVN.")))
        lo_ = int(g.rng.integers(0, 60))
        s[lo_:lo_ + 30] = bytes(s[lo_:lo_ + 30]).lower()
        out.append(("nce_iupac_%d" % rep, bytes(s)))
    # lengths
    for n in (1, 2, 3, 8, 9, 10, 11, 12, 16, 17, 255, 256, 257, 1023, 1024):
        for rep in range(3):
            s = g.unique_locus(n)
            if n >= 50:
                s = g.sub(s, 0.01)
            out.append(("len_%d_%d" % (n, rep), g.strand(s, rep & 1)))
    # near every end, gap side and the join: the bulk of the corpus
    anchors = [("A", 0, 1), ("A", len(A), -1), ("B", 0, 1), ("B", len(B), -1), ("B", lo, -1), ("B", hi, 1)]
    joined = A + B
    i = 0
    while len(out) < 16000:
        chrom, at, d = anchors[i % len(anchors)]
        s = A if chrom == "A" else B
        n = int(g.rng.choice([36, 50, 76, 101, 101, 101, 150, 250]))
        off = int(g.rng.integers(-20, 200))
        if i % 7 == 6:          # straddle the join
            p = len(A) - int(g.rng.integers(1, n))
            r = joined[p:p + n]
        elif d > 0:
            p = max(at + off - (20 if off < 0 else 0), 20 - n)     # at least 20 bases on the sequence
            r = (g.rand(-p) + s[:p + n]) if p < 0 else s[p:p + n]
        else:
            p = min(at - off - n, len(s) - 20)
            r = s[p:] + g.rand(p + n - len(s)) if p + n > len(s) else s[p:p + n]
        r = r.replace(b"N", g.rand(1))
        r = bytearray(g.sub(r, 0.01))
        if g.rng.random() < 0.2:
            q = int(g.rng.integers(5, len(r) - 5))
            if g.rng.random() < 0.5:
                del r[q:q + int(g.rng.integers(1, 4))]
            else:
                r[q:q] = g.rand(int(g.rng.integers(1, 4)))
        if g.rng.random() < 0.1:
            r[int(g.rng.integers(0, len(r)))] = ord("N")
        out.append(("near_%s%d_%d" % (chrom, anchors.index((chrom, at, d)), i), g.strand(bytes(r), int(g.rng.integers(0, 2)))))
        i += 1
    return out


def n_blocks(g):
    """The N ceiling on reads that can align: floor(0.15 len) Ns in one block (at an end, in the middle, at a third)
    leave long exact seeds, and the intended alignment (AS = -Ns) passes --score-min; one N more filters the read
    (YF:Z:NS)."""
    out = []
    for n in (20, 40, 60, 100, 101):
        ceil_ = int(0.15000000596046448 * n)
        for extra in (0, 1):
            for rep in range(4):
                s = g.unique_locus(n)
                k = ceil_ + extra
                pos = [list(range(k)), list(range(n - k, n)), list(range((n - k) // 2, (n + k) // 2)),
                       list(range(n // 3 - k // 2, n // 3 - k // 2 + k))][rep]
                out.append(("nce_block_%d_%d_%d" % (n, ceil_ + extra, rep), g.strand(g.mutate_at(s, pos, "N"), rep & 1)))
    return out


def paired_end(g):
    """(name, mate1, mate2): fragments at the ends (one mate overhanging), across the gap, across the join."""
    A, B = g.c["chrA"], g.c["chrB"]
    lo, hi = g.gap, g.gap + GAP_LEN
    out = []
    for i in range(3000):
        kind = i % 5
        flen = int(g.rng.integers(200, 400))
        if kind == 0:      # mate overhanging a sequence start
            s = A if i & 8 else B
            k = int(g.rng.integers(1, 31))
            frag = g.rand(k) + s[:flen - k]
        elif kind == 1:    # mate overhanging a sequence end
            s = A if i & 8 else B
            k = int(g.rng.integers(1, 31))
            frag = s[len(s) - (flen - k):] + g.rand(k)
        elif kind == 2:    # mates on opposite sides of the N gap
            left = int(g.rng.integers(101, 250))
            frag = B[lo - left:lo] + g.rand(GAP_LEN) + B[hi:hi + int(g.rng.integers(101, 250))]
        elif kind == 3:    # fragment across the join
            k = int(g.rng.integers(1, flen))
            frag = A[len(A) - k:] + B[:flen - k]
        else:              # fragment ending inside the gap
            k = int(g.rng.integers(1, 60))
            frag = B[lo - flen + k:lo] + g.rand(k)
        frag = g.sub(frag, 0.005)
        m1, m2 = frag[:101], frag[-101:].translate(COMP)[::-1]
        if g.rng.random() < 0.5:
            m1, m2 = m2, m1
        out.append(("pe%d_%s" % (i, ("ovs", "ove", "gap", "join", "ingap")[kind]), m1, m2))
    return out


def fastq_reads(g):
    """(name, seq, phred values): the whole quality range, mismatches on chosen quality classes and at the ends."""
    classes = {"q01": [0, 1], "q1627": list(range(16, 28)), "q41": list(range(41, 94)), "qall": list(range(0, 94))}
    out = []
    for i in range(4000):
        n = 101 if i % 4 else int(g.rng.choice([40, 76, 150]))
        s = g.unique_locus(n)
        q = g.rng.integers(0, 94, n)
        cls = list(classes)[i % 4]
        nm = int(g.rng.integers(1, 4))
        pos = sorted(int(p) for p in g.rng.choice(np.arange(10, n - 10), nm, replace=False))
        ends = []
        if i % 3 == 0:       # mismatches on the outermost bases: clip or pay
            ends = [0, 1, 2][:int(g.rng.integers(1, 4))] if i & 1 else [n - 1, n - 2][:int(g.rng.integers(1, 3))]
        for p in pos + ends:
            q[p] = int(g.rng.choice(classes[cls]))
        s = g.mutate_at(s, pos + ends)
        out.append(("q_%s_%d" % (cls, i), g.strand(s, i & 1), q[::-1] if i & 1 else q))
    return out


def score_boundary(g, sm):
    """Reads whose intended alignment (the chrA locus) scores minsc, minsc + 1 and minsc - 1 under SCORE_MIN entry sm:
    mismatches cost 6 (FASTA qualities are 'I'), Ns 1, spread over the middle of the read."""
    out = []
    for n in sm[3]:
        m = minsc(sm, n)
        nceil = int(0.15000000596046448 * n)
        for d in (0, 1, -1):
            cost = -(m + d)
            if cost < 0:
                continue
            a, b = divmod(cost, 6)
            if b > nceil or a + b > n - 20:
                continue
            for rep in range(12):
                s = g.unique_locus(n)
                step = (n - 20) / float(a + b + 1)
                pos = [10 + int(round(step * (k + 1))) for k in range(a + b)]
                g.rng.shuffle(pos)
                s = g.mutate_at(g.mutate_at(s, pos[:a]), pos[a:], "N")
                out.append(("sc_%d_%d_%+d_%d" % (n, m, d, rep), g.strand(s, rep & 1)))
    return out


def write_fasta(path, recs):
    with open(path, "wb") as f:
        for name, s in recs:
            f.write(b">%s\n%s\n" % (name.encode(), s))


def write_fastq(path, recs, offset=33):
    with open(path, "wb") as f:
        for name, s, q in recs:
            qq = np.minimum(q, 126 - offset) + offset
            f.write(b"@%s\n%s\n+\n%s\n" % (name.encode(), s, bytes(qq.astype(np.uint8))))


def generate(reference, prefix, seed=11):
    g = Gen(load_contigs(reference), seed)
    se = single_end(g)
    se += n_blocks(Gen(g.c, seed + 1))        # own stream: the other files stay as they were without it
    write_fasta(prefix + "_se.fa", [r for r in se if not r[0].startswith("near_")])
    write_fasta(prefix + "_near.fa", [r for r in se if r[0].startswith("near_")])
    pe = paired_end(g)
    write_fasta(prefix + "_pe_1.fa", [(n, a) for n, a, b in pe])
    write_fasta(prefix + "_pe_2.fa", [(n, b) for n, a, b in pe])
    fq = fastq_reads(g)
    write_fastq(prefix + "_q.fq", fq)
    write_fastq(prefix + "_q64.fq", fq, offset=64)
    for i, sm in enumerate(SCORE_MIN):
        write_fasta(prefix + "_sc%d.fa" % i, score_boundary(g, sm))
    return prefix


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("reference")
    ap.add_argument("out_prefix")
    ap.add_argument("--seed", type=int, default=11)
    a = ap.parse_args()
    generate(a.reference, a.out_prefix, a.seed)


if __name__ == "__main__":
    main()
