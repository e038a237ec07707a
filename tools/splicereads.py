#!/usr/bin/env python3
"""Seeded spliced-read corpus over tests/golden/tiny.fa: junctions at every rule boundary of spliced alignment.

tools/sim_rna.py cuts GT-AG introns of 60-4000 bases and never reaches the intron-length penalty steps, MaxIntronLen,
the --min-intronlen line, the semi-canonical motifs or a sequence end.  This generator cuts every intron from the
reference at a chosen motif, every read name starting with its category:

  motif_*   one junction per read for each motif: GT-AG, CT-AC, GC-AG, CT-GC, AT-AC, GT-AT and non-canonical, both
            read strands
  anchor_*  a 1-30-base anchor left or right of the junction (minAnchorLen 7 canonical, 14 otherwise), clean and with
            a mismatch, an N or a 1-3-base indel inside the anchor
  len_*     intron lengths 19 / 20 / 21 (a deletion or an intron at --min-intronlen), 8103 / 8104 and 22026 / 22027 (the
            intron-length penalty steps), 2^13 and 2^14 +-1 with anchors of 7-9 (MaxIntronLen), 4095 / 4096 ...
            32767 / 32768 (the splice-probability thresholds) and floor / ceil of 0.01 * 2^(2a+4) and 0.01 * 2^(2a)
            for anchors a = 4..10 (intronLen_prob of the junction search)
  multi_*   2-4 junctions with middle exons of 5-40 bases, reads of 101, 150 and 250 bases
  sense_*   a GT-AG junction and a CT-AC junction in one read (opposite senses)
  redge_*   exons within 1-30 bases of a sequence start or end, spliced reads overhanging a sequence end
  gap_*     exons abutting the 137-base N gap of chrB and introns containing it
  join_*    the end of chrA followed by the start of chrB, as if it were a junction

  python tools/splicereads.py tests/golden/tiny.fa OUT [--seed 17]

writes OUT_se.fa (the single-end reads above), OUT_q.fq (FASTQ copies of the anchor reads, low qualities on the
anchor, where a soft clip competes with the splice), OUT_pe_1.fa / OUT_pe_2.fa (fragments across 1-2 junctions, a
mate wholly inside a short exon, mates at sequence ends, fragments longer than -X 1000 only because of an intron),
OUT_ss.txt (85 % of the corpus's introns plus decoys, in tools/sim_rna.py's format) and, from tools/sim_rna.py with
the same seed, OUT_sim.fa / OUT_sim_1.fa / OUT_sim_2.fa / OUT_sim_ss.txt (20 k reads, 10 k pairs).  Deterministic for
a given (reference, seed).  numpy only."""
import argparse
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from edgereads import COMP, GAP_LEN, Gen, load_contigs, write_fasta, write_fastq  # noqa: E402
import sim_rna  # noqa: E402

# motif name -> (first two, last two intron bases, transcript strand of the site list; None: either)
MOTIFS = {"GTAG": (b"GT", b"AG", "+"), "CTAC": (b"CT", b"AC", "-"), "GCAG": (b"GC", b"AG", "+"), "CTGC": (b"CT", b"GC", "-"),
          "ATAC": (b"AT", b"AC", "+"), "GTAT": (b"GT", b"AT", "-"), "non": (None, None, None)}


def _code(a, p):
    return a[p].astype(np.int32) * 256 + a[p + 1]


class SpliceGen(Gen):
    def __init__(self, contigs, seed):
        Gen.__init__(self, contigs, seed)
        self.arr = {k: np.frombuffer(v, np.uint8) for k, v in contigs.items()}
        self.introns = []          # (chrom, last exon base, first base after the intron, strand): the site-file convention

    def _fits(self, a, p, L, motif):
        """Which intron starts p (of lengths L) have the motif and no N at their ends."""
        d, e = _code(a, p), _code(a, p + L - 2)
        m5, m3, _ = MOTIFS[motif]
        if m5 is None:
            ok = np.ones(len(p), bool)
            for x5, x3, _s in MOTIFS.values():
                if x5 is not None:
                    ok &= ~((d == x5[0] * 256 + x5[1]) & (e == x3[0] * 256 + x3[1]))
        else:
            ok = (d == m5[0] * 256 + m5[1]) & (e == m3[0] * 256 + m3[1])
        return ok & (a[p] != 78) & (a[p + 1] != 78) & (a[p + L - 2] != 78) & (a[p + L - 1] != 78)

    def site(self, chrom, L, motif, lo, hi):
        """A random start p in [lo, hi) of an intron of L bases with the given motif, or None."""
        a = self.arr[chrom]
        hi = min(hi, len(a) - L - 1)
        if hi <= lo:
            return None
        p = np.arange(lo, hi)
        cand = p[self._fits(a, p, L, motif)]
        return int(cand[int(self.rng.integers(0, len(cand)))]) if len(cand) else None

    def intron(self, chrom, motif, lens, start=None, end=None):
        """An intron with the given motif starting at `start` or ending before `end` (an int, or a range to choose
        from), its length drawn from range(*lens): (p, L), or None."""
        a = self.arr[chrom]
        L0 = np.arange(*lens)
        at = np.array([start if start is not None else end]).reshape(-1)
        L = np.tile(L0, len(at))
        at = np.repeat(at, len(L0))
        p = at if start is not None else at - L
        keep = (p >= 1) & (p + L < len(a) - 1)
        p, L = p[keep], L[keep]
        ok = np.nonzero(self._fits(a, p, L, motif))[0]
        if not len(ok):
            return None
        k = int(ok[int(self.rng.integers(0, len(ok)))])
        return int(p[k]), int(L[k])

    def note(self, chrom, p, L, motif):
        strand = MOTIFS[motif][2] or "+-"[int(self.rng.integers(0, 2))]
        self.introns.append((chrom, p - 1, p + L, strand))

    def junction(self, L, motif, left, right, chrom="chrA", lo=None, hi=None):
        """The read left exon (left bases) + right exon (right bases) around one intron; (read, chrom, p) or None."""
        s = self.c[chrom]
        lo = left if lo is None else max(lo, left)
        hi = len(s) - L - right if hi is None else min(hi, len(s) - L - right)
        p = self.site(chrom, L, motif, lo, hi)
        if p is None:
            return None
        r = s[p - left:p] + s[p + L:p + L + right]
        if b"N" in r:
            return None
        self.note(chrom, p, L, motif)
        return r, chrom, p

    def chain(self, n, motifs, mid=(5, 41), lens=(60, 3000), chrom="chrA"):
        """A read of n bases over len(motifs) junctions: the first exon ends at a site of motifs[0], every middle exon
        is 5-40 bases up to the next site of the next motif, the last exon fills the read.  None if no such layout."""
        s, a = self.c[chrom], self.arr[chrom]
        first = int(self.rng.integers(10, max(11, n // 3)))
        pos = int(self.rng.integers(2000, len(s) - 30000))
        exons, sites = [], []
        p = pos + first
        for k, m in enumerate(motifs):
            m5, m3, _ = MOTIFS[m]
            pl = self.intron(chrom, m, lens, start=p)
            if pl is None:
                return None
            L = pl[1]
            exons.append((pos, p))
            sites.append((p, L, m))
            pos = p + L
            if k + 1 < len(motifs):
                nxt5 = MOTIFS[motifs[k + 1]][0]
                ks = [j for j in range(*mid) if nxt5 is None or s[pos + j:pos + j + 2] == nxt5]
                if not ks:
                    return None
                p = pos + ks[int(self.rng.integers(0, len(ks)))]
        used = sum(e - b for b, e in exons)
        if used >= n - 5:
            return None
        exons.append((pos, pos + n - used))
        r = b"".join(s[b:e] for b, e in exons)
        if b"N" in r or len(r) != n:
            return None
        for p, L, m in sites:
            self.note(chrom, p, L, m)
        return r


def motif_reads(g):
    out = []
    for m in MOTIFS:
        for rc in (0, 1):
            for L in (60, 500, 3000):
                for left in (20, 50, 81):
                    j = g.junction(L, m, left, 101 - left)
                    if j:
                        out.append(("motif_%s_%d_%d_%d" % (m, L, left, rc), g.strand(j[0], rc)))
    return out


def anchor_reads(g):
    """(name, read, anchor slice in read coordinates before the strand flip, rc)"""
    out = []
    for m in ("GTAG", "CTAC", "GCAG", "non"):
        for a in range(1, 31):
            for side in "LR":
                for var in ("clean", "mm", "n", "ins", "del"):
                    L = int(g.rng.integers(100, 2000))
                    # an insertion of k bases takes k reference bases from the anchor exon, a deletion adds k
                    k = int(g.rng.integers(1, 4)) if var in ("ins", "del") else 0
                    if (var == "ins" and a < k + 2) or (var == "del" and a < 2):
                        continue
                    ex = a - k if var == "ins" else a + k
                    left, right = (ex, 101 - a) if side == "L" else (101 - a, ex)
                    j = g.junction(L, m, left, right)
                    if j is None:
                        continue
                    r = bytearray(j[0])
                    span = (0, ex) if side == "L" else (101 - a, 101 - a + ex)
                    if var in ("mm", "n"):
                        q = int(g.rng.integers(span[0], span[1]))
                        r = bytearray(g.mutate_at(bytes(r), [q], "N" if var == "n" else None))
                    elif var == "ins":
                        q = int(g.rng.integers(span[0] + 1, span[1]))
                        r[q:q] = g.rand(k)
                    elif var == "del":
                        q = int(g.rng.integers(span[0] + 1, span[1] - k))
                        del r[q:q + k]
                    span = (0, a) if side == "L" else (101 - a, 101)
                    rc = int(g.rng.integers(0, 2))
                    out.append(("anchor_%s_%s%d_%s_%d_%d" % (m, side, a, var, L, len(out)), bytes(r), span, rc))
    return out


def length_reads(g):
    out = []
    cases = []
    for L in (19, 20, 21):
        for m in ("GTAG", "non"):
            cases += [(L, m, (30, 70), 3)]
    for L in (8103, 8104, 22026, 22027):
        for m in ("GTAG", "CTAC", "non"):
            cases += [(L, m, (40, 61), 3)]
    for L in (8191, 8192, 8193, 16383, 16384, 16385):
        for m in ("GTAG", "CTAC"):
            for a in (7, 8, 9):
                cases += [(L, m, (a, a + 1), 2)]
    for L in (4095, 4096, 8191, 8192, 16383, 16384, 32767, 32768):
        for m in ("GTAG", "CTAC"):
            cases += [(L, m, (30, 51), 3)]
    for a in range(4, 11):
        for x, ms in ((0.01 * 2 ** (2 * a + 4), ("GTAG", "CTAC")), (0.01 * 2 ** (2 * a), ("GCAG", "non"))):
            for L in sorted({int(math.floor(x)), int(math.ceil(x))}):
                if 2 <= L <= 45000:
                    for m in ms:
                        cases += [(L, m, (a, a + 1), 2)]
    for L, m, (alo, ahi), reps in cases:
        for rep in range(reps):
            a = int(g.rng.integers(alo, ahi))
            left = a if rep & 1 else 101 - a
            j = g.junction(L, m, left, 101 - left)
            if j:
                out.append(("len_%d_%s_a%d_%d" % (L, m, a, rep), g.strand(j[0], (rep >> 1) & 1 if reps > 2 else rep & 1)))
    return out


def multi_reads(g):
    out = []
    for n in (101, 150, 250):
        for k in (2, 3, 4):
            got, tries = 0, 0
            while got < 20 and tries < 2000:
                tries += 1
                ms = [("GTAG", "CTAC", "GCAG", "non")[int(x)] for x in g.rng.choice(4, k, p=[0.55, 0.3, 0.1, 0.05])]
                ms = ms if len(set(MOTIFS[m][2] for m in ms) - {None}) <= 1 else ["GTAG"] * k
                r = g.chain(n, ms)
                if r:
                    out.append(("multi_%d_%d_%s_%d" % (n, k, "-".join(ms), got), g.strand(r, got & 1)))
                    got += 1
    got, tries = 0, 0
    while got < 30 and tries < 3000:
        tries += 1
        ms = ["GTAG", "CTAC"] if got & 2 else ["CTAC", "GTAG"]
        r = g.chain(101 if got % 3 else 150, ms, mid=(20, 41))
        if r:
            out.append(("sense_%s_%d" % ("-".join(ms), got), g.strand(r, got & 1)))
            got += 1
    return out


def edge_reads(g):
    out = []
    lo, hi = g.gap, g.gap + GAP_LEN
    for chrom in ("chrA", "chrB"):
        s = g.c[chrom]
        for k in range(1, 31):
            for rep in range(2):
                m = ("GTAG", "CTAC")[rep]
                # the first exon starts k bases into the sequence
                p, L = g.intron(chrom, m, (100, 3000), start=range(k + 20, k + 70)) or (None, None)
                if p is not None and b"N" not in s[k:p] + s[p + L:p + L + 101 - (p - k)]:
                    g.note(chrom, p, L, m)
                    out.append(("redge_%s_start_%d_%d" % (chrom, k, rep), g.strand(s[k:p] + s[p + L:p + L + 101 - (p - k)], rep)))
                # the last exon ends k bases before the sequence end
                end = len(s) - k
                p, L = g.intron(chrom, m, (100, 3000), end=range(end - 70, end - 20)) or (None, None)
                q = None if p is None else p + L
                if p is not None and b"N" not in s[p - (101 - end + q):p] + s[q:end]:
                    g.note(chrom, p, L, m)
                    out.append(("redge_%s_end_%d_%d" % (chrom, k, rep), g.strand(s[p - (101 - end + q):p] + s[q:end], rep)))
        for k in range(1, 11):       # spliced and overhanging the sequence start / end by k bases
            p, L = g.intron(chrom, "GTAG", (100, 2000), start=range(30 - k, 50 - k)) or (None, None)
            if p is not None and b"N" not in s[p + L:p + L + 61]:
                g.note(chrom, p, L, "GTAG")
                out.append(("redge_%s_ovs_%d" % (chrom, k), g.strand(g.rand(k) + s[:p] + s[p + L:p + L + 61], k & 1)))
            p, L = g.intron(chrom, "GTAG", (100, 2000), end=range(len(s) - 50 + k, len(s) - 30 + k)) or (None, None)
            q = None if p is None else p + L
            if p is not None and b"N" not in s[p - 61:p]:
                g.note(chrom, p, L, "GTAG")
                out.append(("redge_%s_ove_%d" % (chrom, k), g.strand(s[p - 61:p] + s[q:] + g.rand(k), k & 1)))
    B = g.c["chrB"]
    for rep in range(10):
        e = int(g.rng.integers(20, 82))
        L = int(g.rng.integers(GAP_LEN + 40, 2000))
        # an exon ending at the gap's left edge: the intron starts with the gap
        out.append(("gap_abutleft_%d" % rep, g.strand(B[lo - e:lo] + B[lo + L:lo + L + 101 - e], rep & 1)))
        # an exon starting at the gap's right edge: the intron ends with the gap
        out.append(("gap_abutright_%d" % rep, g.strand(B[hi - L - e:hi - L] + B[hi:hi + 101 - e], rep & 1)))
        # an intron containing the gap, with a motif
        L = int(g.rng.integers(GAP_LEN + 300, 3000))
        j = g.junction(L, ("GTAG", "CTAC")[rep & 1], e, 101 - e, "chrB", lo=hi - L + 5, hi=lo - 5)
        if j:
            out.append(("gap_inintron_%d" % rep, g.strand(j[0], rep & 1)))
    A = g.c["chrA"]
    for k in (7, 10, 15, 20, 30, 40, 50, 60, 70, 80, 86, 91, 94):
        for rc in (0, 1):
            out.append(("join_%d_%d" % (k, rc), g.strand(A[len(A) - k:] + B[:101 - k], rc)))
    return out


def fastq_copies(g, anchors):
    """FASTQ copies of the clean and mismatch anchor reads: qualities 30-40, 2-12 on the anchor."""
    out = []
    for name, r, (a, b), rc in anchors:
        if "_clean_" not in name and "_mm_" not in name:
            continue
        q = g.rng.integers(30, 41, len(r))
        q[a:min(b, len(r))] = g.rng.integers(2, 13, max(0, min(b, len(r)) - a))
        out.append(("fq_" + name, g.strand(r, rc), q[::-1].copy() if rc else q))
    return out


def paired_reads(g):
    out = []
    A, B = g.c["chrA"], g.c["chrB"]
    i = 0
    while len(out) < 1500 and i < 20000:
        kind = len(out) % 5
        i += 1
        if kind in (0, 1):           # a fragment across 1 (kind 0) or 2 junctions
            k = kind + 1
            ms = [("GTAG", "CTAC")[int(g.rng.integers(0, 2))]] * k
            r = g.chain(int(g.rng.integers(200, 400)), ms, mid=(60, 200) if k > 1 else (5, 41))
        elif kind == 2:              # one mate wholly inside a short middle exon
            r = g.chain(int(g.rng.integers(220, 320)), ["GTAG", "GTAG"], mid=(105, 140))
        elif kind == 3:              # a fragment starting at a sequence start or ending at a sequence end
            chrom = ("chrA", "chrB")[len(out) & 1]
            s = g.c[chrom]
            e = int(g.rng.integers(120, 200))
            flen = int(g.rng.integers(240, 360))
            if len(out) & 2:
                p, L = g.intron(chrom, "GTAG", (100, 2000), start=range(e, e + 30)) or (None, None)
                r = None if p is None else s[:p] + s[p + L:p + L + flen - p]
            else:
                q = len(s) - e
                p, L = g.intron(chrom, "GTAG", (100, 2000), end=range(q - 30, q)) or (None, None)
                r = None if p is None else s[p - (flen - len(s) + p + L):p] + s[p + L:]
            if r is not None and b"N" not in r:
                g.note(chrom, p, L, "GTAG")
            else:
                r = None
        else:                        # genomic span beyond -X 1000 only through an intron of 800-3000 bases
            r = g.chain(int(g.rng.integers(250, 400)), ["GTAG"], mid=(5, 41), lens=(800, 3000))
        if r is None or len(r) < 202:
            continue
        r = g.sub(r, 0.004)
        m1, m2 = r[:101], r[-101:].translate(COMP)[::-1]
        if g.rng.random() < 0.5:
            m1, m2 = m2, m1
        out.append(("sp%d_%s" % (len(out), ("one", "two", "inexon", "end", "span")[kind]), m1, m2))
    return out


def site_lines(g):
    """85 % of the corpus's introns, decoys, a duplicate and an unknown sequence name, shuffled."""
    keep = [s for s in sorted(set(g.introns)) if g.rng.random() < 0.85]
    decoys = []
    for _ in range(max(20, len(keep) // 5)):
        chrom = ("chrA", "chrB")[int(g.rng.integers(0, 2))]
        p = int(g.rng.integers(100, len(g.c[chrom]) - 5000))
        decoys.append((chrom, p, p + int(g.rng.integers(50, 3000)), "+-"[int(g.rng.integers(0, 2))]))
    sl = keep + decoys
    g.rng.shuffle(sl)
    return ["%s\t%d\t%d\t%s" % s for s in sl[:10]] + ["chrNOPE\t10\t200\t+"] + ["%s\t%d\t%d\t%s" % s for s in sl]


def generate(reference, prefix, seed=17):
    g = SpliceGen(load_contigs(reference), seed)
    anchors = anchor_reads(g)
    se = motif_reads(g) + [(n, g.strand(r, rc)) for n, r, _, rc in anchors] + length_reads(g) + multi_reads(g) + edge_reads(g)
    write_fasta(prefix + "_se.fa", se)
    write_fastq(prefix + "_q.fq", fastq_copies(g, anchors))
    pe = paired_reads(g)
    write_fasta(prefix + "_pe_1.fa", [(n, a) for n, a, b in pe])
    write_fasta(prefix + "_pe_2.fa", [(n, b) for n, a, b in pe])
    open(prefix + "_ss.txt", "w").write("\n".join(site_lines(g)) + "\n")
    ssim, psim, lines = sim_rna.sim(sim_rna.load_fasta(reference), 20000, 10000, seed)
    sim_rna.write(prefix + "_sim", ssim, psim, lines)
    return prefix


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("reference")
    ap.add_argument("out_prefix")
    ap.add_argument("--seed", type=int, default=17)
    a = ap.parse_args()
    generate(a.reference, a.out_prefix, a.seed)


if __name__ == "__main__":
    main()
