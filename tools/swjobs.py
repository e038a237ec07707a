"""Seed-extension jobs for the --bowtie2-dp kernel (csrc/ht2_sw.h), on the committed tests/golden/tiny index.

A job is one call of the dp block of SplicedAligner::hybridSearch: an option set, a read (bases ACGTN, Phred+33
qualities), the strand the read is aligned on, an anchor (tidx, toff, rdoff, len) whose implied offset frames the
rectangle, minsc and the seed of the RandomSource.  `generate(seed)` is deterministic (random.Random only), and
`job_line` is the line oracle/ref_sw reads; the sha1 of those lines identifies the stream.

The jobs are drawn in classes (tags) that each aim at one place where the kernel could go wrong: read lengths
around the warp fill's 32-row blocks and the 256-base maximum, rectangles trimmed at contig ends (reads running past them included) or crossing the
N gap of chrB, indels next to the gap-barrier rows, repeats that make equal-score cells tie, N counts at the
nceil limit, minsc at the u8 / i16 switch and the -15000 refusal, anchors off the read's diagonal (the first
candidates fail) and alignments with more edits than a hit or the backtrace can hold.

usage: python tools/swjobs.py [--seed N] [--jobs out.txt] [--reference]
  --reference runs oracle/_ref/ref_sw on the jobs and writes tests/golden/sw_extend_ref.txt: the sha1 of the
  job stream on the first line, then one result line per job.
"""
import argparse
import hashlib
import os
import random
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
INDEX = os.path.join(GOLDEN, "tiny")
REF_OUT = os.path.join(GOLDEN, "sw_extend_ref.txt")
REF_SW = os.path.join(ROOT, "oracle", "_ref", "ref_sw")
SEED = 20261016

# (name, options of ht2gpu_options_t, the same as (mp_max, mp_min, ignore_quals, np, rdg_const, rdg_linear,
#  rfg_const, rfg_linear, gbar) for the job line)
OPTION_SETS = [
    ("default", {}),
    ("mp42_2", {"mp_max": 42, "mp_min": 2}),
    ("mp3_3_ignore_quals", {"mp_max": 3, "mp_min": 3, "ignore_quals": 1}),
    ("np0", {"np": 0}),
    ("np3", {"np": 3}),
    ("cheap_gaps", {"rdg_const": 1, "rdg_linear": 1, "rfg_const": 1, "rfg_linear": 1}),
    ("costly_gaps", {"rdg_const": 20, "rdg_linear": 10, "rfg_const": 20, "rfg_linear": 10}),
    ("gbar1", {"gbar": 1}),
    ("gbar64", {"gbar": 64}),
]
DEFAULTS = {"mp_max": 6, "mp_min": 2, "ignore_quals": 0, "np": 1, "rdg_const": 5, "rdg_linear": 3,
            "rfg_const": 5, "rfg_linear": 3, "gbar": 4}
SCORING_KEYS = ("mp_max", "mp_min", "ignore_quals", "np", "rdg_const", "rdg_linear", "rfg_const", "rfg_linear", "gbar")
GBAR_HALF = 8     # option set whose --gbar is at or above half of every read of up to 128 bases

LENGTHS = list(range(2, 20)) + [31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, 129, 191, 192, 193, 223, 224, 225, 255, 256]
TOO_LONG = [257, 300]    # aligned by the reference; the device's score planes stop at 256 rows (HT2_ERR_SW)

# classes that tests/test_dp_extension.py counts (each with the minimum it asserts)
CLASS_MIN = {
    "len_short": 200, "len_block": 300, "len_max": 36, "len_too_long": 10, "early": 10,
    "edge_start": 40, "edge_end": 40, "edge_overhang": 60, "edge_clamp": 20, "edge_ngap": 40,
    "indel": 150, "indel_barrier": 60, "repeat": 60, "gbar_half": 30,
    "n_at_ceil": 30, "n_over_ceil": 30, "n_window": 40,
    "minsc_254": 20, "minsc_255": 20, "minsc_opt": 30, "minsc_15000": 10, "minsc_15001": 10,
    "off_diagonal": 60, "cap_edits": 30, "qual_full": 300,
}


def scoring(opt):
    s = dict(DEFAULTS)
    s.update(OPTION_SETS[opt][1])
    return s


def load_fasta(path=os.path.join(GOLDEN, "tiny.fa")):
    seqs, name = {}, None
    for line in open(path):
        line = line.strip()
        if line.startswith(">"):
            name = line[1:].split()[0]
            seqs[name] = []
        elif name is not None:
            seqs[name].append(line.upper())
    return [(n, "".join(v)) for n, v in seqs.items()]


_COMP = {"A": "T", "C": "G", "G": "C", "T": "A", "N": "N"}


def revcomp(s):
    return "".join(_COMP[c] for c in reversed(s))


def mmpen(sc, q):
    """Scoring::mm for a Phred quality q (scoring.h): constant under --ignore-quals, else linear in min(q, 40)."""
    if sc["ignore_quals"]:
        return sc["mp_max"]
    q = min(max(q, 0), 40)
    import numpy as np
    return sc["mp_min"] + int(np.float32(np.float32(q) / np.float32(40.0)) * np.float32(sc["mp_max"] - sc["mp_min"]))


def _repeats(contigs):
    """Homopolymer runs of >= 7 and dinucleotide repeats of >= 4 units: (tidx, start, length)."""
    import re
    out = []
    for t, (_, s) in enumerate(contigs):
        for m in re.finditer(r"(A{7,}|C{7,}|G{7,}|T{7,}|((?:[ACGT]{2}))\2{3,})", s):
            out.append((t, m.start(), m.end() - m.start()))
    return out


class _Gen(object):
    def __init__(self, seed):
        self.r = random.Random(seed)
        self.contigs = load_fasta()
        self.reps = _repeats(self.contigs)
        self.jobs = []

    def base(self, not_=None):
        while True:
            c = "ACGT"[self.r.randrange(4)]
            if c != not_:
                return c

    def refbase(self, tidx, p):
        s = self.contigs[tidx][1]
        return s[p] if 0 <= p < len(s) else "N"

    def quals(self, n, mode):
        r = self.r
        if mode == "full":
            return [r.randrange(94) for _ in range(n)]
        if mode == "high":
            return [40] * n
        return [r.choice((2, 10, 20, 30, 35, 40, 41)) for _ in range(n)]

    def add(self, tags, opt, rdlen, tidx=None, pos=None, fw=None, nsub=None, indels=(), nN=0, shift=0,
            minsc=None, qmode=None, random_read=False, anchor=None, subs_at=None):
        """Build one job.  The read is the reference from `pos` with `indels` ((read row, +k inserted bases |
        -k deleted bases), ...), substitutions and Ns applied, in the orientation it aligns in (S); the read
        itself is S or its reverse complement.  The anchor is a stretch of S placed where S lies (+ shift)."""
        r = self.r
        if tidx is None:
            tidx = r.randrange(len(self.contigs))
        clen = len(self.contigs[tidx][1])
        if pos is None:
            pos = r.randrange(0, clen - rdlen - 30) if clen > rdlen + 60 else 0
        if fw is None:
            fw = r.randrange(2)
        if qmode is None:
            qmode = r.choice(("full", "high", "mixed"))
        ind = dict(indels)
        s, refpos, p = [], [], pos
        while len(s) < rdlen:
            i = len(s)
            k = ind.get(i, 0)
            if k > 0:
                for _ in range(k):
                    if len(s) < rdlen:
                        s.append(self.base()); refpos.append(p)
                ind.pop(i)
                continue
            if k < 0:
                p += -k
                ind.pop(i)
            c = self.refbase(tidx, p)
            s.append(c if c != "N" else self.base()); refpos.append(p)
            p += 1
        if random_read == "homopolymer":      # a quarter of the window matches wherever it goes: no gap pays off
            s = [self.base()] * rdlen
        elif random_read:
            s = [self.base() for _ in range(rdlen)]
        q = self.quals(rdlen, qmode)
        if nsub is None:
            nsub = r.randrange(0, max(1, rdlen // 25) + 1)
        rows = subs_at if subs_at is not None else r.sample(range(rdlen), min(nsub, rdlen))
        for i in rows:
            s[i] = self.base(not_=s[i])
        for i in r.sample(range(rdlen), min(nN, rdlen)):
            s[i] = "N"
        if anchor is None:
            rdoff = r.randrange(rdlen)
            ln = r.randrange(1, rdlen - rdoff + 1)
            if ln >= rdlen:
                ln = rdlen - 1
        else:
            rdoff, ln = anchor
        toff = max(0, refpos[rdoff] + shift)
        if minsc is None:
            minsc = r.choice((-int(0.2 * rdlen), -int(0.6 + 0.6 * rdlen), -int(1.2 * rdlen) - 10, -int(3 * rdlen) - 20))
        S = "".join(s)
        read = S if fw else revcomp(S)
        qread = q if fw else q[::-1]
        job = {"id": len(self.jobs), "opt": opt, "tags": sorted(set(tags)), "fw": fw, "tidx": tidx, "toff": toff,
               "rdoff": rdoff, "len": ln, "minsc": int(minsc), "seed": r.getrandbits(32), "read": read,
               "qual": "".join(chr(33 + x) for x in qread)}
        if rdlen <= 19:
            job["tags"].append("len_short")
        if qmode == "full":                  # Phred 0..93
            job["tags"].append("qual_full")
        self.jobs.append(job)
        return job


def generate(seed=SEED):
    g = _Gen(seed)
    r = g.r
    nopt = len(OPTION_SETS)
    clens = [len(s) for _, s in g.contigs]
    # read lengths: every length of the list under every option set, twice
    for opt in range(nopt):
        for L in LENGTHS:
            for _ in range(2):
                tags = ["len_block"] if L >= 31 else []
                if L >= 255:
                    tags.append("len_max")
                g.add(tags, opt, L)
    for opt in range(0, nopt, 2):
        for L in TOO_LONG:
            g.add(["len_too_long"], opt, L, minsc=-int(0.6 * L))
    # anchors that already span the read: no DP, the caller recurses with the anchor as it is
    for i in range(12):
        L = r.choice((40, 101, 150))
        g.add(["early"], i % nopt, L, anchor=(0, L))
    # anchors at the edges of the text
    for i in range(54):
        opt, L, t = i % nopt, r.choice((20, 33, 64, 101, 150, 224, 256)), i % 2
        g.add(["edge_start"], opt, L, tidx=t, pos=r.randrange(0, 25))
        g.add(["edge_end"], opt, L, tidx=t, pos=clens[t] - L - r.randrange(0, 25))
    # reads that run 1..5 bases past either end of a contig: the rectangle is trimmed to the contig, so the
    # alignment has to fit inside it (mismatches, or gaps outside the barrier rows)
    for i in range(36):
        opt, L, t = i % nopt, r.choice((20, 50, 101, 150)), i % 2
        g.add(["edge_overhang", "edge_end"], opt, L, tidx=t, pos=clens[t] - L + r.randrange(1, 6), minsc=-int(1.5 * L) - 10)
        g.add(["edge_overhang", "edge_start"], opt, L, tidx=t, pos=-r.randrange(1, 6), minsc=-int(1.5 * L) - 10)
    for i in range(27):
        opt, L = i % nopt, r.choice((40, 101, 150, 200))
        rdoff = r.randrange(12, L - 5)
        g.add(["edge_clamp", "edge_start"], opt, L, tidx=i % 2, pos=r.randrange(0, 6), anchor=(rdoff, r.randrange(1, L - rdoff)))
    for i in range(54):
        opt, L = i % nopt, r.choice((30, 64, 101, 150, 256))
        edge = 12000 if i % 2 == 0 else 12137
        g.add(["edge_ngap", "n_window"], opt, L, tidx=1, pos=edge - r.randrange(0, L + 15))
    # gaps: indels of 1..10 bases, some next to the gap-barrier rows
    for i in range(180):
        opt = i % nopt
        L = r.choice((33, 64, 97, 128, 150, 193, 256))
        gb = scoring(opt)["gbar"]
        k = r.randrange(1, 11) * r.choice((1, -1))
        tags = ["indel"]
        if i % 3 == 0 and 2 * gb + 4 < L:
            row = r.choice((gb - 1, gb, gb + 1, L - gb - 2, L - gb - 1, L - gb))
            row = min(max(row, 1), L - 2)
            tags.append("indel_barrier")
        else:
            row = r.randrange(1, L - 1)
        ind = [(row, k)]
        if i % 4 == 0:
            ind.append((min(L - 2, row + r.randrange(3, 30)), r.randrange(1, 4) * r.choice((1, -1))))
        g.add(tags, opt, L, indels=ind, nsub=r.randrange(0, 3))
    # repeats: the read covers a homopolymer / dinucleotide run and carries an indel inside it
    for i in range(90):
        opt = i % nopt
        t, st, ln = g.reps[r.randrange(len(g.reps))]
        L = r.choice((24, 50, 101, 150))
        pos = max(0, min(clens[t] - L - 1, st - r.randrange(2, max(3, L - ln - 2))))
        row = st - pos + r.randrange(0, ln)
        ind = [] if i % 5 == 0 else [(min(max(row, 1), L - 2), r.choice((1, 2, -1, -2)))]
        g.add(["repeat"], opt, L, tidx=t, pos=pos, indels=ind, nsub=0 if i % 2 else 1)
    # --gbar at or above half of the read
    for i in range(36):
        L = r.choice((8, 16, 33, 64, 100, 128))
        g.add(["gbar_half"], GBAR_HALF, L, indels=[(r.randrange(1, L - 1), r.choice((1, -1)))] if i % 2 else ())
    # Ns in the read: exactly floor(0.15 len) (nCeil L,0,0.15) and one more
    for i in range(80):
        opt, L = i % nopt, r.choice((7, 20, 33, 64, 101, 150, 256))
        nc = int(0.15 * L)
        over = i % 2 == 1
        g.add(["n_over_ceil" if over else "n_at_ceil"], opt, L, nN=nc + (1 if over else 0), minsc=-int(1.5 * L) - 10)
    # minsc at the u8 / i16 switch, at the optimum and one above it, at the -15000 refusal
    for i in range(27):
        opt, L = i % nopt, r.choice((101, 150, 200, 256))
        g.add(["minsc_254"], opt, L, minsc=-254, nsub=r.randrange(0, 8))
        g.add(["minsc_255"], opt, L, minsc=-255, nsub=r.randrange(0, 8))
    for i in range(45):
        opt, L = i % nopt, r.choice((20, 64, 101, 150))
        sc = scoring(opt)
        rows = r.sample(range(2, L - 2), r.randrange(1, 4))
        # the constructed alignment's score with 'high' qualities: mismatches only, rows well inside the read
        opt_score = -sum(mmpen(sc, 40) for _ in rows)
        g.add(["minsc_opt"], opt, L, subs_at=rows, qmode="high", minsc=opt_score + (i % 2))
    for i in range(12):
        opt, L = i % nopt, r.choice((64, 150, 256))
        g.add(["minsc_15000"], opt, L, minsc=-15000)
        g.add(["minsc_15001"], opt, L, minsc=-15001)
    # anchors 11..40 columns off the read's diagonal: the best cells lie off the core diagonals
    for i in range(90):
        opt, L = i % nopt, r.choice((30, 64, 101, 150, 256))
        shift = r.randrange(11, 41) * r.choice((1, -1))
        g.add(["off_diagonal"], opt, L, shift=shift, minsc=-int(r.choice((1.0, 2.0, 4.0)) * L) - 40,
              indels=[(r.randrange(1, L - 1), r.randrange(1, 8) * r.choice((1, -1)))] if i % 3 == 0 else ())
    # edit capacity: reads unrelated to the window, long enough for > 128 and > 160 edits
    for i in range(36):
        opt = (0, 6, 2, 4)[i % 4]
        L = r.choice((180, 200, 210)) if i % 2 else r.choice((240, 250, 256))
        g.add(["cap_edits"], opt, L, random_read="homopolymer" if i % 3 == 0 else True, nsub=0, minsc=r.choice((-3000, -15000)))
    return g.jobs


def job_line(job):
    sc = scoring(job["opt"])
    vals = [job["id"]] + [sc[k] for k in SCORING_KEYS] + [job["fw"], job["tidx"], job["toff"], job["rdoff"], job["len"],
                                                         job["minsc"], job["seed"], job["read"], job["qual"]]
    return " ".join(str(v) for v in vals)


def stream_sha1(jobs):
    h = hashlib.sha1()
    for j in jobs:
        h.update((job_line(j) + "\n").encode())
    return h.hexdigest()


def write_jobs(jobs, path):
    with open(path, "w") as f:
        for j in jobs:
            f.write(job_line(j) + "\n")


def run_reference(jobs, exe=REF_SW):
    """oracle/_ref/ref_sw on the jobs -> its output lines."""
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "jobs.txt")
        write_jobs(jobs, p)
        out = subprocess.run([exe, INDEX, p], check=True, stdout=subprocess.PIPE).stdout.decode()
    return out.splitlines()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seed", type=int, default=SEED)
    ap.add_argument("--jobs", help="write the job lines (the input of oracle/_ref/ref_sw) here")
    ap.add_argument("--reference", action="store_true", help="write tests/golden/sw_extend_ref.txt")
    a = ap.parse_args()
    jobs = generate(a.seed)
    if a.jobs:
        write_jobs(jobs, a.jobs)
    counts = {}
    for j in jobs:
        for t in j["tags"]:
            counts[t] = counts.get(t, 0) + 1
    print("%d jobs, sha1 %s" % (len(jobs), stream_sha1(jobs)))
    print(" ".join("%s=%d" % kv for kv in sorted(counts.items())))
    if a.reference:
        lines = run_reference(jobs)
        if len(lines) != len(jobs):
            sys.exit("ref_sw answered %d of %d jobs" % (len(lines), len(jobs)))
        with open(REF_OUT, "w") as f:
            f.write("sha1 %s jobs %d seed %d\n" % (stream_sha1(jobs), len(jobs), a.seed))
            for l in lines:
                f.write(l + "\n")
        print("wrote", REF_OUT)


if __name__ == "__main__":
    main()
