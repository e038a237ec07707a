#!/usr/bin/env python3
"""Random option / read-set parity campaign: the host build of the state machine (tests/hostsim, the same
HT2_HD code the kernels run) against the unmodified reference (oracle/_ref/hisat2-align-s) on the same
reads.  CPU only.  Every SAM difference must be confined to reads the host build flagged with a capacity
error; anything else is reported as UNEXPLAINED.

  python tools/fuzz_parity.py SEED N            # tiny fixtures (tests/golden), all options incl. presets
  python tools/fuzz_parity.py SEED N --big      # chr22 sets (oracle/_ref/data/, oracle/make_data.sh), dp-centred
  ... --spliced                                   # spliced mode (--no-temp-splicesite) instead of --no-spliced-alignment

Option spelling follows the reference's parser quirks exactly like the CLI does (hisat2_b200_main.cpp):
--sp reads both bounds from the first number, --mp re-enables quality-aware penalties under
--ignore-quals, --sensitive / --very-sensitive as hisat2.cpp:1889-1909 applies them."""
import os, random, subprocess, sys, tempfile
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")
D = os.path.join(ROOT, "oracle", "_ref", "data")
R = os.path.join(ROOT, "oracle", "_ref", "hisat2-align-s")
TMP = tempfile.mkdtemp(prefix="ht2fuzz")


def build_hostsim():
    out = os.path.join(TMP, "ht2_hostsim")
    c = os.path.join(ROOT, "hisat2_b200", "csrc")
    subprocess.run(["g++", "-O2", "-std=c++14"] + (["-DHT2_ENABLE_SPLICED"] if "--spliced" in sys.argv else []) +
                   ["-o", out, os.path.join(ROOT, "tests", "hostsim", "ht2_hostsim.cpp"),
                    os.path.join(c, "ht2_index.cpp"), os.path.join(c, "ht2_host.cpp"), "-lpthread"], check=True)
    return out


def fq_from_fa(fa, fq, seed):
    r = np.random.default_rng(seed)
    recs, name, seq = [], None, []
    for l in open(fa):
        if l.startswith(">"):
            if name is not None:
                recs.append((name, "".join(seq)))
            name, seq = l[1:].strip(), []
        else:
            seq.append(l.strip())
    recs.append((name, "".join(seq)))
    with open(fq, "wb") as f:
        for n, s in recs:
            q = r.integers(20, 41, len(s))
            for _ in range(int(r.integers(0, 3))):
                a = int(r.integers(0, max(1, len(s)))); b = min(len(s), a + int(r.integers(1, 30))); q[a:b] = r.integers(2, 12, b - a)
            f.write(b"@" + n.encode() + b"\n" + s.encode() + b"\n+\n" + bytes((q + 33).astype(np.uint8)) + b"\n")


SPLICED = "--spliced" in sys.argv   # spliced mode with --no-temp-splicesite (host build with -DHT2_ENABLE_SPLICED)


def compare(hs, index, fmt, flags, hostopts, f1, f2, threads=1):
    inp = ["-1", f1, "-2", f2] if f2 else ["-U", f1]
    rs, hsam = os.path.join(TMP, "r.sam"), os.path.join(TMP, "h.sam")
    mode = "--no-temp-splicesite" if SPLICED else "--no-spliced-alignment"
    if SPLICED:
        hostopts = list(hostopts) + ["spliced=1"]
    subprocess.run([R, mode, fmt, "-x", index, "-p", str(threads), "--reorder"] + flags + inp + ["-S", rs],
                   stderr=subprocess.DEVNULL, check=True)
    env = dict(os.environ)
    if hostopts:
        env["HT2_OPTS"] = ",".join(hostopts)
    rc = subprocess.run([hs, index, f1, hsam] + ([f2] if f2 else []), stderr=subprocess.PIPE, env=env)
    flagged = set(l.split("(")[1].split(")")[0].split("/")[0] for l in rc.stderr.decode().splitlines() if "err=" in l)
    a = [l for l in open(rs, "rb") if not l.startswith(b"@PG")]
    b = [l for l in open(hsam, "rb") if not l.startswith(b"@PG")]
    sa, sb = set(a), set(b)
    diff = set(l.split(b"\t")[0].decode() for l in a if l not in sb) | set(l.split(b"\t")[0].decode() for l in b if l not in sa)
    return flagged, diff, diff - flagged


def apply_preset(preset, ho):
    ho = [h for h in ho if not h.startswith("score_min")]
    kk = [int(h.split("=")[1]) for h in ho if h.startswith("khits")]
    if preset == "--sensitive":
        if not any(h.startswith("bowtie2_dp") for h in ho):
            ho.append("bowtie2_dp=1")
        if kk and kk[0] < 10:
            ho = [h for h in ho if not h.startswith("khits")] + ["khits=10"]
        ho.append("score_min=L:0:-0.5")
    else:
        ho = [h for h in ho if not h.startswith("bowtie2_dp")] + ["bowtie2_dp=2"]
        if not kk or kk[0] < 30:
            ho = [h for h in ho if not h.startswith("khits")] + ["khits=30"]
        ho.append("score_min=L:0:-1")
    return ho


OPTS = [("khits", [1, 2, 3, 7, 20]), ("mp", [(6, 2), (4, 2), (3, 3), (8, 1)]), ("np", [1, 2, 0]), ("rdg", [(5, 3), (3, 2), (8, 1)]),
        ("rfg", [(5, 3), (2, 2), (7, 4)]), ("sp", [(2, 2), (3, 3), (1, 1)]), ("ignore_quals", [1]), ("nofw", [1]), ("norc", [1]),
        ("secondary", [1]), ("dp", [1, 2, 2]), ("score_min", [("L", 0, -0.5), ("L", 0, -1), ("C", -30, 0), ("G", -5, -8), ("S", -3, -4), ("L", -10, -0.3)]),
        ("gbar", [1, 2, 8, 20]), ("preset", ["--sensitive", "--very-sensitive"]),
        ("no_mixed", [1]), ("no_discordant", [1]), ("frag", [(0, 300), (100, 500), (250, 260), (0, 2000)])]
if "--spliced" in sys.argv:   # options that only matter in spliced mode
    OPTS += [("pen_cansplice", [1, 3]), ("pen_noncansplice", [0, 5, 20]), ("intronlen", [(20, 2000), (50, 100000), (30, 500000)])]


def draw(rng, names, paired):
    flags, ho, preset = [], [], None
    for name, vals in names:
        if name in ("no_mixed", "no_discordant", "frag") and not paired:
            continue
        v = rng.choice(vals)
        if name == "khits": flags += ["-k", str(v)]; ho.append("khits=%d" % v)
        elif name == "mp": flags += ["--mp", "%d,%d" % v]; ho += ["mp_max=%d" % v[0], "mp_min=%d" % v[1]]
        elif name == "np": flags += ["--np", str(v)]; ho.append("np=%d" % v)
        elif name == "rdg": flags += ["--rdg", "%d,%d" % v]; ho += ["rdg_const=%d" % v[0], "rdg_linear=%d" % v[1]]
        elif name == "rfg": flags += ["--rfg", "%d,%d" % v]; ho += ["rfg_const=%d" % v[0], "rfg_linear=%d" % v[1]]
        elif name == "sp": flags += ["--sp", "%d,%d" % v]; ho += ["sp_max=%d" % v[0], "sp_min=%d" % v[0]]
        elif name == "frag": flags += ["-I", str(v[0]), "-X", str(v[1])]; ho += ["min_frag=%d" % v[0], "max_frag=%d" % v[1]]
        elif name == "dp": flags += ["--bowtie2-dp", str(v)]; ho.append("bowtie2_dp=%d" % v)
        elif name == "score_min": flags += ["--score-min", "%s,%g,%g" % v]; ho.append("score_min=%s:%g:%g" % v)
        elif name == "gbar": flags += ["--gbar", str(v)]; ho.append("gbar=%d" % v)
        elif name == "preset": flags += [v]; preset = v
        elif name == "pen_cansplice": flags += ["--pen-cansplice", str(v)]; ho.append("pen_cansplice=%d" % v)
        elif name == "pen_noncansplice": flags += ["--pen-noncansplice", str(v)]; ho.append("pen_noncansplice=%d" % v)
        elif name == "intronlen": flags += ["--min-intronlen", str(v[0]), "--max-intronlen", str(v[1])]; ho += ["min_intronlen=%d" % v[0], "max_intronlen=%d" % v[1]]
        else: flags += ["--" + name.replace("_", "-")]; ho.append(name + "=1")
    if any(h.startswith("mp_max") for h in ho):
        ho = [h for h in ho if not h.startswith("ignore_quals")]
    if preset:
        ho = apply_preset(preset, ho)
    return flags, ho


def main():
    seed, n = int(sys.argv[1]), int(sys.argv[2])
    big = "--big" in sys.argv
    rng = random.Random(seed)
    hs = build_hostsim()
    bad = 0
    tiny_sets = {"tiny": [("tiny_se.fa", None), ("tiny_pe_1.fa", "tiny_pe_2.fa"), ("tiny_rna.fa", None)],
                 "tiny_snp": [("tiny_alt_1.fa", None), ("tiny_alt_1.fa", "tiny_alt_2.fa"), ("tiny_se.fa", None)]}
    big_sets = [("22_20-21M", "hard20k_1.fa", None), ("22_20-21M", "hard20k_1.fa", "hard20k_2.fa"), ("22_20-21M", "len150_1.fa", None),
                ("22_20-21M", "len36_1.fa", "len36_2.fa"), ("22_20-21M_snp", "alt20k_1.fa", "alt20k_2.fa"),
                ("22_20-21M_snp", "hard20k_1.fa", None), ("22_20-21M", "len250_1.fa", None)]
    for it in range(n):
        if big:
            idx, f1, f2 = rng.choice(big_sets)
            index, fmt = os.path.join(D, idx), "-f"
            a1, a2 = os.path.join(D, f1), os.path.join(D, f2) if f2 else None
            names = [o for o in OPTS if o[0] in ("dp", "score_min", "gbar", "rdg", "rfg", "mp", "khits", "secondary") and rng.random() < 0.5]
            if not any(o[0] == "dp" for o in names):
                names.append(OPTS[10])
        else:
            idx = rng.choice(list(tiny_sets)); f1, f2 = rng.choice(tiny_sets[idx])
            index = os.path.join(G, idx)
            a1, a2 = os.path.join(G, f1), os.path.join(G, f2) if f2 else None
            fmt = "-f"
            if rng.random() < 0.5:
                fmt = "-q"
                q1 = os.path.join(TMP, "a1.fq"); fq_from_fa(a1, q1, it * 2 + 1); a1 = q1
                if a2:
                    q2 = os.path.join(TMP, "a2.fq"); fq_from_fa(a2, q2, it * 2 + 2); a2 = q2
            names = rng.sample(OPTS, rng.randint(0, 4))
        flags, ho = draw(rng, names, a2 is not None)
        flagged, diff, unexplained = compare(hs, index, fmt, flags, ho, a1, a2, threads=6 if big else 1)
        print(it, idx, f1, "PE" if a2 else "SE", fmt, " ".join(flags), "flagged=%d diffreads=%d UNEXPLAINED=%d" % (len(flagged), len(diff), len(unexplained)), flush=True)
        if unexplained:
            bad += 1
            print("   e.g.", sorted(unexplained)[:5])
    print("bad", bad)
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
