#!/usr/bin/env python3
"""Regenerate the committed golden fixtures with the UNMODIFIED reference
(oracle/_ref, built by oracle/Makefile from /root/reference).

  tiny.fa            two small references cut from the example region
                     (chrA with a mutated duplicate -> multi-mappers, chrB with
                     an N gap -> several rstarts fragments)
  tiny.{1..8}.ht2    hisat2-build-s --ftabchars 7 tiny.fa tiny   (linear index)
  tiny_se.fa         700 single-end reads: clean, 2% substitutions, indels, Ns,
                     ragged lengths, a few unalignable
  tiny_se.sam        hisat2-align-s --no-spliced-alignment -f -x tiny -U tiny_se.fa
  tiny_pe_{1,2}.fa / tiny_pe.sam   300 pairs, same flags with -1/-2
  tiny_dump.txt      oracle/_ref/ref_dump tiny tiny_se.fa 1   (kernel-level vectors)
  tiny.snp           seeded SNP list (single / deletion / insertion) over tiny.fa
  tiny_snp.{1..8}.ht2  hisat2-build-s --ftabchars 7 --snp tiny.snp tiny.fa tiny_snp  (GRAPH index)
  tiny_snp_dump.txt  ref_dump on the graph index: H/C lines plus G lines (node range, in-edge list)
  tiny_snp_{se,pe,se_fq}.sam  hisat2-align-s --no-spliced-alignment -x tiny_snp on the tiny read sets (Zs:Z tags)
Run from the repo root:  python tests/golden/make_golden.py
"""
import os, subprocess, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import simreads
G = os.path.join(ROOT, "tests", "golden")
REF = os.path.join(ROOT, "oracle", "_ref")

def main():
    _, seq = simreads.load_fasta_codes(os.path.join(ROOT, "oracle", "_ref", "data", "22_20-21M.fa"))
    rng = np.random.default_rng(11)
    def mutate(a, rate):
        a = a.copy()
        m = rng.random(len(a)) < rate
        a[m] = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, m.sum())]
        return a
    s1 = seq[100000:125000]; s2 = seq[300000:315000]
    chrA = np.concatenate([s1, s2, mutate(s1[5000:15000], 0.01)])
    s3 = seq[700000:712000]; s4 = seq[820000:838000]
    chrB = np.concatenate([s3, np.full(137, ord("N"), np.uint8), s4])
    with open(os.path.join(G, "tiny.fa"), "wb") as f:
        for name, s in (("chrA test contig", chrA), ("chrB", chrB)):
            f.write(b">" + name.encode() + b"\n")
            for i in range(0, len(s), 60):
                f.write(s[i:i + 60].tobytes() + b"\n")
    subprocess.run([os.path.join(REF, "hisat2-build-s"), "-q", "--ftabchars", "7", "tiny.fa", "tiny"], check=True, cwd=G,
                   stdout=subprocess.DEVNULL)
    # reads: sample from the concatenation of both contigs (N-containing fragments are skipped by simulate)
    cat = np.concatenate([chrA, np.full(500, ord("N"), np.uint8), chrB])
    a1, _ = simreads.simulate(cat, 250, seed=21, fmin=120, fmax=300, sub=0.0)
    b1, _ = simreads.simulate(cat, 250, seed=22, fmin=120, fmax=300, sub=0.02)
    c1, _ = simreads.simulate(cat, 180, seed=23, fmin=120, fmax=300, sub=0.01)
    rnd = rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), (20, 101))
    se = [r.tobytes() for r in a1] + [r.tobytes() for r in b1] + \
        simreads.add_noise(c1, 5, indel=0.006, nrate=0.004, ragged=True) + [r.tobytes() for r in rnd]
    simreads.write_fasta_list(os.path.join(G, "tiny_se.fa"), se, prefix="s")
    p1, p2 = simreads.simulate(cat, 300, seed=31, fmin=150, fmax=400, sub=0.01)
    q1 = simreads.add_noise(p1, 6, indel=0.002, nrate=0.001)
    q2 = simreads.add_noise(p2, 7, indel=0.002, nrate=0.001)
    simreads.write_fasta_list(os.path.join(G, "tiny_pe_1.fa"), q1, prefix="p")
    simreads.write_fasta_list(os.path.join(G, "tiny_pe_2.fa"), q2, prefix="p")
    al = os.path.join(REF, "hisat2-align-s")
    def sam(args, out):
        subprocess.run([al, "--no-spliced-alignment", "-f", "-x", "tiny"] + args + ["-S", out + ".tmp"], check=True, cwd=G,
                       stderr=subprocess.DEVNULL)
        with open(os.path.join(G, out + ".tmp")) as fi, open(os.path.join(G, out), "w") as fo:
            fo.writelines(l for l in fi if not l.startswith("@PG"))
        os.remove(os.path.join(G, out + ".tmp"))
    sam(["-U", "tiny_se.fa"], "tiny_se.sam")
    sam(["-1", "tiny_pe_1.fa", "-2", "tiny_pe_2.fa"], "tiny_pe.sam")
    # kernel-level vectors: reads 0..99 (clean), 250..349 (2% subs), 500..599 (indels/Ns/ragged)
    keep = set(list(range(0, 100)) + list(range(250, 350)) + list(range(500, 600)))
    for mode, name in (("1", "tiny_dump.txt"), ("0", "tiny_dump_spliced.txt")):
        out = subprocess.run([os.path.join(REF, "ref_dump"), "tiny", "tiny_se.fa", mode], check=True, cwd=G,
                             stdout=subprocess.PIPE).stdout.decode().splitlines(True)
        with open(os.path.join(G, name), "w") as fo:
            fo.writelines(l for l in out if int(l.split()[1]) in keep)

def graph():
    """Graph (SNP) fixture: SNPs every ~150 bp; the dump reads carry alt alleles in half of the cases."""
    names, seqs = [], []
    cur = None
    for l in open(os.path.join(G, "tiny.fa")):
        if l.startswith(">"):
            names.append(l[1:].split()[0]); seqs.append([])
        else:
            seqs[-1].append(l.strip())
    seqs = ["".join(x) for x in seqs]
    rng = np.random.default_rng(77)
    lines = []
    k = 0
    for name, sq in zip(names, seqs):
        pos = 60
        while pos + 40 < len(sq):
            window = sq[pos - 5:pos + 12]
            if "N" not in window:
                t = rng.random()
                if t < 0.75:
                    alt = "ACGT"[(("ACGT".index(sq[pos])) + int(rng.integers(1, 4))) % 4]
                    lines.append("ts%d\tsingle\t%s\t%d\t%s" % (k, name, pos, alt))
                elif t < 0.88:
                    lines.append("ts%d\tdeletion\t%s\t%d\t%d" % (k, name, pos, int(rng.integers(1, 4))))
                else:
                    ins = "".join("ACGT"[int(x)] for x in rng.integers(0, 4, int(rng.integers(1, 4))))
                    lines.append("ts%d\tinsertion\t%s\t%d\t%s" % (k, name, pos, ins))
                k += 1
            pos += int(rng.integers(90, 220))
    open(os.path.join(G, "tiny.snp"), "w").write("\n".join(lines) + "\n")
    subprocess.run([os.path.join(REF, "hisat2-build-s"), "-q", "--ftabchars", "7", "--snp", "tiny.snp", "tiny.fa", "tiny_snp"],
                   check=True, cwd=G, stdout=subprocess.DEVNULL)
    keep = set(list(range(0, 100)) + list(range(250, 350)) + list(range(500, 600)))
    out = subprocess.run([os.path.join(REF, "ref_dump"), "tiny_snp", "tiny_se.fa", "1"], check=True, cwd=G,
                         stdout=subprocess.PIPE).stdout.decode().splitlines(True)
    with open(os.path.join(G, "tiny_snp_dump.txt"), "w") as fo:
        fo.writelines(l for l in out if int(l.split()[1]) in keep)
    graph_sams()


def graph_sams():
    """full-path goldens on the graph index (ALT-aware extension, Zs:Z)"""
    al = os.path.join(REF, "hisat2-align-s")
    # tiny_alt_{1,2}.fa: reads sampled from the reference with half of the ALTs applied (tools/altreads.py --seed 4)
    subprocess.run([sys.executable, os.path.join(ROOT, "tools", "altreads.py"), os.path.join(G, "tiny.fa"), os.path.join(G, "tiny.snp"),
                    "400", os.path.join(G, "tiny_alt"), "--seed", "4", "--paired"], check=True)
    for args, outname in ((["-f", "-U", "tiny_se.fa"], "tiny_snp_se.sam"), (["-f", "-1", "tiny_pe_1.fa", "-2", "tiny_pe_2.fa"], "tiny_snp_pe.sam"),
                          (["-q", "-U", "tiny_se.fq"], "tiny_snp_se_fq.sam"), (["-f", "-U", "tiny_alt_1.fa"], "tiny_snp_alt_se.sam"),
                          (["-f", "-1", "tiny_alt_1.fa", "-2", "tiny_alt_2.fa"], "tiny_snp_alt_pe.sam")):
        subprocess.run([al, "--no-spliced-alignment", "-x", "tiny_snp"] + args + ["-S", outname + ".tmp"], check=True, cwd=G,
                       stderr=subprocess.DEVNULL)
        with open(os.path.join(G, outname + ".tmp")) as fi, open(os.path.join(G, outname), "w") as fo:
            fo.writelines(l for l in fi if not l.startswith("@PG"))
        os.remove(os.path.join(G, outname + ".tmp"))


def fastq():
    """FASTQ fixture: the first 400 single-end reads and 150 pairs with seeded Phred+33 qualities
    (bimodal: mostly 30-40, stretches of 2-15) so that quality-aware mismatch / soft-clip penalties matter."""
    rng = np.random.default_rng(99)
    def quals(n):
        q = rng.integers(28, 41, n)
        for _ in range(int(rng.integers(0, 4))):
            a = int(rng.integers(0, n)); b = min(n, a + int(rng.integers(1, 25)))
            q[a:b] = rng.integers(2, 16, b - a)
        return bytes((q + 33).astype(np.uint8))
    def conv(fa, fq, limit):
        recs, name, seq = [], None, []
        for l in open(os.path.join(G, fa)):
            if l.startswith(">"):
                if name is not None: recs.append((name, "".join(seq)))
                name, seq = l[1:].strip(), []
            else: seq.append(l.strip())
        recs.append((name, "".join(seq)))
        with open(os.path.join(G, fq), "wb") as f:
            for name, sq in recs[:limit]:
                f.write(b"@" + name.encode() + b"\n" + sq.encode() + b"\n+\n" + quals(len(sq)) + b"\n")
    conv("tiny_se.fa", "tiny_se.fq", 400)
    conv("tiny_pe_1.fa", "tiny_pe_1.fq", 150)
    conv("tiny_pe_2.fa", "tiny_pe_2.fq", 150)
    al = os.path.join(REF, "hisat2-align-s")
    def sam(args, out):
        subprocess.run([al, "--no-spliced-alignment", "-q", "-x", "tiny"] + args + ["-S", out + ".tmp"], check=True, cwd=G,
                       stderr=subprocess.DEVNULL)
        with open(os.path.join(G, out + ".tmp")) as fi, open(os.path.join(G, out), "w") as fo:
            fo.writelines(l for l in fi if not l.startswith("@PG"))
        os.remove(os.path.join(G, out + ".tmp"))
    sam(["-U", "tiny_se.fq"], "tiny_se_fq.sam")
    sam(["-1", "tiny_pe_1.fq", "-2", "tiny_pe_2.fq"], "tiny_pe_fq.sam")


OPTION_CASES = [
    # (ht2gpu_options_t fields, reference command-line flags, paired)
    ("khits=1", ["-k", "1"], False),
    ("khits=12", ["-k", "12"], False),
    ("mp_max=4,mp_min=2,np=2", ["--mp", "4,2", "--np", "2"], False),
    ("rdg_const=3,rdg_linear=2,rfg_const=4,rfg_linear=2", ["--rdg", "3,2", "--rfg", "4,2"], False),
    # the reference reads BOTH soft-clip bounds from the first number (aligner_seed_policy.cpp:438-441)
    ("sp_max=3,sp_min=3", ["--sp", "3,1"], False),
    ("ignore_quals=1", ["--ignore-quals"], False),
    ("nofw=1", ["--nofw"], False),
    ("norc=1", ["--norc"], False),
    ("secondary=1", ["--secondary"], False),
    ("no_mixed=1", ["--no-mixed"], True),
    ("no_discordant=1", ["--no-discordant"], True),
    ("min_frag=150,max_frag=320", ["-I", "150", "-X", "320"], True),
    ("nofw=1", ["--nofw"], True),
    ("khits=3", ["-k", "3"], True),
    # "--mp a,b" becomes MMP=Q,a,b, which switches back to quality-aware penalties even under
    # --ignore-quals (aligner_seed_policy.cpp:396-418); the CLI clears ignore_quals when --mp is given
    ("mp_max=4,mp_min=2", ["--mp", "4,2", "--ignore-quals"], False),
    # --score-min and the --bowtie2-dp seed extension (spliced_aligner.h:209-297); the presets are spelled
    # out the way hisat2.cpp:1892-1909 applies them (an omitted -k stays the index default under --sensitive)
    ("score_min_type=71,score_min_const=-5,score_min_coeff=-8", ["--score-min", "G,-5,-8"], False),
    ("bowtie2_dp=2", ["--bowtie2-dp", "2"], False),
    ("bowtie2_dp=1,score_min_type=76,score_min_const=0,score_min_coeff=-0.5", ["--sensitive"], False),
    ("bowtie2_dp=2,khits=30,score_min_type=76,score_min_const=0,score_min_coeff=-1", ["--very-sensitive"], True),
    ("bowtie2_dp=2,gbar=10,score_min_type=76,score_min_const=0,score_min_coeff=-0.6,rdg_const=4,rdg_linear=2",
     ["--bowtie2-dp", "2", "--gbar", "10", "--score-min", "L,0,-0.6", "--rdg", "4,2"], True),
    ("bowtie2_dp=1,khits=10,score_min_type=76,score_min_const=0,score_min_coeff=-0.5", ["--sensitive", "-k", "4"], True),
    # graph index, reads carrying ALT alleles (FASTA)
    ("bowtie2_dp=2,khits=30,score_min_type=76,score_min_const=0,score_min_coeff=-1", ["--very-sensitive"], False, "snp"),
    ("bowtie2_dp=2", ["--bowtie2-dp", "2"], True, "snp"),
]
OPTION_SETS = {   # name -> (index, format flag, SE file, PE files)
    "tiny": ("tiny", "-q", "tiny_se.fq", ("tiny_pe_1.fq", "tiny_pe_2.fq")),
    "snp": ("tiny_snp", "-f", "tiny_alt_1.fa", ("tiny_alt_1.fa", "tiny_alt_2.fa")),
}


def spliced():
    """Spliced mode (the reference's default) with --no-temp-splicesite, i.e. with an empty splice-site DB
    (hisat2.cpp:4092-4093): order-independent, the parity target of SURVEY 8(e).  Golden SAM for the tiny
    fixtures; the chr22-scale sets are compared against the reference run in place (tools/fuzz_parity.py)."""
    al = os.path.join(REF, "hisat2-align-s")
    # RNA-like reads: 101 bases over one or two GT..AG (or, one in five, arbitrary) "introns" of tiny.fa, 0.5 % substitutions
    import random
    rng = random.Random(11)
    refs, name = {}, None
    for l in open(os.path.join(G, "tiny.fa")):
        if l.startswith(">"):
            name = l[1:].split()[0]; refs[name] = []
        else:
            refs[name].append(l.strip().upper())
    refs = {k: "".join(v) for k, v in refs.items()}
    comp = {"A": "T", "C": "G", "G": "C", "T": "A", "N": "N"}
    recs = []
    while len(recs) < 400:
        chrom = rng.choice(list(refs)); seq = refs[chrom]
        nint = rng.choice([1, 1, 1, 2]); pos = rng.randrange(0, len(seq) - 12000); parts = []; left = 101; ok = True
        for k in range(nint + 1):
            ln = left if k == nint else rng.randrange(12, left - 12 * (nint - k))
            parts.append(seq[pos:pos + ln]); left -= ln; pos += ln
            if k < nint:
                if rng.random() < 0.8:
                    g = seq.find("GT", pos, pos + 1)
                    if g != pos:
                        ok = False; break
                    e = -1
                    for _ in range(50):
                        cand = pos + rng.randrange(60, 4000)
                        a = seq.find("AG", cand, cand + 200)
                        if a > 0:
                            e = a + 2; break
                    if e < 0:
                        ok = False; break
                    pos = e
                else:
                    pos += rng.randrange(30, 3000)
        rd = "".join(parts)
        if not ok or len(rd) != 101 or "N" in rd:
            continue
        rd = "".join(rng.choice("ACGT".replace(c, "")) if rng.random() < 0.005 else c for c in rd)
        if rng.random() < 0.5:
            rd = "".join(comp[c] for c in reversed(rd))
        recs.append(rd)
    with open(os.path.join(G, "tiny_rna.fa"), "w") as f:
        for i, r in enumerate(recs):
            f.write(">t%d\n%s\n" % (i, r))
    for idx, fmt, args, out in (("tiny", "-f", ["-U", "tiny_rna.fa"], "tiny_spliced_rna.sam"),
                                ("tiny", "-f", ["-U", "tiny_se.fa"], "tiny_spliced_se.sam"),
                                ("tiny", "-q", ["-1", "tiny_pe_1.fq", "-2", "tiny_pe_2.fq"], "tiny_spliced_pe_fq.sam"),
                                ("tiny_snp", "-f", ["-1", "tiny_alt_1.fa", "-2", "tiny_alt_2.fa"], "tiny_snp_spliced_alt_pe.sam")):
        subprocess.run([al, "--no-temp-splicesite", fmt, "-x", idx] + args + ["-S", "spl.tmp"], check=True, cwd=G, stderr=subprocess.DEVNULL)
        data = b"".join(l for l in open(os.path.join(G, "spl.tmp"), "rb") if not l.startswith(b"@PG"))
        open(os.path.join(G, out), "wb").write(data)
        print(out, data.count(b"\n"), "records,", sum(1 for l in data.splitlines() if not l.startswith(b"@") and b"N" in l.split(b"\t")[5]), "spliced")
    os.remove(os.path.join(G, "spl.tmp"))


def known_splice():
    """Spliced mode with a POPULATED, read-only splice-site DB: --no-temp-splicesite --known-splicesite-infile (and
    --novel-splicesite-infile).  Reads and sites from tools/sim_rna.py (seed 23): 600 single-end reads, many with only
    1-11 bases beyond a junction, 300 pairs with mates in different exons, 1104 site lines (85 % of the introns used,
    decoys, duplicates, an unknown sequence name)."""
    import sim_rna
    al = os.path.join(REF, "hisat2-align-s")
    refs = sim_rna.load_fasta(os.path.join(G, "tiny.fa"))
    se, pairs, lines = sim_rna.sim(refs, 600, 300, 23)
    sim_rna.write(os.path.join(G, "tiny_ss_rna"), se, pairs, lines)
    ss = open(os.path.join(G, "tiny_ss_rna_ss.txt")).read().splitlines()
    open(os.path.join(G, "tiny_ss_known.txt"), "w").write("\n".join(ss[:300]) + "\n")
    open(os.path.join(G, "tiny_ss_novel.txt"), "w").write("\n".join(ss[250:]) + "\n")
    K = ["--no-temp-splicesite", "--known-splicesite-infile", "tiny_ss_rna_ss.txt"]
    for idx, flags, args, out in (("tiny", K, ["-U", "tiny_ss_rna.fa"], "tiny_ss_rna_se.sam"),
                                  ("tiny", K, ["-1", "tiny_ss_rna_1.fa", "-2", "tiny_ss_rna_2.fa"], "tiny_ss_rna_pe.sam"),
                                  ("tiny_snp", K, ["-1", "tiny_ss_rna_1.fa", "-2", "tiny_ss_rna_2.fa"], "tiny_snp_ss_rna_pe.sam"),
                                  ("tiny", K + ["-k", "20", "--secondary"], ["-U", "tiny_ss_rna.fa"], "tiny_ss_rna_se_k20_secondary.sam"),
                                  ("tiny", ["--no-temp-splicesite", "--known-splicesite-infile", "tiny_ss_known.txt", "--novel-splicesite-infile", "tiny_ss_novel.txt"],
                                   ["-1", "tiny_ss_rna_1.fa", "-2", "tiny_ss_rna_2.fa"], "tiny_ss_rna_pe_known_novel.sam")):
        subprocess.run([al, "-f", "-x", idx] + flags + args + ["-S", "ss.tmp"], check=True, cwd=G, stderr=subprocess.DEVNULL)
        data = b"".join(l for l in open(os.path.join(G, "ss.tmp"), "rb") if not l.startswith(b"@PG"))
        open(os.path.join(G, out), "wb").write(data)
        print(out, data.count(b"\n"), "records,", sum(1 for l in data.splitlines() if not l.startswith(b"@") and b"N" in l.split(b"\t")[5]), "spliced")
    os.remove(os.path.join(G, "ss.tmp"))
    # --novel-splicesite-outfile (first pass of the two-pass use; no DB loaded, so the SAM is that of --no-temp-splicesite)
    for args, out in ((["-1", "tiny_ss_rna_1.fa", "-2", "tiny_ss_rna_2.fa"], "tiny_ss_rna_pe_novel_out.txt"), (["-U", "tiny_rna.fa"], "tiny_rna_novel_out.txt")):
        subprocess.run([al, "-f", "-x", "tiny", "--no-temp-splicesite", "--novel-splicesite-outfile", out] + args + ["-S", "/dev/null"], check=True, cwd=G,
                       stderr=subprocess.DEVNULL)
        print(out, sum(1 for _ in open(os.path.join(G, out))), "sites")
    # read-count cutoffs of SpliceSiteDB::print: tiny_rna.fa plus a renamed copy of its first 200 reads
    lines = open(os.path.join(G, "tiny_rna.fa")).read().splitlines(True)
    open(os.path.join(G, "dup.tmp.fa"), "w").write("".join(lines) + "".join(l.replace(">t", ">dup", 1) if l.startswith(">") else l for l in lines[:400]))
    subprocess.run([al, "-f", "-x", "tiny", "--no-temp-splicesite", "--novel-splicesite-outfile", "tiny_rna_dup_novel_out.txt", "-U", "dup.tmp.fa", "-S", "/dev/null"],
                   check=True, cwd=G, stderr=subprocess.DEVNULL)
    os.remove(os.path.join(G, "dup.tmp.fa"))


def options():
    """md5 of the reference's SAM (minus @PG) for every option case -> option_matrix.json."""
    import hashlib, json
    al = os.path.join(REF, "hisat2-align-s")
    out = []
    for case in OPTION_CASES:
        opts, flags, paired = case[:3]
        setname = case[3] if len(case) > 3 else "tiny"
        index, fmt, se, pe = OPTION_SETS[setname]
        inp = ["-1", pe[0], "-2", pe[1]] if paired else ["-U", se]
        subprocess.run([al, "--no-spliced-alignment", fmt, "-x", index] + flags + inp + ["-S", "opt.tmp"], check=True, cwd=G,
                       stderr=subprocess.DEVNULL)
        data = b"".join(l for l in open(os.path.join(G, "opt.tmp"), "rb") if not l.startswith(b"@PG"))
        out.append({"options": opts, "flags": flags, "paired": paired, "md5": hashlib.md5(data).hexdigest(),
                    "records": data.count(b"\n"), "index": index, "format": fmt, "reads": list(pe) if paired else [se]})
    os.remove(os.path.join(G, "opt.tmp"))
    json.dump(out, open(os.path.join(G, "option_matrix.json"), "w"), indent=1)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "spliced":
        spliced()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "known_splice":
        known_splice()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "options":
        options()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "fastq":
        fastq()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "graph_sams":
        graph_sams()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "graph":
        graph()
        sys.exit(0)
    main()
