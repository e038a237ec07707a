#!/usr/bin/env python3
"""Mate orientation, N ceiling, soft-clipping, quality encoding and match bonus options against the unmodified
reference: --fr / --rf / --ff, --n-ceil, --no-softclip, --solexa-quals / --int-quals and --ma.

  python tools/scoring_options_ref.py      # writes tests/golden/scoring_options_sets.json

The expected values come from oracle/_ref/hisat2-align-s (oracle/Makefile), run with --reorder on read sets derived
from tools/refsets.py's sets (generate): both mates reverse-complemented (an RF library), mate 2 reverse-complemented
(an FF library), reads with seeded runs of N, and tests/golden's FASTQ fixtures with their qualities re-encoded as
Solexa-64 characters or as integers (requal).  The JSON keeps, per case, the md5 of the SAM without @PG (and
without the records of refsets' flagged reads), the alignment summary the reference prints, and, for the argument
errors, the first line it prints to stderr with its exit status; the routed --un-conc / --al-conc files of the
READ_FILE_CASES; and the exit status of the quality errors."""
import json
import os
import random
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import refsets  # noqa: E402

GOLDEN = refsets.GOLDEN
OUT = os.path.join(GOLDEN, "scoring_options_sets.json")
NRICH_SEED = 31
COMP = str.maketrans("ACGTNacgtn", "TGCANtgcan")


# case -> dict(src: a refsets.output_input source, xform: None | "rf" (both mates reverse-complemented) | "ff" (mate 2
#              reverse-complemented) | "nrich" (seeded N runs), flags: reference flags, opts: Index options)
def _orient(src, o, xform, *extra, **opts):
    return dict(src=src, xform=xform, flags=["--" + o] + list(extra), opts=dict(opts, pe_orient=o))


def _nceil(src, arg, t, c, l, *extra, **opts):
    return dict(src=src, xform="nrich", flags=["--n-ceil", arg] + list(extra),
                opts=dict(opts, n_ceil_type=t, n_ceil_const=c, n_ceil_coeff=l))


INT_MAX = 2 ** 31 - 1
F15 = float.fromhex("0x1.3333340000000p-3")   # (double)0.15f, the coefficient a token left out keeps
CASES = {
    "fr_pe_reads": _orient(("paired", "reads"), "fr", None),
    "rf_pe_reads_rf": _orient(("paired", "reads"), "rf", "rf"),
    "ff_pe_reads_ff": _orient(("paired", "reads"), "ff", "ff"),
    "rf_pe_reads_fr": _orient(("paired", "reads"), "rf", None),   # an FR library under --rf: no concordant pairs
    "ff_pe_reads_fr": _orient(("paired", "reads"), "ff", None),
    "fr_pe_hard20k": _orient(("paired", "hard20k"), "fr", None),
    "rf_pe_hard20k_rf": _orient(("paired", "hard20k"), "rf", "rf"),
    "ff_pe_hard20k_ff": _orient(("paired", "hard20k"), "ff", "ff"),
    "ff_pe_hard20k_ff_nomixed": _orient(("paired", "hard20k"), "ff", "ff", "--no-mixed", no_mixed=1),
    "ff_pe_hard20k_ff_nodisc": _orient(("paired", "hard20k"), "ff", "ff", "--no-discordant", no_discordant=1),
    "rf_pe_hard20k_rf_norc": _orient(("paired", "hard20k"), "rf", "rf", "--norc", norc=1),
    "rf_graph_pe_alt20k_rf": _orient(("graph_pe", "alt20k"), "rf", "rf"),
    "rf_se_reads": _orient(("se", "reads"), "rf", None),        # unpaired reads: no change
    "rf_sensitive_hard20k_rf": _orient(("paired", "hard20k"), "rf", "rf", "--sensitive", bowtie2_dp=1, score_min_type=ord("L"),
                                       score_min_const=0.0, score_min_coeff=-0.5),
    "ff_spliced_ss_sim_pe_ff": _orient(("spliced", "ss_sim_pe"), "ff", "ff"),
    "rf_spliced_ss_sim_pe_rf_strand": dict(_orient(("spliced", "ss_sim_pe"), "rf", "rf", "--rna-strandness", "RF"), out=dict(rna_strandness="RF")),
    "nceil_default_se": dict(src=("se", "reads"), xform="nrich", flags=[], opts={}),
    "nceil_default_pe": dict(src=("paired", "reads"), xform="nrich", flags=[], opts={}),
    "nceil_C_se": _nceil(("se", "reads"), "3", "C", 3.0, F15),
    "nceil_L_se": _nceil(("se", "reads"), "L,0,0.05", "L", 0.0, 0.05),
    "nceil_L2_pe": _nceil(("paired", "reads"), "L,2", "L", 2.0, F15),
    "nceil_S_pe": _nceil(("paired", "reads"), "S,1,1.5", "S", 1.0, 1.5),
    "nceil_G_pe": _nceil(("paired", "reads"), "G,-1,2.5", "G", -1.0, 2.5),
    "nceil_G_graph_se": _nceil(("graph_se", "alt20k"), "Log,0,1", "G", 0.0, 1.0),
    "nceil_zero_se": _nceil(("se", "reads"), "C,0", "C", 0.0, F15),
    "nceil_comma_se": _nceil(("se", "reads"), ",", "C", 0.0, F15),   # one empty token: C with the default constant
    "nceil_big_se": _nceil(("se", "reads"), "L,0,2", "L", 0.0, 2.0),
    "nceil_sensitive_pe": _nceil(("paired", "reads"), "L,0,0.3", "L", 0.0, 0.3, "--sensitive", bowtie2_dp=1, score_min_type=ord("L"),
                                 score_min_const=0.0, score_min_coeff=-0.5),
    "nceil_dp2_se": _nceil(("se", "reads"), "L,1,0.05", "L", 1.0, 0.05, "--bowtie2-dp", "2", bowtie2_dp=2),
    "ma_se_reads": dict(src=("se", "reads"), xform=None, flags=["--ma", "3"], opts={}),
    "ma_last_wins_se_reads": dict(src=("se", "reads"), xform=None, flags=["--ma", "3", "--ma", "0"], opts={}),
}
NOSC = dict(sp_max=INT_MAX, sp_min=INT_MAX)


def _nosc(src, *extra, **opts):
    return dict(src=src, xform=None, flags=["--no-softclip"] + list(extra), opts=dict(NOSC, **opts))


def _qual(kind, xform, *flags, **reads):
    return dict(src=("golden", kind), xform=xform, flags=list(flags), opts={}, reads=reads)


CASES.update({
    "nosc_edge_se": _nosc(("edge", "se")),
    "nosc_edge_near": _nosc(("edge", "near")),
    "nosc_edge_pe": _nosc(("edge", "pe")),
    "nosc_edge_fq": _nosc(("edge", "fq")),
    "nosc_edge_se_dp": _nosc(("edge", "se"), "--bowtie2-dp", "2", bowtie2_dp=2),
    "nosc_graph_se_alt20k": _nosc(("graph_se", "alt20k")),
    "nosc_sensitive_hard20k": _nosc(("paired", "hard20k"), "--sensitive", bowtie2_dp=1, score_min_type=ord("L"),
                                    score_min_const=0.0, score_min_coeff=-0.5),
    "nosc_then_sp_edge_se": dict(src=("edge", "se"), xform=None, flags=["--no-softclip", "--sp", "3,1"], opts=dict(sp_max=3, sp_min=3)),
    "sp_then_nosc_edge_se": dict(src=("edge", "se"), xform=None, flags=["--sp", "3,1", "--no-softclip"], opts=NOSC),
    "qual_solexa_se": _qual("se", "solexa", "--solexa-quals", solexa_quals=1),
    "qual_solexa_pe": _qual("pe", "solexa", "--solexa-quals", solexa_quals=1),
    "qual_solexa_phred64": _qual("se", "solexa", "--phred64", "--solexa-quals", phred64=1, solexa_quals=1),
    "qual_solexa_then_phred33": _qual("se", "solexa", "--solexa-quals", "--phred33"),
    "qual_int_se": _qual("se", "int", "--int-quals", int_quals=1),
    "qual_int_pe_trim": _qual("pe", "int", "--integer-quals", "-5", "3", "-3", "5", int_quals=1, trim5=3, trim3=5),
    "qual_int_phred64": _qual("se", "int", "--int-quals", "--phred64", int_quals=1, phred64=1),
    "qual_int_solexa_se": _qual("se", "int_solexa", "--int-quals", "--solexa-quals", int_quals=1, solexa_quals=1),
})
# --un-conc / --al-conc under --rf: the routing follows the concordant pairs of the orientation (recorded under "files")
READ_FILE_CASES = ("rf_pe_reads_rf", "rf_pe_reads_fr")
# argument errors: reference flags -> the first line of its stderr and its exit status (recorded under "errors")
ERRORS = {
    "nceil_four_tokens": ["--n-ceil", "L,0,0.1,4"],
    "nceil_bad_type": ["--n-ceil", "X,1"],
    "ma_two_tokens": ["--ma", "1,2"],
}
# quality errors: (fixture, re-encoding, reference flags) -> its exit status (recorded under "qual_errors")
QUAL_ERRORS = {
    "int_fewer": ("se", "int_fewer", ["--int-quals"]),
    "int_more": ("se", "int_more", ["--int-quals"]),
    "int_negative": ("se", "int_negative", ["--int-quals"]),
    "solexa_space": ("se", "solexa_space", ["--solexa-quals"]),
}
GOLDEN_FQ = {"se": ["tiny_se.fq"], "pe": ["tiny_pe_1.fq", "tiny_pe_2.fq"]}


def requal(src, dst, how, seed):
    """tests/golden/<src> with its quality lines re-encoded (binary, seeded): "solexa" as 64-based Solexa characters from
    -15 to 62 (below -10 reads as Phred 0); "int" / "int_solexa" as space-separated integers (Phred up to 120, clamped
    at 93 by the reader; Solexa from -15 to 62), some lines with a leading space (an empty first token reads as 0) or
    one value more than bases; the error re-encodings put one bad line at the 5th record."""
    rng = random.Random("%d:%s:%s" % (seed, how, src))
    lines = open(os.path.join(GOLDEN, src), "rb").read().split(b"\n")
    for i in range(3, len(lines), 4):
        n = len(lines[i - 2])
        bad = i == 4 * 4 + 3
        if how == "solexa" or (how == "solexa_space" and not bad):
            lines[i] = bytes(64 + rng.randint(-15, 62) for _ in range(n))
        elif how == "solexa_space":
            lines[i] = b"J" * (n - 1) + b" "
        else:
            lo, hi = (-15, 62) if how == "int_solexa" else (0, 120)
            v = [rng.randint(lo, hi) for _ in range(n)]
            if how == "int_fewer" and bad:
                v = v[:-1]
            elif how == "int_more" and bad:
                v += [30, 30]
            elif how == "int_negative" and bad:
                v[3] = -2
            elif rng.randrange(5) == 0:
                v.append(rng.randint(0, 40))    # one value more than bases: cut
            t = " ".join(str(x) for x in v)
            if rng.randrange(7) == 0 and not bad and v and len(v) == n + 1:
                t = " " + " ".join(str(x) for x in v[1:])   # a leading space: the empty first token is quality 0
            lines[i] = t.encode()
    with open(dst, "wb") as o:
        o.write(b"\n".join(lines))


def generate(d):
    """Every read set the CASES use, untransformed, under d; returns d."""
    refsets.generate(d, ("reads", "hard20k", "alt20k"))
    refsets.generate_spliced(d)
    refsets.generate_edge(d)
    return d


def _records(path):
    return [(r.split("\n", 1)[0], r.split("\n", 1)[1].replace("\n", "")) for r in open(path).read().split(">")[1:]]


def _write(path, recs):
    with open(path, "w") as o:
        for n, s in recs:
            o.write(">%s\n%s\n" % (n, s))


def transform(d, fs, xform):
    """The read files of a case: fs as given, or written under d by the case's transform."""
    if xform is None:
        return fs
    out = []
    for m, f in enumerate(fs):
        dst = os.path.join(d, "%s_%s" % (xform, os.path.basename(f)))
        out.append(dst)
        if os.path.exists(dst):
            continue
        rng = random.Random("%d:%s" % (NRICH_SEED, os.path.basename(f)))   # each file alike, whichever case writes it
        recs = _records(f)
        if xform == "rf" or (xform == "ff" and m == 1):
            recs = [(n, s.translate(COMP)[::-1]) for n, s in recs]
        elif xform == "nrich":   # per read: no N, a few scattered, or a run of up to 40 % of the read
            new = []
            for n, s in recs:
                k = rng.randrange(4)
                s = list(s)
                if k == 1:
                    for _ in range(rng.randint(1, 12)):
                        s[rng.randrange(len(s))] = "N"
                elif k >= 2:
                    ln = rng.randint(1, max(1, len(s) * 2 // 5))
                    st = rng.randrange(len(s) - ln + 1)
                    s[st:st + ln] = "N" * ln
                new.append((n, "".join(s)))
            recs = new
        _write(dst, recs)
    return out


def case_input(d, case):
    """(index, read files, format flag, reference flags, Index options, known-splice-site file or None) of a case
    under generate(d)."""
    c = CASES[case]
    if c["src"][0] == "golden":
        return "tiny", golden_fq(d, c["src"][1], c["xform"]), "-q", ["--no-spliced-alignment"] + c["flags"], dict(c["opts"]), None
    index, fs, fmt, base, opts, ss = refsets.output_input(d, c["src"])
    return index, transform(d, fs, c["xform"]), fmt, base + c["flags"], dict(opts, **c["opts"]), ss


def golden_fq(d, kind, how):
    """The FASTQ fixtures of kind "se" / "pe" re-encoded by requal under d."""
    out = []
    for f in GOLDEN_FQ[kind]:
        dst = os.path.join(d, "%s_%s" % (how, f))
        if not os.path.exists(dst):
            requal(f, dst, how, NRICH_SEED)
        out.append(dst)
    return out


def flagged(case):
    """The reads of a case's source that hit a fixed device capacity (refsets' `flagged`): no md5 covers their records."""
    src, fl = CASES[case]["src"], refsets.load_expected()["flagged"]
    dp = "_dp" if "--bowtie2-dp" in CASES[case]["flags"] else ""
    return fl.get("spliced/" + src[1], []) if src[0] == "spliced" else fl.get("edge/" + src[1] + dp, []) if src[0] == "edge" else []


def reference_run(d, case):
    """(SAM, stderr) of the reference on a case (--reorder)."""
    index, fs, fmt, flags, _, _ = case_input(d, case)
    out = os.path.join(d, "ref.sam")
    reads = ["-1", fs[0], "-2", fs[1]] if len(fs) == 2 else ["-U", fs[0]]
    r = subprocess.run([refsets.REFBIN, fmt, "-x", os.path.join(GOLDEN, index)] + flags + reads +
                       ["-S", out, "-p", str(min(16, os.cpu_count() or 1)), "--reorder"], check=True, stderr=subprocess.PIPE)
    return open(out, "rb").read(), r.stderr.decode()


def reference_error(d, flags):
    """(first line of the reference's stderr, exit status) for argument errors on a small input."""
    refsets.generate(d, ("reads",))
    r = subprocess.run([refsets.REFBIN, "-f", "-x", os.path.join(GOLDEN, "tiny"), "--no-spliced-alignment"] + flags +
                       ["-U", os.path.join(d, "reads_1.fa"), "-S", os.path.join(d, "err.sam")], stderr=subprocess.PIPE)
    return r.stderr.decode().splitlines()[0], r.returncode


def reference_read_files(d, case):
    """{file: md5} of the reference's --un-conc / --al-conc mates on a case, as the hisat2 wrapper routes them."""
    import readfiles_ref
    index, fs, fmt, flags, _, _ = case_input(d, case)
    r = subprocess.run([refsets.REFBIN, fmt, "-x", os.path.join(GOLDEN, index)] + flags + ["-1", fs[0], "-2", fs[1]] +
                       ["-p", str(min(16, os.cpu_count() or 1)), "--reorder", "--passthrough"],
                       check=True, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
    _, files = readfiles_ref.route(r.stdout)
    return {k: v["md5"] for k, v in readfiles_ref.summarize(files).items() if k.startswith(("un_conc", "al_conc/"))}


def reference_qual_error(d, err):
    kind, how, flags = QUAL_ERRORS[err]
    fs = golden_fq(d, kind, how)
    r = subprocess.run([refsets.REFBIN, "-q", "-x", os.path.join(GOLDEN, "tiny"), "--no-spliced-alignment"] + flags +
                       ["-U", fs[0], "-S", os.path.join(d, "err.sam")], stderr=subprocess.PIPE)
    return r.returncode


def load_expected():
    return json.load(open(OUT))


def main():
    md5, summary, warnings, errors, files, qual_errors = {}, {}, {}, {}, {}, {}
    with tempfile.TemporaryDirectory() as d:
        generate(d)
        for case in sorted(CASES):
            sam, err = reference_run(d, case)
            md5[case] = refsets.sam_md5(sam, flagged(case))
            summary[case] = refsets.summary_text(err.encode())
            warnings[case] = [l for l in err.splitlines() if l.startswith("Warning: Match bonus")]
        for name, flags in sorted(ERRORS.items()):
            errors[name] = reference_error(d, flags)
        for case in READ_FILE_CASES:
            files[case] = reference_read_files(d, case)
        for err in sorted(QUAL_ERRORS):
            qual_errors[err] = reference_qual_error(d, err)
    json.dump({"md5": md5, "summary": summary, "warnings": warnings, "errors": errors, "files": files, "qual_errors": qual_errors},
              open(OUT, "w"), indent=1, sort_keys=True)
    open(OUT, "a").write("\n")


if __name__ == "__main__":
    main()
