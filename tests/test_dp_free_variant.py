"""The aligner compiled without the --bowtie2-dp extension against the one that reads the option (CPU,
tests/hostsim/ht2_nodpsim.cpp).

The pool kernel of a DNA-only run on a linear index is built twice: Ht2AlignerT<.., .., DP = false> when the handle's
--bowtie2-dp mode is 0, DP = true otherwise (ht2_gpu.cu launchAlign).  With the option off the two must hand on the
same alignments, edits, pairs, RNG state and work counters for every read; with it on, only the DP = true side may
enter the extension (the DP-free kernel is never launched then, and must not be able to run it by accident).

On the device both sides are covered by the GPU suites that compare SAM with the reference byte for byte with and
without --bowtie2-dp.
"""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def nodpsim(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("nodpsim") / "ht2_nodpsim")
    c = os.path.join(ROOT, "hisat2_b200", "csrc")
    subprocess.run(["g++", "-O2", "-std=c++14", "-o", exe, os.path.join(ROOT, "tests", "hostsim", "ht2_nodpsim.cpp"),
                    os.path.join(c, "ht2_index.cpp"), os.path.join(c, "ht2_host.cpp"), "-lpthread"], check=True)
    return exe


def run(nodpsim, mode):
    r = subprocess.run([nodpsim, os.path.join(GOLDEN, "tiny"), os.path.join(GOLDEN, "tiny_pe_1.fq"),
                        os.path.join(GOLDEN, "tiny_pe_2.fq"), str(mode)], stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    assert r.returncode == 0, r.stderr.decode()[-4000:]
    return tuple(map(int, r.stdout.split()))


def test_dp_free_aligner_equals_dp_aligner_with_the_option_off(nodpsim):
    pairs, differ, alns, ran_dp = run(nodpsim, 0)
    assert pairs >= 100 and alns > pairs      # the fixture aligns: most pairs report both mates
    assert differ == 0
    assert ran_dp == 0


@pytest.mark.parametrize("mode", [1, 2])
def test_only_the_dp_aligner_enters_the_extension(nodpsim, mode):
    # the helper exits 1 when the DP-free aligner touches the DP scratch
    pairs, differ, alns, ran_dp = run(nodpsim, mode)
    assert pairs >= 100
    assert ran_dp > 0
