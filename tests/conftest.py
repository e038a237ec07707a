import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")
REFDIR = os.path.join(ROOT, "oracle", "_ref")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def lib():
    """The built CUDA library (compiled here with nvcc if missing)."""
    from hisat2_b200 import build, api
    build.build_lib()
    return api.load_library()


@pytest.fixture(scope="session")
def oracle_bin(tmp_path_factory):
    """oracle/ht2_oracle.c compiled as a command-line tool."""
    out = str(tmp_path_factory.mktemp("oracle") / "ht2_oracle")
    subprocess.run(["gcc", "-O2", "-std=gnu99", "-DHT2_ORACLE_MAIN", "-o", out,
                    os.path.join(ROOT, "oracle", "ht2_oracle.c")], check=True)
    return out


@pytest.fixture(scope="session")
def hostsim_bin(tmp_path_factory):
    """TEST-ONLY host build of the state machine (tests/hostsim)."""
    out = str(tmp_path_factory.mktemp("hostsim") / "ht2_hostsim")
    c = os.path.join(ROOT, "hisat2_b200", "csrc")
    subprocess.run(["g++", "-O2", "-std=c++14", "-o", out, os.path.join(ROOT, "tests", "hostsim", "ht2_hostsim.cpp"),
                    os.path.join(c, "ht2_index.cpp"), os.path.join(c, "ht2_host.cpp")], check=True)
    return out


@pytest.fixture(scope="session")
def hostsim_spliced_bin(tmp_path_factory):
    """TEST-ONLY host build with -DHT2_ENABLE_SPLICED: the spliced-alignment pieces (splice edits, the spliced
    branch of combineWith, splice scoring, N/XS:A in SAM) that are not in the CUDA library yet (DESIGN.md 8.2)."""
    out = str(tmp_path_factory.mktemp("hostsim_spl") / "ht2_hostsim_spliced")
    c = os.path.join(ROOT, "hisat2_b200", "csrc")
    subprocess.run(["g++", "-O2", "-std=c++14", "-DHT2_ENABLE_SPLICED", "-o", out, os.path.join(ROOT, "tests", "hostsim", "ht2_hostsim.cpp"),
                    os.path.join(c, "ht2_index.cpp"), os.path.join(c, "ht2_host.cpp"), "-lpthread"], check=True)
    return out


def sam_lines(data):
    if isinstance(data, str):
        data = data.encode()
    return [l for l in data.splitlines() if not l.startswith(b"@PG")]
