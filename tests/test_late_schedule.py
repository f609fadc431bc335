"""Host-side logic of the cascade parser (no GPU): the late-stage feature schedule of k_cascade.

ht_api.cu's parse_cascade re-arranges the features of every late stage into chunks of 32 records so that the 32
shared-memory addresses of each load slot fall into different banks.  The order of an exact integer sum is free, but
every feature must appear exactly once with its points and its alpha; the host-only self-test checks that.
"""
import json
import subprocess
from pathlib import Path

import pytest

from headtrackr_b200 import _lib

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "headtrackr_b200" / "csrc"


@pytest.fixture(scope="module")
def selftest(tmp_path_factory):
    exe = tmp_path_factory.mktemp("selftest") / "ht_selftest"
    subprocess.check_call([_lib.nvcc(), "-DHT_HOST_SELFTEST", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-O1", "-std=c++17", "-fmad=false", "-o", str(exe), str(CSRC / "ht_api.cu")],
                          stderr=subprocess.DEVNULL)
    out = subprocess.check_output([str(exe), str(ROOT / "headtrackr_b200" / "data" / "cascade_face.bin")], text=True)
    return json.loads(out)


def test_schedule_is_a_permutation_of_the_features(selftest):
    assert selftest["bad"] == 0
    assert selftest["n_stages"] == 16 and selftest["n_features"] == 2015
    assert selftest["fast"] == 1 and selftest["late_first"] == 8


def test_schedule_is_nearly_conflict_free(selftest):
    # 7,952 point loads of stages 8..15 in < 600 load instructions that touch shared memory, < 10 conflicts
    assert selftest["point_loads"] == 7952
    assert selftest["bank_conflicts"] == selftest["late_conflicts"] < 10
    assert selftest["load_instr_with_traffic"] < 600
