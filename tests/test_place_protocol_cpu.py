"""The critical placement of the solve kernel (csrc/mpc_place.h: admission on a per-SM word, takes from the light part and the
heavy leftovers) on the CPU: threads play the CTAs of a launch, start in random order, some on SMs without a word
(tests/emu/place_stress.cpp).  Every instance must be taken exactly once, a heavy SM must keep at most 1 + cotenants CTAs, and
every run must finish within its time bound -- a deadlock here would be a hang of the solve kernel."""
import os
import subprocess

import pytest

from tests.conftest import ROOT


@pytest.fixture(scope="module")
def place_stress(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "emu", "place_stress.cpp")
    exe = str(tmp_path_factory.mktemp("place_stress") / "place_stress")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-pthread", "-o", exe, src])
    return exe


# (SMs, CTAs per SM, SMs without a word, instances, H): a headline-like launch, more heavy instances than SMs with a word, a
# heavy part that is the whole batch, one CTA per SM, and no heavy part
SHAPES = [(16, 4, 0, 200, 6), (16, 4, 5, 64, 14), (8, 4, 0, 8, 8), (8, 1, 2, 40, 4), (8, 2, 0, 33, 0), (4, 4, 4, 20, 3)]


@pytest.mark.parametrize("shape", SHAPES, ids=["x".join(map(str, s)) for s in SHAPES])
@pytest.mark.parametrize("cotenants", [0, 1, 3])
def test_every_instance_is_taken_once_and_heavy_sms_keep_the_cap(place_stress, shape, cotenants):
    for seed in range(4):
        r = subprocess.run([place_stress, *map(str, shape), str(cotenants), str(seed)], capture_output=True, text=True, timeout=60)
        assert r.returncode == 0, f"seed {seed}: status {r.returncode} (2: deadlock)\n{r.stdout}{r.stderr}"
        assert "0 errors" in r.stdout
