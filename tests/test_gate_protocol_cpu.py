"""The phase-gate protocol of the solve kernel (csrc/mpc_gate.h: arrive / join / leave of the per-SM barrier) on the CPU:
threads play the CTAs of one SM, join, arrive in and out of phase and leave at random points (tests/emu/gate_stress.cpp).
Each barrier must open only when all its members have arrived, and every run must finish within its time bound -- a deadlock
here would be a hang of the solve kernel."""
import os
import subprocess

import pytest

from tests.conftest import ROOT


@pytest.fixture(scope="module")
def gate_stress(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "emu", "gate_stress.cpp")
    exe = str(tmp_path_factory.mktemp("gate_stress") / "gate_stress")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-pthread", "-o", exe, src])
    return exe


@pytest.mark.parametrize("threads", [1, 2, 3, 4, 8, 16])
@pytest.mark.parametrize("gates", [2, 3])
@pytest.mark.parametrize("tail", [0, 1])   # after the queue drains: leave when alone / leave in any case
def test_gates_open_only_when_every_member_arrived(gate_stress, threads, gates, tail):
    for seed in range(3):
        r = subprocess.run([gate_stress, str(threads), str(gates), "2000", str(seed), str(tail)], capture_output=True, text=True,
                           timeout=60)
        assert r.returncode == 0, f"seed {seed}: status {r.returncode} (2: deadlock)\n{r.stdout}{r.stderr}"
        assert "0 errors" in r.stdout
