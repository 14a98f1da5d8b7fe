"""MPCB200_OPT_CRITICAL_PLACEMENT on the GPU: the heaviest instances of a history-ordered batch on SMs of their own change only
which CTA runs which instance, so every output is bit for bit what the solve without it gives, and no instance is lost when CTAs
of a heavy SM exit without one.  Every handle solves twice, the second time with the robots moved on, so that the second solve
is ordered by the first one's iteration counts and an instance it skipped would keep the first solve's outputs."""
import numpy as np
import pytest
import torch

from mpc_local_planner_b200 import capi, configs

pytestmark = pytest.mark.gpu

OUT = ("u_seq", "x_seq", "dt", "status", "kkt_err", "iters")


def _moved(data, t):
    d = dict(data)
    d["x0"] = data["x0"] + t * (data["xf"] - data["x0"]) * np.array([1.0, 1.0, 0.0])
    return d


def _two_solves(cid, B, place, order=1, K=0):
    cfg = configs.config_for(cid, tol=1e-6)
    data = configs.generate(cid, B)
    s = capi.BatchSolver(cfg, B * max(K, 1))
    s.set_option(capi.OPT_CRITICAL_PLACEMENT, place)
    s.set_option(capi.OPT_ORDER_BY_HISTORY, order)
    outs = []
    for t in range(2):
        d = _moved(data, 0.05 * t)
        if K:
            outs.append(s.step_multistart(d["x0"], d["xf"], K, 1.0, d["u_prev"], d["u_prev_dt"], d["obstacles"], d["viapoints"]))
        else:
            outs.append(s.step(d["x0"], d["xf"], d["u_prev"], d["u_prev_dt"], d["obstacles"], d["viapoints"]))
    s.close()
    return outs


def _same(a, b, what):
    for k in OUT:
        assert np.array_equal(a[k], b[k]), f"{what}: {k} differs"
    if "winner" in a:
        assert np.array_equal(a["winner"], b["winner"]), f"{what}: winner differs"


# (cfg 3 runs two CTAs per SM: B = 512 keeps it within the two instances per CTA slot that the launch places)
@pytest.mark.parametrize("cid, B, order, K", [(2, 1024, 1, 0), (3, 512, 1, 0), (4, 1024, 1, 0), (2, 512, 1, 2), (2, 1024, 0, 0)],
                         ids=["cfg2", "cfg3", "cfg4", "multistart-K2", "index-order"])
def test_placement_does_not_change_results(cid, B, order, K):
    on, off = _two_solves(cid, B, 1, order, K), _two_solves(cid, B, 0, order, K)
    for t in range(2):
        _same(on[t], off[t], f"cfg {cid} B {B} solve {t}")


@pytest.mark.parametrize("size", ["sms+1", "2sms", "1024", "4096"])
def test_every_instance_is_solved(size):
    """(B = 4096 is above the two instances per CTA slot that the launch places: the take step of before)"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = {"sms+1": sms + 1, "2sms": 2 * sms, "1024": 1024, "4096": 4096}[size]
    on, off = _two_solves(2, B, 1), _two_solves(2, B, 0)
    for t in range(2):
        _same(on[t], off[t], f"B {B} solve {t}")
    assert (on[1]["iters"] > 0).all()
    # the second solve's outputs are its own: an instance it never took would still hold the first solve's
    assert not np.array_equal(on[1]["x_seq"], on[0]["x_seq"])
    moved = np.array([not np.array_equal(on[1]["x_seq"][i], on[0]["x_seq"][i]) for i in range(B)])
    assert moved.mean() > 0.99
