"""The device-memory entry points (mpcb200_*_async) on a box without a GPU: declared, exported, bound, and argument errors
without a handle."""
import ctypes as C
import os
import re

import pytest

from mpc_local_planner_b200 import capi
from tests.conftest import ROOT

ASYNC = ["mpcb200_step_batch_async", "mpcb200_step_batch_costmap_async", "mpcb200_check_feasible_async"]


def test_async_symbols_declared_exported_and_bound(cuda_lib):
    hdr = open(os.path.join(ROOT, "include", "mpcb200.h")).read()
    declared = set(re.findall(r"\b(mpcb200_[a-z0-9_]+)\s*\(", hdr))
    assert re.search(r"#define\s+MPCB200_ASYNC_LINE_OBSTACLES\s+1u", hdr)
    assert capi.ASYNC_LINE_OBSTACLES == 1
    for sym in ASYNC:
        assert sym in declared, sym
        assert sym in capi.EXPORTS, sym
        assert getattr(cuda_lib, sym).argtypes, f"{sym} has no ctypes signature"


def test_null_handle_is_invalid(cuda_lib):
    d = C.c_void_p(0)
    assert cuda_lib.mpcb200_step_batch_async(None, 1, None, None, None, 0.0, None, None, None, None, 0,
                                             None, None, None, None, None, None) == capi.E_INVALID
    m = capi.Costmaps(4, 4, 0.1, None, None)
    assert cuda_lib.mpcb200_step_batch_costmap_async(None, 1, None, None, None, 0.0, C.byref(m), 0.3, 16, None, None, None,
                                                     None, None, None, None, None, None, None) == capi.E_INVALID
    assert cuda_lib.mpcb200_check_feasible_async(None, 1, C.byref(m), d, 3, None, 0, 0.2, 0.0, 0.1, -1, d) == capi.E_INVALID


def test_tensor_checks_come_before_the_call():
    """the wrapper's checks of the tensors it is given need no device: a wrong type, dtype or device is a ValueError"""
    torch = pytest.importorskip("torch")
    import numpy as np
    with pytest.raises(ValueError, match="torch CUDA tensor"):
        capi._tensor_ptr(np.zeros((2, 3)), "x0", torch.float64, 0, (2, 3))
    with pytest.raises(ValueError, match="cuda:0"):
        capi._tensor_ptr(torch.zeros((2, 3), dtype=torch.float64), "x0", torch.float64, 0, (2, 3))
    assert capi._tensor_ptr(None, "x_init", torch.float64, 0, (2, 3), optional=True) is None
    with pytest.raises(ValueError, match="required"):
        capi._tensor_ptr(None, "x0", torch.float64, 0, (2, 3))
