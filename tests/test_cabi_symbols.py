"""The C-ABI library loads without a GPU and exports every symbol include/momentum_b200.h declares."""
import ctypes
import os
import re

import pytest

from momentum_b200 import solver as ms

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g

    g.build()
    return ctypes.CDLL(ms.DEFAULT_LIB)


def test_header_symbols_exported(lib):
    header = open(os.path.join(ROOT, "include", "momentum_b200.h")).read()
    declared = sorted(set(re.findall(r"\b(mb2_[a-z0-9_]+)\s*\(", header)))
    assert len(declared) >= 35
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in momentum_b200.h but not exported"
    assert sorted(ms.CABI_SYMBOLS) == declared
    # the launch reports of the per-instance character kernels (tests/test_instance_launch_variants.py)
    assert {"mb2_character_get_instance_launch", "mb2_solver_function_get_input_gradient_launch"} <= set(declared)
    # every binding takes as many arguments as its prototype declares (comments dropped: some hold commas or calls)
    prototypes = dict(re.findall(r"\b(mb2_[a-z0-9_]+)\s*\(([^)]*)\)", re.sub(r"/\*.*?\*/", "", header, flags=re.S)))
    for name, (_, argtypes) in ms.CABI_SIGNATURES.items():
        params = prototypes[name].strip()
        assert len(argtypes) == (0 if params in ("", "void") else params.count(",") + 1), (name, params, argtypes)


def test_no_cpu_fallback_without_device(lib):
    """Without a usable sm_90 device every compute entry point must fail loudly (no CPU path)."""
    import numpy as np
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from momentum_b200 import character as mc

    lib.mb2_device_count.restype = ctypes.c_int
    assert lib.mb2_device_count() == 0
    with pytest.raises(ms.MomentumB200Error, match="no usable sm_90 CUDA device|cuda"):
        ms.DeviceCharacter(mc.create_test_character(3))


def test_invalid_character_is_rejected_like_mt_check(lib):
    from momentum_b200 import character as mc

    ch = mc.create_test_character(4)
    ch.parents = ch.parents.copy()
    ch.parents[1] = 3  # child before parent: skeleton.h:23-24 ordering violated
    with pytest.raises(ms.MomentumB200Error, match="topologically sorted"):
        ms.DeviceCharacter(ch)
