"""The backward of skin_with_blend_shapes over several slices of its rest-point scratch, on the device.

The skel-state gradient writes the shaped rest points of a slice of instances to at most 256 MiB of scratch (DESIGN, "Scratch and handles
of the character operations"). Instances on both sides of each slice boundary must meet test_blend_shape_skinning's float64 bounds and
give the same bits as in a batch of their own.
"""
import pytest
import torch

from momentum_b200 import solver as ms
from tests import test_blend_shape_skinning as tbs
from tests import test_skinning as tsn


@pytest.mark.gpu
def test_backward_in_several_slices_meets_the_bounds():
    """bodyhands300's 20 100 vertices take 236 KiB of shaped rest points each, so 2400 instances need three slices."""
    ch, Kp = tbs._fixture("bodyhands300_k16")
    dc = ms.DeviceCharacter(ch, 0)
    B, V = 2400, ch.skinning.num_vertices
    assert B * V * 3 * 4 > 2 * (256 << 20)
    per_slice = (256 << 20) // (V * 3 * 4)
    st, w = tsn._states(ch, B, 71), tbs._weights(B, Kp, 72)
    std, wd = tbs._dev(st), tbs._dev(w)
    Gd = torch.randn(B, V, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(73))
    gs, gw = tbs._device_backward(dc, std, wd, Gd)
    sub = [0, per_slice - 1, per_slice, 2 * per_slice - 1, 2 * per_slice, B - 1]  # both sides of each slice boundary
    tbs._check(tbs._ratios(ch, st[sub], w[sub], Gd[sub].cpu().numpy(), None, gs[sub].cpu().numpy(), gw[sub].cpu().numpy()), "slices")
    gs_alone, gw_alone = tbs._device_backward(dc, std[sub].contiguous(), wd[sub].contiguous(), Gd[sub].contiguous())
    assert torch.equal(gs_alone, gs[sub]) and torch.equal(gw_alone, gw[sub])
