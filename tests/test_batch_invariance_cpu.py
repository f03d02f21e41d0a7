"""Batch invariance of the deterministic plans without a GPU: every workspace query of a deterministic inference op that takes
B is B times its one-image size, i.e. an image's partial sums get the same slots -- and so the same grouping and order of
additions -- whatever batch it is in.  (The conv_tc2 / conv_tc3 queries take a plan, which needs a device; the GPU suite
checks those on real plans.)"""
import pytest

from pdae_b200 import _native

BATCHES = [1, 2, 7, 64, 256]
LEVELS = [4, 8, 16, 64]           # square levels of the UNets and encoders


def _linear(query, *shape):
    one = query(1, *shape)
    assert one > 0, shape
    for B in BATCHES:
        assert query(B, *shape) == B * one, (query.__name__, B, shape)


@pytest.mark.parametrize("S", LEVELS)
@pytest.mark.parametrize("C", [64, 128, 256, 512, 768])
def test_stats_workspace_is_linear_in_batch(S, C):
    _linear(_native.lib().pdae_stats_det_workspace_bytes, S * S, C)


@pytest.mark.parametrize("HW", [6 * 6, 12 * 12, 24 * 24, 48 * 48, 128 * 128])
def test_stats_workspace_is_linear_in_batch_off_powers_of_two(HW):
    _linear(_native.lib().pdae_stats_det_workspace_bytes, HW, 128)


@pytest.mark.parametrize("S", [16, 48, 64, 128])
@pytest.mark.parametrize("stride", [1, 2])
def test_stem_workspace_is_linear_in_batch(S, stride):
    for Cout in (64, 128):
        _linear(_native.lib().pdae_stem_conv_det_workspace_bytes, S, S, Cout, stride)


@pytest.mark.parametrize("S", LEVELS + [40, 48])
def test_metric_workspaces_are_linear_in_batch(S):
    L = _native.lib()
    _linear(L.pdae_mse_det_workspace_bytes, 3 * S * S)
    _linear(L.pdae_ssim_det_workspace_bytes, 3, S, S)
