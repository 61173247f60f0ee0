"""Host-side parts of the two-direction channel scan (vmambair_b200.cross_scan.cross_selective_scanC): the fused-path bounds, the
CrossScanC / CrossMergeC pair, and the SS2D_1.cforward_corev2 variant check.  No GPU needed."""
import pytest
import torch

import vmambair_b200.archs as archs
from vmambair_b200 import _lib, ops
from vmambair_b200 import cross_scan as cs


@pytest.mark.parametrize("C", [48, 96, 192, 384])
def test_every_realsr_channel_call_fits_the_fused_kernels(C):
    R = -(-C // 16)
    assert ops.cross_scan_c_supported(1, C, R, 16)
    assert 0 < _lib.lib().vmb_cross_selective_scan_c_smem_bytes(1, C, R, 16) <= 227 * 1024


@pytest.mark.parametrize("shape", [(1, 4096, 4, 16), (1, 48, 3, 24), (17, 32, 2, 8)])
def test_shapes_beyond_the_bounds_are_rejected(shape):
    assert not ops.cross_scan_c_supported(*shape)


def test_cross_scan_c_and_merge_c_are_adjoint_gathers():
    x = torch.randn(2, 3, 11, dtype=torch.float64, requires_grad=True)
    xs = cs.CrossScanC.apply(x)
    assert torch.equal(xs[:, 0], x.detach()) and torch.equal(xs[:, 1], x.detach().flip(-1))
    assert torch.autograd.gradcheck(cs.CrossScanC.apply, (x,))
    ys = torch.randn(2, 2, 3, 11, dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(cs.CrossMergeC.apply, (ys,))


def test_cforward_corev2_is_realsr_only():
    m = archs.SS2D_1(d_model=16, ssm_ratio=1, variant="sisr")
    with pytest.raises(NotImplementedError, match="realsr"):
        m.cforward_corev2(torch.randn(1, 16, 4, 4), channel_first=True)
