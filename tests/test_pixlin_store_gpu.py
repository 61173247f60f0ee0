"""pixlin's 16-bit outputs are its fp32 epilogue values rounded once: the same call with out_dtype=float32, rounded to the I/O
dtype, matches bit for bit -- bias, SiLU range and residual included, on both pixel-tile sizes and with a partial last tile."""
import pytest
import torch

from vmambair_b200 import ops

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("B,K,M,P", [(8, 96, 256, 4096), (2, 48, 160, 1024), (1, 96, 96, 200)])
def test_16bit_output_is_the_fp32_epilogue_rounded(B, K, M, P, dtype):
    g = torch.Generator().manual_seed(B * 1000 + K + P)
    x = torch.randn(B, K, P, generator=g).to(DEV, dtype)
    w = ops.pad_weight((torch.randn(M, K, generator=g) / K ** 0.5).to(DEV, dtype))
    bias = torch.randn(M, generator=g).to(DEV)
    res = torch.randn(B, M, P, generator=g).to(DEV, dtype)
    kw = dict(bias=bias, residual=res, act=(M // 2, M))
    got = ops.pixlin(x, w, **kw)
    ref = ops.pixlin(x, w, out_dtype=torch.float32, **kw).to(dtype)
    assert torch.equal(got.view(torch.int16), ref.view(torch.int16))
