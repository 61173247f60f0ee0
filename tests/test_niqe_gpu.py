"""vmambair_b200.niqe (csrc/niqe.cu) against the reference's results (tests/golden/niqe_ref.npz) and against oracle/niqe_ref.py fed
the GPU's own planes and r(gamma) table.  Bounds: scores within 1e-4 relative of the reference; the scale-1 MSCN map bit for bit for integer inputs; the half plane within
2 ulp of cv2's; features and scores within 1e-12 of the oracle with identical alphas; the table within 1e-13 of scipy's."""
import math

import numpy as np
import pytest
import torch

from oracle import metrics_ref, niqe_ref
from vmambair_b200 import metrics, niqe, ops

from .test_niqe_cpu import ALPHA_COLS, CASES, G, PARAMS, SCORED, case, half_of

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ACOLS = [s + a for s in (0, 18) for a in ALPHA_COLS]


def params():
    return niqe.load_params(PARAMS)


def view(name):
    """the case's image on the GPU as calculate_niqe stages it -> (view, convert_to)"""
    img, _, order, conv = case(name)
    if order == "HW":
        return metrics._device_image(img, "HWC", DEV), None
    return metrics._device_image(img, order, DEV), conv


def run(name):
    v, conv = view(name)
    return niqe._run(v, case(name)[1], conv, params(), planes=True)


def scene(seed, b, h, w):
    g = torch.Generator().manual_seed(seed)
    y = torch.linspace(0, 6, h)[:, None, None]
    x = torch.linspace(0, 9, w)[None, :, None]
    base = 0.5 + 0.3 * torch.sin(x + y * torch.rand(1, 1, 3, generator=g) * 3)
    img = base[None] + 0.1 * torch.randn(b, h, w, 3, generator=g)
    return (img.clamp(0, 1) * 255).round().to(torch.uint8).to(DEV)


@pytest.mark.parametrize("name", SCORED)
def test_calculate_niqe_matches_the_reference(name):
    img, crop, order, conv = case(name)
    got = niqe.calculate_niqe(img, crop, input_order=order, convert_to=conv, params=params())
    want = G[f"{name}/score"]
    assert isinstance(got, np.ndarray) and got.shape == want.shape == (1, 1) and got.dtype == want.dtype == np.float64
    assert math.isclose(float(got[0, 0]), float(want[0, 0]), rel_tol=1e-4)


def test_degenerate_cases_raise_in_the_dropin_and_give_nan_batched():
    for name, err in (("one_block", np.linalg.LinAlgError), ("small", ValueError), ("small_after_crop", ValueError)):
        img, crop, order, conv = case(name)
        with pytest.raises(err):
            niqe.calculate_niqe(img, crop, input_order=order, convert_to=conv, params=params())
        t = torch.from_numpy(img)[None].to(DEV)
        assert torch.isnan(niqe.niqe(t, crop, conv, params=params())).all()
    flat = torch.full((2, 192, 192, 3), 77, dtype=torch.uint8, device=DEV)  # every block flat: no NaN-free row
    assert torch.isnan(niqe.niqe(flat, params=params())).all()


def test_flat_and_clipped_blocks_follow_the_reference():
    """NaN betas and alpha 0.2 where a distribution has no negative or no positive value; the covariance over NaN-free rows"""
    r = run("flat_clipped")
    f = r["features"][0].cpu().numpy()
    want = G["flat_clipped/features"]
    assert np.array_equal(np.isnan(f), np.isnan(want))
    nan_rows = np.isnan(f).any(axis=1)
    assert (f[nan_rows][:, [0, 18]] == 0.2).any()
    assert math.isclose(r["score"].item(), float(G["flat_clipped/score"][0, 0]), rel_tol=1e-4)


@pytest.mark.parametrize("name", [c for c in CASES if f"{c}/mscn" in G])
def test_scale1_mscn_is_the_references_bit_for_bit(name):
    assert np.array_equal(run(name)["mscn"][0].cpu().numpy(), G[f"{name}/mscn"])


@pytest.mark.parametrize("name", SCORED)
def test_half_plane_within_two_ulp_of_cv2(name):
    got = run(name)["half"][0].cpu().numpy()
    want = half_of(name)
    ulp = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
    assert got.shape == want.shape and ulp.max() <= 2


def test_table_matches_scipys():
    t = niqe._table(DEV).cpu().numpy()
    assert np.max(np.abs(t / G["r_gam"] - 1)) < 1e-13
    assert np.all(np.diff(t) > 0)


@pytest.mark.parametrize("name", SCORED)
def test_matches_the_oracle_on_the_gpus_planes(name):
    r = run(name)
    p = params()
    plane, half, tab = (r[k][0].cpu().numpy() if k != "table" else r[k].cpu().numpy() for k in ("plane", "half", "table"))
    assert np.array_equal(r["mscn"][0].cpu().numpy(), niqe_ref.mscn(plane, p.window))
    assert np.array_equal(r["mscn_half"][0].cpu().numpy(), niqe_ref.mscn(half, p.window))
    got = r["features"][0].cpu().numpy()
    want = niqe_ref.features(plane, half, p.window, tab)
    assert np.array_equal(got[:, ACOLS], want[:, ACOLS])
    assert np.allclose(got, want, rtol=1e-12, atol=1e-14, equal_nan=True)
    assert math.isclose(r["score"].item(), niqe_ref.score(got, p.mu, p.cov), rel_tol=1e-12)


def test_y_plane_is_to_y_channel_and_the_plane_input_is_kept():
    img, crop, _, _ = case("u8_crop4")
    v, _ = view("u8_crop4")
    plane = niqe._run(v, crop, "y", params(), planes=True)["plane"][0].cpu().numpy()
    y = metrics_ref.to_y_channel(img.astype(np.float64))[crop:-crop, crop:-crop]
    assert np.array_equal(plane, y[:plane.shape[0], :plane.shape[1]])
    hw = case("f32_hw")[0]
    plane = run("f32_hw")["plane"][0].cpu().numpy()
    assert np.array_equal(plane, hw[:plane.shape[0], :plane.shape[1]])


def test_batch_equals_each_image_alone_and_quantized_outputs():
    x = scene(1, 3, 230, 310)
    both = niqe.niqe(x, 3, params=params())
    feats = niqe.niqe_features(x, 3, params=params())
    assert both.shape == (3,) and both.dtype == torch.float64 and feats.shape == (3, 6, 36)
    for i in range(3):
        assert torch.equal(niqe.niqe(x[i:i + 1], 3, params=params()), both[i:i + 1])
        assert torch.equal(niqe.niqe_features(x[i:i + 1], 3, params=params()), feats[i:i + 1])
    # a network output (RGB, (B, 3, H, W)) through tensor2img equals its uint8 BGR image
    out = torch.rand(2, 3, 200, 200, generator=torch.Generator().manual_seed(3)).to(DEV) * 1.2 - 0.1
    u8 = torch.from_numpy(np.stack([metrics_ref.tensor2img(o) for o in out.cpu().numpy()])).to(DEV)
    for conv in ("y", "gray"):
        assert torch.equal(niqe.niqe(out, 0, conv, quantize=True, params=params()), niqe.niqe(u8, 0, conv, params=params()))


def test_bitwise_reproducible_deterministic_without_host_sync():
    x = scene(2, 2, 200, 300)
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        a = niqe.niqe(x, params=params()), niqe.niqe_features(x, params=params())
        torch.cuda.set_sync_debug_mode("error")
        try:
            b = niqe.niqe(x, params=params()), niqe.niqe_features(x, params=params())
        finally:
            torch.cuda.set_sync_debug_mode(0)
    finally:
        torch.use_deterministic_algorithms(old)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_cuda_graph_replays_equal_to_eager():
    x0 = scene(4, 2, 200, 300)
    x = x0.clone()
    want = niqe.niqe(x0, params=params())
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        niqe.niqe(x, params=params())
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        got = niqe.niqe(x, params=params())
    x.copy_(scene(5, 2, 200, 300))
    graph.replay()
    other = got.clone()
    x.copy_(x0)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(got, want) and not torch.equal(other, want)


def test_at_most_four_launches_per_call():
    for b in (1, 5):
        x = scene(6, b, 200, 200)
        n0 = ops.launch_count()
        niqe.niqe(x, params=params())
        assert ops.launch_count() - n0 <= 4
        n0 = ops.launch_count()
        niqe.niqe(x, params=params())
        assert ops.launch_count() - n0 == 3  # the table is built once per device


def test_input_validation():
    x = scene(7, 1, 100, 100)
    with pytest.raises(ValueError, match="niqe"):
        niqe.niqe(x[0], params=params())
    with pytest.raises(ValueError, match="convert_to"):
        niqe.niqe(x[..., :1], convert_to="gray", params=params())
    with pytest.raises(ValueError, match="crop_border"):
        niqe.niqe(x, crop_border=-1, params=params())
