"""NIQE without a GPU: oracle/niqe_ref.py against the reference's own results (tests/golden/niqe_ref.npz, made by
tests/golden/make_golden_niqe.py from the real calculate_niqe with scipy and cv2 on oracle/niqe_ref.case_image's seeded inputs), fed
the reference's planes and r(gamma) table;
parameter loading and argument checks of vmambair_b200.niqe."""
import hashlib
import math
import os

import numpy as np
import pytest

from oracle import metrics_ref, niqe_ref
from vmambair_b200 import niqe

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
G = np.load(os.path.join(GOLDEN, "niqe_ref.npz"))
PARAMS = os.path.join(GOLDEN, "niqe_pris_params.npz")
CASES = [str(c) for c in G["cases"]]
SCORED = [c for c in CASES if str(G[f"{c}/raises"]) == ""]
ALPHA_COLS = [0, 2, 6, 10, 14]  # alpha of each fit within a scale's 18 features; the fit's other columns follow it
FIT_COLS = [(0, [1]), (2, [3, 4, 5]), (6, [7, 8, 9]), (10, [11, 12, 13]), (14, [15, 16, 17])]


def case(name):
    """-> (the input as the reference received it, crop_border, input_order, convert_to); the input is rebuilt from its seed and must
    have the bytes the reference scored"""
    crop, order, conv = (str(x) for x in G[f"{name}/meta"])
    seed, h, w, c, dtype, flat = (str(x) for x in G[f"{name}/spec"])
    img = niqe_ref.case_image(int(seed), int(h), int(w), int(c), dtype, bool(int(flat)))
    img = np.ascontiguousarray(img.transpose(2, 0, 1)) if order == "CHW" else img
    assert hashlib.sha256(img.tobytes()).hexdigest() == str(G[f"{name}/img_sha256"]), name
    return img, int(crop), order, conv


def plane_of(name):
    """the float32 plane the reference's niqe() filters: stored for 'gray'; to_y_channel (bit for bit, oracle/metrics_ref.py) or
    the float32 input itself otherwise; cropped and cut to whole blocks"""
    if f"{name}/plane" in G:
        return G[f"{name}/plane"]
    img, crop, order, _ = case(name)
    if order == "HW":
        p = img.astype(np.float32)
    else:
        a = img[..., None] if img.ndim == 2 else img
        a = a.transpose(1, 2, 0) if order == "CHW" else a
        p = metrics_ref.to_y_channel(a.astype(np.float32).astype(np.float64))
    if crop:
        p = p[crop:-crop, crop:-crop]
    h, w = p.shape[0] // 96 * 96, p.shape[1] // 96 * 96
    return p[:h, :w]


def half_of(name):
    """cv2's half plane of the case: stored as its ulp offset from the float32 2 x 2 mean of the plane"""
    m = niqe_ref.half_plane(plane_of(name))
    return (m.view(np.int32) + G[f"{name}/half_ulp"].astype(np.int32)).view(np.float32)


def params():
    return niqe.load_params(PARAMS)


def compare_features(got, want, rtol=1e-4):
    """alpha within one table step; every other entry of a fit whose alpha agrees to rtol; NaN where the reference has NaN
    -> (fits whose alpha moved one step, fits)"""
    assert got.shape == want.shape
    assert np.array_equal(np.isnan(got), np.isnan(want))
    moved = total = 0
    for s in (0, 18):
        for a, rest in FIT_COLS:
            steps = np.rint(np.abs(got[:, s + a] - want[:, s + a]) / 0.001)
            assert steps.max() <= 1, steps.max()
            assert np.allclose(got[:, s + a], want[:, s + a], rtol=0, atol=1e-9 + 0.001 * steps.max())
            same = steps == 0
            moved += int((~same).sum())
            total += same.size
            for c in rest:
                g, w = got[same, s + c], want[same, s + c]
                ok = np.isnan(w) | (np.abs(g - w) <= rtol * np.abs(w) + 1e-9)
                assert ok.all(), (s + c, np.nanmax(np.abs(g - w) / np.abs(w)))
    return moved, total


@pytest.mark.parametrize("name", SCORED + ["one_block"])
def test_oracle_reproduces_reference_features(name):
    p = params()
    plane = plane_of(name)
    got = niqe_ref.features(plane, half_of(name), p.window, G["r_gam"])
    compare_features(got, G[f"{name}/features"])


def test_oracle_alpha_moves_on_at_most_one_percent_of_fits():
    """the reference's float32 means move rhatnorm by ~1e-6 relative: near a midpoint of two table entries alpha takes the other"""
    p = params()
    counts = [compare_features(niqe_ref.features(plane_of(n), half_of(n), p.window, G["r_gam"]), G[f"{n}/features"])
              for n in SCORED + ["one_block"]]
    moved, total = (sum(c) for c in zip(*counts))
    assert moved <= 0.01 * total, (moved, total)


@pytest.mark.parametrize("name", SCORED)
def test_oracle_reproduces_reference_scores(name):
    p = params()
    f = niqe_ref.features(plane_of(name), half_of(name), p.window, G["r_gam"])
    want = float(G[f"{name}/score"].reshape(()))
    assert math.isclose(niqe_ref.score(f, p.mu, p.cov), want, rel_tol=1e-4)
    assert math.isclose(niqe_ref.score(G[f"{name}/features"], p.mu, p.cov), want, rel_tol=1e-12)  # the score step alone


@pytest.mark.parametrize("name", [c for c in CASES if f"{c}/mscn" in G])
def test_oracle_mscn_is_scipys_bit_for_bit(name):
    got = niqe_ref.mscn(plane_of(name), params().window)
    assert np.array_equal(got, G[f"{name}/mscn"])


def test_flat_case_has_nan_betas_and_alpha_point_two():
    f = G["flat_clipped/features"]
    nan_rows = np.isnan(f).any(axis=1)
    assert nan_rows.any() and (~nan_rows).sum() >= 2
    assert (f[nan_rows][:, [0, 18]] == 0.2).any()  # an empty side: np.argmin of all-NaN distances is 0
    assert np.isnan(niqe_ref.score(G["one_block/features"], params().mu, params().cov))


def test_oracle_table_matches_scipys():
    t = niqe_ref.table()
    assert t.shape == (9801,) and np.all(np.diff(t) > 0)  # strictly increasing: a search finds np.argmin's entry
    assert np.max(np.abs(t / G["r_gam"] - 1)) < 1e-13
    assert np.array_equal(niqe_ref.gam(np.arange(9801)), np.arange(0.2, 10.001, 0.001))


def test_half_planes_are_within_two_ulp_of_the_float32_mean():
    for name in SCORED:
        assert np.abs(G[f"{name}/half_ulp"]).max() <= 2, name


def test_expected_raises_recorded():
    assert str(G["one_block/raises"]) == "LinAlgError"
    assert str(G["small/raises"]) == "cv2.error" and str(G["small_after_crop/raises"]) == "cv2.error"


def test_load_params_path_default_cache_and_errors(tmp_path, monkeypatch):
    p = niqe.load_params(PARAMS)
    assert p is niqe.load_params(PARAMS)
    assert p.mu.shape == (36,) and p.cov.shape == (36, 36) and p.window.shape == (7, 7)
    assert hashlib.sha256(open(PARAMS, "rb").read()).hexdigest() == str(G["params_sha256"])
    monkeypatch.chdir(tmp_path)
    with pytest.raises(FileNotFoundError, match="basicsr/metrics/niqe_pris_params.npz"):
        niqe.load_params()
    with pytest.raises(FileNotFoundError, match="missing.npz"):
        niqe.load_params("missing.npz")
    d = tmp_path / "basicsr" / "metrics"
    d.mkdir(parents=True)
    (d / "niqe_pris_params.npz").write_bytes(open(PARAMS, "rb").read())
    q = niqe.load_params()
    assert np.array_equal(q.cov, p.cov) and np.array_equal(q.window, p.window)
    with pytest.raises(ValueError, match="36"):
        niqe.NiqeParams(p.mu[:35], p.cov, p.window)


def test_argument_errors():
    img = np.zeros((100, 100, 3), np.uint8)
    with pytest.raises(TypeError):
        niqe.calculate_niqe(img.tolist(), 0)
    with pytest.raises(ValueError, match="input_order"):
        niqe.calculate_niqe(img, 0, input_order="WHC")
    with pytest.raises(ValueError, match="convert_to"):
        niqe.calculate_niqe(img, 0, convert_to="rgb")
    with pytest.raises(ValueError, match="convert_to"):
        niqe._convert("gray", 1)
    with pytest.raises(ValueError, match="convert_to"):
        niqe._convert(None, 3)
