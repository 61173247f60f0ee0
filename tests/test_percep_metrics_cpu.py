"""vmambair_b200.lpips and .dists on the CPU: the DISTS restatement (oracle/dists_ref.py) against the real reference's float64 scores
(tests/golden/dists_ref.npz), the drop-ins' state_dict layouts and seeded draws, the pinned constants, the weight lookups (never a
download) and the errors of the constructors and the forwards."""
import os

import numpy as np
import pytest
import torch
import torchvision

from oracle import dists_ref, lpips_ref
from vmambair_b200 import _pmetric, dists, lpips
from vmambair_b200.dists import DISTS, calculate_dists
from vmambair_b200.lpips import LPIPS, calculate_lpips

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "dists_ref.npz"))
SEED = 5  # make_golden_dists.SEED


def _gold_convs():
    convs = lpips_ref.seeded_vgg16_convs(int(GOLD["vgg_seed"]))
    np.testing.assert_allclose(lpips_ref.checksums(convs).numpy(), GOLD["vgg_checksums"], rtol=1e-12, atol=0)
    return [(w.double(), b.double()) for w, b in convs]


@pytest.mark.parametrize("weights", ["real", "seed"])
@pytest.mark.parametrize("shape", ["a", "b"])
def test_dists_restatement_matches_the_reference(weights, shape):
    x, y = (torch.from_numpy(GOLD[f"{v}_{shape}"]).double() for v in "xy")
    a, b = (torch.from_numpy(GOLD[f"{weights}_{v}"]) for v in ("alpha", "beta"))
    convs = _gold_convs()
    got = dists_ref.dists(convs, a, b, x, y)
    np.testing.assert_allclose(got.numpy(), GOLD[f"score_{weights}_{shape}"], rtol=0, atol=1e-10)
    np.testing.assert_allclose(dists_ref.feature_sums(convs, x).numpy(), GOLD[f"feat_{shape}"], rtol=1e-10, atol=0)


def test_dists_seeded_construction_and_state_dict_are_the_references():
    torch.manual_seed(SEED)
    m = DISTS(load_weights=False, vgg_weights=None)
    sd = m.state_dict()
    assert list(sd) == list(GOLD["keys"])
    assert [str(tuple(v.shape)) for v in sd.values()] == list(GOLD["shapes"])
    assert np.array_equal(m.alpha.detach().numpy(), GOLD["seed_alpha"])
    assert np.array_equal(m.beta.detach().numpy(), GOLD["seed_beta"])
    # a reference-constructed state_dict (its keys and shapes) loads strictly, and ours loads into the reference's layout
    ref_sd = {k: torch.full(eval(s), float(i)) for i, (k, s) in enumerate(zip(GOLD["keys"], GOLD["shapes"]))}
    m.load_state_dict(ref_sd, strict=True)
    assert all(torch.equal(m.state_dict()[k], v) for k, v in ref_sd.items())


def test_dists_restatement_runs_on_the_drop_ins_state_dict():
    torch.manual_seed(SEED)
    m = DISTS(load_weights=False, vgg_weights=None)
    x, y = torch.rand(2, 3, 9, 11, dtype=torch.float64), torch.rand(2, 3, 9, 11, dtype=torch.float64)
    s = dists_ref.dists_from_state_dict(m.state_dict(), x, y)
    assert s.shape == (2,) and torch.isfinite(s).all()


def test_l2pool_taps_are_the_normalised_hanning_window():
    a = np.hanning(5)[1:-1]
    g = np.outer(a, a) / np.outer(a, a).sum()
    m = dists.L2pooling(channels=64)
    assert m.filter.shape == (64, 1, 3, 3)
    assert np.array_equal(m.filter[0, 0].numpy(), g.astype(np.float32))
    assert np.array_equal(np.outer(dists.TAPS, dists.TAPS), g) and dists.TAPS == dists_ref.TAPS


def test_lpips_constants_and_cuts():
    m = LPIPS(pretrained=False, pnet_rand=True)
    assert torch.equal(m.scaling_layer.shift.flatten(), torch.tensor([-.030, -.088, -.188]))
    assert torch.equal(m.scaling_layer.scale.flatten(), torch.tensor([.458, .448, .450]))
    assert lpips.SLICES == ((0, 4), (4, 9), (9, 16), (16, 23), (23, 30)) == lpips_ref.SLICES
    kinds = [type(f).__name__ for f in torchvision.models.vgg16(weights=None).features]
    assert [kinds[i] for i in _pmetric.CONVS] == ["Conv2d"] * 13 == [kinds[i] for i in lpips_ref.CONV_INDEX]
    assert all(kinds[i] == "ReLU" and kinds[i - 1] == "Conv2d" for i in _pmetric.FEATURE_RELUS)
    assert [hi - 1 for _, hi in lpips.SLICES] == list(_pmetric.FEATURE_RELUS)  # each slice ends at its feature's ReLU
    assert [lo for lo, _ in dists.STAGES[1:]] == [4, 9, 16, 23] and all(kinds[i] == "MaxPool2d" for i in (4, 9, 16, 23))
    assert dists.MEAN == dists_ref.MEAN and dists.STD == dists_ref.STD


def test_lpips_state_dict_is_lpips():
    want = ["scaling_layer.shift", "scaling_layer.scale"]
    for k, (lo, hi) in enumerate(lpips.SLICES, 1):
        want += [f"net.slice{k}.{i}.{p}" for i in range(lo, hi) if i in _pmetric.CONVS for p in ("weight", "bias")]
    want += [f"lin{k}.model.1.weight" for k in range(5)] + [f"lins.{k}.model.1.weight" for k in range(5)]
    sd = LPIPS(pretrained=False, pnet_rand=True).state_dict()
    assert list(sd) == want
    assert [tuple(sd[f"lin{k}.model.1.weight"].shape) for k in range(5)] == [(1, c, 1, 1) for c in (64, 128, 256, 512, 512)]
    assert "lin0.model.0.weight" in LPIPS(pretrained=False, pnet_rand=True, use_dropout=False).state_dict()


@pytest.fixture
def no_download(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("tried to download")
    monkeypatch.setattr(torch.hub, "download_url_to_file", refuse)
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", refuse)


@pytest.fixture
def no_lpips_package(monkeypatch, tmp_path):
    monkeypatch.setattr(lpips, "lpips_package_weights", lambda version="0.1", net="vgg": str(tmp_path / "pkg" / "weights" / "v0.1" /
                                                                                             "vgg.pth"))
    return str(tmp_path / "pkg" / "weights" / "v0.1" / "vgg.pth")


def test_lpips_lin_weights_lookup(tmp_path, no_lpips_package, no_download):
    with pytest.raises(FileNotFoundError) as e:
        LPIPS(pretrained=True, pnet_rand=True)
    assert no_lpips_package in str(e.value) and "model_path None" in str(e.value)
    missing = str(tmp_path / "nowhere.pth")
    with pytest.raises(FileNotFoundError) as e:
        LPIPS(pretrained=True, pnet_rand=True, model_path=missing)
    assert missing in str(e.value) and no_lpips_package in str(e.value)
    torch.manual_seed(0)
    lins = {f"lin{k}.model.1.weight": torch.rand(1, c, 1, 1) for k, c in enumerate((64, 128, 256, 512, 512))}
    torch.save(lins, tmp_path / "vgg.pth")
    m = LPIPS(pretrained=True, pnet_rand=True, model_path=str(tmp_path / "vgg.pth"), verbose=False)
    assert all(torch.equal(m.state_dict()[k], v) for k, v in lins.items())
    assert all(torch.equal(m.lins[k].model[1].weight, lins[f"lin{k}.model.1.weight"]) for k in range(5))
    os.makedirs(os.path.dirname(no_lpips_package))
    torch.save(lins, no_lpips_package)
    m = LPIPS(pretrained=True, pnet_rand=True, verbose=False)
    assert torch.equal(m.lin4.model[1].weight, lins["lin4.model.1.weight"])


def test_vgg_trunk_lookup(tmp_path, monkeypatch, no_download):
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "hub"))
    for make in (lambda: LPIPS(pretrained=False), lambda: DISTS(load_weights=False)):
        with pytest.raises(FileNotFoundError) as e:
            make()
        assert os.path.join("experiments", "pretrained_models", "vgg16-397923af.pth") in str(e.value)
        assert os.path.join(str(tmp_path / "hub"), "checkpoints", "vgg16-397923af.pth") in str(e.value)
    torch.manual_seed(1)
    feats = torchvision.models.vgg16(weights=None).features
    os.makedirs("experiments/pretrained_models")
    torch.save({f"features.{k}": v for k, v in feats.state_dict().items()}, "experiments/pretrained_models/vgg16-397923af.pth")
    lp, di = LPIPS(pretrained=False), DISTS(load_weights=False)
    for i in _pmetric.CONVS:
        assert torch.equal(lp.net.module(i).weight, feats[i].weight) and torch.equal(di._module(i).bias, feats[i].bias)


def test_dists_weights_lookup(tmp_path, monkeypatch, no_download):
    monkeypatch.chdir(tmp_path)
    with pytest.raises(FileNotFoundError) as e:
        DISTS(vgg_weights=None)
    assert dists.DEFAULT_WEIGHTS in str(e.value) and "weights_path None" in str(e.value)
    w = {"alpha": torch.rand(1, 1475, 1, 1), "beta": torch.rand(1, 1475, 1, 1)}
    os.makedirs(os.path.dirname(dists.DEFAULT_WEIGHTS))
    torch.save(w, dists.DEFAULT_WEIGHTS)
    assert torch.equal(DISTS(vgg_weights=None).alpha, w["alpha"])
    missing = str(tmp_path / "nowhere.pt")
    with pytest.raises(FileNotFoundError) as e:
        DISTS(vgg_weights=None, weights_path=missing)
    assert missing in str(e.value) and dists.DEFAULT_WEIGHTS in str(e.value)
    torch.save({"alpha": w["beta"], "beta": w["alpha"]}, tmp_path / "other.pt")
    assert torch.equal(DISTS(vgg_weights=None, weights_path=str(tmp_path / "other.pt")).beta, w["alpha"])


@pytest.mark.parametrize("kw", [dict(net="alex"), dict(net="squeeze"), dict(lpips=False), dict(spatial=True), dict(version="0.0"),
                                dict(pnet_tune=True)])
def test_lpips_unsupported_options(kw):
    with pytest.raises(NotImplementedError):
        LPIPS(pretrained=False, pnet_rand=True, **kw)


def test_unsupported_calls():
    d = DISTS(load_weights=False, vgg_weights=None)
    x = torch.rand(1, 3, 16, 16)
    with pytest.raises(NotImplementedError):
        d(x, x, require_grad=True)
    xg = x.clone().requires_grad_()
    with pytest.raises(NotImplementedError):
        d(xg, x)
    with pytest.raises(NotImplementedError):
        LPIPS(pretrained=False, pnet_rand=True)(xg, x)


@pytest.mark.parametrize("x,y", [
    (torch.rand(2, 3, 32, 32), torch.rand(2, 3, 32, 33)),         # shapes differ
    (torch.rand(2, 1, 32, 32), torch.rand(2, 1, 32, 32)),         # not 3 channels
    (torch.rand(3, 32, 32), torch.rand(3, 32, 32)),               # not 4-D
    (torch.rand(2, 3, 32, 32).double(), torch.rand(2, 3, 32, 32).double()),  # not float32
    (torch.rand(2, 3, 32, 32), torch.rand(2, 3, 32, 32)),         # not on CUDA
])
def test_bad_inputs_raise_value_error(x, y):
    with pytest.raises(ValueError):
        LPIPS(pretrained=False, pnet_rand=True)(x, y)
    with pytest.raises(ValueError):
        DISTS(load_weights=False, vgg_weights=None)(x, y)


def test_evaluation_loop_rejects_bad_images():
    lp, di = LPIPS(pretrained=False, pnet_rand=True), DISTS(load_weights=False, vgg_weights=None)
    img = np.zeros((32, 32, 3), np.uint8)
    for f, m in ((calculate_lpips, lp), (calculate_dists, di)):
        with pytest.raises(ValueError):
            f(img.astype(np.float32), img.astype(np.float32), m)
        with pytest.raises(ValueError):
            f(img[..., :1], img[..., :1], m)
        with pytest.raises(TypeError):
            f(img.tolist(), img.tolist(), m)
        with pytest.raises(ValueError):
            f(torch.zeros(1, 32, 32, 3, dtype=torch.uint8), torch.zeros(1, 32, 32, 3, dtype=torch.uint8), m)  # not on CUDA
