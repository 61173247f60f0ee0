"""vmambair_b200.perceptual on the CPU: basicsr's state_dict layout for every VGG type and several layer sets, the weight lookup
(a path, both 'auto' locations, never a download) and the errors of the constructor and the forward."""
import os

import pytest
import torch
import torchvision

from vmambair_b200.perceptual import PerceptualLoss, layer_names

RECIPE = {"conv1_2": 0.1, "conv2_2": 0.1, "conv3_4": 1, "conv4_4": 1, "conv5_4": 1}
CHANNELS = (64, 128, 256, 512, 512)
CONVS = {"vgg11": (1, 1, 2, 2, 2), "vgg13": (2, 2, 2, 2, 2), "vgg16": (2, 2, 3, 3, 3), "vgg19": (2, 2, 4, 4, 4)}


def _basicsr_layout(vgg_type, layers, use_input_norm=True):
    """{key: shape} of basicsr's PerceptualLoss state_dict, written out from the VGG configurations"""
    out = {"vgg.mean": (1, 3, 1, 1), "vgg.std": (1, 3, 1, 1)} if use_input_norm else {}
    order = []
    cin = 3
    for i, (n, c) in enumerate(zip(CONVS[vgg_type], CHANNELS), 1):
        for j in range(1, n + 1):
            order += [(f"conv{i}_{j}", cin, c), (f"relu{i}_{j}", None, None)]
            cin = c
        order.append((f"pool{i}", None, None))
    cut = max(i for i, (name, _, _) in enumerate(order) if name in layers)
    for name, ci, co in order[:cut + 1]:
        if ci is not None:
            out[f"vgg.vgg_net.{name}.weight"] = (co, ci, 3, 3)
            out[f"vgg.vgg_net.{name}.bias"] = (co,)
    return out


@pytest.mark.parametrize("vgg_type", ["vgg11", "vgg13", "vgg16", "vgg19"])
@pytest.mark.parametrize("layers", [RECIPE, {"relu1_1": 1.0, "pool2": 0.5, "relu3_2": 1.0}, {"conv1_1": 1.0}])
def test_state_dict_is_basicsrs(vgg_type, layers):
    names = layer_names(vgg_type)
    if any(k not in names for k in layers):  # conv3_4 / conv4_4 / conv5_4 exist in vgg19 only
        with pytest.raises(ValueError):
            PerceptualLoss(layers, vgg_type=vgg_type, weights=None)
        return
    loss = PerceptualLoss(layers, vgg_type=vgg_type, weights=None)
    sd = loss.state_dict()
    assert list(sd) == list(_basicsr_layout(vgg_type, layers))
    assert {k: tuple(v.shape) for k, v in sd.items()} == _basicsr_layout(vgg_type, layers)
    assert torch.equal(sd["vgg.mean"].flatten(), torch.tensor([0.485, 0.456, 0.406]))
    assert torch.equal(sd["vgg.std"].flatten(), torch.tensor([0.229, 0.224, 0.225]))
    assert all(not p.requires_grad for p in loss.parameters()) and not loss.vgg.vgg_net.training


def test_layer_names_follow_torchvision_features():
    for vgg_type in CONVS:
        feats = getattr(torchvision.models, vgg_type)(weights=None).features
        kinds = [type(m).__name__ for m in feats]
        names = layer_names(vgg_type)
        assert len(names) == len(kinds)
        assert all(n.startswith({"Conv2d": "conv", "ReLU": "relu", "MaxPool2d": "pool"}[k]) for n, k in zip(names, kinds))


def test_without_input_norm_has_no_mean_and_std():
    sd = PerceptualLoss({"conv1_1": 1.0}, use_input_norm=False, weights=None).state_dict()
    assert list(sd) == list(_basicsr_layout("vgg19", {"conv1_1": 1.0}, use_input_norm=False))


@pytest.fixture
def vgg19_file(tmp_path):
    torch.manual_seed(0)
    feats = torchvision.models.vgg19(weights=None).features
    sd = {f"features.{k}": v for k, v in feats.state_dict().items()}
    path = tmp_path / "vgg19-dcbb9e9d.pth"
    torch.save(sd, path)
    return path, sd


def _check_loaded(loss, sd):
    for i, name in enumerate(layer_names("vgg19")[:len(loss.vgg.vgg_net)]):
        if name.startswith("conv"):
            assert torch.equal(loss.vgg.vgg_net[i].weight, sd[f"features.{i}.weight"])
            assert torch.equal(loss.vgg.vgg_net[i].bias, sd[f"features.{i}.bias"])


@pytest.fixture
def no_download(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("PerceptualLoss tried to download")
    monkeypatch.setattr(torch.hub, "download_url_to_file", refuse)
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", refuse)
    import torchvision.models._api as api
    monkeypatch.setattr(api, "load_state_dict_from_url", refuse, raising=False)


def test_weights_path_loads_a_torchvision_state_dict(vgg19_file, no_download):
    path, sd = vgg19_file
    _check_loaded(PerceptualLoss(RECIPE, weights=str(path)), sd)


def test_weights_path_missing_keys_raise(tmp_path, vgg19_file):
    path, sd = vgg19_file
    short = tmp_path / "short.pth"
    torch.save({k: v for k, v in sd.items() if k != "features.34.weight"}, short)  # conv5_4
    with pytest.raises(KeyError):
        PerceptualLoss(RECIPE, weights=str(short))
    PerceptualLoss({"conv5_3": 1.0}, weights=str(short))  # the cut network does not need it


def test_auto_finds_experiments_pretrained_models(tmp_path, monkeypatch, vgg19_file, no_download):
    path, sd = vgg19_file
    work = tmp_path / "work"
    (work / "experiments" / "pretrained_models").mkdir(parents=True)
    os.replace(path, work / "experiments" / "pretrained_models" / path.name)
    monkeypatch.chdir(work)
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "empty_hub"))
    _check_loaded(PerceptualLoss(RECIPE), sd)


def test_auto_finds_the_hub_cache(tmp_path, monkeypatch, vgg19_file, no_download):
    path, sd = vgg19_file
    (tmp_path / "hub" / "checkpoints").mkdir(parents=True)
    os.replace(path, tmp_path / "hub" / "checkpoints" / path.name)
    (tmp_path / "work").mkdir()
    monkeypatch.chdir(tmp_path / "work")
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "hub"))
    _check_loaded(PerceptualLoss(RECIPE), sd)


def test_auto_without_a_file_raises_and_does_not_download(tmp_path, monkeypatch, no_download):
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "hub"))
    with pytest.raises(FileNotFoundError) as e:
        PerceptualLoss(RECIPE)
    msg = str(e.value)
    assert os.path.join("experiments", "pretrained_models", "vgg19-dcbb9e9d.pth") in msg
    assert os.path.join(str(tmp_path / "hub"), "checkpoints", "vgg19-dcbb9e9d.pth") in msg


def test_out_of_scope_options_raise():
    with pytest.raises(NotImplementedError, match="style"):
        PerceptualLoss(RECIPE, style_weight=1.0, weights=None)
    with pytest.raises(NotImplementedError, match="batch norm"):
        PerceptualLoss(RECIPE, vgg_type="vgg19_bn", weights=None)
    with pytest.raises(NotImplementedError):
        PerceptualLoss(RECIPE, criterion="huber", weights=None)
    with pytest.raises(ValueError):
        PerceptualLoss({"conv6_1": 1.0}, weights=None)


@pytest.mark.parametrize("x,gt", [
    (torch.rand(2, 3, 32, 32), torch.rand(2, 3, 32, 33)),         # shapes differ
    (torch.rand(2, 1, 32, 32), torch.rand(2, 1, 32, 32)),         # not 3 channels
    (torch.rand(3, 32, 32), torch.rand(3, 32, 32)),               # not 4-D
    (torch.rand(2, 3, 8, 32), torch.rand(2, 3, 8, 32)),           # H < 2 ** 4 for conv5_4
    (torch.rand(2, 3, 32, 32).double(), torch.rand(2, 3, 32, 32).double()),  # not float32
    (torch.rand(2, 3, 32, 32), torch.rand(2, 3, 32, 32)),         # not on CUDA
])
def test_bad_inputs_raise_value_error(x, gt):
    loss = PerceptualLoss(RECIPE, weights=None)
    with pytest.raises(ValueError):
        loss(x, gt)


def test_zero_perceptual_weight_returns_none():
    loss = PerceptualLoss(RECIPE, perceptual_weight=0.0, weights=None)
    assert loss(torch.rand(1, 3, 16, 16), torch.rand(1, 3, 16, 16)) == (None, None)
