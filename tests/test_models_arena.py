"""Model zoo parity (tensor counts / parameter counts of the reference models), split drivers, arenas."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from draco_b200.models import (FC_NN, FC_NN_Split, LeNet, LeNetSplit, ResNet18, ResNetSplit18, available_networks,
                               build_model)
from draco_b200.parallel.arena import TILE, ArenaLayout, ModelBinder

EXPECTED = {
    "LeNet": (8, 431080), "FC": (6, 1033510), "ResNet18": (62, 11173962), "ResNet34": (110, 21282122),
    "ResNet50": (161, 23520842), "ResNet101": (314, 42512970), "ResNet152": (467, 58156618),
    "VGG11": (38, 9756426), "VGG16": (58, 15253578),
}


@pytest.mark.parametrize("name", sorted(EXPECTED))
def test_parameter_counts_match_reference(name):
    m = build_model(name)
    ps = list(m.parameters())
    assert (len(ps), sum(p.numel() for p in ps)) == EXPECTED[name]


def test_registry_covers_reference_networks():
    for n in ["LeNet", "FC", "ResNet18", "ResNet34", "ResNet50", "ResNet101", "ResNet152", "VGG11", "VGG13", "VGG16"]:
        assert n in available_networks()
    with pytest.raises(ValueError):
        build_model("AlexNet")


def test_lenet_and_fc_quirks():
    torch.manual_seed(0)
    x = torch.randn(4, 1, 28, 28)
    m = LeNet()
    # pool BEFORE relu, no activation between fc1 and fc2 (reference lenet.py:27-41)
    h = F.relu(F.max_pool2d(m.conv1(x), 2, 2))
    h = F.relu(F.max_pool2d(m.conv2(h), 2, 2)).reshape(4, -1)
    assert torch.allclose(m(x), m.fc2(m.fc1(h)), atol=1e-6)
    fc = FC_NN()
    out = fc(x)
    assert out.shape == (4, 10) and out.min() >= 0 and out.max() <= 1      # sigmoid on the logits (fc_nn.py:38)


@pytest.mark.parametrize("ctor,shape", [(LeNetSplit, (1, 28, 28)), (FC_NN_Split, (1, 28, 28)), (ResNetSplit18, (3, 32, 32))])
def test_split_backward_drivers(ctor, shape):
    torch.manual_seed(0)
    m = ctor()
    x = torch.randn(2, *shape)
    y = torch.tensor([1, 3])
    seen = []
    loss = F.cross_entropy(m(x), y)
    grads = m.backward_normal(loss, on_ready=lambda i, p: seen.append(i))
    n = len(list(m.parameters()))
    assert sorted(seen) == list(range(n)) and len(grads) == n
    assert seen[0] >= n - 2, "the classifier's gradients must become ready first (reverse layer order)"
    ref = [g.clone() for g in grads]
    m.zero_grad()
    coded = m.backward_coded(F.cross_entropy(m(x), y))
    for a, b in zip(reversed(coded), ref):
        assert torch.allclose(a, b, atol=1e-6)
    m.zero_grad()
    m.backward_single(F.cross_entropy(m(x), y))
    assert all(p.grad is not None for p in m.parameters())


def test_arena_layout_and_binder_roundtrip():
    torch.manual_seed(0)
    m = ResNet18()
    ref = [p.detach().clone() for p in m.parameters()]
    L = ArenaLayout.from_model(m, bf16=False, channels_last=True)
    assert L.ntensors == 62 and L.total % TILE == 0 and L.num_params == 11173962
    assert all(s.offset % TILE == 0 for s in L.specs)
    assert L.tile_tensor_np[0] == 0 and L.tile_tensor_np[-1] == 61
    assert L.valid_mask().sum() == L.num_params
    b = ModelBinder(m, L, "cpu", bf16=False)
    for p, r in zip(m.parameters(), ref):
        assert torch.equal(p.detach(), r)                       # logical values preserved
    # parameters alias the arena
    b.params_f32.zero_()
    assert all(float(p.abs().sum()) == 0 for p in m.parameters())
    conv = L.view(b.params_f32, 0)
    assert conv.shape == (64, 3, 3, 3) and conv.is_contiguous(memory_format=torch.channels_last)
    g32, g16 = b.new_grad_arenas()
    b.bind_grads(g32, g16)
    with torch.no_grad():
        L.flatten_into(b.params_f32, ref)
    out = m(torch.randn(2, 3, 32, 32))
    out.sum().backward()
    assert float(g32.abs().sum()) > 0                           # autograd accumulated into the arena
    assert g32[~torch.from_numpy(L.valid_mask())].abs().sum() == 0   # padding untouched


def test_binder_bf16_policy_on_cpu():
    m = ResNet18()
    L = ArenaLayout.from_model(m, bf16=True)
    bn = [s for s in L.specs if "bn" in s.name or "shortcut.1" in s.name]
    assert bn and all(not s.is_bf16 for s in bn)
    assert all(s.is_bf16 for s in L.specs if "conv" in s.name or s.name.startswith("linear"))
    b = ModelBinder(m, L, "cpu", bf16=True)
    assert m.conv1.weight.dtype == torch.bfloat16 and m.bn1.weight.dtype == torch.float32
    assert m.bn1.running_mean.dtype == torch.float32
