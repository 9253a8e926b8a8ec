"""Layer-wise wgmma MLP (csrc/dense_tc.cu, BF16x3) against a plain PyTorch reference of the same network evaluated in
fp64: outputs, parameter gradients (torch flat order) and input gradients, ragged batches, widths that are not
multiples of the tile sizes, gradient accumulation, several live forward passes (slots).
Bars: outputs 4e-6 relative to the output scale (FP32-accurate six-term products; FP32 accumulation over up to 256
inputs per layer, three layers), gradients 1e-4 relative L2
(two-plane deltas, three-term products)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ACTS = {"relu": torch.nn.ReLU, "gelu": torch.nn.GELU, "elu": torch.nn.ELU, "tanh": torch.nn.Tanh}


def _ref_net(sizes, act, seed):
    torch.manual_seed(seed)
    layers = []
    for j in range(len(sizes) - 1):
        layers.append(torch.nn.Linear(sizes[j], sizes[j + 1]))
        if j < len(sizes) - 2:
            layers.append(ACTS[act]())
    return torch.nn.Sequential(*layers)


@pytest.mark.parametrize("sizes,act,B", [
    ([7, 256, 256, 256, 2], "gelu", 1000),        # DSAC-shaped (obs + act -> mean, std)
    ([247, 256, 256, 2], "elu", 8192),            # C3 policy (obs 246 + time)
    ([6, 64, 64, 30], "relu", 333),               # FiniteHorizonFullPolicy-shaped: act_dim * pre_horizon outputs
    ([19, 100, 37, 5], "tanh", 129),              # nothing aligned
    ([4, 256, 1], "gelu", 1),
])
def test_forward_backward_against_fp64(sizes, act, B):
    from gops_b200.ops.layerwise_mlp import LayerwiseMlp
    ref = _ref_net(sizes, act, seed=B)
    flat = torch.cat([p.detach().reshape(-1) for p in ref.parameters()]).cuda()
    net = LayerwiseMlp(sizes, act, max_batch=B, slots=2)
    assert net.nparam == flat.numel()
    net.pack(flat)
    g = torch.Generator().manual_seed(B + 1)
    x = torch.randn(B, sizes[0], generator=g)
    dy = torch.randn(B, sizes[-1], generator=g) / B
    ref64 = ref.double()
    x64 = x.double().requires_grad_(True)
    y64 = ref64(x64)
    (y64 * dy.double()).sum().backward()
    xg = x.cuda()
    y = net.forward(xg, slot=1)
    scale = float(y64.abs().max())
    assert float((y.cpu().double() - y64.detach()).abs().max()) <= 4e-6 * max(1.0, scale)
    grad = torch.zeros(net.nparam, device="cuda")
    dx = net.backward(dy.cuda(), slot=1, grad=grad, want_dx=True)
    torch.cuda.synchronize()
    g64 = torch.cat([p.grad.reshape(-1) for p in ref64.parameters()])
    err = float((grad.cpu().double() - g64).norm() / g64.norm())
    assert err < 1e-4, err
    errx = float((dx.cpu().double() - x64.grad).norm() / x64.grad.norm())
    assert errx < 1e-4, errx
    # accumulate on top, from a second live forward pass in another slot
    x2 = torch.randn(B, sizes[0], generator=g).cuda()
    net.forward(x2, slot=0)
    net.backward(dy.cuda(), slot=0, grad=grad, accumulate=True)
    x264 = x2.cpu().double()
    for p in ref64.parameters():
        p.grad = None
    (ref64(x264) * dy.double()).sum().backward()
    g64b = g64 + torch.cat([p.grad.reshape(-1) for p in ref64.parameters()])
    assert float((grad.cpu().double() - g64b).norm() / g64b.norm()) < 1e-4


def test_deterministic_and_inference_mode():
    from gops_b200.ops.layerwise_mlp import LayerwiseMlp
    sizes, B = [7, 256, 256, 256, 2], 4096
    ref = _ref_net(sizes, "gelu", 3)
    flat = torch.cat([p.detach().reshape(-1) for p in ref.parameters()]).cuda()
    net = LayerwiseMlp(sizes, "gelu", max_batch=B)
    net.pack(flat)
    x = torch.randn(B, 7, generator=torch.Generator().manual_seed(1)).cuda()
    dy = torch.randn(B, 2, generator=torch.Generator().manual_seed(2)).cuda()
    g1, g2 = torch.zeros(net.nparam, device="cuda"), torch.zeros(net.nparam, device="cuda")
    y1 = net.forward(x).clone()
    net.backward(dy, grad=g1)
    y2 = net.forward(x)
    net.backward(dy, grad=g2)
    assert torch.equal(y1, y2) and torch.equal(g1, g2)
    y3 = net.forward(x, train=False)
    assert torch.equal(y1, y3)
