"""CPU checks of the arithmetic the tensor-core paths rely on (no GPU, no oracle):

* BF16x3 (csrc/mlp_tc_full.cuh): x = b0 + b1 + b2 with round-to-nearest bf16 planes leaves a residual <= 2^-24 |x|, and
  the six product terms of order <= 2 reproduce x*y to <= 2^-23 relative -- FP32-level, better than 3xTF32.
* 3xTF32 (csrc/mma_tiles.cuh, mlp_tc.cuh): hi = round-to-nearest (ties away) onto the TF32 grid by integer add + mask,
  lo = x - hi exact; hi*hi + hi*lo + lo*hi is within 2^-21 of x*y.
* Truncating accumulation: adding N equal-sign terms into an FP32 accumulator with round-toward-zero loses ~N * 2^-25
  relative -- the reason the tensor-core weight gradients are added into an FP32 round-to-nearest partial every
  horizon step (DESIGN.md 3).
"""
import numpy as np
import torch


def _bf16(x):
    return x.to(torch.bfloat16).to(torch.float32)


def _split3(x):
    b0 = _bf16(x)
    r1 = x - b0
    b1 = _bf16(r1)
    r2 = r1 - b1
    return b0, b1, _bf16(r2)


def _tf32_split(x):
    bits = x.view(torch.int32)
    hi = ((bits + 0x1000) & ~0x1FFF).view(torch.float32)      # == (bits + 0x1000) & 0xffffe000
    return hi, x - hi


def test_bf16x3_split_and_six_term_product():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(200000, generator=g) * torch.exp(torch.randn(200000, generator=g) * 3)
    y = torch.randn(200000, generator=g) * torch.exp(torch.randn(200000, generator=g) * 3)
    xs, ys = _split3(x), _split3(y)
    res = (x.double() - sum(p.double() for p in xs)).abs() / x.double().abs()
    assert float(res.max()) <= 2.0 ** -24
    terms = [(0, 0), (0, 1), (1, 0), (1, 1), (0, 2), (2, 0)]
    prod = sum(xs[i].double() * ys[j].double() for i, j in terms)
    rel = (prod - x.double() * y.double()).abs() / (x.double() * y.double()).abs()
    assert float(rel.max()) <= 2.0 ** -23, float(rel.max())
    # every partial product of two bf16 values is exact in fp32 (8 + 8 significant bits)
    p00 = xs[0] * ys[0]
    assert torch.equal(p00.double(), xs[0].double() * ys[0].double())


def test_3xtf32_split_product():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(200000, generator=g) * 7
    y = torch.randn(200000, generator=g) * 0.3
    xh, xl = _tf32_split(x)
    yh, yl = _tf32_split(y)
    assert torch.equal((xh + xl), x)                                   # exact split
    assert int((xh.view(torch.int32) & 0x1FFF).abs().max()) == 0       # hi on the TF32 grid
    assert float((xl.abs() / x.abs()).max()) <= 2.0 ** -11 + 1e-12     # round-to-nearest: |lo| <= ulp_tf32 / 2
    # the tensor core truncates the lo operands to TF32 as well
    trunc = lambda t: (t.view(torch.int32) & ~0x1FFF).view(torch.float32)
    prod = xh.double() * yh.double() + xh.double() * trunc(yl).double() + trunc(xl).double() * yh.double()
    rel = (prod - x.double() * y.double()).abs() / (x.double() * y.double()).abs()
    assert float(rel.max()) <= 2.0 ** -20, float(rel.max())


def test_truncating_accumulation_bias_grows_with_chain_length():
    """Round-toward-zero accumulation (what a tensor core does when it adds a product into its accumulator): the relative
    loss of a sum of N positive terms grows ~ N * 2^-25; 128-long chains stay at the 1e-6 level, 1e4-long ones reach 1e-4."""
    rng = np.random.default_rng(2)

    def rz_sum(terms):
        acc = np.float32(0.0)
        for t in terms:
            exact = np.float64(acc) + np.float64(t)
            r = np.float32(exact)
            if abs(np.float64(r)) > abs(exact):              # round-to-nearest went away from zero: step back
                r = np.nextafter(r, np.float32(0.0), dtype=np.float32)
            acc = r
        return np.float64(acc)

    def rel_loss(n):
        t = (1.0 + rng.random(n)).astype(np.float32)
        return (np.sum(t.astype(np.float64)) - rz_sum(t)) / np.sum(t.astype(np.float64))

    short, long_ = rel_loss(128), rel_loss(13000)
    assert 0 <= short < 8e-6
    assert 5e-5 < long_ < 1e-3
    assert long_ > 20 * short


def test_bf16x3_mlp_forward_emulation_is_fp32_accurate():
    """The wgmma rollout path's layer arithmetic emulated on the CPU (bf16x3 planes of activations and weights, six
    product terms, FP32-or-better accumulation): a 7 -> 64 -> 64 -> 1 gelu policy stays within 2e-6 of float64 --
    the same margin the GPU parity tests hold -- while plain bf16 operands are
    three orders of magnitude worse (SURVEY F8: why a split is needed at all)."""
    g = torch.Generator().manual_seed(3)
    B = 4096
    x = torch.randn(B, 7, generator=g) * 1.5
    W1, b1 = torch.randn(64, 7, generator=g) * 0.4, torch.randn(64, generator=g) * 0.1
    W2, b2 = torch.randn(64, 64, generator=g) * 0.15, torch.randn(64, generator=g) * 0.1
    W3, b3 = torch.randn(1, 64, generator=g) * 0.2, torch.randn(1, generator=g) * 0.1
    gelu = torch.nn.functional.gelu

    def mm6(a, w):          # a [B, K], w [N, K]: six-term BF16x3 product, accumulated in float64, rounded to fp32
        as_, ws = _split3(a), _split3(w)
        acc = sum(as_[i].double() @ ws[j].double().T for i, j in [(2, 0), (0, 2), (1, 1), (1, 0), (0, 1), (0, 0)])
        return acc.float()

    def mm1(a, w):          # single bf16 plane
        return (_bf16(a).double() @ _bf16(w).double().T).float()

    def net(mm):
        h1 = gelu(mm(x, W1) + b1)
        h2 = gelu(mm(h1, W2) + b2)
        return (h2 @ W3.T + b3).double()

    ref = (gelu(gelu(x.double() @ W1.double().T + b1.double()) @ W2.double().T + b2.double()) @ W3.double().T
           + b3.double())
    err3 = float((net(mm6) - ref).abs().max())
    err1 = float((net(mm1) - ref).abs().max())
    assert err3 < 2e-6, err3
    assert err1 > 100 * err3, (err1, err3)
