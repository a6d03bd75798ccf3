"""``moe_experts_mxfp8_reference`` (the PyTorch emulation of the MX-FP8 experts, the oracle of test_moe_fp8_gpu.py)
against the fp32 ``moe_experts_reference``, on the CPU."""
import math

import torch

from torchacc_b200.ops.moe import moe_experts_mxfp8_reference, moe_experts_reference


def _exact_case(T=64, H=128, Fd=128, E=4, k=2, seed=0):
    """Inputs on which every rounding of the fp8 path is exact, so both references must agree bit for bit:
    x[t] = 1 at feature 0 and +-1 at one other feature; gate rows (64, 0, ...), so g = 64 and silu(g) = 64 in fp32;
    up rows (a, 0, ...) with a in {0, +-1, +-2, +-4}, so h = 64 a; one weight of +-1 or +-2 per down-projection row, so
    y has at most 4 significant bits; routing weights 3/4 and 1/4.  Every GEMM operand is then q 2^s with |q| <= 8 (or
    a power of two), which the quantiser represents exactly, and every sum is exact in bf16."""
    g = torch.Generator().manual_seed(seed)
    x = torch.zeros(T, H)
    x[:, 0] = 1
    j = torch.randint(1, H, (T,), generator=g)
    x[torch.arange(T), j] = torch.randint(0, 2, (T,), generator=g).float() * 2 - 1
    wgu = torch.zeros(E, 2 * Fd, H)
    wgu[:, :Fd, 0] = 64
    choices = torch.tensor([0.0, 1, -1, 2, -2, 4, -4])
    wgu[:, Fd:, 0] = choices[torch.randint(0, len(choices), (E, Fd), generator=g)]
    wd = torch.zeros(E, H, Fd)
    cols = torch.stack([torch.randperm(Fd, generator=g)[:H] if H <= Fd else torch.randint(0, Fd, (H,), generator=g)
                        for _ in range(E)])
    vals = torch.tensor([1.0, -1, 2, -2])[torch.randint(0, 4, (E, H), generator=g)]
    wd.scatter_(2, cols[:, :, None], vals[:, :, None])
    ids = torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(T)])
    w = torch.tensor([0.75, 0.25]).expand(T, k).contiguous()
    bf = torch.bfloat16
    return x.to(bf), ids, w, wgu.to(bf), wd.to(bf)


def test_mxfp8_reference_equals_bf16_reference_on_exact_inputs():
    x, ids, w, wgu, wd = _exact_case()
    got = moe_experts_mxfp8_reference(x, ids, w, wgu, wd)
    ref = moe_experts_reference(x, ids, w, wgu, wd)
    assert got.dtype == ref.dtype == torch.bfloat16
    assert torch.equal(got, ref)
    assert ref.abs().max() > 0
    ids2 = ids.clone()
    ids2[::5, 1] = 4                                                  # HF's "no expert" sentinel adds nothing
    assert torch.equal(moe_experts_mxfp8_reference(x, ids2, w, wgu, wd), moe_experts_reference(x, ids2, w, wgu, wd))


def test_mxfp8_reference_gradients_close_to_fp32_autograd():
    """On Gaussian data the emulated fp8 experts stay within a relative norm of 0.085 of the fp32 ones: sqrt(2) times
    the 0.06 bound of one fp8 linear layer, since every output goes through two chained fp8 GEMMs with independent
    quantisation errors.  A wrong expert, transpose or scale orientation would be off by O(1)."""
    torch.manual_seed(0)
    T, H, Fd, E, k = 256, 128, 128, 4, 2
    x = torch.randn(T, H).bfloat16()
    w, ids = torch.topk(torch.softmax(torch.randn(T, E), -1), k, -1)
    w = w / w.sum(-1, keepdim=True)
    wgu = (torch.randn(E, 2 * Fd, H) / math.sqrt(H)).bfloat16()
    wd = (torch.randn(E, H, Fd) / math.sqrt(Fd)).bfloat16()
    dout = torch.randn(T, H).bfloat16()
    out, dx, dw, dgu, dd = moe_experts_mxfp8_reference(x, ids, w, wgu, wd, dout=dout)
    leaves = [t.float().requires_grad_(True) for t in (x, w, wgu, wd)]
    ref = moe_experts_reference(leaves[0], ids, leaves[1], leaves[2], leaves[3])
    ref.backward(dout.float())
    for name, a, b in (("out", out, ref.detach()), ("dx", dx, leaves[0].grad), ("dweights", dw, leaves[1].grad),
                       ("dW_gate_up", dgu, leaves[2].grad), ("dW_down", dd, leaves[3].grad)):
        rel = float((a.double() - b.double()).norm() / b.double().norm())
        assert rel < 0.085, (name, rel)
