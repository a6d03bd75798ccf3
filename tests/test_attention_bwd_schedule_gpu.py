"""The head-dim-64 main backward kernel (128-row query tiles) at the shapes that reach the edges of its schedule: the
Q/dO ring wrapping after 1, 2 and 3 iterations, GQA groups, ragged varlen sequences, a sliding window and Sq != Sk,
plus the flagship attention shape.  On each: dK and dV bitwise equal between the default and the deterministic
backward (they share the kernel's dK / dV arithmetic), and dQ / dK / dV within the fp64-derived bounds of
test_attention_kernels_gpu.py."""
import pytest
import torch

from test_attention_kernels_gpu import _case, _fixed

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _native_backend():
    from torchacc_b200.ops import attention as A
    A.set_attention_backend("native")
    yield
    A.set_attention_backend("auto")


def _both(tag, cu_q, cu_k, Hq, Hk, causal=True, window=(-1, -1), regime="peaked", dtype=torch.bfloat16, seed=0):
    _case(tag, cu_q, cu_k, Hq, Hk, 64, dtype, causal, window, regime, dets=(False, True), seed=seed)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("n_iter", [1, 2, 3])
def test_ring_wrap(n_iter, dtype):
    """Every CTA runs n_iter iterations (non-causal, one q head per kv head, n_iter query tiles; the last one ragged),
    so the 2-stage Q/dO ring and the double-buffered dQ staging end in every phase."""
    cu_q, cu_k = _fixed(2, 128 * n_iter - 5, 200)
    _both(f"wrap n={n_iter} {str(dtype)[6:]}", cu_q, cu_k, 2, 2, causal=False, dtype=dtype, seed=n_iter)


@pytest.mark.parametrize("group", [1, 4, 8])
def test_gqa_group(group):
    cu_q, cu_k = _fixed(2, 300, 300)
    _both(f"gqa group={group}", cu_q, cu_k, 8, 8 // group, seed=group)


def test_ragged_varlen():
    lens = [37, 200, 5, 300, 128, 1, 129]
    cu = [0] + torch.tensor(lens).cumsum(0).tolist()
    _both("varlen", cu, cu, 4, 2, regime="probe", seed=5)


def test_sliding_window():
    cu_q, cu_k = _fixed(2, 600, 600)
    _both("window (100, 0)", cu_q, cu_k, 4, 2, window=(100, 0), seed=6)


@pytest.mark.parametrize("sq,sk", [(200, 520), (520, 200)])
def test_sq_ne_sk(sq, sk):
    cu_q, cu_k = _fixed(2, sq, sk)
    _both(f"Sq={sq} Sk={sk}", cu_q, cu_k, 4, 2, seed=sq)


def test_flagship_attention_shape():
    """B = 2, S = 4096, 32 query / 8 kv heads, D = 64, causal: the attention shape of the default benchmark."""
    cu_q, cu_k = _fixed(2, 4096, 4096)
    _both("flagship D=64", cu_q, cu_k, 32, 8, regime="flat", seed=1)
