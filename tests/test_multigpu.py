"""Multi-GPU tests (run under torchrun on >= 2 GPUs; collected but skipped elsewhere).

    torchrun --nproc-per-node 2 --master-addr 127.0.0.1 -m pytest tests/test_multigpu.py -m multigpu -q

Covers: peer-memory collectives vs NCCL, FSDP / TP / CP parity against a single-GPU run of the same model."""
import os

import pytest
import torch
import torch.distributed as dist

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]

WORLD = int(os.environ.get("WORLD_SIZE", "1"))


@pytest.fixture(scope="module", autouse=True)
def _pg():
    if WORLD < 2:
        pytest.skip("launch with torchrun on >= 2 GPUs")
    rank = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(rank)
    if not dist.is_initialized():
        dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    yield
    dist.barrier()


def _dev():
    return torch.device("cuda", int(os.environ["LOCAL_RANK"]))


def test_symm_collectives_match_nccl():
    from torchacc_b200.parallel.symm_mem import SymmCollectives, symm_available
    g = dist.group.WORLD
    assert symm_available(g)
    c = SymmCollectives(g, WORLD, dist.get_rank(), _dev())
    torch.manual_seed(dist.get_rank())
    for n in (4096, 1 << 20, (1 << 22) + 1024):
        shard = c.alloc(n, torch.bfloat16)
        shard.copy_(torch.randn(n, device=_dev()).bfloat16())
        full = torch.empty(n * WORLD, dtype=torch.bfloat16, device=_dev())
        ref = torch.empty_like(full)
        c.all_gather(shard, full)
        dist.all_gather_into_tensor(ref, shard)
        assert torch.equal(full, ref), f"all_gather n={n}"
        big = c.alloc(n * WORLD, torch.bfloat16)
        big.copy_(torch.randn(n * WORLD, device=_dev()).bfloat16())
        out = torch.empty(n, dtype=torch.float32, device=_dev())
        c.reduce_scatter(big, out, 1.0 / WORLD)
        tmp = big.float() / WORLD
        ref32 = torch.empty(n, dtype=torch.float32, device=_dev())
        dist.reduce_scatter_tensor(ref32, tmp)
        assert torch.allclose(out, ref32, atol=1e-5, rtol=1e-5), f"reduce_scatter n={n}"
        inp = torch.randn(n * WORLD, device=_dev()).bfloat16()
        o1, o2 = torch.empty_like(inp), torch.empty_like(inp)
        c.all_to_all(inp, o1)
        dist.all_to_all_single(o2, inp)
        assert torch.equal(o1, o2), f"all_to_all n={n}"
    t = torch.full((5,), float(dist.get_rank() + 1), device=_dev())
    c.all_reduce(t)
    assert torch.allclose(t, torch.full_like(t, WORLD * (WORLD + 1) / 2))
    big = torch.randn(8 * WORLD * 40000, device=_dev())
    ref = big.clone()
    c.all_reduce(big)
    dist.all_reduce(ref)
    assert torch.allclose(big, ref, atol=1e-4, rtol=1e-4)


def test_carried_collectives_match_reference():
    """Parameter all-gather and gradient reduce-scatter carried by wgmma GEMM launches (csrc/fused/carry.cuh): results
    equal the NCCL collectives, the GEMMs that carried them are still correct, the fused sum of squares matches, and
    the counters prove slices really rode inside GEMM kernels (not only in the stand-alone flush)."""
    from torchacc_b200.ops.linear import gemm
    from torchacc_b200.parallel.carry import BACKGROUND, CarryRuntime, make_carry
    from torchacc_b200.parallel.symm_mem import SymmCollectives, symm_available
    from torchacc_b200 import _native as nat
    g = dist.group.WORLD
    assert symm_available(g)
    c = SymmCollectives(g, WORLD, dist.get_rank(), _dev())
    rt = make_carry(c, _dev())
    assert rt is not None
    prev_sched = nat.require().tb_gemm_sched_mode(-1)
    nat.set_gemm_scheduler(False)
    torch.manual_seed(100 + dist.get_rank())
    n = (6 << 20) + 128 * 7                      # elements per shard; not a multiple of the 8 KB chunk
    shard = c.alloc(n, torch.bfloat16)
    shard.copy_(torch.randn(n, device=_dev()).bfloat16())
    grads = c.alloc(n * WORLD, torch.bfloat16)
    grads.copy_(torch.randn(n * WORLD, device=_dev()).bfloat16())
    full = torch.zeros(n * WORLD, dtype=torch.bfloat16, device=_dev())
    out = torch.full((n,), 7.0, dtype=torch.float32, device=_dev())
    a = torch.randn(4096, 4096, device=_dev()).bfloat16()
    b = torch.randn(4096, 4096, device=_dev()).bfloat16()
    ref_y = (a.float() @ b.float().t())
    CarryRuntime.counters(reset=True)
    rt.arm_stats()
    rt.publish_params()                           # "my shards are final" (once per step in the engine)
    jg = rt.push_gather(shard, full)
    e = rt.publish_grads()                        # "my gradient buffer is final" ...
    ys0 = gemm(a, b)                              # ... the job may be enqueued later than that
    jr = rt.push_reduce(grads, out, 1.0 / WORLD, accumulate=False, epoch=e)
    ys = [gemm(a, b) for _ in range(6)]           # 6 x 137 GFLOP: carries most of the 2 x 12 MB x (W-1)
    rt.flush()                                    # whatever is left
    rt.wait_done(jg[1], jg[2])
    rt.wait_done(jr[1], jr[2])
    torch.cuda.synchronize()
    cnt = CarryRuntime.counters()
    assert cnt["chunks_carried"] > 0 and cnt["launches_carrying"] > 0, cnt
    ref_full = torch.empty_like(full)
    dist.all_gather_into_tensor(ref_full, shard)
    assert torch.equal(full, ref_full)
    ref_out = torch.empty(n, dtype=torch.float32, device=_dev())
    dist.reduce_scatter_tensor(ref_out, grads.float() / WORLD)
    assert torch.allclose(out, ref_out, atol=1e-5, rtol=1e-5), float((out - ref_out).abs().max())
    assert torch.allclose(rt.stats[0], (ref_out.double() ** 2).sum().float(), rtol=1e-4), (rt.stats, (ref_out ** 2).sum())
    assert float(rt.stats[1]) == 0.0
    for y in ys + [ys0]:
        assert torch.allclose(y.float(), ref_y, atol=2.0, rtol=2e-2)
    # accumulate into the existing shard + everything through the stand-alone kernel
    jr2 = rt.push_reduce(grads, out, 1.0 / WORLD, accumulate=True, epoch=rt.publish_grads())
    rt.flush(jr2[0], BACKGROUND)
    rt.wait_done(jr2[1], jr2[2])
    torch.cuda.synchronize()
    assert torch.allclose(out, 2 * ref_out, atol=2e-5, rtol=1e-5)
    nat.set_gemm_scheduler(bool(prev_sched))


def _tiny(dtype=torch.bfloat16):
    from torchacc_b200.models import build_llama
    torch.manual_seed(0)
    with torch.device(_dev()):
        return build_llama("tiny", hidden_size=512, intermediate_size=1024, num_hidden_layers=2, num_attention_heads=8,
                           num_key_value_heads=2 * max(1, WORLD // 2), head_dim=64, vocab_size=2048,
                           max_position_embeddings=512, dtype=dtype)


def _train(cfg_fn, steps=4, split_batch=True):
    import torchacc_b200 as ta
    model = _tiny()
    cfg = ta.Config()
    cfg.compute.bf16 = True
    cfg_fn(cfg)
    model = ta.accelerate(model, config=cfg)
    opt = ta.optim.FusedAdamW(model.parameters(), lr=1e-3)
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 2048, (2 * WORLD, 128), generator=g).to(_dev())
    local = ids.chunk(WORLD)[dist.get_rank()] if split_batch else ids
    losses = []
    for _ in range(steps):
        out = model(input_ids=local, labels=local)
        out["loss"].backward()
        model.clip_grad_norm_(1.0)
        opt.step()
        model.zero_grad()
        l = out["loss"].detach().float().clone()
        if split_batch:
            dist.all_reduce(l)
            l /= WORLD
        losses.append(float(l))
    return losses


def _single_gpu_reference(steps=4):
    """Same model/data on one GPU (every rank computes it redundantly with a private, non-distributed config)."""
    import torchacc_b200 as ta
    from torchacc_b200.parallel.fsdp import ShardingEngine, shard_model
    model = _tiny()
    eng = ShardingEngine(_dev(), compute_dtype=torch.bfloat16, strategy="NO_SHARD", grad_mode="compat")
    from torchacc_b200.models import LlamaDecoderLayer
    root = shard_model(model, eng, (LlamaDecoderLayer,), ())
    opt = ta.optim.FusedAdamW(eng.flat_parameters(), lr=1e-3)
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 2048, (2 * WORLD, 128), generator=g).to(_dev())
    losses = []
    for _ in range(steps):
        out = root(input_ids=ids, labels=ids)
        out["loss"].backward()
        eng.clip_grad_norm_(1.0)
        opt.step()
        eng.zero_grad()
        losses.append(float(out["loss"]))
    return losses


def test_fsdp_matches_single_gpu():
    ref = _single_gpu_reference()

    def cfg(c):
        c.dist.fsdp.size = WORLD
        c.dist.fsdp.wrap_layer_cls = {"LlamaDecoderLayer"}
        c.memory.gc = True
    got = _train(cfg)
    assert all(abs(a - b) < 5e-2 for a, b in zip(got, ref)), (got, ref)
    assert got[-1] < got[0]


def test_fsdp_nccl_fallback_matches():
    ref = _single_gpu_reference()

    def cfg(c):
        c.dist.fsdp.size = WORLD
        c.dist.fsdp.wrap_layer_cls = {"LlamaDecoderLayer"}
        c.dist.fsdp.fused_collectives = False
    got = _train(cfg)
    assert all(abs(a - b) < 5e-2 for a, b in zip(got, ref)), (got, ref)


def test_tensor_parallel_matches_single_gpu():
    ref = _single_gpu_reference()

    def cfg(c):
        c.dist.tp.size = WORLD
    got = _train(cfg, split_batch=False)
    assert all(abs(a - b) < 5e-2 for a, b in zip(got, ref)), (got, ref)


@pytest.mark.parametrize("mode", ["ulysses", "ring"])
def test_context_parallel_matches_single_gpu(mode):
    ref = _single_gpu_reference(steps=2)

    def cfg(c):
        c.dist.sp.size = WORLD
        c.dist.sp.mode = mode
    import torchacc_b200 as ta
    got = _train(cfg, steps=2, split_batch=False)
    # each rank reports the loss of its sequence shard: average over the group
    t = torch.tensor(got, device=_dev())
    dist.all_reduce(t)
    got = (t / WORLD).tolist()
    assert all(abs(a - b) < 6e-2 for a, b in zip(got, ref)), (got, ref)


def test_fused_tp_kernels_match_unfused():
    """all-gather->GEMM and GEMM->reduce-scatter (one kernel each, peer memory) vs NCCL collective + plain GEMM."""
    from torchacc_b200.parallel.fused_tp import make_fused_tp
    f = make_fused_tp(dist.group.WORLD, _dev())
    assert f is not None
    torch.manual_seed(100 + dist.get_rank())
    rows, K, N = 512, 1024, 768
    for it in range(3):   # several calls: exercises buffer / counter / epoch reuse
        x = (torch.randn(rows, K, device=_dev()) * 0.5).bfloat16()
        torch.manual_seed(7 + it)
        w = (torch.randn(N, K, device=_dev()) * 0.05).bfloat16()     # same weight on every rank
        y, xf = f.ag_gemm(x, w)
        ref_x = torch.empty(rows * WORLD, K, dtype=torch.bfloat16, device=_dev())
        dist.all_gather_into_tensor(ref_x, x)
        assert torch.equal(xf, ref_x), "gathered activation differs"
        ref_y = ref_x.float() @ w.float().t()
        assert torch.allclose(y.float(), ref_y, atol=0.15, rtol=3e-2), float((y.float() - ref_y).abs().max())
        # MN-major B (the dgrad form): y2 = gather(x) @ w2 with w2 stored [K, N2]
        w2 = (torch.randn(K, 512, device=_dev()) * 0.05).bfloat16()
        dist.broadcast(w2, 0)
        y2, _ = f.ag_gemm(x, w2, b_mn_major=True)
        assert torch.allclose(y2.float(), ref_x.float() @ w2.float(), atol=0.15, rtol=3e-2)
        # GEMM -> reduce-scatter
        torch.manual_seed(200 + dist.get_rank() + 10 * it)
        a = (torch.randn(rows * WORLD, K, device=_dev()) * 0.5).bfloat16()
        wl = (torch.randn(N, K, device=_dev()) * 0.05).bfloat16()
        res = torch.randn(rows, N, device=_dev()).bfloat16()
        out = f.gemm_rs(a, wl, residual=res)
        part = (a.float() @ wl.float().t()).bfloat16().float()
        ref = torch.empty(rows, N, device=_dev())
        dist.reduce_scatter_tensor(ref, part)
        ref = ref + res.float()
        assert torch.allclose(out.float(), ref, atol=0.25, rtol=3e-2), float((out.float() - ref).abs().max())


def test_pipeline_parallel_matches_single_gpu():
    """1F1B over NCCL p2p (activations and gradients on separate communicators: one communicator runs its p2p
    operations in issue order, and early-posted receives would otherwise deadlock the 2-stage schedule)."""
    import torchacc_b200 as ta
    ref = _single_gpu_reference(steps=3)
    model = _tiny()
    cfg = ta.Config()
    cfg.compute.bf16 = True
    cfg.dist.pp.size = WORLD
    cfg.dist.pp.num_micro_batches = 2
    cfg.dist.pp.split_points = [f"model.layers.{max(1, i * 2 // WORLD)}" for i in range(1, WORLD)] if WORLD == 2 else None
    if WORLD != 2:
        pytest.skip("the tiny 2-layer model splits into exactly 2 stages")
    model = ta.accelerate(model, config=cfg)
    opt = ta.optim.FusedAdamW(model.parameters(), lr=1e-3)
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 2048, (2 * WORLD, 128), generator=g).to(_dev())
    losses = []
    for _ in range(3):
        loss = model.forward_backward(input_ids=ids, labels=ids, output_fn=lambda out: out["loss"])
        model.clip_grad_norm_(1.0)
        opt.step()
        model.zero_grad()
        t = torch.zeros(1, device=_dev()) if loss is None else loss.detach().float().reshape(1).clone()
        dist.all_reduce(t, op=dist.ReduceOp.MAX)     # only the last stage holds the loss (it is positive)
        losses.append(float(t))
    assert all(abs(a - b) < 6e-2 for a, b in zip(losses, ref)), (losses, ref)
