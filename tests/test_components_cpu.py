"""CPU unit tests: AsyncLoader bucketing, PP schedules, checkpoint surgery, reference-path ops, amp, offload API."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

import torchacc_b200 as ta


# ---- AsyncLoader -------------------------------------------------------------------------------------------------
def test_async_loader_bucketing_and_order():
    batches = [{"input_ids": torch.full((2, n), i), "attention_mask": torch.ones(2, n, dtype=torch.long),
                "labels": torch.full((2, n), i)} for i, n in enumerate([5, 17, 33, 64, 70])]
    loader = ta.AsyncLoader(batches, torch.device("cpu"), buckets=[16, 32, 64])
    out = list(loader)
    assert len(out) == len(loader) == 5
    assert [b["input_ids"].shape[-1] for b in out] == [16, 32, 64, 64, 70]    # 70 opens a new bucket
    for i, b in enumerate(out):
        n = [5, 17, 33, 64, 70][i]
        assert (b["input_ids"][:, :n] == i).all() and (b["input_ids"][:, n:] == 0).all()
        assert (b["labels"][:, n:] == -100).all() and (b["attention_mask"][:, n:] == 0).all()


def test_async_loader_uniform_buckets_and_tuples():
    from torchacc_b200.core.async_loader import closest_bucket, uniform_buckets
    assert uniform_buckets(128, 4) == [32, 64, 96, 128]
    assert closest_bucket([32, 64, 96, 128], 65) == 96
    data = [(torch.randn(3, 40), torch.tensor([1, 2, 3])) for _ in range(3)]
    out = list(ta.AsyncLoader(data, torch.device("cpu"), max_length=128, num_buckets=4, pad_value_dict={}))
    assert out[0][0].shape == (3, 64) and out[0][1].shape == (3,)
    # no bucketing configured: batches pass through untouched
    out = list(ta.AsyncLoader(data, torch.device("cpu")))
    assert out[0][0].shape == (3, 40)


def test_async_loader_propagates_errors():
    def gen():
        yield {"x": torch.zeros(2, 4)}
        raise RuntimeError("boom")
    it = iter(ta.AsyncLoader(gen(), torch.device("cpu")))
    next(it)
    with pytest.raises(RuntimeError, match="boom"):
        next(it)


# ---- pipeline schedules -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("stages,mbs", [(2, 4), (4, 4), (4, 8), (3, 2), (4, 1)])
@pytest.mark.parametrize("algo", ["1f1b", "gpipe"])
def test_pipeline_schedule_is_consistent(stages, mbs, algo):
    """Simulate all stages: every send has a matching posted receive in order, each micro-batch is forwarded before
    it is backwarded, and the simulation never deadlocks."""
    from torchacc_b200.parallel.pp import schedule as S
    streams = [[ins for step in S.create_scheduler(algo, True, mbs, stages, s) for ins in step] for s in range(stages)]
    pos = [0] * stages
    act_q = [[] for _ in range(stages)]    # activations in flight towards stage i
    grad_q = [[] for _ in range(stages)]   # gradients in flight towards stage i
    fwd_done = [set() for _ in range(stages)]
    bwd_done = [set() for _ in range(stages)]
    progressed = True
    while progressed:
        progressed = False
        for s in range(stages):
            while pos[s] < len(streams[s]):
                ins = streams[s][pos[s]]
                if isinstance(ins, S.WaitRecvActivation):
                    if ins.micro_batch not in act_q[s]:
                        break
                    act_q[s].remove(ins.micro_batch)
                elif isinstance(ins, S.WaitRecvGrad):
                    if ins.micro_batch not in grad_q[s]:
                        break
                    grad_q[s].remove(ins.micro_batch)
                elif isinstance(ins, S.ForwardPass):
                    fwd_done[s].add(ins.micro_batch)
                elif isinstance(ins, S.BackwardPass):
                    assert ins.micro_batch in fwd_done[s]
                    bwd_done[s].add(ins.micro_batch)
                elif isinstance(ins, S.SendActivation):
                    act_q[s + 1].append(ins.micro_batch)
                elif isinstance(ins, S.SendGrad):
                    grad_q[s - 1].append(ins.micro_batch)
                pos[s] += 1
                progressed = True
    for s in range(stages):
        assert pos[s] == len(streams[s]), f"stage {s} stuck at {streams[s][pos[s]]}"
        assert fwd_done[s] == bwd_done[s] == set(range(mbs))


def test_1f1b_buffer_count_and_warmup():
    from torchacc_b200.parallel.pp import schedule as S
    sch = S.OneFOneBTrain(8, 4, 0)
    assert sch.num_pipe_buffers() == 4
    flat = [i for st in sch for i in st]
    first_bwd = next(i for i, x in enumerate(flat) if isinstance(x, S.BackwardPass))
    n_fwd_before = sum(isinstance(x, S.ForwardPass) for x in flat[:first_bwd])
    assert n_fwd_before == 4          # stages - stage_id - 1 warm-up forwards + the first steady-state forward
    assert isinstance(S.create_scheduler(S.Algo.PipeDreamFlush, False, 2, 2, 0), S.ForwardOnly)


def test_microbatch_split():
    import inspect
    from torchacc_b200.parallel.pp.microbatch import bind_args_to_kwargs, split_kwargs_into_chunks

    def f(self, x, y=None, flag=True):
        pass
    kw = bind_args_to_kwargs((torch.arange(8).view(4, 2),), {"y": torch.arange(4)}, inspect.signature(f))
    chunks = split_kwargs_into_chunks({**kw, "flag": False}, 2)
    assert chunks[1]["x"].tolist() == [[4, 5], [6, 7]] and chunks[1]["y"].tolist() == [2, 3] and chunks[0]["flag"] is False
    with pytest.raises(ValueError):
        split_kwargs_into_chunks({"x": torch.zeros(3, 2)}, 2)


# ---- checkpoint surgery ------------------------------------------------------------------------------------------
def _engine_model():
    from torchacc_b200.models import build_llama
    torch.manual_seed(0)
    m = build_llama("tiny", hidden_size=32, intermediate_size=64, num_hidden_layers=2, num_attention_heads=2,
                    num_key_value_heads=1, head_dim=16, vocab_size=64, max_position_embeddings=32)
    cfg = ta.Config()
    cfg.compute.bf16 = True
    cfg.dist.fsdp.wrap_layer_cls = {"LlamaDecoderLayer"}
    return ta.accelerate(m, config=cfg), m


def test_checkpoint_consolidate_and_reshard_roundtrip(tmp_path):
    from torchacc_b200.parallel import state_dict_utils as U
    model, raw = _engine_model()
    opt = torch.optim.AdamW(model.parameters(), lr=1e-2)
    ids = torch.randint(0, 64, (2, 16))
    for _ in range(2):
        model(ids, labels=ids)["loss"].backward()
        opt.step()
        model.zero_grad()
    inner = model._inner_engine_module()
    d = tmp_path / "ckpt"
    d.mkdir()
    torch.save({"model": inner.sharded_state_dict(), "shard_metadata": inner.get_shard_metadata()},
               d / "rank0-of-1-model.pth")
    torch.save(inner.sharded_optim_state_dict(opt), d / "rank0-of-1-optim.pth")
    full = inner.full_state_dict(rank0_only=False)
    # reshard 1 -> 4, then consolidate the 4 shards again: identical tensors
    U.consolidate_and_reshard_fsdp_checkpoint(str(d), "rank*-of-1-model.pth", "rank*-of-1-optim.pth",
                                              save_dir=str(d / "r4"), reshard_num=4)
    files = sorted(os.listdir(d / "r4"))
    assert files == [f"rank{r}-of-4-{k}.pth" for r in range(4) for k in ("model", "optim")] or len(files) == 8
    back, _ = U.consolidate_and_reshard_fsdp_model_dict(str(d / "r4"), "rank*-of-4-model.pth", save_model=False)
    for k, v in full.items():
        assert torch.equal(back[k], v), k
    sm = torch.load(d / "r4" / "rank2-of-4-model.pth", weights_only=False)["shard_metadata"]
    assert sm["world_size"] == 4 and sm["rank"] == 2 and sm["units"][0]["padded"] % (128 * 4) == 0
    fo = inner.full_optim_state_dict(opt, rank0_only=False)
    back_o, _ = U.consolidate_and_reshard_fsdp_optim_dict(str(d / "r4"), "rank*-of-4-optim.pth", save_optimizer=False)
    for name, st in fo["state"].items():
        assert torch.equal(back_o["state"][name]["exp_avg"], st["exp_avg"]), name
    # CLI: consolidate to single files
    from torchacc_b200.utils.consolidate_and_reshard_ckpts import main
    main(["--ckpt_dir", str(d), "--model_ckpt_name_pattern", "rank*-of-1-model.pth", "--optimizer_ckpt_name_pattern",
          "rank*-of-1-optim.pth", "--save_dir", str(d / "full")])
    cons = torch.load(d / "full" / "model_consolidated.pth", weights_only=False)["model"]
    assert all(torch.equal(cons[k], full[k]) for k in full)
    main(["--ckpt_dir", str(d), "--ckpt_type", "optimizer", "--optimizer_ckpt_name_pattern", "rank*-of-1-optim.pth",
          "--save_dir", str(d / "full")])
    assert os.path.exists(d / "full" / "optimizer_consolidated.pth")


def test_optimizer_state_load_roundtrip():
    model, _ = _engine_model()
    opt = torch.optim.AdamW(model.parameters(), lr=1e-2)
    ids = torch.randint(0, 64, (2, 16))
    model(ids, labels=ids)["loss"].backward()
    opt.step()
    model.zero_grad()
    full = model.full_optim_state_dict(opt, rank0_only=False)
    sharded = model.sharded_optim_state_dict(opt)
    model2, _ = _engine_model()
    opt2 = torch.optim.AdamW(model2.parameters(), lr=1e-2)
    opt2.load_state_dict(model2.optim_state_dict_to_load(full, rank0_only=False))
    opt3 = torch.optim.AdamW(model2.parameters(), lr=1e-2)
    opt3.load_state_dict(model2.optim_state_dict_to_load(sharded))
    for a, b, c in zip(opt.state_dict()["state"].values(), opt2.state_dict()["state"].values(),
                       opt3.state_dict()["state"].values()):
        assert torch.equal(a["exp_avg"], b["exp_avg"]) and torch.equal(a["exp_avg_sq"], c["exp_avg_sq"])


@pytest.mark.parametrize("optimizer", ["fused", "torch"])
def test_optimizer_zero_grad_equals_model_zero_grad(optimizer):
    """reference loop (benchmarks/transformer.py:162-184): only ``optimizer.zero_grad()`` is called.  The engine must
    not carry gradient state past it (round-1 advisor finding: stale gradients were summed into the next step)."""
    import torchacc_b200 as ta
    ids = torch.randint(0, 64, (2, 16), generator=torch.Generator().manual_seed(3))

    def run(use_opt_zero):
        model, _ = _engine_model()
        opt = ta.optim.FusedAdamW(model.parameters(), lr=1e-2) if optimizer == "fused" \
            else torch.optim.AdamW(model.parameters(), lr=1e-2)
        norms = []
        for _ in range(3):
            model(ids, labels=ids)["loss"].backward()
            norms.append(float(model.clip_grad_norm_(1e9)))
            opt.step()
            (opt if use_opt_zero else model).zero_grad()
        return norms, [p.detach().clone() for p in model.parameters()]

    n_a, p_a = run(True)
    n_b, p_b = run(False)
    assert n_a == pytest.approx(n_b, rel=1e-6), (n_a, n_b)
    for a, b in zip(p_a, p_b):
        assert torch.equal(a, b)


def test_load_checkpoints_validates_every_shard(tmp_path):
    from torchacc_b200.parallel import state_dict_utils as U
    meta = {"world_size": 2, "rank": 0, "units": [], "pad_multiple": 128}
    torch.save({"model": {}, "shard_metadata": meta}, tmp_path / "rank0-of-2-model.pth")
    torch.save({"model": {}, "shard_metadata": dict(meta, rank=0)}, tmp_path / "rank1-of-2-model.pth")  # wrong rank
    with pytest.raises(ValueError):
        U.load_checkpoints(str(tmp_path), "rank*-of-2-model.pth")


# ---- reference-path ops ------------------------------------------------------------------------------------------
def test_reference_ops_match_torch():
    from torchacc_b200.ops import rmsnorm, swiglu, fused_linear_cross_entropy, rope_tables, rope_qkv_
    x, w = torch.randn(7, 32), torch.rand(32) + 0.5
    y, _ = rmsnorm(x, w, 1e-6)
    assert torch.allclose(y, x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6) * w, atol=1e-5)
    y2, h = rmsnorm(x, w, 1e-6, residual=x)
    assert torch.allclose(h, 2 * x)
    gu = torch.randn(5, 16)
    assert torch.allclose(swiglu(gu), F.silu(gu[:, :8]) * gu[:, 8:], atol=1e-6)
    hid, wt, lab = torch.randn(9, 12), torch.randn(20, 12), torch.randint(0, 20, (9,))
    lab[0] = -100
    assert torch.allclose(fused_linear_cross_entropy(hid, wt, lab), F.cross_entropy(hid @ wt.t(), lab, ignore_index=-100),
                          atol=1e-5)
    cos, sin = rope_tables(16, 8, 10000.0)
    qkv = torch.randn(6, (2 + 2) * 8)
    out = rope_qkv_(qkv.clone(), 2, 1, 8, cos, sin, None, 6)
    assert torch.equal(out[:, 24:], qkv[:, 24:])                       # v untouched
    q0 = qkv[0, :8]
    assert torch.allclose(out[0, :8], q0, atol=1e-6)                    # position 0: identity rotation


def test_attention_reference_masks_and_variants():
    from torchacc_b200.ops import attention as A
    torch.manual_seed(0)
    q, k, v = torch.randn(2, 10, 4, 8), torch.randn(2, 10, 2, 8), torch.randn(2, 10, 2, 8)
    out = A.flash_attn_func(q, k, v, causal=True)
    ref = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2).repeat_interleave(2, 1),
                                         v.transpose(1, 2).repeat_interleave(2, 1), is_causal=True).transpose(1, 2)
    assert torch.allclose(out, ref, atol=1e-5)
    o, lse, _ = A.flash_attn_func(q, k, v, window_size=(2, 0), return_attn_probs=True)
    assert lse.shape == (2, 4, 10)
    mask = torch.tensor([[1] * 10, [1] * 6 + [0] * 4])
    ov = A.flash_attn_varlen_func(q, k, v, mask, causal=True)
    assert torch.allclose(ov[1, :6], A.flash_attn_func(q[1:, :6], k[1:, :6], v[1:, :6], causal=True)[0], atol=1e-5)
    assert (ov[1, 6:] == 0).all()
    pos = torch.cat([torch.arange(4), torch.arange(6)])[None]
    op = A.flash_attn_varlen_position_ids_func(q[:1], k[:1], v[:1], pos, causal=True)
    assert torch.allclose(op[:, 4:], A.flash_attn_func(q[:1, 4:], k[:1, 4:], v[:1, 4:], causal=True), atol=1e-5)
    qkv = torch.stack([q, q, q], 2)
    assert A.flash_attn_varlen_qkvpacked_xla(qkv, mask).shape == q.shape
    assert ta.ops.flash_attn_xla is A.flash_attn_func


def test_sdpa_shim_honours_scale_and_mask():
    from torchacc_b200.ops.sdpa import scaled_dot_product_attention as sdpa
    q, k, v = (torch.randn(1, 2, 6, 8, dtype=torch.bfloat16) for _ in range(3))
    a = sdpa(q, k, v, is_causal=True, scale=0.5)
    b = F.scaled_dot_product_attention(q, k, v, is_causal=True, scale=0.5)
    assert torch.allclose(a.float(), b.float(), atol=3e-2)
    m = torch.ones(6, 6, dtype=torch.bool).tril()
    assert torch.allclose(sdpa(q, k, v, attn_mask=m).float(), F.scaled_dot_product_attention(q, k, v, attn_mask=m).float())


# ---- amp / misc --------------------------------------------------------------------------------------------------
def test_grad_scaler_skips_on_inf_and_backs_off():
    p = torch.nn.Parameter(torch.ones(4))
    opt = ta.optim.FusedAdamW([p], lr=0.1)
    sc = ta.amp.GradScaler(init_scale=8.0, growth_interval=1)
    loss = (p * 2).sum()
    sc.scale(loss).backward()
    assert torch.allclose(p.grad, torch.full((4,), 16.0))
    sc.step(opt)
    sc.update()
    assert sc.get_scale() == 16.0 and not torch.allclose(p.detach(), torch.ones(4))
    before = p.detach().clone()
    p.grad = torch.tensor([float("inf"), 1, 1, 1])
    sc.step(opt)
    sc.update()
    assert torch.equal(p.detach(), before) and sc.get_scale() == 8.0


def test_core_aliases_and_patches():
    assert ta.lazy_device().type in ("cpu", "cuda") and not ta.is_lazy_device(ta.lazy_device())
    assert not ta.is_lazy_tensor(torch.zeros(1))
    ta.sync(wait=True)
    ta.mark_step()
    x = ta.mark_dynamic(torch.zeros(2, 5), 1, 8)
    assert x._tb_dynamic_bounds == {1: 8}
    with pytest.raises(ValueError):
        ta.mark_dynamic(torch.zeros(2, 9), 1, 8)
    ta.utils.patch.patch_autocast()
    with torch.autocast("xla", dtype=torch.bfloat16):
        pass
    ta.utils.patch.unpatch_all()
    ta.utils.decompose.replace_decompose()
    assert ta.utils.import_utils.is_torch_xla_available() in (True, False)


def test_cpu_offload_context_is_transparent_on_cpu():
    ctx, sync = ta.utils.cpu_offload.get_cpu_offload_context(num_offload_layers=1)
    lin = [torch.nn.Linear(8, 8) for _ in range(3)]
    x = torch.randn(4, 8, requires_grad=True)
    h = x
    for l in lin:
        with ctx:
            h = torch.relu(l(h))
        h = sync(h)
    h.sum().backward()
    h2 = x.detach().clone().requires_grad_()
    y = h2
    for l in lin:
        y = torch.relu(l(y))
    y.sum().backward()
    assert torch.allclose(x.grad, h2.grad)


def test_gradient_checkpoint_wraps_named_classes():
    from torchacc_b200.models import build_llama
    from torchacc_b200.utils.checkpoint import CheckpointedModule, gradient_checkpoint
    m = build_llama("tiny", hidden_size=32, intermediate_size=64, num_hidden_layers=3, num_attention_heads=2,
                    num_key_value_heads=1, head_dim=16, vocab_size=64, max_position_embeddings=32)
    gradient_checkpoint(m, {"LlamaDecoderLayer"}, gc_cnt=2)
    kinds = [isinstance(l, CheckpointedModule) for l in m.model.layers]
    assert kinds == [True, True, False]
    ids = torch.randint(0, 64, (2, 8))
    m(ids, labels=ids)["loss"].backward()


def test_partitioners():
    from torchacc_b200.utils.utils import partition_balanced, partition_uniform
    assert partition_uniform(10, 3) == [0, 4, 7, 10]
    b = partition_balanced([1, 1, 1, 10, 1, 1], 3)
    assert b[0] == 0 and b[-1] == 6 and len(b) == 4


def test_throughput_meter_and_memory_stats():
    import time
    import torchacc_b200 as ta
    from torchacc_b200.models import build_llama
    m = ta.utils.ThroughputMeter(torch.device("cpu"))
    for _ in range(3):
        with m.step(1000):
            time.sleep(0.01)
    s = m.summary()
    assert s["steps"] == 3 and 20_000 < s["tokens_per_s"] < 400_000, s
    model = build_llama("tiny", hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
                        num_key_value_heads=2, head_dim=16, vocab_size=128, max_position_embeddings=64)
    model = ta.accelerate(model, config=ta.Config())
    st = ta.utils.memory_stats(model)
    n_params = sum(p.numel() for p in model.parameters())
    assert abs(st["engine_master_shards"] * (1 << 30) - 4 * n_params) < 1e-3 * 4 * n_params + 4096, st


def test_trace_summary_tool(tmp_path):
    """tools/trace_summary.py on a synthetic two-stream chrome trace: overlap accounting."""
    import json
    import subprocess
    import sys
    ev = [
        {"ph": "X", "cat": "kernel", "name": "void tb::gemm_bf16_kernel<2>(...)", "ts": 0, "dur": 1000, "args": {"stream": 7}},
        {"ph": "X", "cat": "kernel", "name": "tb::multi_copy_tma_kernel(...)", "ts": 500, "dur": 1000, "args": {"stream": 21}},
        {"ph": "X", "cat": "kernel", "name": "void tb::flash_fwd_kernel<128>(...)", "ts": 2000, "dur": 500, "args": {"stream": 7}},
    ]
    p = tmp_path / "t.json"
    p.write_text(json.dumps({"traceEvents": ev}))
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "tools", "trace_summary.py"), str(p)], capture_output=True,
                         text=True, check=True).stdout
    assert "step span 2.50 ms" in out and "GPU busy (any stream) 2.00 ms" in out, out
    assert "communication kernels busy 1.00 ms, of which 0.50 ms" in out, out


def test_sliding_window_model_matches_masked_reference():
    """Mistral-style local attention in the native model == explicit banded causal mask."""
    from torchacc_b200.models import build_llama, llama_config
    assert llama_config("mistral-7b").sliding_window == 4096
    torch.manual_seed(0)
    kw = dict(hidden_size=64, intermediate_size=128, num_hidden_layers=1, num_attention_heads=4, num_key_value_heads=2,
              head_dim=16, vocab_size=97, max_position_embeddings=64)
    m_win = build_llama("tiny", sliding_window=8, **kw)
    m_full = build_llama("tiny", **kw)
    m_full.load_state_dict(m_win.state_dict())
    ids = torch.randint(0, 97, (2, 32))
    a = m_win(ids, return_logits=True)["logits"]
    b = m_full(ids, return_logits=True)["logits"]
    # the first `window` positions see the same keys in both models, later ones do not
    assert torch.allclose(a[:, :8], b[:, :8], atol=1e-5)
    assert not torch.allclose(a[:, 16:], b[:, 16:], atol=1e-4)
    # and the windowed output equals attention with an explicit band mask
    from torchacc_b200.ops.attention import attention_reference
    q = torch.randn(1, 32, 4, 16)
    k = torch.randn(1, 32, 2, 16)
    v = torch.randn(1, 32, 2, 16)
    out, _ = attention_reference(q, k, v, 16 ** -0.5, True, (7, 0))
    kk, vv = k.repeat_interleave(2, 2), v.repeat_interleave(2, 2)
    i = torch.arange(32)
    band = (i[None, :] <= i[:, None]) & (i[None, :] >= i[:, None] - 7)
    ref = torch.nn.functional.scaled_dot_product_attention(q.transpose(1, 2), kk.transpose(1, 2), vv.transpose(1, 2),
                                                           attn_mask=band).transpose(1, 2)
    assert torch.allclose(out, ref, atol=1e-5)


# ---- fx tracing + parameter lifting (reference utils/trace.py:21-175) ----------------------------------------------
class _TraceToy(torch.nn.Module):

    def __init__(self):
        super().__init__()
        self.a, self.b = torch.nn.Linear(8, 8), torch.nn.Linear(8, 8)
        self.scale = torch.nn.Parameter(torch.randn(8))
        self.register_buffer("shift", torch.randn(8))

    def forward(self, x, flag=None):
        h = self.a(x) + self.shift
        return self.b(h) * self.scale


def _split_at(gm, target):
    from torch.fx.passes.split_module import split_module
    stage, cur = {}, 0
    for n in gm.graph.nodes:
        if n.op == "call_module" and n.target == target:
            cur = 1
        stage[n] = cur
    return split_module(gm, gm, lambda n: stage[n])


def test_trace_and_lift_single_use_params():
    from torchacc_b200.utils.trace import lift_single_use_params, trace
    torch.manual_seed(0)
    m = _TraceToy()
    x = torch.randn(3, 8)
    want = m(x)
    gm = trace(m, ["x"])
    split = _split_at(gm, "b")
    assert sum(n.op == "get_attr" for n in split.graph.nodes) == 2
    qmap = lift_single_use_params(split)
    assert qmap == {"submod_0.lifted_shift": "shift", "submod_1.lifted_scale": "scale"}
    assert not any(n.op == "get_attr" for n in split.graph.nodes)       # every stage owns its tensors now
    assert "submod_1.lifted_scale" in dict(split.named_parameters())
    assert "submod_0.lifted_shift" in dict(split.named_buffers())
    assert torch.allclose(split(x), want)
    split(x).sum().backward()
    assert split.submod_1.lifted_scale.grad is not None


def test_trace_hf_llama_block_level():
    """HF forwards cannot be traced whole (kwargs decorators, mask control flow): the block-level trace keeps decoder
    layers as leaves, reproduces the logits, and splits into stages that own their parameters."""
    pytest.importorskip("transformers")
    from transformers import LlamaConfig, LlamaForCausalLM
    from torchacc_b200.utils.patch import unpatch_all
    from torchacc_b200.utils.trace import lift_single_use_params, trace
    hc = LlamaConfig(vocab_size=160, hidden_size=64, intermediate_size=128, num_hidden_layers=2,
                     num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=64,
                     attn_implementation="eager", use_cache=False)
    torch.manual_seed(0)
    m = LlamaForCausalLM(hc)
    ids = torch.randint(0, 160, (2, 16))
    pos = torch.arange(16)[None].expand(2, 16)
    want = m(input_ids=ids, position_ids=pos).logits
    try:
        gm = trace(m, ["input_ids", "position_ids"])
        layer_calls = [n.target for n in gm.graph.nodes if n.op == "call_module" and ".layers." in n.target]
        assert layer_calls == ["model.model.layers.0", "model.model.layers.1"]
        assert torch.allclose(gm(ids, pos), want, atol=1e-5)
        split = _split_at(gm, "model.model.layers.1")
        # norms are leaf modules as well (their forward may be patched onto fused kernels): nothing is fetched at the top level
        assert "model.model.norm" in [n.target for n in gm.graph.nodes if n.op == "call_module"]
        assert lift_single_use_params(split) == {}
        assert torch.allclose(split(ids, pos), want, atol=1e-5)
    finally:
        unpatch_all()


def test_trace_failure_is_loud():
    from torchacc_b200.utils.trace import trace

    class Bad(torch.nn.Module):
        def forward(self, x):
            return x if x.sum() > 0 else -x

    with pytest.raises(Exception):
        trace(Bad(), ["x"])


def test_graft_entry_build_compiles_library_and_harnesses():
    """``__graft_entry__.build()`` is the driver's build check: the in-tree library AND the stand-alone nvcc harnesses have
    to compile and link on a GPU-less host (the harness silently stopped linking once when the GEMM gained a dependency)."""
    import shutil
    if shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"):
        pytest.skip("nvcc not available")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    harness = os.path.join(root, "build", "gemm_test")
    if os.path.exists(harness):
        os.remove(harness)                      # force the link step
    sys.path.insert(0, root)
    try:
        import __graft_entry__ as g
        g.build()
    finally:
        sys.path.remove(root)
    assert os.path.exists(harness)
    assert os.path.exists(os.path.join(root, "torchacc_b200", "_C.so"))


def test_step_watchdog_dumps_stacks_of_a_hung_step(tmp_path):
    """Fault injection for SURVEY 5.3: a step that blocks longer than its budget produces a stack dump naming the blocked
    frame (and, with exit=True, ends the process instead of hanging the job); a step inside the budget prints nothing."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "hang.py"
    script.write_text(
        "import sys, time\n"
        f"sys.path.insert(0, {root!r})\n"
        "from torchacc_b200.utils.watchdog import StepWatchdog\n"
        "def fast_step():\n    time.sleep(0.05)\n"
        "def blocked_in_collective():\n    time.sleep(30)\n"
        "with StepWatchdog(5):\n    fast_step()\n"
        "print('fast ok', flush=True)\n"
        "with StepWatchdog(0.5, exit=True):\n    blocked_in_collective()\n"
        "print('not reached', flush=True)\n")
    r = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=60)
    assert "fast ok" in r.stdout and "not reached" not in r.stdout
    assert r.returncode != 0                                        # exit=True: the hung process is terminated
    assert "blocked_in_collective" in r.stderr and "Timeout" in r.stderr
    assert "fast_step" not in r.stderr                               # the healthy step left no dump


def test_attn_params_layout_matches_the_library():
    """The attention entry points take one ``AttnParams`` struct through ctypes, so nothing checks argument counts or
    types: the Python mirror must have the C struct's size and every field at the C offset, in declaration order."""
    import ctypes
    from torchacc_b200 import _native as nat
    from torchacc_b200.ops.attention import AttnParams
    L = nat.lib()
    if L is None:
        pytest.skip("native library not built")
    out = (nat.i64 * 64)()
    n = L.tb_attn_params_layout(out, 64)
    expected = [ctypes.sizeof(AttnParams)] + [getattr(AttnParams, name).offset for name, _ in AttnParams._fields_]
    assert list(out[:n]) == expected


def test_carry_queue_slices_jobs_by_flop_budget():
    """Host side of the carried collectives (csrc/fused/carry.cu, C++): jobs are cut into chunk ranges proportional to the
    FLOPs of the GEMM that takes them along, foreground jobs before background jobs, at most two slices per launch, every
    chunk handed out exactly once.  Pure host logic: runs without a GPU (pointers are never dereferenced)."""
    import ctypes
    from torchacc_b200 import _native as nat
    from torchacc_b200.parallel import carry as C
    L = nat.lib()
    if L is None or not hasattr(L, "tb_carry_take_probe"):
        pytest.skip("native library not built")
    out = (nat.i64 * 8)()

    def drain():
        while L.tb_carry_take_probe(1e18, out) > 0:
            pass
    drain()
    old = L.tb_carry_bytes_per_flop(1e-4)                 # 1e-4 bytes of NVLink traffic per GEMM FLOP
    try:
        world = 2
        ptrs = (nat.u64 * world)(0x1000, 0x2000)
        pads = (nat.u64 * world)(0x3000, 0x4000)
        nbytes = 8 << 20                                   # 8 MiB shard per rank

        def push(kind, background):
            return L.tb_carry_push(kind, ptrs, 0x5000, pads, nbytes, 0, world, C.CH_GATHER, 1, 0, 0.5, 1, 1, 0, 0,
                                   int(background), C.CH_PARAMS, 1)
        bg = push(1, True)                                 # background gather (prefetch)
        fg = push(2, False)                                # foreground reduce-scatter
        assert fg > bg > 0
        # gather: 8 KB chunks, own shard included -> 2 * 1024 chunks; reduce: (8 KB / world) per source and chunk -> 2048
        assert L.tb_carry_pending(0, C.BACKGROUND) == 2048 and L.tb_carry_pending(0, C.FOREGROUND) == 2048
        cost = {2: 4096 * world, 1: 8192 * (world - 1) / world}   # wire bytes per chunk: reduce / gather
        nxt = {2: 0, 1: 0}                                           # next expected chunk of each job
        launches = 0
        while L.tb_carry_pending(0, C.ALL_QUEUES) > 0:
            flops = float(1 << (34 + launches % 4))                  # GEMMs of different sizes
            budget = flops * 1e-4
            n = L.tb_carry_take_probe(flops, out)
            assert 1 <= n <= 2
            spent = 0.0
            for i in range(n):
                kind, lo, hi, chunk_bytes = (int(out[4 * i + k]) for k in range(4))
                assert chunk_bytes == (4096 if kind == 2 else 8192)
                assert lo == nxt[kind] and hi > lo                   # contiguous, every chunk exactly once
                nxt[kind] = hi
                spent += (hi - lo) * cost[kind]
                if kind == 1:                                        # background work only once the foreground job is done
                    assert nxt[2] == 2048 or i == 1                  # ... or with what is left of this launch's budget
            assert spent <= budget                                   # never more traffic than the GEMM can hide
            if nxt[1] < 2048:                                        # unless the queue ran dry the budget is used up
                assert budget - spent < max(cost.values())
            if launches == 0:
                assert int(out[0]) == 2 and int(out[1]) == 0         # the foreground job goes first
            launches += 1
        assert nxt == {2: 2048, 1: 2048} and launches > 3
        assert L.tb_carry_take_probe(1e12, out) == 0                 # empty queue: the GEMM carries nothing
    finally:
        drain()
        L.tb_carry_bytes_per_flop(old)
        stats = (nat.i64 * 4)()
        L.tb_carry_stats(stats, 1)


def test_pp_boundary_header_roundtrip_with_tuple_values():
    """Stage-boundary protocol: named values may be tensors or flat tuples of tensors (HF's rotary (cos, sin) pair); the
    single int64 header of a shape epoch carries dtype / shape / requires_grad and the grouping."""
    from torchacc_b200.parallel.pp import p2p
    hidden = torch.randn(2, 5, 8, requires_grad=True)
    cos, sin = torch.randn(1, 5, 4), torch.randn(1, 5, 4)
    ids = torch.zeros(2, 5, dtype=torch.int64)
    flat, groups = p2p.flatten_values([hidden, (cos, sin), ids])
    assert len(flat) == 4 and groups == [(0, False), (1, True), (1, True), (2, False)]
    metas = p2p.decode_header(p2p.encode_header(flat, "cpu", groups))
    assert [m.shape for m in metas] == [(2, 5, 8), (1, 5, 4), (1, 5, 4), (2, 5)]
    assert [m.dtype for m in metas] == [torch.float32, torch.float32, torch.float32, torch.int64]
    assert [m.requires_grad for m in metas] == [True, False, False, False]
    back = p2p.unflatten_values(flat, metas)
    assert back[0] is hidden and isinstance(back[1], tuple) and back[1][0] is cos and back[1][1] is sin and back[2] is ids
    with pytest.raises(TypeError):
        p2p.flatten_values([hidden, {"a": cos}])
    with pytest.raises(TypeError):
        p2p.flatten_values([(cos, 3)])
