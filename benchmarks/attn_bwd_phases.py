"""Phase profile of the head-dim-64 attention backward main kernel (flash_bwd_kernel) on the flagship attention shape.

Runs one causal forward + backward with the instrumented instantiation (tb_attn_bwd_set_profile): one elected thread
per MMA warpgroup writes clock64() at the end of every phase of every iteration, the TMA producer at its empty-wait
and its issue, for the key tiles of kv head 0 of sequence 0 (the heaviest and the lightest key tiles of a causal run
and everything between).  Prints, for the default (dQ reduce-add) and the deterministic (dK / dV only) kernel, the
median and p90 cycles of every phase over the interior iterations, the same for the diagonal iterations (per-element
key masking), and the prologue, epilogue and per-iteration totals.  The card name and power limit go with the numbers.

Cycles are SM clocks: the stamps cost a few instructions on one thread per warpgroup, so the profiled kernel is a
little slower than the shipped one; compare its numbers with each other, and kernel times with attn_bench.py.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# phase that ends at each warpgroup slot of an iteration, in the order of flash_bwd_kernel's schedule
PHASES = ["Q/dO full-wait", "issue S^T, dP^T", "load statistics", "barrier 1", "wait S^T + dP^T",
          "P^T, dS^T (+ smem store)", "barrier 2", "issue dQ, dV, dK", "stage dQ, reduce-add", "final wait"]
HEAD, WG_SLOTS = 8, 10                     # kProfHead, kProfWgSlots (csrc/attn/flash_bwd.cu)
SLOTS = 2 * WG_SLOTS + 2                   # kProfSlots
TILE = 128                                 # keys per CTA = query rows per iteration at D = 64


def device_desc():
    import subprocess
    desc = {"gpu": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
        pl, clk = r.stdout.strip().splitlines()[0].split(",")
        desc["power_limit_w"], desc["max_sm_clock_mhz"] = float(pl), float(clk)
    except Exception:
        desc["power_limit_w"] = desc["max_sm_clock_mhz"] = None
    return desc


def analyse(rec, S, group):
    """Per-phase cycle samples from the records [ctas, words] (int64) of one causal run."""
    interior = {p: [] for p in PHASES}
    diagonal = {p: [] for p in PHASES}
    iters_int, iters_diag, prologue, epilogue, producer_wait = [], [], [], [], []
    for jt in range(rec.shape[0]):
        n_iter = int(rec[jt, 0])
        if n_iter == 0:
            continue
        n_qt = n_iter // group
        it_lo = jt   # causal, Sq == Sk: query tile jt is the first that sees key tile jt
        body = rec[jt, HEAD:HEAD + min(n_iter, (rec.shape[1] - HEAD) // SLOTS) * SLOTS].reshape(-1, SLOTS)
        prologue.append(int(rec[jt, 3] - rec[jt, 2]))
        for wg in range(2):
            st = body[:, wg * WG_SLOTS:(wg + 1) * WG_SLOTS]
            used = [i for i in range(WG_SLOTS) if st[0, i] != 0]
            prev = int(rec[jt, 3])                       # K/V landed
            for it in range(st.shape[0]):
                diag = (it_lo + it % n_qt) == jt         # the query tile on the diagonal: per-element masking
                tgt = diagonal if diag else interior
                start = prev
                for i in used:
                    tgt[PHASES[i]].append(int(st[it, i]) - prev)
                    prev = int(st[it, i])
                (iters_diag if diag else iters_int).append(prev - start)
            epilogue.append(int(rec[jt, 4 + wg]) - prev)
        producer_wait += [int(body[it, 2 * WG_SLOTS] - (body[it - 1, 2 * WG_SLOTS + 1] if it else rec[jt, 2]))
                          for it in range(body.shape[0])]
    return interior, diagonal, iters_int, iters_diag, prologue, epilogue, producer_wait


def stats(xs):
    if not xs:
        return None
    a = np.asarray(xs, dtype=np.float64)
    return {"median": round(float(np.median(a))), "p90": round(float(np.percentile(a, 90))), "n": len(xs)}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--batch", type=int, default=2)
    p.add_argument("--seq", type=int, default=4096)
    p.add_argument("--hq", type=int, default=32)
    p.add_argument("--hk", type=int, default=8)
    p.add_argument("--out", default="", help="also write the JSON summary here")
    a = p.parse_args()
    from torchacc_b200 import _native as nat
    from torchacc_b200.ops import attention as A
    nat.register_signatures({"tb_attn_bwd_set_profile": ([nat.u64, nat.i64], nat.i64)})
    L = nat.require()
    A.set_attention_backend("native")
    B, S, Hq, Hk, D = a.batch, a.seq, a.hq, a.hk, 64
    torch.manual_seed(0)
    q = torch.randn(B, S, Hq, D, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    k = torch.randn(B, S, Hk, D, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    v = torch.randn(B, S, Hk, D, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    do = torch.randn(B, S, Hq, D, device="cuda", dtype=torch.bfloat16)
    ctas = (S + TILE - 1) // TILE
    out = {"shape": [B, S, Hq, Hk, D], "device": device_desc(), "kernels": {}}
    for det in (False, True):
        words = L.tb_attn_bwd_set_profile(0, 0)
        buf = torch.zeros(ctas, words, dtype=torch.int64, device="cuda")
        for _ in range(2):   # the second run is the one kept: instruction caches and the L2 warm
            buf.zero_()
            L.tb_attn_bwd_set_profile(buf.data_ptr(), ctas)
            try:
                A.flash_attn_func(q, k, v, causal=True, deterministic=det).backward(do)
                torch.cuda.synchronize()
            finally:
                L.tb_attn_bwd_set_profile(0, 0)
        rec = buf.cpu().numpy()
        interior, diagonal, it_i, it_d, pro, epi, pw = analyse(rec, S, Hq // Hk)
        name = "kDQ=false (deterministic)" if det else "kDQ=true (default)"
        res = {"phases_interior": {k_: stats(v_) for k_, v_ in interior.items() if v_},
               "phases_diagonal": {k_: stats(v_) for k_, v_ in diagonal.items() if v_},
               "iteration_interior": stats(it_i), "iteration_diagonal": stats(it_d),
               "prologue_to_kv_landed": stats(pro), "epilogue": stats(epi), "producer_empty_wait": stats(pw),
               "cta_cycles_max": int((rec[:, 4:6].max(axis=1) - rec[:, 2]).max())}
        out["kernels"][name] = res
        print(f"\n== {name}: cycles per phase (one MMA warpgroup, medians / p90)", flush=True)
        print(f"{'phase':24s} {'interior':>16s} {'diagonal':>16s}")
        for ph in PHASES:
            si, sd = res["phases_interior"].get(ph), res["phases_diagonal"].get(ph)
            if si is None:
                continue
            print(f"{ph:24s} {si['median']:>7d} / {si['p90']:<7d} {sd['median']:>7d} / {sd['p90']:<7d}")
        si, sd = res["iteration_interior"], res["iteration_diagonal"]
        print(f"{'iteration':24s} {si['median']:>7d} / {si['p90']:<7d} {sd['median']:>7d} / {sd['p90']:<7d}")
        for key in ("prologue_to_kv_landed", "epilogue", "producer_empty_wait"):
            print(f"{key:24s} {res[key]['median']:>7d} / {res[key]['p90']:<7d}")
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
