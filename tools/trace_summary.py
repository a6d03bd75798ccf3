#!/usr/bin/env python
"""Summarise a torch-profiler chrome trace of one training step (bench.py --trace):

  * GPU busy time (union over streams) vs the span of the step, per-stream busy time
  * time per kernel family, and how much of the communication kernels' time is hidden behind compute kernels
  * the largest idle gaps on the busiest (compute) stream with the neighbouring kernels

    python tools/trace_summary.py trace.json [--top 25]
"""
import argparse
import gzip
import json
from collections import defaultdict

COMM = ("all_gather_kernel", "reduce_scatter_kernel", "all_to_all_kernel", "multi_copy_tma_kernel",
        "reduce_scatter_tma_kernel", "nccl", "rs_reduce")


def family(name: str) -> str:
    n = name
    for key, fam in (("gemm_bf16_kernel", "gemm (wgmma)"), ("flash_fwd", "attention fwd"), ("flash_bwd", "attention bwd"),
                     ("attn_bwd_pre", "attention bwd pre/post"), ("convert", "attention bwd pre/post"),
                     ("adamw", "adamw"), ("rmsnorm", "rmsnorm"), ("rope", "rope"), ("swiglu", "swiglu"),
                     ("cross_entropy", "cross-entropy"), ("sqnorm", "grad-norm"), ("multi_copy_tma_kernel", "symm all-gather / all-to-all (TMA)"),
                     ("reduce_scatter_tma_kernel", "symm reduce-scatter (TMA)"), ("all_gather_kernel", "symm all-gather"),
                     ("reduce_scatter_kernel", "symm reduce-scatter"), ("all_to_all_kernel", "symm all-to-all"),
                     ("nccl", "nccl"), ("Memcpy", "memcpy"), ("Memset", "memset")):
        if key in n:
            return fam
    if "at::native" in n or "elementwise" in n or "vectorized" in n:
        return "torch elementwise/other"
    return n[:60]


def union(iv):
    iv = sorted(iv)
    tot, cur_s, cur_e = 0.0, None, None
    merged = []
    for s, e in iv:
        if cur_e is None or s > cur_e:
            if cur_e is not None:
                merged.append((cur_s, cur_e))
                tot += cur_e - cur_s
            cur_s, cur_e = s, e
        else:
            cur_e = max(cur_e, e)
    if cur_e is not None:
        merged.append((cur_s, cur_e))
        tot += cur_e - cur_s
    return tot, merged


def overlap(a_merged, b_merged):
    i = j = 0
    tot = 0.0
    while i < len(a_merged) and j < len(b_merged):
        s = max(a_merged[i][0], b_merged[j][0])
        e = min(a_merged[i][1], b_merged[j][1])
        if e > s:
            tot += e - s
        if a_merged[i][1] < b_merged[j][1]:
            i += 1
        else:
            j += 1
    return tot


def comm_exposure(trace_path: str) -> dict:
    """{'step_ms', 'comm_busy_ms', 'comm_overlapped_ms', 'exposed_comm_ms'} of one traced step (bench.py uses this)."""
    op = gzip.open if trace_path.endswith(".gz") else open
    with op(trace_path, "rt") as f:
        ev = json.load(f)["traceEvents"]
    ks = [e for e in ev if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
    if not ks:
        return {}
    # the step proper starts with the first compute kernel (a collective may spin in its entry barrier before that
    # while the slowest rank starts profiling)
    comp = [(e["ts"], e["ts"] + e["dur"]) for e in ks if not any(c in e["name"] for c in COMM)]
    comm = [(e["ts"], e["ts"] + e["dur"]) for e in ks if any(c in e["name"] for c in COMM)]
    if not comp:
        return {}
    t0 = min(s for s, _ in comp)
    t1 = max(e for _, e in comp + comm)
    comm = [(max(s, t0), e) for s, e in comm if e > t0]
    ct, cm = union(comm)
    _, pm = union(comp)
    ov = overlap(cm, pm)
    return {"step_ms": (t1 - t0) / 1e3, "comm_busy_ms": ct / 1e3, "comm_overlapped_ms": ov / 1e3,
            "exposed_comm_ms": (ct - ov) / 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("trace")
    ap.add_argument("--top", type=int, default=25)
    a = ap.parse_args()
    op = gzip.open if a.trace.endswith(".gz") else open
    with op(a.trace, "rt") as f:
        ev = json.load(f)["traceEvents"]
    ks = [e for e in ev if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
    if not ks:
        print("no GPU activity in trace")
        return
    t0 = min(e["ts"] for e in ks)
    t1 = max(e["ts"] + e["dur"] for e in ks)
    span = t1 - t0
    by_stream = defaultdict(list)
    fam_t = defaultdict(float)
    fam_n = defaultdict(int)
    comm_iv, comp_iv = [], []
    for e in ks:
        s, d = e["ts"], e["dur"]
        st = e.get("args", {}).get("stream", e.get("tid"))
        by_stream[st].append((s, s + d, e["name"]))
        fam = family(e["name"])
        fam_t[fam] += d
        fam_n[fam] += 1
        (comm_iv if any(c in e["name"] for c in COMM) else comp_iv).append((s, s + d))
    busy, merged_all = union([(s, e) for v in by_stream.values() for s, e, _ in v])
    print(f"step span {span / 1e3:.2f} ms, GPU busy (any stream) {busy / 1e3:.2f} ms ({100 * busy / span:.1f} %), "
          f"{len(ks)} GPU activities on {len(by_stream)} streams")
    print("\nper stream: busy ms, share of span, #kernels")
    for st, v in sorted(by_stream.items(), key=lambda kv: -sum(e - s for s, e, _ in kv[1])):
        b, _ = union([(s, e) for s, e, _ in v])
        print(f"  stream {st}: {b / 1e3:9.2f} ms  {100 * b / span:5.1f} %  {len(v)}")
    ct, cm = union(comm_iv)
    pt, pm = union(comp_iv)
    ov = overlap(cm, pm)
    print(f"\ncompute kernels busy {pt / 1e3:.2f} ms; communication kernels busy {ct / 1e3:.2f} ms, of which "
          f"{ov / 1e3:.2f} ms ({100 * ov / max(ct, 1e-9):.1f} %) overlap compute; exposed communication "
          f"{(ct - ov) / 1e3:.2f} ms ({100 * (ct - ov) / span:.1f} % of the step)")
    print(f"\nkernel families (sum of durations; overlapping streams can exceed the span)")
    for fam, t in sorted(fam_t.items(), key=lambda kv: -kv[1])[:a.top]:
        print(f"  {t / 1e3:9.2f} ms  {100 * t / span:5.1f} %  x{fam_n[fam]:<5d} {fam}")
    main_st = max(by_stream.items(), key=lambda kv: sum(e - s for s, e, _ in kv[1]))[0]
    v = sorted(by_stream[main_st])
    gaps = []
    for (s0, e0, n0), (s1, e1, n1) in zip(v, v[1:]):
        if s1 - e0 > 20:
            gaps.append((s1 - e0, e0 - t0, n0[:50], n1[:50]))
    tot_gap = sum(g[0] for g in gaps)
    print(f"\nidle gaps > 20 us on stream {main_st}: {len(gaps)} gaps, {tot_gap / 1e3:.2f} ms total; largest:")
    for g in sorted(gaps, reverse=True)[:15]:
        print(f"  {g[0] / 1e3:7.3f} ms at +{g[1] / 1e3:8.2f} ms  after [{g[2]}]  before [{g[3]}]")


if __name__ == "__main__":
    main()
