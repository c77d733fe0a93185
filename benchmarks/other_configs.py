#!/usr/bin/env python
"""Timing of the non-headline BASELINE.json configs on one GPU (parity for these is in tests/;
they are not bench.py lines).  Prints one JSON object per config.

  config 2: 3-layer SAGEConv(mean), synthetic power-law 10 M nodes / 100 M edges, h = 256, fp32
  config 3: GATConv 8 heads x 16, ogbn-products-shaped synthetic (2.4 M nodes / 123 M edges), bf16 features
  config 5: RGCNConv 4 relations, 5 M nodes / 50 M edges (single GPU here), h = 64, fp32

  config 6: SURVEY section 8(f) rank 1 -- PNA-style [mean, min, max, std] multi-aggregation on the headline graph
            (10 M nodes / 100 M edges, F = 256, fp32): ONE sweep (csrc/multi_aggr.cu) vs one pass per aggregation

    python benchmarks/other_configs.py [--configs 2,3,5,6] [--steps 3]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import synth_graph  # noqa: E402


def timed(fn, steps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="2,3,5")
    ap.add_argument("--steps", type=int, default=3)
    args = ap.parse_args()
    from pytorch_geometric_b200 import functional as Fn
    from pytorch_geometric_b200.graph import CSRGraph
    from pytorch_geometric_b200.nn import GATConv, RGCNConv, SAGEConv
    dev = torch.device("cuda", 0)
    todo = {int(c) for c in args.configs.split(",")}
    if os.environ.get("B200MP_ATTN_STAGED") is not None:          # A/B switch of the cp.async-staged kernels (and the hit mask)
        from pytorch_geometric_b200 import ops as _o
        _o.set_option("attn_staged", int(os.environ["B200MP_ATTN_STAGED"]))
    if os.environ.get("B200MP_MULTI_TUNE"):
        from pytorch_geometric_b200 import ops as _o
        _o.set_option("multi_tune", int(os.environ["B200MP_MULTI_TUNE"]))
    if os.environ.get("B200MP_MULTI_MASK") == "0":
        from pytorch_geometric_b200 import ops as _o
        _o.MULTI_HIT_MASK = False

    if 2 in todo:
        N, E, F = 10_000_000, 100_000_000, 256
        ei = synth_graph(N, E, 2, dev)
        g = CSRGraph(ei[0], ei[1], N, N)
        g.build_transpose()
        del ei
        convs = torch.nn.ModuleList([SAGEConv(F, F) for _ in range(3)]).to(dev)
        x = torch.randn(N, F, device=dev)
        gout = torch.randn(N, F, device=dev)

        def step():
            for c in convs:
                c.zero_grad(set_to_none=True)
            h = x
            for i, c in enumerate(convs):
                h = c(h, g)
                if i < 2:
                    h = h.relu_()
            h.backward(gout)

        ms = timed(step, args.steps)
        print(json.dumps({"config": 2, "what": "3-layer SAGEConv(mean) fwd+bwd, N=10M, E=100M, h=256, fp32",
                          "ms_per_step": ms, "edge_layers_per_s": 3 * E / (ms * 1e-3)}))
        del g, convs, x, gout
        torch.cuda.empty_cache()

    if 3 in todo:
        N, E, H, C = 2_400_000, 123_000_000, 8, 16
        ei = synth_graph(N, E, 3, dev)
        conv = GATConv(128, C, heads=H).to(dev)
        g = conv.graph_for(ei, N)                      # remove + add self loops, CSR
        g.build_transpose()
        _ = g.t2csr
        del ei
        deg = g.in_degree()
        xh = torch.randn(N, H * C, device=dev).bfloat16()
        a_s = torch.randn(N, H, device=dev)
        a_d = torch.randn(N, H, device=dev)
        ms_f = timed(lambda: Fn.gat_attention(g, xh, a_s, a_d, H, C, 0.2), args.steps)
        xh32 = xh.float().requires_grad_()
        a_s.requires_grad_()
        a_d.requires_grad_()
        gout = torch.randn(N, H * C, device=dev)

        def step():
            xh32.grad = a_s.grad = a_d.grad = None
            Fn.gat_attention(g, xh32, a_s, a_d, H, C, 0.2).backward(gout)

        ms_fb = timed(step, args.steps)
        Ep = g.num_edges
        bytes_fwd = Ep * (H * C * 2 + H * 4 + 4) + N * (H * C * 2 + 3 * H * 4)
        print(json.dumps({"config": 3, "what": "fused GAT attention+aggregation, N=2.4M, E=123M (+N loops), 8x16",
                          "max_in_degree": int(deg.max()), "fwd_ms_bf16": ms_f,
                          "fwd_algorithmic_GBps": bytes_fwd / (ms_f * 1e-3) / 1e9, "fwd_bwd_ms_fp32": ms_fb,
                          "edges_per_s_fwd_bwd": E / (ms_fb * 1e-3)}))
        del g, xh, xh32, a_s, a_d, gout
        torch.cuda.empty_cache()

    if 6 in todo:
        N, E, F = 10_000_000, 100_000_000, 256
        ei = synth_graph(N, E, 2, dev)
        g = CSRGraph(ei[0], ei[1], N, N)
        g.build_transpose()
        del ei
        x = torch.randn(N, F, device=dev)
        aggrs = ["mean", "min", "max", "std"]
        ms_fused = timed(lambda: Fn.multi_aggregate(g, x, aggrs), args.steps)

        def separate():
            mean = Fn.aggregate(g, x, "mean")
            mn = Fn.aggregate(g, x, "min")
            mx = Fn.aggregate(g, x, "max")
            sq = Fn.aggregate(g, x * x, "mean")
            return mean, mn, mx, (sq - mean * mean).clamp_(min=1e-5).sqrt_()

        ms_sep = timed(separate, args.steps)
        xg = x.clone().requires_grad_()
        gouts = [torch.randn(N, F, device=dev) for _ in aggrs]

        def step():
            xg.grad = None
            torch.autograd.backward(Fn.multi_aggregate(g, xg, aggrs), gouts)

        ms_fb = timed(step, args.steps)
        from pytorch_geometric_b200 import ops as _ops
        _ops.PROFILE.reset(True)                                # one more step with per-call events: the breakdown
        step()
        prof = {k: round(v["ms_total"], 3) for k, v in _ops.PROFILE.summary().items()}
        _ops.PROFILE.reset(False)
        bytes_fwd = E * (F * 4 + 4) + N * F * 4 * len(aggrs) + (N + 1) * 4
        res = {"config": 6, "what": "multi-aggregation [mean,min,max,std], N=10M, E=100M, F=256, fp32",
               "fused_fwd_ms": ms_fused, "separate_fwd_ms": ms_sep,
               "fused_fwd_algorithmic_GBps": bytes_fwd / (ms_fused * 1e-3) / 1e9, "fused_fwd_bwd_ms": ms_fb,
               "fwd_bwd_breakdown_ms": prof,
               "staged": os.environ.get("B200MP_ATTN_STAGED", "1"), "hit_mask": os.environ.get("B200MP_MULTI_MASK", "1"),
               "multi_tune": os.environ.get("B200MP_MULTI_TUNE", "6")}
        del x, xg, gouts
        torch.cuda.empty_cache()
        # segment form (what PNAConv / MultiAggregation see): materialised messages [E, 64] sorted by destination
        Fm = 64
        msg = torch.randn(E, Fm, device=dev)
        where = (g.rowptr, g.dst_csr, g.plan)
        ms_seg = timed(lambda: Fn.multi_aggregate(where, msg, aggrs), args.steps)

        def separate_seg():
            mean = Fn.segment(msg, g.rowptr, "mean")
            mn = Fn.segment(msg, g.rowptr, "min")
            mx = Fn.segment(msg, g.rowptr, "max")
            sq = Fn.segment(msg * msg, g.rowptr, "mean")
            return mean, mn, mx, (sq - mean * mean).clamp_(min=1e-5).sqrt_()

        ms_seg_sep = timed(separate_seg, args.steps)
        mg = msg.clone().requires_grad_()
        gouts = [torch.randn(N, Fm, device=dev) for _ in aggrs]

        def step_seg():
            mg.grad = None
            torch.autograd.backward(Fn.multi_aggregate(where, mg, aggrs), gouts)

        ms_seg_fb = timed(step_seg, args.steps)
        res.update(segment_F=Fm, segment_fused_fwd_ms=ms_seg, segment_separate_fwd_ms=ms_seg_sep,
                   segment_fused_fwd_algorithmic_GBps=(E * Fm * 4 + N * Fm * 4 * len(aggrs) + (N + 1) * 4) / (ms_seg * 1e-3) / 1e9,
                   segment_fused_fwd_bwd_ms=ms_seg_fb)
        print(json.dumps(res))
        del g, msg, mg, gouts
        torch.cuda.empty_cache()

    if 5 in todo:
        N, E, R, F = 5_000_000, 50_000_000, 4, 64
        ei = synth_graph(N, E, 5, dev)
        et = torch.randint(0, R, (E, ), device=dev)
        conv = RGCNConv(F, F, R).to(dev)
        g = conv.relation_graph(ei, et, N)
        g.build_transpose()
        del ei, et
        x = torch.randn(N, F, device=dev).requires_grad_()
        gout = torch.randn(N, F, device=dev)

        def step():
            x.grad = None
            conv.zero_grad(set_to_none=True)
            conv(x, g).backward(gout)

        ms = timed(step, args.steps)
        print(json.dumps({"config": 5, "what": "RGCNConv(mean) 4 relations fwd+bwd, N=5M, E=50M, h=64, fp32, 1 GPU",
                          "ms_per_step": ms, "edges_per_s": E / (ms * 1e-3)}))


if __name__ == "__main__":
    main()
