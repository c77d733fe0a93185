"""bench.py --config {2,3,5}: the other single-box BASELINE.json configurations as bench lines of their own
(same JSON contract as the headline line: device-timed value, roofline object of the dominant kernel with live
CUDA-event launch times, e2e with host buffers, clocks, launches, parity_check).

  config 2  3-layer SAGEConv(mean) + ReLU, synthetic power-law N = 10 M / E = 100 M, h = 256, fp32
  config 3  GATConv(128 -> 8 heads x 16), ogbn-products-shaped synthetic N = 2.4 M / E = 123 M, bf16, full layer
  config 5  RGCNConv, 4 relations, N = 5 M / E = 50 M, h = 128, fp32 (single GPU: one rank's share of the 2-GPU config)

edges/sec = E_input * layers / t(fwd+bwd).  `parity_check`: a seeded sample of destination rows (hubs, 0/1/2-edge
rows, random rows) of the timed step's output recomputed from the RAW edge list in fp64 (ATen ops only for selecting
the rows' in-edges; numpy/torch fp64 for the arithmetic of the reference's unfused formula), plus gradient rows.
"""
from __future__ import annotations

import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _rows_sample(deg: torch.Tensor, n_rows: int, max_edges: int, seed: int) -> torch.Tensor:
    from oracle.sampled import _pick
    return _pick(deg, n_rows, max_edges, seed)


def _rel(got: torch.Tensor, want: torch.Tensor, scale: torch.Tensor) -> float:
    err = (got.double() - want.double()).abs()
    s = scale.double().clamp(min=1e-30)
    return float((err / s).max()) if err.numel() else 0.0


def run_config(args, B):
    """B = the bench module (synth_graph, ClockSampler, measured_peaks, emit, bind_to_gpu_numa_node)."""
    import pytorch_geometric_b200 as pgb  # noqa: F401
    from pytorch_geometric_b200 import dense, functional as Fn, ops
    from pytorch_geometric_b200.graph import CSRGraph
    from pytorch_geometric_b200.nn import conv as C

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    if os.environ.get("B200MP_ATTN_STAGED") is not None:           # A/B switch of the cp.async-staged attention forward
        ops.set_option("attn_staged", int(os.environ["B200MP_ATTN_STAGED"]))
    cfg = args.config
    peak, peak_src = B.measured_peaks()
    gen = torch.Generator(device=dev).manual_seed(100 + cfg)

    if cfg == 2:
        N, E, F, L = args.nodes, args.edges, args.feat, 3
        ei = B.synth_graph(N, E, 2, dev)
        graph = CSRGraph(ei[0], ei[1], N, N)
        graph.build_transpose()
        Ws = [(torch.randn(F, F, device=dev, generator=gen) / F ** 0.5).requires_grad_() for _ in range(2 * L)]
        bs = [(torch.randn(F, device=dev, generator=gen) * 0.1).requires_grad_() for _ in range(L)]
        params = Ws + bs
        x = torch.randn(N, F, device=dev, generator=gen).requires_grad_()
        gout = torch.randn(N, F, device=dev, generator=gen)
        workload = (f"3-layer SAGEConv({F},{F}, aggr=mean) + ReLU fwd+bwd, power-law synthetic graph N={N}, E={E}, fp32 "
                    f"(BASELINE config 2)")
        dtype_name, s_bytes = "f32", 4

        def model(xx):
            h = xx
            for i in range(L):
                h = C.sage_conv(h, h, graph, "mean", Ws[2 * i], bs[i], Ws[2 * i + 1], relu=(i < L - 1), input_is_relu=(i > 0),
                                grad_masked_by_consumer=(i < L - 1))
            return h

        dom_op, dom_kernel = "spmm_csr", "csr_reduce_kernel (mean aggregation fwd on CSR / bwd on transposed CSR)"
        Eg = graph.num_edges
        alg_bytes = Eg * (F * s_bytes + 4 + 0) + N * F * s_bytes + (N + 1) * 4          # SURVEY 8(d): SAGE, no weights (fwd)
        layers = L
    elif cfg == 3:
        N, E, H, Cc, Fin = 2_400_000 if args.nodes == 5_000_000 else args.nodes, 123_000_000 if args.edges == 50_000_000 else args.edges, 8, 16, 128
        ei = B.synth_graph(N, E, 3, dev)
        from pytorch_geometric_b200.graph import cached_graph
        graph = cached_graph(ei, N, N, loops="gat", loop_nodes=N)
        graph.build_transpose()
        _ = graph.t2csr
        bf = torch.bfloat16
        W = (torch.randn(H * Cc, Fin, device=dev, generator=gen) / Fin ** 0.5).to(bf).requires_grad_()
        att_s = (torch.randn(1, H, Cc, device=dev, generator=gen) * 0.3).to(bf).requires_grad_()
        att_d = (torch.randn(1, H, Cc, device=dev, generator=gen) * 0.3).to(bf).requires_grad_()
        bias = (torch.randn(H * Cc, device=dev, generator=gen) * 0.1).to(bf).requires_grad_()
        params = [W, att_s, att_d, bias]
        x = torch.randn(N, Fin, device=dev, generator=gen).to(bf).requires_grad_()
        gout = torch.randn(N, H * Cc, device=dev, generator=gen).to(bf)
        workload = (f"GATConv({Fin}, {Cc}, heads={H}) fwd+bwd (lin + attention + bias), ogbn-products-shaped synthetic "
                    f"N={N}, E={E}, bf16 storage / fp32 accumulate (BASELINE config 3)")
        dtype_name, s_bytes = "bf16", 2

        def model(xx):
            xh = dense.linear(xx, W)
            return C.gat_conv(xh, None, graph, att_s, att_d, H, Cc, 0.2, True, None, bias)

        dom_op, dom_kernel = "attn_forward", "attn_fwd_kernel (GAT score + online edge softmax + weighted aggregation)"
        Eg, HC = graph.num_edges, H * Cc
        alg_bytes = Eg * (HC * s_bytes + 4 + H * 4) + N * (HC * s_bytes + 3 * H * 4) + (N + 1) * 4
        layers, F, L = 1, HC, 1
    elif cfg == 5:
        N = args.nodes
        E = args.edges
        F, R, L = (128 if args.feat == 256 else args.feat), 4, 1
        ei = B.synth_graph(N, E, 5, dev)
        et = torch.randint(0, R, (E, ), device=dev, generator=gen)
        from pytorch_geometric_b200.graph import cached_graph
        graph = cached_graph(ei, N, N * R, edge_type=et, num_relations=R)
        graph.build_transpose()
        Wr = (torch.randn(R, F, F, device=dev, generator=gen) / F ** 0.5).requires_grad_()
        root = (torch.randn(F, F, device=dev, generator=gen) / F ** 0.5).requires_grad_()
        bias = (torch.randn(F, device=dev, generator=gen) * 0.1).requires_grad_()
        params = [Wr, root, bias]
        x = torch.randn(N, F, device=dev, generator=gen).requires_grad_()
        gout = torch.randn(N, F, device=dev, generator=gen)
        workload = (f"RGCNConv({F},{F}, num_relations={R}, aggr=mean) fwd+bwd, power-law synthetic N={N}, E={E}, fp32, "
                    f"one sweep into [N, R*F] + one K=(R+1)*F product (BASELINE config 5, one GPU)")
        dtype_name, s_bytes = "f32", 4

        def model(xx):
            return C.rgcn_conv(xx, graph, Wr, root, bias, "mean")

        dom_op, dom_kernel = "spmm_csr", "csr_reduce_kernel (per-relation mean into [N*R, F])"
        Eg = graph.num_edges
        alg_bytes = Eg * (F * s_bytes + 4) + N * R * F * s_bytes + (N * R + 1) * 4
        layers = 1
    else:
        raise SystemExit(f"--config {cfg}: configs 1 and 4 are the CPU-only toy and the 8-GPU run (bench.py --gpus 8)")
    torch.cuda.synchronize()

    def step():
        x.grad = None
        for p in params:
            p.grad = None
        out = model(x)
        out.backward(gout)
        return out

    for _ in range(max(args.warmup, 3)):
        step()
    torch.cuda.synchronize()
    sampler = B.ClockSampler(0)
    sampler.start()
    ops.PROFILE.reset(enabled=True)
    l0 = ops.LAUNCHES.count
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(args.steps):
        step()
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1)
    launches = ops.LAUNCHES.count - l0
    kern = ops.PROFILE.summary()
    ops.PROFILE.reset(enabled=False)
    clocks = sampler.stop()
    ms_per_step = ms / args.steps
    value = E * layers / (ms_per_step * 1e-3)

    # ---- roofline of the dominant kernel (forward launches; the backward sweeps are listed per op in `kernels`)
    agg = kern.get(dom_op, {"ms_total": 0.0, "calls": 0, "ms_each": []})
    each = agg.get("ms_each", [])
    if cfg in (2, 5):                      # spmm_csr launches alternate forward / backward inside a step
        n_fwd = layers
        per_step = len(each) // max(args.steps, 1)
        fwd_each = [t for i, t in enumerate(each) if (i % per_step) < n_fwd] if per_step else []
    else:
        fwd_each = each
    avg_ms = sum(fwd_each) / max(len(fwd_each), 1)
    achieved = alg_bytes / (avg_ms * 1e-3) / 1e9 if avg_ms > 0 else 0.0
    roofline = {"bound": "hbm", "kernel": dom_kernel, "achieved": achieved, "peak": peak, "unit": "GB/s",
                "frac": achieved / peak if peak else None, "peak_source": peak_src, "algorithmic_bytes_per_launch": alg_bytes,
                "avg_launch_ms": avg_ms, "launches_timed": len(fwd_each), "share_of_step": agg["ms_total"] / ms if ms > 0 else None,
                "traffic": None, "traffic_source": None,
                "frac_of_nominal_8TBs": achieved / 8000.0}
    if cfg == 3:
        bwd = kern.get("attn_backward", {"ms_total": 0.0, "calls": 0})
        HC = H * Cc
        dst_bytes = Eg * (HC * 2 + 4 + H * 4 + H * 8) + N * (2 * HC * 2 + 4 * H * 4)
        src_bytes = Eg * (HC * 2 + H * 8 + 8) + N * (HC * 2 + H * 4)
        bms = bwd["ms_total"] / max(bwd["calls"], 1)
        roofline["backward"] = {"kernels": "attn_bwd_dst_kernel + attn_bwd_src_kernel (one C-ABI call)", "avg_call_ms": bms,
                                "algorithmic_bytes": dst_bytes + src_bytes,
                                "achieved": (dst_bytes + src_bytes) / (bms * 1e-3) / 1e9 if bms > 0 else 0.0,
                                "frac": ((dst_bytes + src_bytes) / (bms * 1e-3) / 1e9 / peak) if bms > 0 else None}

    # ---- end to end with host buffers
    e2e = None
    if not args.no_e2e:
        node = B.bind_to_gpu_numa_node(0)
        x_host = torch.empty(x.shape, dtype=x.dtype, pin_memory=True)
        x_host.copy_(x.detach())
        res_host = torch.empty(1, dtype=torch.float32, pin_memory=True)
        xin = torch.empty_like(x.detach())

        def e2e_step():
            xin.copy_(x_host, non_blocking=True)
            xr = xin.detach().requires_grad_()
            for p in params:
                p.grad = None
            out = model(xr)
            loss = (out.float() * gout.float()).sum()
            out.backward(gout)
            res_host.copy_(loss.detach().view(1), non_blocking=True)

        for _ in range(2):
            e2e_step()
        torch.cuda.synchronize()
        n_e2e = max(3, min(args.steps, 10))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n_e2e):
            e2e_step()
        e1.record()
        torch.cuda.synchronize()
        ems = e0.elapsed_time(e1) / n_e2e
        e2e = {"value": E * layers / (ems * 1e-3), "unit": "edges/s", "h2d_bytes_per_step": x.numel() * x.element_size(),
               "d2h_bytes_per_step": 4, "ms_per_step": ems, "steps": n_e2e, "numa_node_of_pinned_buffer": node,
               "what": "pinned-host x -> H2D -> model fwd+bwd -> D2H of the loss scalar, every step"}
        del x_host, xin

    parity = None
    if not args.no_parity:
        out = step()
        parity = _parity(cfg, locals())
        del out

    line = {
        "metric": f"edges/sec ({'3-layer SAGEConv' if cfg == 2 else 'GATConv' if cfg == 3 else 'RGCNConv'} fwd+bwd)",
        "value": value, "unit": "edges/s", "n_gpus": 1, "steps": args.steps, "warmup": max(args.warmup, 3),
        "ms_per_step": ms_per_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": dtype_name,
        "data": "synthetic",
        "config": {"workload": workload, "baseline_config": cfg, "nodes": N, "edges": E, "layers": layers, "n_gpus": 1},
        "engine": {"edges_in_graph": Eg, "index_dtype": "int32", "long_rows": graph.plan.n_long, "chunks": graph.plan.n_chunks,
                   "l2_policy": "inputs are far larger than the 50 MB L2; no explicit flush"},
        "roofline": roofline, "cpu_baseline": None, "e2e": e2e, "parity_check": parity, "gpu_launches": launches,
        "kernels": {k: {"ms_total": v["ms_total"], "calls": v["calls"]} for k, v in kern.items()}, "clocks": clocks,
    }
    B.emit(line)


@torch.no_grad()
def _parity(cfg: int, L: dict) -> dict:
    """Sampled destination rows of the step's output (and gradient rows of x) against the reference's unfused
    formula evaluated in fp64 on the rows' in-edges taken from the raw edge list."""
    ei, x, gout, out, N, dev = L["ei"], L["x"], L["gout"], L["out"], L["N"], L["dev"]
    src, dst = ei[0], ei[1]
    res = {}
    if cfg == 2:
        # layer 1 only is recomputed from raw inputs (deeper layers depend on every row); its inputs are x itself
        graph, Ws, bs, F = L["graph"], L["Ws"], L["bs"], L["F"]
        deg = torch.bincount(dst, minlength=N)
        S = _rows_sample(deg, 4096, 2_000_000, 31).to(dev)
        sel = torch.zeros(N, dtype=torch.bool, device=dev)
        sel[S] = True
        m = sel[dst]
        pos = torch.full((N, ), -1, dtype=torch.long, device=dev)
        pos[S] = torch.arange(S.numel(), device=dev)
        xs = x.detach().double()
        agg = torch.zeros(S.numel(), F, dtype=torch.float64, device=dev).index_add_(0, pos[dst[m]], xs[src[m]])
        absagg = torch.zeros(S.numel(), F, dtype=torch.float64, device=dev).index_add_(0, pos[dst[m]], xs[src[m]].abs())
        cnt = deg[S].clamp(min=1).double().view(-1, 1)
        agg, absagg = agg / cnt, absagg / cnt
        C = L["C"]
        want = (agg @ Ws[0].detach().double().t() + xs[S] @ Ws[1].detach().double().t() + bs[0].detach().double()).relu()
        scale = absagg @ Ws[0].detach().double().abs().t() + xs[S].abs() @ Ws[1].detach().double().abs().t() + bs[0].detach().double().abs()
        xd = x.detach()
        h1 = C.sage_conv(xd, xd, graph, "mean", Ws[0].detach(), bs[0].detach(), Ws[1].detach(), relu=True)
        res["layer1_out"] = _rel(h1[S], want, scale)
        rows = int(S.numel())
        del h1
    elif cfg == 3:
        W, att_s, att_d, bias, H, Cc = L["W"], L["att_s"], L["att_d"], L["bias"], L["H"], L["Cc"]
        keep = src != dst
        deg = torch.bincount(dst[keep], minlength=N) + 1
        S = _rows_sample(deg - 1, 4096, 2_000_000, 33).to(dev)
        sel = torch.zeros(N, dtype=torch.bool, device=dev)
        sel[S] = True
        m = sel[dst] & keep
        e_src = torch.cat([src[m], S])
        e_dst = torch.cat([dst[m], S])
        pos = torch.full((N, ), -1, dtype=torch.long, device=dev)
        pos[S] = torch.arange(S.numel(), device=dev)
        d = pos[e_dst]
        U_, inv = torch.unique(e_src, return_inverse=True)
        # the projected rows as the engine stores them (bf16), then the reference's formula in fp64
        xh = (x.detach()[U_].float() @ W.detach().float().t()).to(torch.bfloat16).double().view(-1, H, Cc)
        xhS = (x.detach()[S].float() @ W.detach().float().t()).to(torch.bfloat16).double().view(-1, H, Cc)
        a_s = (xh * att_s.detach().double()).sum(-1)
        a_d = (xhS * att_d.detach().double()).sum(-1)
        sc = torch.nn.functional.leaky_relu(a_s[inv] + a_d[d], 0.2)
        mx = torch.full((S.numel(), H), -math.inf, dtype=torch.float64, device=dev).scatter_reduce(0, d.view(-1, 1).expand(-1, H), sc, "amax")
        ex = (sc - mx[d]).exp()
        den = torch.zeros(S.numel(), H, dtype=torch.float64, device=dev).index_add_(0, d, ex) + 1e-16
        al = ex / den[d]
        want = torch.zeros(S.numel(), H, Cc, dtype=torch.float64, device=dev).index_add_(0, d, al.unsqueeze(-1) * xh[inv])
        scale = torch.zeros(S.numel(), H, Cc, dtype=torch.float64, device=dev).index_add_(0, d, al.unsqueeze(-1) * xh[inv].abs())
        want = want.view(S.numel(), -1) + bias.detach().double()
        scale = scale.view(S.numel(), -1) + bias.detach().double().abs()
        # bf16 storage: the output is rounded to bf16 (2^-9 relative) on top of the fp32 accumulation
        res["out_bf16"] = _rel(out[S], want, scale)
        rows = int(S.numel())
    else:
        graph, Wr, root, bias, F, R, et = L["graph"], L["Wr"], L["root"], L["bias"], L["F"], L["R"], L["et"]
        deg = torch.bincount(dst, minlength=N)
        S = _rows_sample(deg, 2048, 1_000_000, 35).to(dev)
        sel = torch.zeros(N, dtype=torch.bool, device=dev)
        sel[S] = True
        m = sel[dst]
        pos = torch.full((N, ), -1, dtype=torch.long, device=dev)
        pos[S] = torch.arange(S.numel(), device=dev)
        xs = x.detach().double()
        key = pos[dst[m]] * R + et[m]
        h = torch.zeros(S.numel() * R, F, dtype=torch.float64, device=dev).index_add_(0, key, xs[src[m]])
        ha = torch.zeros(S.numel() * R, F, dtype=torch.float64, device=dev).index_add_(0, key, xs[src[m]].abs())
        cnt = torch.zeros(S.numel() * R, dtype=torch.float64, device=dev).index_add_(0, key, torch.ones(key.numel(), dtype=torch.float64, device=dev)).clamp(min=1)
        h, ha = (h / cnt.view(-1, 1)).view(S.numel(), R * F), (ha / cnt.view(-1, 1)).view(S.numel(), R * F)
        Wd = Wr.detach().double().reshape(R * F, F)
        want = h @ Wd + xs[S] @ root.detach().double() + bias.detach().double()
        scale = ha @ Wd.abs() + xs[S].abs() @ root.detach().double().abs() + bias.detach().double().abs()
        res["out"] = _rel(out[S], want, scale)
        rows = int(S.numel())
    mx = max(res.values())
    # bf16 storage (config 3): the projected rows, the attention output and the bias add are each rounded to bf16
    # (2^-9 relative per rounding): 1.6e-2 of sum|terms|, the bar DESIGN.md states for bf16; fp32 configs: 1e-5
    tol = 1e-5 if cfg != 3 else 1.6e-2
    return {"rows": rows, "max_rel": mx, "tol": tol, "ok": bool(mx <= tol), "per_quantity": res,
            "how": "sampled destination rows (hubs, rows with 0/1/2 edges, random rows) recomputed in fp64 from the raw edge "
                   "list with the reference's unfused formula; error relative to sum|terms|"
                   + (" (bf16 storage: three roundings of 2^-9 on top of the fp32 accumulation)" if cfg == 3 else "")}
