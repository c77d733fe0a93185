"""The other A/B switches of the library, selected in-process instead of through B200MP_ATTN_STAGED /
B200MP_MULTI_TUNE for a whole session: every setting is checked against float64 at the tolerances of
test_gpu_attention.py and test_gpu_multi_aggr.py, and settings that run the same kernel template with another CTA size
(hence the same per-row summation order) must agree bit for bit."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from pytorch_geometric_b200 import functional as Fn  # noqa: E402
from pytorch_geometric_b200._lib import lib  # noqa: E402
from pytorch_geometric_b200.graph import CSRGraph  # noqa: E402
from test_gpu_attention import _problem, ref_attention  # noqa: E402
from test_gpu_csr_variants import engine_option  # noqa: E402,F401  (fixture)
from test_gpu_multi_aggr import test_gather_mode_vs_oracle as gather_mode_vs_oracle  # noqa: E402

DEV = "cuda"

# n_vec = H * C * element size / 16; the staged sweeps take 4 < n_vec <= 32
ATTN_CASES = [("gat", 8, 16, torch.float32),      # n_vec 32: staged
              ("gatv2", 8, 16, torch.bfloat16),   # n_vec 16: staged
              ("dot", 4, 8, torch.float32),       # n_vec 8: staged
              ("dot", 2, 128, torch.float32),     # n_vec 64: register form under every setting
              ("gat", 3, 4, torch.float32)]       # n_vec 3: register form under every setting


@pytest.mark.parametrize("mode,H,C,dtype", ATTN_CASES)
def test_attention_under_every_attn_staged(engine_option, mode, H, C, dtype):
    """attn_staged 0 (register loop), 1 (staged, 4-warp CTAs) and 2 (staged, one-warp CTAs), forward and backward with
    hub rows cut at chunk = 16, against the unfused float64 formula.  1 and 2 launch the same kernel templates with
    128- and 32-thread CTAs, so out, alpha and every gradient must be bit-identical between them."""
    p = _problem(mode, H, C, dtype, seed=H * 31 + C + len(mode))
    n_src, n_dst = p["v"].size(0), p["gout"].size(0)
    names = [n for n in ("v", "k", "q", "s_src", "s_dst", "att") if n in p]
    scale = 1.0 / math.sqrt(C)
    ref_in = {n: p[n].clone().to(DEV).requires_grad_() for n in names}
    ref_out, ref_alpha = ref_attention(mode, p["src"].to(DEV), p["dst"].to(DEV), n_dst, H, C, slope=0.2, scale=scale,
                                       **ref_in)
    ref_out.backward(p["gout"].to(DEV))
    graph = CSRGraph(p["src"].to(DEV), p["dst"].to(DEV), n_src, n_dst, chunk=16)
    assert graph.plan.n_long > 0
    perm = graph.perm.long()
    fp32 = dtype == torch.float32
    results = {}
    for staged in (0, 1, 2):
        engine_option("attn_staged", staged)
        ours = {n: (p[n].to(dtype) if n in ("v", "k", "q") else p[n].float()).to(DEV).requires_grad_() for n in names}
        out, alpha = Fn.attention(mode, graph, H, C, negative_slope=0.2, scale=scale, return_alpha=True, **ours)
        out.backward(p["gout"].to(dtype).to(DEV))

        def close(a, b, what, t):
            a, b = a.detach().double(), b.detach().double()
            err = (a - b).abs().max().item()
            assert err <= t * max(b.abs().max().item(), 1e-3), f"attn_staged={staged} {what}: max err {err:.3e}"

        close(out, ref_out, "out", 2e-5 if fp32 else 1.5e-2)
        close(alpha, ref_alpha[perm], "alpha", 1e-4 if fp32 else 1.5e-2)
        for n in names:
            close(ours[n].grad, ref_in[n].grad, "grad_" + n, 2e-4 if fp32 else 3e-2)
        results[staged] = [out, alpha] + [ours[n].grad for n in names]
    for i, (a, b) in enumerate(zip(results[1], results[2])):
        assert torch.equal(a, b), f"attn_staged 1 and 2 differ in output {i} ({(['out', 'alpha'] + names)[i]})"


@pytest.mark.parametrize("F", [96, 132, 256])
def test_multi_aggregation_under_multi_tune_and_attn_staged(engine_option, F):
    """The graph-mode multi-aggregation check of test_gpu_multi_aggr.py (sum, mean, min, max, var, std, forward and
    backward, chunk = 16) under multi_tune 5 / 6 x attn_staged 0 / 2.  At these fp32 widths the backward takes the
    hit-bit path exactly when attn_staged != 0 (b200mp_multi_aggr_mask_supported).  multi_tune 5 and 6 launch the same
    row-sweep and staged-backward templates with 128- and 32-thread CTAs, so for one attn_staged value every output and
    the input gradient must be bit-identical between them."""
    rng = np.random.default_rng(F)
    N, E = 700, 20000
    src = torch.from_numpy(rng.integers(0, N, size=E)).to(DEV)
    dst = torch.from_numpy(((rng.random(E) ** 3) * (N - 5)).astype(np.int64)).to(DEV)
    x = torch.from_numpy(rng.standard_normal((N, F)).astype(np.float32) * (rng.random((N, F)) > 0.2)).to(DEV)
    gouts = [torch.randn(N, F, device=DEV, generator=torch.Generator(device=DEV).manual_seed(k)) for k in range(6)]
    aggrs = ["sum", "mean", "min", "max", "var", "std"]
    g = CSRGraph(src, dst, N, N, chunk=16)
    for staged in (0, 2):
        engine_option("attn_staged", staged)
        assert bool(lib().b200mp_multi_aggr_mask_supported(F, 0, 0)) == (staged != 0)
        runs = {}
        for tune in (5, 6):
            engine_option("multi_tune", tune)
            gather_mode_vs_oracle(F, torch.float32, 16)
            xt = x.clone().requires_grad_()
            outs = Fn.multi_aggregate(g, xt, aggrs)
            torch.autograd.backward(outs, gouts)
            runs[tune] = list(outs) + [xt.grad]
        for name, a, b in zip(aggrs + ["grad_x"], runs[5], runs[6]):
            assert torch.equal(a, b), f"attn_staged={staged}: multi_tune 5 and 6 differ in {name}"
