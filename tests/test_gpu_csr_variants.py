"""Every selectable variant of the CSR gather-reduce (csrc/csr_reduce.cuh, csr_tma.cuh, csr_dispatch.cuh) against each
other and against a float64 reference of the same operation on the storage-rounded inputs.

Variants: the lane-group kernel (spmm_impl 0 = auto, 1 = forced), the TMA-fed persistent kernel (spmm_impl 2, legal for
512 B <= row_bytes <= 2 KB), the launch variants spmm_tune 1-3 of the G = 32 / VPL = 2 sum shape, and the scalar fallback
(taken for odd widths and for any matrix that is not 16-byte aligned).  All of them walk a row in CSR order with fp32
__fmul_rn / __fadd_rn, cut hub rows at the same chunk boundaries and fold the chunks with the same csr_combine_kernel, so
their outputs must be bit-identical; each test proves once, with torch.profiler, that the kernel it names is the one
that ran.  Then the addressing modes (halo segment, peer table), the accumulate / ReLU-mask epilogue, the bf16 rounding
contract forward and backward, the edge-weight gradient (SDDMM) and non-finite inputs."""
import os
import re

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import pytorch_geometric_b200 as pgb  # noqa: E402
from pytorch_geometric_b200 import ops  # noqa: E402
from pytorch_geometric_b200._lib import B200MPError, lib  # noqa: E402
from pytorch_geometric_b200.graph import CSRGraph  # noqa: E402

DEV = "cuda"
REDUCES = ("sum", "mean", "min", "max")
BF16_HALF_ULP = 2.0 ** -8          # round-to-nearest bf16: |round(v) - v| <= 2^-8 |v|

# ------------------------------------------------------------------ engine options
# The options are process-wide.  conftest.py sets attn_staged / multi_tune from the environment for a whole session; the
# others start at the library default.  There is no getter, so a test restores the value by that same rule.
_OPTION_ENV = {"attn_staged": "B200MP_ATTN_STAGED", "multi_tune": "B200MP_MULTI_TUNE"}
_OPTION_DEFAULT = {"spmm_impl": 0, "spmm_tune": 0, "attn_staged": 2, "multi_tune": 6}


def session_option(name):
    env = _OPTION_ENV.get(name)
    if env is not None and os.environ.get(env) is not None:
        return int(os.environ[env])
    return _OPTION_DEFAULT[name]


@pytest.fixture
def engine_option():
    """engine_option(name, value) sets a library option for the rest of the test; every option touched is put back to
    its session value afterwards, whether the test passed or not."""
    touched = set()

    def set_option(name, value):
        touched.add(name)
        ops.set_option(name, value)

    try:
        yield set_option
    finally:
        for name in touched:
            ops.set_option(name, session_option(name))


# ------------------------------------------------------------------ which kernel ran
def kernels_launched(fn, attempts=8):
    """Names of the CUDA kernels `fn` launched (torch.profiler, CUDA activity).  The profiler now and then returns a
    session without some of its kernel records, so `fn` (which must be idempotent) is profiled again, up to `attempts`
    times, until a gather-reduce kernel shows up."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(attempts):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        if any(re.search(r"csr_\w+_kernel<", n) and "csr_combine_kernel" not in n for n in names):
            break
    return names


def _template_args(name):
    m = re.search(r"(csr_\w+_kernel)<(.*?)>\(", name)
    return (m.group(1), [a.strip() for a in m.group(2).split(",")]) if m else (None, [])


def assert_kernel(names, kernel, **args):
    """Exactly one gather-reduce kernel ran besides csr_combine_kernel, it is `kernel`, and its template arguments at
    the given positions (a0 = first) are the expected ones."""
    main = [_template_args(n) for n in names if re.search(r"csr_\w+_kernel<", n) and "csr_combine_kernel" not in n]
    assert len(main) == 1 and main[0][0] == kernel, f"expected {kernel}{args}, launched {names}"
    for k, v in args.items():
        assert main[0][1][int(k[1:])] == str(v), f"{kernel}: template argument {k} is not {v} in {names}"


def lane_bucket(n_vec):
    """(G, VPL) of csr_reduce_dispatch for a row of n_vec 16-byte vectors."""
    for lim, g in ((1, 1), (2, 2), (4, 4), (8, 8), (16, 16), (32, 32)):
        if n_vec <= lim:
            return g, 1
    return (32, 2) if n_vec <= 64 else (32, 4)


TUNE_LAUNCH = {1: (4, 256, 1), 2: (4, 256, 4), 3: (1, 256, 8)}          # spmm_tune k -> (UNR, BLOCK, MINB)


def expect_kernel(names, variant, dtype, F, reduce="sum"):
    kind, k = variant
    row_bytes = F * torch.empty(0, dtype=dtype).element_size()
    if kind == "scalar" or row_bytes % 16:
        return assert_kernel(names, "csr_reduce_scalar_kernel")
    n_vec = row_bytes // 16
    if kind == "impl" and k == 2 and 512 <= row_bytes <= 2048:
        return assert_kernel(names, "csr_tma_kernel", a2=1 if n_vec <= 32 else (2 if n_vec <= 64 else 4))
    g, vpl = lane_bucket(n_vec)
    if kind == "tune" and reduce in ("sum", "mean"):
        unr, block, minb = TUNE_LAUNCH[k]
    else:
        unr, block, minb = (1 if vpl >= 4 else 4 // vpl), 128, (12 if dtype == torch.float32 else 8)
    assert_kernel(names, "csr_reduce_kernel", a2=g, a3=vpl, a6=unr, a7=block, a8=minb)


# ------------------------------------------------------------------ inputs
def stress_csr(seed, n_src=300):
    """Row degrees built for the TMA kernel's 32-row work units: 205 rows (not a multiple of 32, last unit partial);
    unit 0 has hub rows at lanes 0, 15 and 31 and two adjacent ones (20, 21); unit 1 is all empty; unit 2 ends in
    trailing empty rows after a 70-edge row; unit 3 starts with empty rows and ends with a 33-edge row; the partial
    last unit has a hub at its second-to-last lane and an empty last row.  'Hub' means above chunk = 16 edges."""
    rng = np.random.default_rng(seed)
    n_rows = 32 * 6 + 13
    deg = rng.integers(0, 9, size=n_rows)
    deg[rng.random(n_rows) < 0.2] = 0
    deg[[0, 15, 20, 21, 31]] = [40, 37, 23, 90, 50]
    deg[32:64] = 0
    deg[67] = 70
    deg[74:96] = 0
    deg[96:101] = 0
    deg[127] = 33
    deg[201:203] = 0
    deg[203], deg[204] = 45, 0
    rowptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    col = rng.integers(0, n_src, size=int(rowptr[-1])).astype(np.int64)
    w = (rng.random(col.size) + 0.5).astype(np.float32)
    return rowptr, col, w, n_src


def rounded(a, dtype):
    """CPU tensor of `a` rounded to the storage dtype (the values the kernel reads)."""
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dtype)


def misaligned(t):
    """A contiguous copy of t whose storage starts one element past a 16-byte boundary."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


def messages(rowptr, col, w, x, reduce):
    """(destination of each edge, float64 message rows): min / max messages are the fp32 products the kernel forms."""
    rp = torch.as_tensor(rowptr)
    dst = torch.repeat_interleave(torch.arange(rp.numel() - 1), rp[1:] - rp[:-1])
    xs = x.float()[torch.as_tensor(col)]
    if w is None:
        return dst, xs.double()
    wt = torch.as_tensor(w).view(-1, 1)
    return dst, ((wt * xs).double() if reduce in ("min", "max") else xs.double() * wt.double())


def reference(rowptr, col, w, x, reduce, n_rows, gather=True):
    """float64 gather + reduce and the sum of |terms| per output element (the scale of a sum's rounding error)."""
    if gather:
        dst, msg = messages(rowptr, col, w, x, reduce)
    else:
        rp = torch.as_tensor(rowptr)
        dst, msg = torch.repeat_interleave(torch.arange(rp.numel() - 1), rp[1:] - rp[:-1]), x.double()
    F = msg.size(1)
    z = torch.zeros(n_rows, F, dtype=torch.float64)
    scale = z.index_add(0, dst, msg.abs())
    if reduce in ("sum", "mean"):
        out = z.index_add(0, dst, msg)
        if reduce == "mean":
            cnt = torch.bincount(dst, minlength=n_rows).clamp(min=1).double().view(-1, 1)
            out, scale = out / cnt, scale / cnt
    else:
        out = z.scatter_reduce(0, dst.view(-1, 1).expand(-1, F), msg, "amin" if reduce == "min" else "amax",
                               include_self=False)
    return out, scale


def check_reference(got, ref, scale, reduce, dtype, bias=None, what=""):
    """min / max: exactly the fp32 extremum (+ fp32 bias) rounded once to the storage dtype.  sum / mean: within
    1e-5 * sum|terms| of the float64 value (fp32 accumulation), plus one bf16 rounding for bf16 output."""
    got = got.detach().cpu()
    if reduce in ("min", "max"):
        r = ref.float()
        if bias is not None:
            r = r + bias.cpu()
        want = r.to(dtype)
        assert torch.equal(got, want), f"{what}: {reduce} differs at {torch.nonzero(got != want)[:5].tolist()}"
        return
    r = ref + (bias.cpu().double() if bias is not None else 0.0)
    tol = 1e-5 * scale + 1e-7 * r.abs() + 1e-30
    if dtype == torch.bfloat16:
        tol = tol + BF16_HALF_ULP * r.abs()
    err = (got.double() - r).abs()
    assert (err <= tol).all(), f"{what}: {reduce} max err {err.max().item():.3e}, worst ratio {(err / tol).max().item():.2f}"


def device_csr(rowptr, col, w, idx_dtype):
    return (torch.from_numpy(rowptr).to(DEV, idx_dtype), torch.from_numpy(col).to(DEV, idx_dtype),
            None if w is None else torch.from_numpy(w).to(DEV))


def variants(dtype, F, reduce, gather=True):
    """The kernel variants that exist for this call: ('impl', 0 | 1 | 2), ('tune', 1..3), ('scalar', 0)."""
    row_bytes = F * torch.empty(0, dtype=dtype).element_size()
    vs = [("impl", 0), ("impl", 1)]
    if row_bytes % 16 == 0:
        if 512 <= row_bytes <= 2048:
            vs.append(("impl", 2))
        if gather and 32 < row_bytes // 16 <= 64 and reduce in ("sum", "mean"):
            vs += [("tune", 1), ("tune", 2), ("tune", 3)]
        vs.append(("scalar", 0))
    return vs


def select(engine_option, variant):
    kind, k = variant
    engine_option("spmm_impl", k if kind == "impl" else 0)
    engine_option("spmm_tune", k if kind == "tune" else 0)


SENTINEL = float("nan")            # output rows a kernel forgets to write stay NaN: never equal, never close


# ------------------------------------------------------------------ A. the variant matrix
A_SHAPES = ([(torch.float32, F) for F in (1, 3, 4, 8, 12, 16, 32, 64, 128, 132, 256, 512)] +
            [(torch.bfloat16, F) for F in (5, 12, 8, 16, 32, 64, 128, 256, 264, 512, 1024)])


@pytest.mark.parametrize("dtype,F", A_SHAPES, ids=[f"{str(d)[6:]}-F{F}" for d, F in A_SHAPES])
def test_spmm_variants_bit_identical_and_match_fp64(engine_option, dtype, F):
    """Every variant of b200mp_spmm_csr x {sum, mean, min, max} x {unweighted, weighted} x {int32, int64} x {no plan,
    chunk = 16} x {no bias, bias}: bit-identical to each other (and int32 == int64), and one of them against float64.
    bf16 sum / mean are held to one bf16 rounding, min / max to exactly round_bf16(max_e fp32(w * x))."""
    rowptr, col, w, n_src = stress_csr(F)
    n_rows = rowptr.size - 1
    rng = np.random.default_rng(F + 1)
    x_cpu = rounded(rng.standard_normal((n_src, F)), dtype)
    x = x_cpu.to(DEV)
    bias_t = torch.from_numpy(rng.standard_normal(F).astype(np.float32)).to(DEV)
    proven = set()
    for reduce in REDUCES:
        vs = variants(dtype, F, reduce)
        for weighted in (False, True):
            ref, scale = reference(rowptr, col, w if weighted else None, x_cpu, reduce, n_rows)
            by_idx = {}
            for idx_dtype in (torch.int32, torch.int64):
                rp, cl, val = device_csr(rowptr, col, w if weighted else None, idx_dtype)
                for chunk in (None, 16):
                    plan = ops.LongRowPlan(rp, chunk) if chunk else None
                    if chunk:
                        assert plan.n_long == 8
                    for bias in (None, bias_t):
                        outs = []
                        for v in vs:
                            select(engine_option, v)
                            xv = misaligned(x) if v[0] == "scalar" else x
                            out = torch.full((n_rows, F), SENTINEL, dtype=dtype, device=DEV)

                            def call():
                                ops.spmm_csr(rp, cl, val, xv, n_rows, reduce, plan, out=out, bias=bias)
                            if (v, reduce in ("sum", "mean")) not in proven:
                                proven.add((v, reduce in ("sum", "mean")))
                                expect_kernel(kernels_launched(call), v, dtype, F, reduce)
                            else:
                                call()
                            outs.append(out)
                        tag = f"{reduce} w={weighted} {idx_dtype} chunk={chunk} bias={bias is not None}"
                        for v, o in zip(vs[1:], outs[1:]):
                            assert torch.equal(o, outs[0]), f"{tag}: {v} differs from {vs[0]}"
                        check_reference(outs[0], ref, scale, reduce, dtype, bias, tag)
                        key = (chunk, bias is not None)
                        if key in by_idx:
                            assert torch.equal(by_idx[key], outs[0]), f"{tag}: int32 and int64 indices differ"
                        by_idx[key] = outs[0]


SEG_SHAPES = [(torch.float32, 128), (torch.float32, 132), (torch.float32, 512), (torch.bfloat16, 256),
              (torch.bfloat16, 1024), (torch.float32, 6)]


@pytest.mark.parametrize("dtype,F", SEG_SHAPES, ids=[f"{str(d)[6:]}-F{F}" for d, F in SEG_SHAPES])
def test_segment_variants_bit_identical_and_match_fp64(engine_option, dtype, F):
    """The non-gather entry (b200mp_segment_csr) under spmm_impl 0 / 1 / 2 and the scalar fallback, with and without
    a chunk plan, int32 and int64 offsets."""
    rowptr, _, _, _ = stress_csr(F + 7)
    n_rows, E = rowptr.size - 1, int(rowptr[-1])
    src_cpu = rounded(np.random.default_rng(F).standard_normal((E, F)), dtype)
    src = src_cpu.to(DEV)
    proven = set()
    for reduce in REDUCES:
        ref, scale = reference(rowptr, None, None, src_cpu, reduce, n_rows, gather=False)
        vs = [v for v in variants(dtype, F, reduce, gather=False)]
        for idx_dtype in (torch.int32, torch.int64):
            ptr = torch.from_numpy(rowptr).to(DEV, idx_dtype)
            for chunk in (None, 16):
                plan = ops.LongRowPlan(ptr, chunk) if chunk else None
                outs = []
                for v in vs:
                    select(engine_option, v)
                    sv = misaligned(src) if v[0] == "scalar" else src
                    res = []
                    if v not in proven:
                        proven.add(v)
                        names = kernels_launched(lambda: res.append(ops.segment_csr(sv, ptr, reduce, plan)))
                        expect_kernel(names, v, dtype, F, reduce)
                        if v == ("impl", 2):
                            assert_kernel(names, "csr_tma_kernel", a4="false")
                    else:
                        res.append(ops.segment_csr(sv, ptr, reduce, plan))
                    outs.append(res[-1])
                tag = f"segment {reduce} {idx_dtype} chunk={chunk}"
                for v, o in zip(vs[1:], outs[1:]):
                    assert torch.equal(o, outs[0]), f"{tag}: {v} differs from {vs[0]}"
                check_reference(outs[0], ref, scale, reduce, dtype, None, tag)


# ------------------------------------------------------------------ B. addressing and epilogue modes
@pytest.mark.parametrize("dtype,F", [(torch.float32, 256), (torch.float32, 132), (torch.bfloat16, 512),
                                     (torch.float32, 16), (torch.bfloat16, 12)])
def test_halo_segment_equals_the_concatenated_matrix(engine_option, dtype, F):
    """x_halo: columns >= split (77, not a multiple of 32) are read from a second matrix.  Bit-identical to the same
    call on torch.cat([x, x_halo]) under the lane-group kernel, the TMA kernel, the scalar kernel (misaligned x) and a
    misaligned halo alone (which must also fall back to the scalar kernel)."""
    rowptr, col, w, n_src = stress_csr(3)
    n_rows, split = rowptr.size - 1, 77
    x_all = rounded(np.random.default_rng(F).standard_normal((n_src, F)), dtype).to(DEV)
    x_loc, x_halo = x_all[:split].clone(), x_all[split:].clone()
    rp, cl, val = device_csr(rowptr, col, w, torch.int32)
    bias = torch.linspace(-1, 1, F, device=DEV)
    vec = (F * x_all.element_size()) % 16 == 0
    cases = [("impl", 1, False, False), ("impl", 2, False, False)]
    if vec:
        cases += [("scalar", 0, True, False), ("halo", 0, False, True), ("halo", 2, False, True)]
    for reduce in REDUCES:
        for chunk in (None, 16):
            plan = ops.LongRowPlan(rp, chunk) if chunk else None
            for kind, k, mis_x, mis_h in cases:
                engine_option("spmm_impl", k)
                want = ops.spmm_csr(rp, cl, val, x_all, n_rows, reduce, plan, bias=bias)
                xl = misaligned(x_loc) if mis_x else x_loc
                xh = misaligned(x_halo) if mis_h else x_halo
                res = []
                names = kernels_launched(lambda: res.append(ops.spmm_csr(rp, cl, val, xl, n_rows, reduce, plan, bias=bias,
                                                                        x_halo=xh)))
                if reduce == "sum" and chunk is None:
                    expect_kernel(names, ("scalar", 0) if (mis_x or mis_h) else ("impl", k), dtype, F)
                assert torch.equal(res[-1], want), f"{reduce} chunk={chunk} {kind}{k}"


def _peer_shards(dtype, F, n_local, sizes, seed):
    g = torch.Generator().manual_seed(seed)
    shards = [torch.randn(n, F, generator=g).to(dtype).to(DEV) for n in sizes]
    table = torch.tensor([s.data_ptr() for s in shards], dtype=torch.int64, device=DEV)
    return shards, table


@pytest.mark.parametrize("dtype,F", [(torch.float32, 256), (torch.float32, 16), (torch.bfloat16, 128),
                                     (torch.bfloat16, 1024)])
def test_peer_table_equals_the_concatenated_matrix(engine_option, dtype, F):
    """peer_ptrs: the source matrix as R separate shards of peer_rows rows, addressed through a device table of their
    base pointers (one device stands in for R GPUs).  Full shards and a shorter last shard, with a chunk plan and
    bias, bit-identical to the aggregate over torch.cat(shards); spmm_impl 2 must not take the TMA kernel here."""
    n_local = 100
    for sizes in ((100, 100, 100), (100, 100, 37)):
        shards, table = _peer_shards(dtype, F, n_local, sizes, seed=F + sizes[-1])
        x_cat = torch.cat(shards)
        rowptr, col, w, _ = stress_csr(F, n_src=sum(sizes))
        n_rows = rowptr.size - 1
        rp, cl, val = device_csr(rowptr, col, w, torch.int64)
        bias = torch.linspace(-2, 2, F, device=DEV)
        for impl in (0, 2):
            engine_option("spmm_impl", impl)
            for reduce in REDUCES:
                for chunk in (None, 16):
                    plan = ops.LongRowPlan(rp, chunk) if chunk else None
                    want = ops.spmm_csr(rp, cl, val, x_cat, n_rows, reduce, plan, bias=bias)
                    res = []

                    def call():
                        res.append(ops.spmm_csr(rp, cl, val, shards[0], n_rows, reduce, plan, bias=bias,
                                                peer_ptrs=table.data_ptr(), peer_rows=n_local))
                    if reduce == "max" and chunk == 16 and len(set(sizes)) > 1:
                        expect_kernel(kernels_launched(call), ("impl", 1), dtype, F, reduce)
                    else:
                        call()
                    assert torch.equal(res[-1], want), f"shards {sizes} impl={impl} {reduce} chunk={chunk}"


def test_peer_table_refuses_a_misaligned_x_or_out():
    """The scalar fallback has no peer-table addressing (it would read x[c] with the global column id), so a peer-table
    call whose x, out or ReLU mask is not 16-byte aligned is refused on the host: B200MP_ERR_INVALID_ARG, no launch."""
    F, n_local = 64, 50
    shards, table = _peer_shards(torch.float32, F, n_local, (50, 50), seed=1)
    rowptr, col, _, _ = stress_csr(2, n_src=100)
    n_rows = rowptr.size - 1
    rp, cl, _ = device_csr(rowptr, col, None, torch.int32)
    out_ok = torch.zeros(n_rows, F, device=DEV)
    calls = {
        "x": lambda: ops.spmm_csr(rp, cl, None, misaligned(shards[0]), n_rows, "sum", peer_ptrs=table.data_ptr(),
                                  peer_rows=n_local),
        "out": lambda: ops.spmm_csr(rp, cl, None, shards[0], n_rows, "sum", out=misaligned(out_ok),
                                    peer_ptrs=table.data_ptr(), peer_rows=n_local),
        "relu_mask": lambda: ops.spmm_csr(rp, cl, None, shards[0], n_rows, "sum", out=out_ok.clone(), accumulate=True,
                                          relu_mask=misaligned(out_ok), peer_ptrs=table.data_ptr(), peer_rows=n_local),
    }
    for what, call in calls.items():
        errors = []

        def guarded():
            try:
                call()
            except B200MPError as e:
                errors.append(str(e))
            # positive control in the same profiler session: the aligned call's kernel is recorded, and only it
            ops.spmm_csr(rp, cl, None, shards[0], n_rows, "sum", out=out_ok, peer_ptrs=table.data_ptr(),
                         peer_rows=n_local)
        names = kernels_launched(guarded)
        assert errors and "invalid argument" in errors[0], f"misaligned {what}: {errors}"
        assert len([n for n in names if "csr_" in n]) == 1, f"misaligned {what}: launched {names}"
        expect_kernel(names, ("impl", 0), torch.float32, F)
    # the C ABI itself: B200MP_ERR_INVALID_ARG (-1)
    x_mis, out = misaligned(shards[0]), torch.zeros(n_rows, F, device=DEV)
    rc = lib().b200mp_spmm_csr(rp.data_ptr(), cl.data_ptr(), None, x_mis.data_ptr(), out.data_ptr(), n_rows, 100, F, 0,
                               None, None, 0, 0, 0, None, None, None, 0, 0, table.data_ptr(), n_local, None, 0, 0,
                               torch.cuda.current_stream().cuda_stream)
    assert rc == -1
    torch.cuda.synchronize()
    assert torch.equal(out, torch.zeros_like(out))
    # the aligned call is accepted and equals the concatenated matrix
    got = ops.spmm_csr(rp, cl, None, shards[0], n_rows, "sum", peer_ptrs=table.data_ptr(), peer_rows=n_local)
    assert torch.equal(got, ops.spmm_csr(rp, cl, None, torch.cat(shards), n_rows, "sum"))


@pytest.mark.parametrize("dtype,F", [(torch.float32, 64), (torch.float32, 256), (torch.bfloat16, 512),
                                     (torch.bfloat16, 16), (torch.float32, 5)])
def test_accumulate_and_relu_mask(engine_option, dtype, F):
    """accumulate: out[i] = round(out[i] + acc_fp32[i]) for rows with edges, rows without edges untouched; with
    relu_mask, every row (empty ones too) is then zeroed where mask <= 0.  acc_fp32 is the fp32 sum itself, taken from
    the fp32 kernel on the same storage-rounded values (same order, same chunks => the same bits).  Hub rows go
    through csr_combine_kernel (chunk = 16); the vector kernel and the scalar kernel (misaligned x, and a misaligned
    mask alone) are both covered; spmm_impl 2 must not take the TMA kernel (it has no accumulate epilogue)."""
    rowptr, col, w, n_src = stress_csr(F + 11)
    n_rows = rowptr.size - 1
    rng = np.random.default_rng(F)
    x = rounded(rng.standard_normal((n_src, F)), dtype).to(DEV)
    out0 = rounded(rng.standard_normal((n_rows, F)), dtype).to(DEV)
    mask = rounded(rng.standard_normal((n_rows, F)) * (rng.random((n_rows, F)) < 0.8), dtype).to(DEV)
    deg = torch.from_numpy(np.diff(rowptr)).to(DEV).view(-1, 1)
    rp, cl, val = device_csr(rowptr, col, w, torch.int32)
    vec = (F * x.element_size()) % 16 == 0
    for chunk in (None, 16):
        plan = ops.LongRowPlan(rp, chunk) if chunk else None
        acc32 = ops.spmm_csr(rp, cl, val, x.float(), n_rows, "sum", plan)
        summed = torch.where(deg > 0, (out0.float() + acc32).to(dtype), out0)
        masked = torch.where(mask > 0, summed, torch.zeros_like(summed))
        for impl, mis_x, mis_m in ((0, False, False), (2, False, False), (0, True, False), (0, False, True)):
            if not vec and (mis_x or mis_m):
                continue
            engine_option("spmm_impl", impl)
            xv = misaligned(x) if mis_x else x
            for m in (None, misaligned(mask) if mis_m else mask):
                if mis_m and m is None:
                    continue
                out = out0.clone()

                def call():
                    out.copy_(out0)
                    ops.spmm_csr(rp, cl, val, xv, n_rows, "sum", plan, out=out, accumulate=True, relu_mask=m)
                if chunk == 16:
                    expect_kernel(kernels_launched(call), ("scalar", 0) if (mis_x or mis_m) else ("impl", 1), dtype, F)
                else:
                    call()
                assert torch.equal(out, masked if m is not None else summed), \
                    f"chunk={chunk} impl={impl} misaligned x={mis_x} mask={mis_m} relu_mask={m is not None}"


# ------------------------------------------------------------------ C. bf16 backward and the edge-weight gradient
def _coarse_graph(seed, N=260, E=5000):
    rng = np.random.default_rng(seed)
    src = rng.integers(0, N, size=E)
    dst = ((rng.random(E) ** 2.5) * (N - 4)).astype(np.int64)          # hubs near 0, the last rows empty
    return rng, src, dst, N


@pytest.mark.parametrize("F", [5, 64, 256, 512])
@pytest.mark.parametrize("weighted", [False, True])
def test_bf16_backward_vs_fp64(F, weighted):
    """bf16 backward of sum, mean, min and max on a coarse value grid (real ties, exact zeros) against float64.
    min / max follow the engine's rule: the ties of out[i, f] are the edges whose product, rounded to bf16, equals
    out[i, f], plus one when out[i, f] == 0 (count_self_zero), and the gradient is split evenly among them.  The
    weights carry bits below bf16 precision, so a tie test on the unrounded product would find no tie at all."""
    rng, src, dst, N = _coarse_graph(F + weighted)
    x = torch.from_numpy(np.round(rng.standard_normal((N, F)) * 2) / 2).float().bfloat16()
    w = torch.from_numpy(rng.choice(np.array([0.75, 1.0, 1.0078125, 1.25], np.float32), size=src.size))
    gout = torch.randn(N, F, generator=torch.Generator().manual_seed(F)).bfloat16()
    g = CSRGraph(torch.from_numpy(src).to(DEV), torch.from_numpy(dst).to(DEV), N, N,
                 w.to(DEV) if weighted else None, chunk=32)
    assert g.plan.n_long > 0
    s, d = torch.from_numpy(src), torch.from_numpy(dst)
    wd = w.double() if weighted else torch.ones(src.size, dtype=torch.float64)
    deg = torch.bincount(d, minlength=N).double()
    for reduce in REDUCES:
        xt = x.to(DEV).requires_grad_()
        out = pgb.aggregate(g, xt, reduce)
        out.backward(gout.to(DEV))
        go = gout.double()
        if reduce in ("sum", "mean"):
            coef = wd / (deg[d].clamp(min=1) if reduce == "mean" else 1.0)
            terms = coef.view(-1, 1) * go[d]
        else:
            prod = ((w.view(-1, 1) if weighted else 1.0) * x.float()[s]).bfloat16().double()
            o = out.detach().cpu().double()
            hit = prod == o[d]
            ties = torch.zeros(N, F, dtype=torch.float64).index_add(0, d, hit.double()) + (o == 0).double()
            terms = torch.where(hit, wd.view(-1, 1) * go[d] / ties[d], torch.zeros_like(go[d]))
        ref = torch.zeros(N, F, dtype=torch.float64).index_add(0, s, terms)
        scale = torch.zeros(N, F, dtype=torch.float64).index_add(0, s, terms.abs())
        assert torch.isfinite(xt.grad).all(), f"{reduce}: non-finite gradient (a tie count of zero?)"
        err = (xt.grad.cpu().double() - ref).abs()
        tol = BF16_HALF_ULP * ref.abs() + 1e-5 * scale + 1e-30
        assert (err <= tol).all(), f"{reduce}: max err {err.max().item():.3e} ratio {(err / tol).max().item():.2f}"


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("F", [1, 33, 256, 300, 1024])
def test_sddmm_edge_weight_gradient_vs_fp64(F, dtype):
    """b200mp_sddmm_csr: dot[e] = <a[row(e)], b[col[e]]> in CSR order -- up to 8 values per lane stay in registers,
    wider rows are re-read -- and the edge-weight gradient of sum / mean aggregation built on it."""
    rng, src, dst, N = _coarse_graph(F, E=3000)
    gen = torch.Generator().manual_seed(F)
    a = torch.randn(N, F, generator=gen).to(dtype)
    b = torch.randn(N, F, generator=gen).to(dtype)
    g = CSRGraph(torch.from_numpy(src).to(DEV), torch.from_numpy(dst).to(DEV), N, N)
    dot = ops.sddmm_csr(g.rowptr, g.col, a.to(DEV), b.to(DEV)).cpu().double()
    rp = g.rowptr.long().cpu()
    row = torch.repeat_interleave(torch.arange(N), rp[1:] - rp[:-1])
    cl = g.col.long().cpu()
    ref = (a.double()[row] * b.double()[cl]).sum(1)
    scale = (a.double()[row].abs() * b.double()[cl].abs()).sum(1)
    assert ((dot - ref).abs() <= 1e-5 * scale + 1e-30).all(), f"sddmm max err {(dot - ref).abs().max().item():.3e}"
    w = torch.from_numpy((rng.random(src.size) + 0.5).astype(np.float32))
    deg = torch.bincount(torch.from_numpy(dst), minlength=N).double()
    for reduce in ("sum", "mean"):
        wt = w.to(DEV).requires_grad_()
        out = pgb.aggregate(g, b.to(DEV), reduce, edge_weight=wt)
        out.backward(a.to(DEV))
        d, s = torch.from_numpy(dst), torch.from_numpy(src)
        gw = (a.double()[d] * b.double()[s]).sum(1)
        gscale = (a.double()[d].abs() * b.double()[s].abs()).sum(1)
        if reduce == "mean":
            gw, gscale = gw / deg[d], gscale / deg[d]
        err = (wt.grad.cpu().double() - gw).abs()
        assert (err <= 1e-5 * gscale + 1e-30).all(), f"{reduce} weight grad max err {err.max().item():.3e}"


# ------------------------------------------------------------------ D. non-finite inputs
def _nonfinite(a, seed):
    """Feature 0 is -inf everywhere (rows whose messages are all -inf), feature 1 +inf everywhere, and about 2% of
    the other entries each NaN, +inf or -inf."""
    rng = np.random.default_rng(seed)
    a = a.copy()
    a[:, 0], a[:, 1] = -np.inf, np.inf
    r = rng.random(a.shape)
    a[:, 2:][r[:, 2:] < 0.02] = np.nan
    a[:, 2:][(r[:, 2:] >= 0.02) & (r[:, 2:] < 0.04)] = np.inf
    a[:, 2:][(r[:, 2:] >= 0.04) & (r[:, 2:] < 0.06)] = -np.inf
    return a


def aten_reference(dst, msg, reduce, n_rows):
    """ATen's own CPU scatter_reduce_(include_self=False) on a zero tensor, in float64."""
    F = msg.size(1)
    op = {"sum": "sum", "mean": "mean", "min": "amin", "max": "amax"}[reduce]
    return torch.zeros(n_rows, F, dtype=torch.float64).scatter_reduce_(0, dst.view(-1, 1).expand(-1, F), msg, op,
                                                                      include_self=False)


def assert_nonfinite_match(got, ref, reduce, dtype, what):
    got = got.detach().cpu().double()
    for name, f in (("nan", torch.isnan), ("+inf", torch.isposinf), ("-inf", torch.isneginf)):
        bad = f(got) != f(ref)
        assert not bad.any(), f"{what}: {name} pattern differs at {torch.nonzero(bad)[:5].tolist()}"
    fin = torch.isfinite(ref)
    if reduce in ("min", "max"):
        assert torch.equal(got[fin], ref.float().to(dtype).double()[fin]), what
    else:
        tol = 1e-4 * ref[fin].abs().max() + 1e-6 + (BF16_HALF_ULP * ref[fin].abs() if dtype == torch.bfloat16 else 0)
        assert ((got[fin] - ref[fin]).abs() <= tol).all(), what


@pytest.mark.parametrize("dtype,F", [(torch.float32, 5), (torch.float32, 128), (torch.bfloat16, 256)])
def test_non_finite_inputs(engine_option, dtype, F):
    """NaN propagates through min and max as ATen's amax / amin do; +-inf survives the gather path (and the weight
    product); a row whose messages are all -inf gives what ATen gives; the segment path maps +-inf of min / max to 0.
    Under spmm_impl 0 / 1 / 2 and through the chunked hub path, whose partials carry NaN / inf into
    csr_combine_kernel."""
    rowptr, col, w, n_src = stress_csr(F + 5)
    n_rows = rowptr.size - 1
    x_cpu = rounded(_nonfinite(np.random.default_rng(F).standard_normal((n_src, F)), F), dtype)
    E = int(rowptr[-1])
    src_cpu = rounded(_nonfinite(np.random.default_rng(F + 1).standard_normal((E, F)), F + 1), dtype)
    x, src = x_cpu.to(DEV), src_cpu.to(DEV)
    rp_cpu = torch.from_numpy(rowptr)
    seg_dst = torch.repeat_interleave(torch.arange(n_rows), rp_cpu[1:] - rp_cpu[:-1])
    rp, cl, val = device_csr(rowptr, col, w, torch.int32)
    for reduce in REDUCES:
        refs = {wt: aten_reference(*messages(rowptr, col, w if wt else None, x_cpu, reduce), reduce, n_rows)
                for wt in (False, True)}
        seg_ref = aten_reference(seg_dst, src_cpu.double(), reduce, n_rows)
        if reduce in ("min", "max"):
            seg_ref[torch.isinf(seg_ref)] = 0.0
        for chunk in (None, 16):
            plan = ops.LongRowPlan(rp, chunk) if chunk else None
            first = {}
            for impl in (0, 1, 2):
                engine_option("spmm_impl", impl)
                for wt in (False, True):
                    out = torch.full((n_rows, F), 7.0, dtype=dtype, device=DEV)
                    ops.spmm_csr(rp, cl, val if wt else None, x, n_rows, reduce, plan, out=out)
                    what = f"gather {reduce} weighted={wt} chunk={chunk} impl={impl}"
                    assert_nonfinite_match(out, refs[wt], reduce, dtype, what)
                    torch.testing.assert_close(out, first.setdefault(wt, out), rtol=0, atol=0, equal_nan=True, msg=what)
                seg = ops.segment_csr(src, rp, reduce, plan)
                what = f"segment {reduce} chunk={chunk} impl={impl}"
                assert_nonfinite_match(seg, seg_ref, reduce, dtype, what)
                torch.testing.assert_close(seg, first.setdefault("seg", seg), rtol=0, atol=0, equal_nan=True, msg=what)
