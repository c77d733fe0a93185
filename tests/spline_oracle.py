"""fp64 restatement of the B-spline basis and weighting that SplineConv takes from pyg_lib.ops (spline_conv.py:15-18,
150-153), written from the convention of torch-spline-conv's basis kernels: for slot s in [0, (degree + 1)^D), with
dimension 0 varying fastest,

    v_d = pseudo[e, d] * (kernel_size[d] - degree * is_open_spline[d])       computed in fp32, as the CUDA kernel does,
    k_d = (s // (degree + 1)^d) % (degree + 1)                               so floor(v_d) and the indices are bit-exact
    weight_index = sum_d ((floor(v_d) + k_d) mod kernel_size[d]) * prod_{d' < d} kernel_size[d']
    basis = prod_d B_degree(v_d - floor(v_d), k_d)

Everything after v is fp64.  The numpy functions are the oracle of the GPU tests; `torch_spline_basis` /
`torch_spline_weighting` state the same thing with torch autograd, to be bound into the unmodified reference module
on the CPU (where pyg-lib is absent) for the golden data."""
import numpy as np
import torch


def piece(degree: int, t, k: int):
    if degree == 1:
        return 1.0 - t - k + 2.0 * t * k
    if degree == 2:
        return (0.5 * t * t - t + 0.5, -t * t + t + 0.5, 0.5 * t * t)[k]
    return ((1.0 - t) ** 3 / 6.0, (3.0 * t ** 3 - 6.0 * t * t + 4.0) / 6.0,
            (-3.0 * t ** 3 + 3.0 * t * t + 3.0 * t + 1.0) / 6.0, t ** 3 / 6.0)[k]


def piece_grad(degree: int, t, k: int):
    if degree == 1:
        return np.full_like(t, 2.0 * k - 1.0)
    if degree == 2:
        return (t - 1.0, -2.0 * t + 1.0, t)[k]
    return (-0.5 * (1.0 - t) ** 2, 1.5 * t * t - 2.0 * t, -1.5 * t * t + t + 0.5, 0.5 * t * t)[k]


def _v(pseudo, kernel_size, is_open_spline, degree):
    ks = np.maximum(np.asarray(kernel_size, dtype=np.int64), 1)
    scale = (ks - degree * (np.asarray(is_open_spline) != 0)).astype(np.float32)
    v = np.asarray(pseudo, dtype=np.float32) * scale[None, :]              # one fp32 multiply
    return v, ks, scale


def _digits(s: int, dim: int, degree: int):
    out = []
    for _ in range(dim):
        out.append(s % (degree + 1))
        s //= degree + 1
    return out


def spline_basis(pseudo, kernel_size, is_open_spline, degree: int):
    """(basis [E, S] fp64, weight_index [E, S] int64)."""
    v, ks, _ = _v(pseudo, kernel_size, is_open_spline, degree)
    E, D = v.shape
    fl = np.floor(v)
    t = (v - fl).astype(np.float64)
    fi = fl.astype(np.int64)
    S = (degree + 1) ** D
    basis = np.ones((E, S))
    wi = np.zeros((E, S), dtype=np.int64)
    for s in range(S):
        off = 1
        for d, km in enumerate(_digits(s, D, degree)):
            wi[:, s] += ((fi[:, d] + km) % ks[d]) * off                     # numpy's % is non-negative here
            off *= int(ks[d])
            basis[:, s] *= piece(degree, t[:, d], km)
    return basis, wi


def spline_basis_grad(grad_basis, pseudo, kernel_size, is_open_spline, degree: int):
    """grad_pseudo [E, D] fp64 = sum_s grad_basis[e, s] d basis[e, s] / d pseudo[e, d]."""
    v, ks, scale = _v(pseudo, kernel_size, is_open_spline, degree)
    E, D = v.shape
    t = (v - np.floor(v)).astype(np.float64)
    g = np.asarray(grad_basis, dtype=np.float64)
    out = np.zeros((E, D))
    for s in range(g.shape[1]):
        ks_ = _digits(s, D, degree)
        for dg in range(D):
            prod = np.ones(E)
            for d, km in enumerate(ks_):
                prod = prod * (piece_grad(degree, t[:, d], km) * float(scale[d]) if d == dg else piece(degree, t[:, d], km))
            out[:, dg] += g[:, s] * prod
    return out


def spline_weighting(x, weight, basis, wi):
    """out [E, F_out] fp64 = sum_s basis[e, s] x[e] @ weight[wi[e, s]]."""
    x, w, b = (np.asarray(a, dtype=np.float64) for a in (x, weight, basis))
    out = np.zeros((x.shape[0], w.shape[2]))
    for s in range(b.shape[1]):
        out += b[:, s:s + 1] * np.einsum("ef,efo->eo", x, w[wi[:, s]])
    return out


def spline_weighting_grads(grad_out, x, weight, basis, wi):
    """(grad_x, grad_weight, grad_basis) in fp64."""
    g, x, w, b = (np.asarray(a, dtype=np.float64) for a in (grad_out, x, weight, basis))
    gx = np.zeros_like(x)
    gw = np.zeros_like(w)
    gb = np.zeros_like(b)
    for s in range(b.shape[1]):
        ws = w[wi[:, s]]                                                    # [E, F_in, F_out]
        gx += b[:, s:s + 1] * np.einsum("eo,efo->ef", g, ws)
        gb[:, s] = np.einsum("ef,efo,eo->e", x, ws, g)
        np.add.at(gw, wi[:, s], b[:, s, None, None] * x[:, :, None] * g[:, None, :])
    return gx, gw, gb


def torch_spline_basis(pseudo: torch.Tensor, kernel_size: torch.Tensor, is_open_spline: torch.Tensor, degree: int):
    """The same basis with torch autograd (floor is piecewise constant), fp64 after v; basis in pseudo's dtype."""
    ks = kernel_size.clamp(min=1).to(torch.int64)
    scale = (ks - degree * (is_open_spline != 0).to(torch.int64)).to(torch.float32)
    v32 = pseudo.to(torch.float32) * scale
    fl = torch.floor(v32.detach())
    v = v32.to(torch.float64)
    t = v - fl.to(torch.float64)
    E, D = pseudo.shape
    S = (degree + 1) ** D
    cols, idx = [], []
    for s in range(S):
        b = torch.ones(E, dtype=torch.float64)
        w = torch.zeros(E, dtype=torch.int64)
        off = 1
        for d, km in enumerate(_digits(s, D, degree)):
            w = w + torch.remainder(fl[:, d].to(torch.int64) + km, int(ks[d])) * off
            off *= int(ks[d])
            b = b * piece(degree, t[:, d], km)
        cols.append(b)
        idx.append(w)
    return torch.stack(cols, 1).to(pseudo.dtype), torch.stack(idx, 1)


def torch_spline_weighting(x: torch.Tensor, weight: torch.Tensor, basis: torch.Tensor, weight_index: torch.Tensor):
    out = 0
    for s in range(basis.size(1)):
        out = out + basis[:, s:s + 1].double() * torch.einsum("ef,efo->eo", x.double(), weight[weight_index[:, s]].double())
    return out.to(x.dtype)
