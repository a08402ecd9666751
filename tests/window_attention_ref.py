"""fp64 reference of the shifted-window attention kernels (window_attention_sm90.cu), built from the models' own
``torch.roll`` / ``window_partition`` / ``relative_position_index`` / ``shifted_window_mask``, so it shares no
coordinate math with the kernels.

The backward forms ``delta_i = sum_j P_ij dP_ij`` as the kernel does (exactly here), and each check is
``|out - ref| <= bound`` per element.  The bounds scale "magnitude" tensors: the same fp64 sums with
every factor replaced by its absolute value, so a bound is what the rounding of each term can add up to.

Kernel rounding points, each at most 2^-9 relative (bf16 round to nearest):
- forward: P rounded to bf16 for P.V (``2^-9 sum_j P_ij |V_jd|``), O rounded to bf16 (``2^-9 |O|``).  The scores are
  fp32 sums of bf16 products; in cosine mode ``q^.k^`` misses the lo*lo product, ``<= d 2^-18`` for unit vectors,
  which tau = 100 turns into a logit error below 2^-11, i.e. a relative error of P below 2^-11.
- backward: P^T and dS rounded to bf16 before the dV, dK, dQ products; dS = P (dP - delta) with fp32 P (recomputed
  from the fp32 lse, relative error ~2^-20), dP and delta.  The outputs are rounded to bf16.
The bound ``2^-6 * magnitude + 2^-8 * |ref|`` covers four such 2^-8 terms; a wrong bias entry, mask region, token or
head moves an element by percents of its magnitude.

The table and tau gradients sum the fp32 dS, which is never rounded to bf16: its error is that of P (the exponent, and
in cosine mode the missing lo*lo product, below 2^-11 relative at tau = 100) and of the fp32 sums, so they are held to
``2^-10 * magnitude`` (DS_TOL).
"""
import torch

from libai_b200.models.swin_transformer import relative_position_index, shifted_window_mask, window_partition

TOL = 2.0 ** -6
DS_TOL = 2.0 ** -10
OUT_TOL = 2.0 ** -8


def window_tokens(H, W, ws, shift):
    """``[nW, ws²]`` image-order token of each local position of each window (roll(-shift), then partition)."""
    t = torch.arange(H * W, dtype=torch.float64).view(1, H, W, 1)
    if shift:
        t = torch.roll(t, shifts=(-shift, -shift), dims=(1, 2))
    return window_partition(t, ws).view(-1, ws * ws).long()


def _scores(q, k, table, tau, scale, H, W, ws, shift):
    """z [B, nW, h, N, N], the cosine product (or None) and q^, k^ (or q, k)."""
    N, heads = ws * ws, q.shape[2]
    if tau is None:
        qn, kn, cos = q, k, None
        z = scale * q @ k.transpose(-1, -2)
    else:
        qn = q / q.norm(dim=-1, keepdim=True).clamp_min(1e-12)
        kn = k / k.norm(dim=-1, keepdim=True).clamp_min(1e-12)
        cos = qn @ kn.transpose(-1, -2)
        z = tau.double().view(1, 1, heads, 1, 1) * cos
    rel = relative_position_index((ws, ws)).view(-1).to(q.device)
    z = z + table.double()[rel].view(N, N, heads).permute(2, 0, 1)
    if shift:
        z = z + shifted_window_mask(H, W, ws, shift, q.device).double()[None, :, None]
    return z, cos, qn, kn


def forward(qkv, H, W, ws, shift, heads, scale, table, tau=None):
    """fp64 O [B, H·W, C] and the magnitude of each element (``sum_j P |V|``)."""
    B = qkv.shape[0]
    d = qkv.shape[-1] // (3 * heads)
    tok = window_tokens(H, W, ws, shift).to(qkv.device)
    x = qkv.double().view(B, H * W, 3, heads, d)[:, tok]                    # [B, nW, N, 3, h, d]
    q, k, v = (x[..., s, :, :].transpose(2, 3) for s in range(3))          # [B, nW, h, N, d]
    z, _, _, _ = _scores(q, k, table, tau, scale, H, W, ws, shift)
    p = torch.softmax(z, dim=-1)
    o, mag = p @ v, p @ v.abs()
    out = torch.empty(B, H * W, heads, d, dtype=torch.float64, device=qkv.device)
    out_mag = torch.empty_like(out)
    out[:, tok] = o.transpose(2, 3)
    out_mag[:, tok] = mag.transpose(2, 3)
    return out.view(B, H * W, heads * d), out_mag.view(B, H * W, heads * d)


def backward(dout, qkv, H, W, ws, shift, heads, scale, table, tau=None):
    """fp64 (dqkv, dtable, dtau) and their magnitudes."""
    B = qkv.shape[0]
    d = qkv.shape[-1] // (3 * heads)
    N = ws * ws
    tok = window_tokens(H, W, ws, shift).to(qkv.device)
    x = qkv.double().view(B, H * W, 3, heads, d)[:, tok]
    q, k, v = (x[..., s, :, :].transpose(2, 3) for s in range(3))
    go = dout.double().view(B, H * W, heads, d)[:, tok].transpose(2, 3)
    z, cos, qn, kn = _scores(q, k, table, tau, scale, H, W, ws, shift)
    p = torch.softmax(z, dim=-1)
    dp = go @ v.transpose(-1, -2)
    delta = (p * dp).sum(-1, keepdim=True)
    ds = p * (dp - delta)
    ds_mag = p * (dp.abs() + (p * dp.abs()).sum(-1, keepdim=True))
    dv, dv_mag = p.transpose(-1, -2) @ go, p.transpose(-1, -2) @ go.abs()
    sc = scale if tau is None else tau.double().view(1, 1, heads, 1, 1)
    dq, dq_mag = sc * ds @ kn, sc * ds_mag @ kn.abs()
    dk, dk_mag = sc * ds.transpose(-1, -2) @ qn, sc * ds_mag.transpose(-1, -2) @ qn.abs()
    dtau = dtau_mag = None
    if tau is not None:
        dtau = (ds * cos).sum((0, 1, 3, 4))
        dtau_mag = (ds_mag * cos.abs()).sum((0, 1, 3, 4))

        def jac(g, g_mag, xn, x):
            n = x.norm(dim=-1, keepdim=True)
            inv = 1.0 / n.clamp_min(1e-12)
            proj = (xn * g).sum(-1, keepdim=True)
            proj_mag = (xn.abs() * g_mag).sum(-1, keepdim=True)
            keep = n > 1e-12
            return (torch.where(keep, g - xn * proj, g) * inv,
                    torch.where(keep, g_mag + xn.abs() * proj_mag, g_mag) * inv)

        dq, dq_mag = jac(dq, dq_mag, qn, q)
        dk, dk_mag = jac(dk, dk_mag, kn, k)
    rel = relative_position_index((ws, ws)).view(-1).to(qkv.device)
    dt = torch.zeros((2 * ws - 1) ** 2, heads, dtype=torch.float64, device=qkv.device)
    dt_mag = torch.zeros_like(dt)
    dt.index_add_(0, rel, ds.sum((0, 1)).permute(1, 2, 0).reshape(N * N, heads))
    dt_mag.index_add_(0, rel, ds_mag.sum((0, 1)).permute(1, 2, 0).reshape(N * N, heads))
    dqkv = torch.empty(B, H * W, 3, heads, d, dtype=torch.float64, device=qkv.device)
    dqkv_mag = torch.empty_like(dqkv)
    for s, (g, m) in enumerate(((dq, dq_mag), (dk, dk_mag), (dv, dv_mag))):
        dqkv[:, tok, s] = g.transpose(2, 3)
        dqkv_mag[:, tok, s] = m.transpose(2, 3)
    return (dqkv.view(qkv.shape), dqkv_mag.view(qkv.shape)), (dt, dt_mag), (dtau, dtau_mag)


def assert_close(out, ref, mag, what, tol=TOL, out_tol=OUT_TOL):
    """|out - ref| <= tol * mag + out_tol * |ref| (+ the smallest normal fp32) for every element."""
    out = out.double()
    bound = tol * mag + out_tol * ref.abs() + 1.2e-38
    err = (out - ref).abs()
    bad = err > bound
    if bad.any():
        i = int(torch.nonzero(bad.flatten())[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements out of bound; "
                             f"first at flat index {i}: got {out.flatten()[i].item()}, ref {ref.flatten()[i].item()}, "
                             f"bound {bound.flatten()[i].item()}, max err/bound {(err / bound).max().item():.3g}")
