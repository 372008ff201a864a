"""Float64 restatements of the kernel contracts (TEST INFRASTRUCTURE ONLY).

Every function takes the op's inputs (any dtype, any device), upcasts them to float64 on the CPU and returns the exact
result of the operation -- no bf16 rounding point, no fp32 accumulation.  Backward passes come from torch.autograd in
double wherever the op is the derivative of a forward written here, so a formula that is wrong in a kernel and in
oracle/emu_ops.py alike does not carry over into this module: it imports nothing from the oracle.

Layouts follow include/microdit_b200.h: activations are token rows [B*T, D], per-sample modulation vectors are
[samples, D] column slices, patches are [B*T, C*p*p] with column (c*p + i)*p + j, DiT output tokens are [B*T, p*p*C] with
column (i*p + j)*C + c, attention heads are column blocks of width hd, lse is in log2 units.
"""
from __future__ import annotations

import math

import torch

D64 = torch.float64
LOG2E = 1.0 / math.log(2.0)


def f64(t):
    """Upcast to float64 on the CPU (differentiable: the autograd-derived backward passes call the forwards with
    tensors that require grad)."""
    return None if t is None else t.to("cpu", D64)


def _per_row(m, T, rows):
    """[samples, D] -> [rows, D]: sample s covers rows [s*T, (s+1)*T)."""
    return f64(m).repeat_interleave(T, dim=0)[:rows]


def _grads(fn, inputs, cot):
    """Gradients of <fn(*inputs), cot> with respect to every input (float64 autograd)."""
    with torch.enable_grad():
        xs = [f64(x).detach().clone().requires_grad_(True) for x in inputs]
        out = fn(*xs)
        outs = out if isinstance(out, (tuple, list)) else (out,)
        cots = cot if isinstance(cot, (tuple, list)) else (cot,)
        s = sum((o * f64(c)).sum() for o, c in zip(outs, cots) if c is not None)
        return [g.detach() for g in torch.autograd.grad(s, xs, allow_unused=True)]


# ---------------------------------------------------------------------------------------------------------- GEMM
def matmul(A, B, layout=0):
    """NT: A [.., M, K], B [.., N, K] -> A B^T;  TN: A [.., K, M], B [.., K, N] -> A^T B (batched when 3-D)."""
    A, B = f64(A), f64(B)
    return A @ B.transpose(-1, -2) if layout == 0 else A.transpose(-1, -2) @ B


def gelu(x, act):
    """act 0: x Phi(x) (erf); act 1: the tanh approximation."""
    x = f64(x)
    if act == 0:
        return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))


def gelu_grad(x, act):
    """d gelu / dx in closed form (checked against autograd of gelu() in tests/test_f64_reference_cpu.py)."""
    x = f64(x)
    if act == 0:
        return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)
    k = math.sqrt(2.0 / math.pi)
    t = torch.tanh(k * (x + 0.044715 * x ** 3))
    return 0.5 * (1.0 + t) + 0.5 * x * (1.0 - t * t) * k * (1.0 + 3 * 0.044715 * x * x)


def gemm(A, B, layout=0, *, alpha=1.0, bias=None, res=None, res_mod=0, gate=None, rows_per_gate=0, accumulate=None,
         act=None, aux=None):
    """The GEMM contract of md_gemm_bf16 in exact arithmetic.  acc = alpha * op(A) op(B) (+ bias), then
      * accumulate (EPI_ATOMIC): accumulate + acc;
      * res (EPI_RESID): res[m % res_mod] + gate[m // rows_per_gate] * acc;
      * act with aux (EPI_ACT_GRAD): acc * gelu'(aux);  act alone (EPI_ACT_DUAL): (acc, gelu(acc)).
    bias is [N] or [batch, N]; the accumulate epilogue takes none."""
    if accumulate is not None and bias is not None:
        raise ValueError("the accumulate epilogue (EPI_ATOMIC) takes no bias")
    acc = matmul(A, B, layout) * (alpha if alpha != 0 else 1.0)
    if bias is not None:
        b = f64(bias)
        acc = acc + (b[:, None, :] if b.dim() == 2 else b)
    if accumulate is not None:
        return f64(accumulate) + acc
    if res is not None:
        M = acc.shape[-2]
        if gate is not None:
            acc = acc * _per_row(gate, rows_per_gate, M)
        r = f64(res)
        if res_mod > 0:
            r = r[..., torch.arange(M) % res_mod, :]
        return r + acc
    if aux is not None:
        return acc * gelu_grad(aux, act)
    if act is not None:
        return acc, gelu(acc, act)
    return acc


def interleaved_to_natural(f):
    """Row p of a 32-interleaved w1 | w2 stack [2f, D] is row perm[p] of the natural stack (blocks of 32 rows: w1
    block j, then w2 block j)."""
    p = torch.arange(2 * f)
    blk, inn = p // 64, p % 64
    return torch.where(inn < 32, 32 * blk + inn, f + 32 * blk + inn - 32)


# ---------------------------------------------------------------------------------------------------------- norms
def pending_residual(x, y_add, gate_add, T):
    """x_new = x + gate * y_add (the gated residual a LayerNorm forward folds in)."""
    ya = f64(y_add)
    if gate_add is not None:
        ya = ya * _per_row(gate_add, T, ya.shape[0])
    return f64(x) + ya


def _ln(x, gamma, shift, scale, T, eps):
    mu = x.mean(1, keepdim=True)
    var = ((x - mu) ** 2).mean(1, keepdim=True)
    y = (x - mu) / torch.sqrt(var + eps)
    if gamma is not None:
        y = y * gamma
    if scale is not None:
        y = y * (1.0 + scale.repeat_interleave(T, dim=0)[: x.shape[0]])
    if shift is not None:
        y = y + shift.repeat_interleave(T, dim=0)[: x.shape[0]]
    return y


def ln_fwd(x, *, gamma=None, shift=None, scale=None, T, eps=1e-6, src_rows=None, y_add=None, gate_add=None):
    """LayerNorm + adaLN modulate of the rows x[src_rows] (all rows without src_rows), after the pending residual
    x + gate_add * y_add when y_add is given.  Returns (y, mean, rstd, x_new rows)."""
    xv = f64(x).reshape(-1, f64(x).shape[-1])
    if src_rows is not None:
        xv = xv[src_rows.long().cpu()]
    if y_add is not None:
        ya = f64(y_add).reshape(-1, xv.shape[1])
        if src_rows is not None:
            ya = ya[src_rows.long().cpu()]
        xv = pending_residual(xv, ya, gate_add, T)
    mu = xv.mean(1)
    rstd = 1.0 / torch.sqrt(((xv - mu[:, None]) ** 2).mean(1) + eps)
    y = _ln(xv, f64(gamma), f64(shift), f64(scale), T, eps)
    return y, mu, rstd, xv


def ln_bwd(dy, x, *, gamma=None, shift=True, scale=None, T, eps=1e-6, src_rows=None):
    """Autograd of ln_fwd with respect to the normalised rows, gamma, shift and scale (per sample).
    Returns (dx rows, dgamma, dshift, dscale); the entries of absent parameters are None."""
    xv = f64(x).reshape(-1, f64(x).shape[-1])
    if src_rows is not None:
        xv = xv[src_rows.long().cpu()]
    rows, D = xv.shape
    ns = rows // T
    g = f64(gamma) if gamma is not None else None
    sh = torch.zeros(ns, D, dtype=D64) if shift else None
    sc = f64(scale) if scale is not None else None
    ins = [xv] + [v for v in (g, sh, sc) if v is not None]

    def fn(xv, *rest):
        it = iter(rest)
        gg = next(it) if g is not None else None
        ss = next(it) if sh is not None else None
        cc = next(it) if sc is not None else None
        return _ln(xv, gg, ss, cc, T, eps)
    grads = iter(_grads(fn, ins, dy))
    dx = next(grads)
    dg = next(grads) if g is not None else None
    dsh = next(grads) if sh is not None else None
    dsc = next(grads) if sc is not None else None
    return dx, dg, dsh, dsc


def scatter_rows(dx_rows, src_rows, total_rows):
    """dx [total_rows, D] with dx[src_rows[i]] += dx_rows[i] (the gather's adjoint)."""
    out = torch.zeros(total_rows, dx_rows.shape[1], dtype=D64)
    return out.index_add_(0, src_rows.long().cpu(), f64(dx_rows))


def gate_bwd(dres, *, y=None, gate=None, T):
    """Backward of res + gate * y at the residual gradient dres: (dy = gate * dres, dgate = sum_t dres * y)."""
    d = f64(dres)
    rows, D = d.shape
    dy = d * _per_row(gate, T, rows) if gate is not None else d.clone()
    dgate = (d * f64(y)).reshape(rows // T, T, D).sum(1) if y is not None else None
    return dy, dgate


def rownorm_fwd(x, eps=1e-6):
    """Per-row normalisation without affine parameters: (xhat, rstd)."""
    x = f64(x)
    mu = x.mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x - mu) ** 2).mean(1, keepdim=True) + eps)
    return (x - mu) * rstd, rstd[:, 0]


def rownorm_bwd(dy, xhat, rstd):
    """VJP of rownorm_fwd at the row whose normalisation is xhat: rstd (g - mean g - xhat mean(g xhat)).  Its agreement
    with autograd of rownorm_fwd is checked in tests/test_f64_reference_cpu.py."""
    d, xh, r = f64(dy), f64(xhat), f64(rstd)
    return r[:, None] * (d - d.mean(1, keepdim=True) - xh * (d * xh).mean(1, keepdim=True))


# ---------------------------------------------------------------------------------------------------------- FFN tails
def swiglu_fwd(u):
    """u [rows, 2f] = [u1 | u2] -> silu(u1) * u2."""
    u = f64(u)
    f = u.shape[1] // 2
    a, b = u[:, :f], u[:, f:]
    return a / (1.0 + torch.exp(-a)) * b


def swiglu_bwd(dh, u):
    return _grads(swiglu_fwd, [u], dh)[0]


def act_fwd(x, act):
    return gelu(x, act)


def act_bwd(dact, x, act):
    return _grads(lambda v: gelu(v, act), [x], dact)[0]


# ---------------------------------------------------------------------------------------------------------- attention
def _heads(x, B, T, H, hd):
    return f64(x)[:, : H * hd].reshape(B, T, H, hd).permute(0, 2, 1, 3)


def _unheads(x):
    B, H, T, hd = x.shape
    return x.permute(0, 2, 1, 3).reshape(B * T, H * hd)


def _attn(q, k, v, hd):
    s = q @ k.transpose(-1, -2) / math.sqrt(hd)
    lse = torch.logsumexp(s, -1)
    return torch.exp(s - lse[..., None]) @ v, lse


def attn_fwd(q, k, v, B, H, Tq, Tk, hd):
    """softmax(q k^T / sqrt(hd)) v per (sample, head): (o [B*Tq, H*hd], lse [B, H, Tq] in log2 units)."""
    o, lse = _attn(_heads(q, B, Tq, H, hd), _heads(k, B, Tk, H, hd), _heads(v, B, Tk, H, hd), hd)
    return _unheads(o), lse * LOG2E


def attn_bwd(do, q, k, v, B, H, Tq, Tk, hd):
    """(dq, dk, dv) = autograd of attn_fwd's o at the cotangent do."""
    dq, dk, dv = _grads(lambda q, k, v: _attn(q, k, v, hd)[0],
                        [_heads(q, B, Tq, H, hd), _heads(k, B, Tk, H, hd), _heads(v, B, Tk, H, hd)],
                        _heads(do, B, Tq, H, hd))
    return _unheads(dq), _unheads(dk), _unheads(dv)


# ---------------------------------------------------------------------------------------------------------- MoE router
def moe_gate_fwd(x, wg):
    """Router probabilities softmax(x wg^T) [rows, E]."""
    return torch.softmax(f64(x) @ f64(wg).t(), -1)


def _routes(idx, B, E, k, T):
    """(token row b*T + idx[b,e,j], expert row b*k + j of expert e) for every routed slot, flattened in (b, e, j)."""
    idx = idx.long().cpu().reshape(B, E, k)
    b = torch.arange(B)[:, None, None].expand(B, E, k)
    e = torch.arange(E)[None, :, None].expand(B, E, k)
    j = torch.arange(k)[None, None, :].expand(B, E, k)
    return (b * T + idx).reshape(-1), e.reshape(-1), (b * k + j).reshape(-1)


def moe_combine_fwd(h2, gval, idx, B, T, E, k, xres=None, gate=None):
    """ymoe[b*T + t] = sum over the slots (e, j) that routed token t of gval[b,e,j] h2[e, b*k + j];
    xout = xres + gate * ymoe.  Returns (ymoe, xout or None)."""
    h = f64(h2)
    tok, e, r = _routes(idx, B, E, k, T)
    y = torch.zeros(B * T, h.shape[-1], dtype=D64).index_add_(0, tok, f64(gval).reshape(-1)[:, None] * h[e, r])
    xout = None
    if xres is not None:
        xout = f64(xres) + (_per_row(gate, T, B * T) if gate is not None else 1.0) * y
    return y, xout


def moe_combine_bwd(dy, h2, gval, idx, B, T, E, k):
    """Autograd of moe_combine_fwd's ymoe: (dh2 [E, B*k, D], dgval [B, E, k])."""
    dh2, dg = _grads(lambda h, g: moe_combine_fwd(h, g, idx, B, T, E, k)[0], [h2, gval], dy)
    return dh2, dg.reshape(B, E, k)


def moe_dx_bwd(dxin, idx, dgval, probs, wg, B, T, E, k):
    """Backward to the router input x of (gather to the experts, gate values picked from softmax(x wg^T)):
      dscores = softmax-VJP of the gate-value gradients at the routed (token, expert) pairs;
      dx = sum of the expert-input gradients of every slot the token went to + dscores wg.
    Returns (dscores [B*T, E], dx [B*T, D])."""
    tok, e, r = _routes(idx, B, E, k, T)
    dp = torch.zeros(B * T, E, dtype=D64)
    dp[tok, e] = f64(dgval).reshape(-1)
    # probs = softmax(log probs): the softmax VJP through autograd, independent of the closed form
    ds = _grads(lambda s: torch.softmax(s, -1), [torch.log(f64(probs))], dp)[0]
    dx = ds @ f64(wg)
    dx.index_add_(0, tok, f64(dxin)[e, r])
    return ds, dx


def moe_gate_wgrad(dscores, x, accumulate=None):
    g = f64(dscores).t() @ f64(x)
    return g if accumulate is None else f64(accumulate) + g


# ---------------------------------------------------------------------------------------------------------- EDM
def edm_coef(rnd=None, sigma_in=None, p_mean=-1.2, p_std=1.2, sigma_data=0.5):
    """[6, B]: sigma, c_skip, c_out, c_in, c_noise, loss weight (Karras et al. 2022, EDM preconditioning)."""
    sigma = f64(sigma_in).flatten() if sigma_in is not None else torch.exp(f64(rnd).flatten() * p_std + p_mean)
    sd = sigma_data
    s2 = sigma ** 2 + sd ** 2
    return torch.stack([sigma, sd ** 2 / s2, sigma * sd / torch.sqrt(s2), 1.0 / torch.sqrt(s2), torch.log(sigma) / 4,
                        s2 / (sigma * sd) ** 2])


def patchify(x, p, scale=None):
    """[B, C, H, W] -> [B*(H/p)*(W/p), C*p*p], row b*T + h*(W/p) + w, column (c*p + i)*p + j (times scale[b])."""
    x = f64(x)
    B, Cc, H, W = x.shape
    if scale is not None:
        x = x * f64(scale).reshape(B, 1, 1, 1)
    return x.reshape(B, Cc, H // p, p, W // p, p).permute(0, 2, 4, 1, 3, 5).reshape(-1, Cc * p * p)


def patchify_bwd(dpatches, p, shape, scale=None):
    return _grads(lambda x: patchify(x, p, f64(scale) if scale is not None else None),
                  [torch.zeros(shape, dtype=D64)], dpatches)[0]


def unpatchify(ftok, p, shape, keep_rows=None, ids_restore=None, mask_token=None):
    """Token rows [B*Tk, p*p*C] (column (i*p + j)*C + c) -> image [B, C, H, W].  With ids_restore the Tk kept tokens and
    T - Tk mask tokens are put back in image order (token ids_restore[b, t] of [kept | masked] lands at t); with keep_rows
    (the adjoint's view) kept token i of sample b sits at global row keep_rows[b*Tk + i]."""
    B, Cc, H, W = shape
    gh, gw = H // p, W // p
    T = gh * gw
    f = f64(ftok).reshape(B, -1, p * p * Cc)
    Tk = f.shape[1]
    if ids_restore is not None:
        mt = f64(mask_token).reshape(1, 1, -1) if mask_token is not None else torch.zeros(1, 1, p * p * Cc, dtype=D64)
        full = torch.cat([f, mt.expand(B, T - Tk, -1)], 1)
        f = full[torch.arange(B)[:, None], ids_restore.long().cpu().reshape(B, T)]
    elif keep_rows is not None:
        full = torch.zeros(B * T, p * p * Cc, dtype=D64)
        full[keep_rows.long().cpu()] = f.reshape(B * Tk, -1)
        f = full.reshape(B, T, -1)
    return f.reshape(B, gh, gw, p, p, Cc).permute(0, 5, 1, 3, 2, 4).reshape(B, Cc, H, W)


def unpatchify_bwd(dF, p, Tk, keep_rows=None):
    B, Cc, H, W = dF.shape
    z = torch.zeros(B * Tk, p * p * Cc, dtype=D64)
    return _grads(lambda f: unpatchify(f, p, (B, Cc, H, W), keep_rows=keep_rows), [z], dF)[0]


def edm_prepare(lat, eps, p, *, rnd=None, sigma_in=None, p_mean=-1.2, p_std=1.2, sigma_data=0.5):
    """Noised latents xn = lat + sigma eps, DiT input patches of c_in xn, and coef [6, B]."""
    coef = edm_coef(rnd, sigma_in, p_mean, p_std, sigma_data)
    xn = f64(lat) + coef[0].reshape(-1, 1, 1, 1) * f64(eps)
    return xn, patchify(xn, p, coef[3]), coef


def _edm_per_sample(ftok, lat, xn, coef, p, Tk, keep_rows):
    B, Cc, H, W = lat.shape
    T = (H // p) * (W // p)
    D = unpatchify(ftok, p, (B, Cc, H, W), keep_rows=keep_rows) * coef[2].reshape(B, 1, 1, 1) \
        + coef[1].reshape(B, 1, 1, 1) * f64(xn)
    r = patchify(D - f64(lat), p).reshape(B, T, -1)
    if keep_rows is not None:
        r = r.reshape(B * T, -1)[keep_rows.long().cpu()].reshape(B, Tk, -1)
    return coef[5] * (r ** 2).mean((1, 2))


def edm_loss_fwd(ftok, lat, xn, coef, p, Tk, keep_rows=None):
    """Per-sample weighted MSE of D = c_skip xn + c_out F against the clean latents over the kept patches, and its
    mean over the batch: (per_sample [B], loss)."""
    ps = _edm_per_sample(f64(ftok), f64(lat), f64(xn), f64(coef), p, Tk, keep_rows)
    return ps, ps.mean()


def edm_loss_bwd(ftok, lat, xn, coef, gscale, p, Tk, keep_rows=None):
    """gscale * d loss / d ftok."""
    g = _grads(lambda f: _edm_per_sample(f, f64(lat), f64(xn), f64(coef), p, Tk, keep_rows).mean(), [ftok],
               torch.ones((), dtype=D64))[0]
    return float(f64(gscale).flatten()[0]) * g


def edm_output(ftok, p, shape, coef, xn, ids_restore=None, mask_token=None):
    """(F image, D_x = c_skip xn + c_out F)."""
    F = unpatchify(ftok, p, shape, ids_restore=ids_restore, mask_token=mask_token)
    B = shape[0]
    return F, f64(coef)[1].reshape(B, 1, 1, 1) * f64(xn) + f64(coef)[2].reshape(B, 1, 1, 1) * F


def timestep_embed(t, dim):
    """[cos(t f_i) | sin(t f_i)], f_i = 10000^(-i/half), i < half = dim // 2 (a zero last column when dim is odd)."""
    t = f64(t).flatten()
    half = dim // 2
    fr = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=D64) / half)
    a = t[:, None] * fr[None]
    out = torch.cat([torch.cos(a), torch.sin(a)], -1)
    if dim % 2:
        out = torch.cat([out, torch.zeros(t.shape[0], 1, dtype=D64)], -1)
    return out


def timestep_embed_bwd(dfreq, t):
    return _grads(lambda tt: timestep_embed(tt, dfreq.shape[1]), [t], dfreq)[0]


def mean_tokens(x, B, L):
    x = f64(x)
    return x.reshape(B, L, -1).mean(1)


def sumsq(x):
    return (f64(x) ** 2).sum()


def colsum(x):
    return f64(x).sum(0)


def colsum_interleaved(x, half):
    """Column sums of [rows, 2 half] whose columns are the 32-interleaved w1 | w2 order, returned in [b1 | b2] order."""
    out = torch.zeros(2 * half, dtype=D64)
    return out.index_add_(0, interleaved_to_natural(half), f64(x).sum(0))
