"""TEST INFRASTRUCTURE ONLY — plain-PyTorch (fp32 math, bf16 storage) emulation of every `qflux_b200.lib` entry point.

`-m "not gpu"` tests monkey-patch it over `qflux_b200.lib` to exercise the host-side orchestration (launch order, operand wiring,
LoRA registry, gradient offsets) of the fused model on CPU against the oracle.  The emulation is held to the kernels it stands in
for by tests/test_glue_kernels.py (tools/glue_check.py, `-m gpu`): element by element on the same inputs, bit-identical for data
movement and within a stated rounding-flip bound elsewhere.  The `-m gpu` kernel cases themselves compare against independent
fp64 references, not against this file.  It is never imported by the product package.
"""
from __future__ import annotations

import math
import types

import torch
import torch.nn.functional as F

BF = torch.bfloat16
EPI_BIAS, EPI_GELU, EPI_RESID_GATE, EPI_DGELU, EPI_ADD, EPI_ATTN_DO = 0, 1, 2, 3, 4, 5


def _f(t):
    return None if t is None else t.float()


def gemm_problem(A, B, out, *, A2=None, B2=None, kb2=0, a2_col0=0, bias=None, out2=None, resid=None, gate=None,
                 rows_per_batch=0, aux=None, row_bands=None, delta=None, s_offset=0):
    return types.SimpleNamespace(A=A, B=B, out=out, A2=A2, B2=B2, kb2=kb2, a2_col0=a2_col0, bias=bias, out2=out2, resid=resid,
                                 gate=gate, rows_per_batch=rows_per_batch, aux=aux, row_bands=row_bands, delta=delta, s_offset=s_offset)


def _gelu_grad(u):
    k0, k1 = 0.7978845608028654, 0.044715
    t = torch.tanh(k0 * (u + k1 * u ** 3))
    return 0.5 * (1 + t) + 0.5 * u * (1 - t * t) * k0 * (1 + 3 * k1 * u * u)


def gemm(problems, N, K, *, trans_b=False, epilogue=EPI_BIAS, alpha=1.0, lora_group_n=0, block_n=0):
    # like qfx_gemm_bf16: alpha scales the accumulator of BIAS / ADD / DGELU / ATTN_DO only
    assert alpha == 1.0 or epilogue not in (EPI_GELU, EPI_RESID_GATE), "the GELU and RESID_GATE epilogues take alpha = 1 only"
    for p in problems:
        A, W = p.A.float(), p.B.float()
        acc = A @ (W if trans_b else W.t())
        if p.kb2:
            w2 = 64 * p.kb2
            if trans_b:
                acc = acc + p.A2.float()[:, p.a2_col0:p.a2_col0 + w2] @ p.B2.float()[:w2]
            else:
                groups = N // lora_group_n if lora_group_n else 1
                gn = N // groups
                for g in range(groups):
                    a2 = p.A2.float()[:, p.a2_col0 + g * w2: p.a2_col0 + (g + 1) * w2]
                    acc[:, g * gn:(g + 1) * gn] += a2 @ p.B2.float()[g * gn:(g + 1) * gn, :w2].t()
        b = p.bias.float() if p.bias is not None else 0.0
        if epilogue == EPI_BIAS:
            p.out.copy_((acc * alpha + b).to(BF))
        elif epilogue == EPI_GELU:
            u = (acc + b).to(BF)
            p.out2.copy_(u)
            p.out.copy_(F.gelu(u.float(), approximate="tanh").to(BF))
        elif epilogue == EPI_RESID_GATE:
            y = (acc + b).to(BF).float()
            rpb = p.rows_per_batch or A.shape[0]
            g = p.gate.float().repeat_interleave(rpb, 0)[:A.shape[0]]  # row -> gate row // rows_per_batch, as the kernel
            p.out.copy_((p.resid.float() + (g * y).to(BF).float()).to(BF))
            if p.out2 is not None:
                p.out2.copy_(y.to(BF))
        elif epilogue == EPI_ADD:
            p.out.copy_((p.resid.float() + (acc * alpha).to(BF).float()).to(BF))
        elif epilogue == EPI_DGELU:
            p.out.copy_(((acc * alpha).to(BF).float() * _gelu_grad(p.aux.float())).to(BF))
        elif epilogue == EPI_ATTN_DO:  # g = grad wrt the attention output: head-major scatter + delta = rowsum(g * O)
            g = (acc * alpha).to(BF)
            Bsz, H, S, _ = p.out.shape
            tps = p.rows_per_batch
            gb = g.view(-1, tps, H, 128)
            p.out[:gb.shape[0], :, p.s_offset:p.s_offset + tps] = gb.permute(0, 2, 1, 3)
            p.delta[:gb.shape[0], :, p.s_offset:p.s_offset + tps] = (gb.float() * p.aux.float().reshape(-1, tps, H, 128)).sum(-1).permute(0, 2, 1)
            if p.out2 is not None:
                p.out2.copy_(g)
        else:
            raise ValueError(epilogue)
        if p.row_bands is not None:  # ragged row group: rows outside the computed bands are zero-filled (qfx_zero_rows)
            for lo, hi in p.row_bands.host_dead:
                p.out[lo:hi] = 0
                if p.out2 is not None:
                    p.out2[lo:hi] = 0


def ln_modulate_fwd(x, y, shift, scale, rows_per_batch, mean=None, rstd=None, eps=1e-6):
    xf = x.float()
    mu = xf.mean(1, keepdim=True)
    rs = torch.rsqrt(((xf - mu) ** 2).mean(1, keepdim=True) + eps)
    n = ((xf - mu) * rs).to(BF).float()
    sc = (1 + scale.float()).to(BF).float().repeat_interleave(rows_per_batch, 0)
    sh = shift.float().repeat_interleave(rows_per_batch, 0)
    y.copy_(((n * sc).to(BF).float() + sh).to(BF))
    if mean is not None:
        mean.copy_(mu[:, 0])
        rstd.copy_(rs[:, 0])


def ln_modulate_bwd(dy, x, mean, rstd, scale, rows_per_batch, dx, dres=None, gate=None, dx_gated=None):
    sc = (1 + scale.float()).to(BF).float().repeat_interleave(rows_per_batch, 0)
    g = (dy.float() * sc).to(BF).float()
    xh = (x.float() - mean[:, None]) * rstd[:, None]
    d = (rstd[:, None] * (g - g.mean(1, keepdim=True) - xh * (g * xh).mean(1, keepdim=True))).to(BF).float()
    o = (dres.float() + d).to(BF) if dres is not None else d.to(BF)
    if dx_gated is not None:
        dx_gated.copy_((o.float() * gate.float().repeat_interleave(rows_per_batch, 0)).to(BF))
    dx.copy_(o)


def mod_grad(g, rows_per_batch, sum_out=None, m=None, prod_out=None, mean=None, rstd=None):
    B = g.shape[0] // rows_per_batch
    gf = g.float().view(B, rows_per_batch, -1)
    if sum_out is not None:
        sum_out += gf.sum(1)
    if prod_out is not None:
        mf = m.float()
        if mean is not None:
            mf = ((mf - mean[:, None]) * rstd[:, None]).to(BF).float()
        prod_out += (gf * mf.view(B, rows_per_batch, -1)).sum(1)


def gate_mul(a, gate, rows_per_batch, out):
    out.copy_((a.float() * gate.float().repeat_interleave(rows_per_batch, 0)).to(BF))


def add_bf16(a, b, out):
    out.copy_((a.float() + b.float()).to(BF))


def rmsnorm_rows(x, w, y, eps=1e-6):
    xf = x.float()
    r = torch.rsqrt((xf ** 2).mean(1, keepdim=True) + eps)
    y.copy_(((xf * r).to(BF).float() * w.float()).to(BF))


def _rope_apply(n, cs, conj=False):
    """n [..., 128] fp32; cs [..., 64, 2]"""
    x = n.reshape(*n.shape[:-1], 64, 2)
    c, s = cs[..., 0], cs[..., 1]
    if conj:
        s = -s
    return torch.stack([x[..., 0] * c - x[..., 1] * s, x[..., 0] * s + x[..., 1] * c], -1).reshape(n.shape)


def _rope_rows(rope, B, n, s_offset):
    if rope.dim() == 3:
        return rope[s_offset:s_offset + n][None].expand(B, n, 64, 2)
    return rope[:, s_offset:s_offset + n]


def qk_norm_rope_fwd(qkv, wq, wk, rope, Q, K, V, tokens_per_sample, s_offset, eps=1e-6, round_mid=True):
    B, H, S, _ = Q.shape
    n = tokens_per_sample
    x = qkv.float().view(B, n, 3, H, 128)
    cs = _rope_rows(rope, B, n, s_offset)[:, :, None]  # [B,n,1,64,2]
    for which, (w, dst) in enumerate(((wq, Q), (wk, K))):
        f = x[:, :, which]
        r = torch.rsqrt((f ** 2).mean(-1, keepdim=True) + eps)
        nn_ = ((f * r).to(BF).float() * w.float()).to(BF).float() if round_mid else (f * r * w.float()).to(BF).float()
        dst[:, :, s_offset:s_offset + n] = _rope_apply(nn_, cs).to(BF).permute(0, 2, 1, 3)
    V[:, :, s_offset:s_offset + n] = x[:, :, 2].to(BF).permute(0, 2, 1, 3)


def qk_norm_rope_bwd(dQ, dK, dV, qkv, wq, wk, rope, dqkv, tokens_per_sample, s_offset, eps=1e-6, round_mid=True):
    B, H, S, _ = dK.shape
    n = tokens_per_sample
    x = qkv.float().view(B, n, 3, H, 128)
    cs = _rope_rows(rope, B, n, s_offset)[:, :, None]
    out = torch.empty(B, n, 3, H, 128)
    for which, (w, g) in enumerate(((wq, dQ), (wk, dK))):
        go = g[:, :, s_offset:s_offset + n].float().to(BF).float().permute(0, 2, 1, 3)
        gn = _rope_apply(go, cs, conj=True).to(BF).float()
        f = x[:, :, which]
        r = torch.rsqrt((f ** 2).mean(-1, keepdim=True) + eps)
        gw = gn * w.float()
        out[:, :, which] = r * gw - f * (r ** 3) * (gw * f).mean(-1, keepdim=True)
    out[:, :, 2] = dV[:, :, s_offset:s_offset + n].float().permute(0, 2, 1, 3)
    dqkv.copy_(out.reshape(B * n, 3 * H * 128).to(BF))


def gemv_act(x, W, bias, y, act=0):
    xin = F.silu(x.float()).to(BF).float() if act == 1 else x.float()
    y.copy_((xin @ W.float().t() + (bias.float() if bias is not None else 0.0)).to(BF))


def timestep_sinusoid(t_f32, scale, out):
    half = out.shape[1] // 2
    freq = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32) / half)
    arg = scale * (t_f32[:, None].float() * freq[None])
    out.copy_(torch.cat([arg.cos(), arg.sin()], -1).to(BF))


def flow_noisy_input(x0, noise, control, sigma_f32, packed):
    B, L, C = x0.shape
    sg = sigma_f32.to(BF).view(B, 1, 1)
    packed[:, :L] = (1.0 - sg) * x0 + sg * noise
    packed[:, L:] = control


def flow_noisy_input_var(x0, noise, control, sigma_f32, Lt, Lc, packed):
    B = x0.shape[0]
    packed.zero_()
    sg = sigma_f32.to(BF)
    for b in range(B):
        lt, lc = int(Lt[b]), int(Lc[b])
        packed[b, :lt] = (1.0 - sg[b]) * x0[b, :lt] + sg[b] * noise[b, :lt]
        packed[b, lt:lt + lc] = control[b, :lc]


def flow_loss(pred, x0, noise, w, norm, loss, dpred=None, grad_scale=1.0):
    B, L, C = x0.shape
    p = pred.float().view(B, -1, C)
    tgt = (noise - x0).float()
    d = p[:, :L] - tgt
    wt = w.float()[..., None] if w is not None else 1.0
    loss.copy_(((wt * d * d).sum() * norm).reshape(1))
    if dpred is not None:
        g = torch.zeros_like(p)
        g[:, :L] = 2 * norm * wt * d * grad_scale
        dpred.copy_(g.view(dpred.shape).to(BF))


def lora_wgrad(P, Q, G, gs_i, gs_j, r):
    res = P.float().t() @ Q.float()[:, :r]  # [Dp, r]
    Dp = P.shape[1]
    view = torch.as_strided(G, (Dp, r), (gs_i, gs_j))
    view += res


def lora_wgrad_tc(A, B, G_list, gs_i, gs_j, r, mode=0, Dg=0):
    Af, Bf = A.float(), B.float()
    for g, G in enumerate(G_list):
        if mode == 1:
            res = Af[:, g * Dg:(g + 1) * Dg].t() @ Bf[:, g * 64: g * 64 + r]
        else:
            res = Af.t() @ Bf[:, g * 64: g * 64 + r]
        view = torch.as_strided(G, (res.shape[0], r), (gs_i, gs_j))
        view += res


def adamw_tables(members, device):
    return list(members), None


def fused_adamw(tables, grad, exp_avg, exp_avg_sq, sumsq, pre_scale, max_norm, lr, beta1, beta2, eps, weight_decay, step):
    members, _ = tables
    # the C ABI takes the scalars as fp32 and forms 1 - beta, 1 - lr * wd and the bias corrections in fp32 (optimizer.cu)
    f32 = lambda x: float(torch.tensor(x, dtype=torch.float32))
    pre_scale, max_norm, lr, beta1, beta2, eps, weight_decay = (f32(x) for x in (pre_scale, max_norm, lr, beta1, beta2, eps, weight_decay))
    g = grad * pre_scale
    sumsq.copy_((g ** 2).sum().reshape(1))
    coef = 1.0
    if max_norm > 0:
        coef = min(1.0, max_norm / (float(sumsq.sqrt()) + 1e-6))
    g = g * coef
    bc1, bc2 = f32(1 - f32(beta1 ** step)), f32(1 - f32(beta2 ** step))
    omb1, omb2, decay = f32(1 - beta1), f32(1 - beta2), f32(1 - lr * weight_decay)
    for p, off in members:
        n = p.numel()
        gi = g[off: off + n].view(p.shape)
        m, v = exp_avg[off: off + n].view(p.shape), exp_avg_sq[off: off + n].view(p.shape)
        w = p.float() * decay
        m.mul_(beta1).add_(gi, alpha=omb1)
        v.mul_(beta2).addcmul_(gi, gi, value=omb2)
        p.copy_((w - (lr / bc1) * m / (v.sqrt() / f32(bc2 ** 0.5) + eps)).to(BF))


def attn_delta(O, dO, delta, tokens_per_sample, s_offset, dO_joint=None):
    B, H, S = delta.shape
    n = tokens_per_sample
    o, g = O.float().view(B, n, H, 128), dO.float().view(B, n, H, 128)
    delta[:, :, s_offset:s_offset + n] = (o * g).sum(-1).permute(0, 2, 1)
    if dO_joint is not None:
        dO_joint[:, :, s_offset:s_offset + n] = dO.view(B, n, H, 128).permute(0, 2, 1, 3)


def _scores(Q, K, kv_len, scale, txt_len=None, split=0):
    B, H, S, d = Q.shape
    sc = Q.float() @ K.float().transpose(-1, -2) * scale
    pos = torch.arange(S)[None, :]
    mask = torch.ones(B, S, dtype=torch.bool)
    if kv_len is not None:
        mask &= pos < kv_len[:, None].cpu()
    if txt_len is not None:
        mask &= ~((pos >= txt_len[:, None].cpu()) & (pos < split))
    return sc.masked_fill(~mask[:, None, None, :], float("-inf"))


def attn_fwd(Q, K, V, out_txt, out_img, split, lse=None, kv_len=None, scale=None, txt_len=None):
    B, H, S, d = Q.shape
    scale = scale if scale is not None else d ** -0.5
    sc = _scores(Q, K, kv_len, scale, txt_len, split)
    o = (torch.softmax(sc, -1) @ V.float()).permute(0, 2, 1, 3).reshape(B, S, H * d)
    if split > 0:
        out_txt.copy_(o[:, :split].reshape(B * split, H * d).to(BF))
    out_img.copy_(o[:, split:].reshape(B * (S - split), H * d).to(BF))
    if lse is not None:
        lse.copy_(torch.logsumexp(sc, -1) * 1.4426950408889634)


def attn_bwd(Q, K, V, dO, lse, delta, dQ_accum, dK, dV, kv_len=None, scale=None, txt_len=None, split=0):
    B, H, S, d = Q.shape
    scale = scale if scale is not None else d ** -0.5
    sc = _scores(Q, K, kv_len, scale, txt_len, split)
    P = torch.exp2(sc * 1.4426950408889634 - lse[..., None])
    dP = dO.float() @ V.float().transpose(-1, -2)
    dS = P * (dP - delta[..., None]) * scale
    Pb, dSb = P.to(BF).float(), dS.to(BF).float()
    dV.copy_((Pb.transpose(-1, -2) @ dO.float()).to(BF))
    dK.copy_((dSb.transpose(-1, -2) @ Q.float()).to(BF))
    dQ_accum += dSb @ K.float()


def grad_finalize(g_f32, pre_scale, max_norm, sumsq, out_bf16):
    g = g_f32 * pre_scale
    ss = (g * g).sum()
    sumsq.copy_(ss.reshape(1))
    coef = min(1.0, max_norm / (math.sqrt(float(ss)) + 1e-6)) if max_norm > 0 else 1.0
    out_bf16.copy_((g * coef).to(BF))


# ---- stream-pair launches (one CUDA launch over both row groups of a stream-major buffer): emulated as the two single-group calls
def ln_modulate_fwd_pair(x, y, g0, g1, split, mean=None, rstd=None, eps=1e-6):
    for (sh, sc, rpb), sl in ((g0, slice(0, split)), (g1, slice(split, None))):
        ln_modulate_fwd(x[sl], y[sl], sh, sc, rpb, None if mean is None else mean[sl], None if rstd is None else rstd[sl], eps)


def ln_modulate_bwd_pair(dy, x, mean, rstd, g0, g1, split, dx, dres=None, dx_gated=None):
    for (sc, rpb, gate), sl in ((g0, slice(0, split)), (g1, slice(split, None))):
        ln_modulate_bwd(dy[sl], x[sl], mean[sl], rstd[sl], sc, rpb, dx[sl], dres=None if dres is None else dres[sl], gate=gate,
                        dx_gated=None if dx_gated is None else dx_gated[sl])


def qk_norm_rope_fwd_pair(qkv, g0, g1, split, rope, Q, K, V, eps=1e-6, round_mid=True):
    for (wq, wk, tps, so), sl in ((g0, slice(0, split)), (g1, slice(split, None))):
        qk_norm_rope_fwd(qkv[sl], wq, wk, rope, Q, K, V, tps, so, eps=eps, round_mid=round_mid)


def qk_norm_rope_bwd_pair(dQ, dK, dV, qkv, g0, g1, split, rope, dqkv, eps=1e-6, round_mid=True, clear_dq=False):
    for (wq, wk, tps, so), sl in ((g0, slice(0, split)), (g1, slice(split, None))):
        qk_norm_rope_bwd(dQ, dK, dV, qkv[sl], wq, wk, rope, dqkv[sl], tps, so, eps=eps, round_mid=round_mid)
    if clear_dq:  # like the kernel: only the positions the two groups read are zeroed (qfx.h asks the groups to cover all of S)
        for (_, _, tps, so), sl in ((g0, slice(0, split)), (g1, slice(split, None))):
            if qkv[sl].shape[0]:
                dQ[:qkv[sl].shape[0] // tps, :, so:so + tps] = 0


def attn_delta_pair(O, dO, delta, g0, g1, split, dO_joint=None):
    for (tps, so), sl in ((g0, slice(0, split)), (g1, slice(split, None))):
        attn_delta(O[sl], dO[sl], delta, tps, so, dO_joint)


def require_cuda(*tensors):
    return None


_NAMES = ["gemm_problem", "gemm", "ln_modulate_fwd", "ln_modulate_bwd", "mod_grad", "gate_mul", "add_bf16", "rmsnorm_rows", "qk_norm_rope_fwd",
          "qk_norm_rope_bwd", "gemv_act", "timestep_sinusoid", "flow_noisy_input", "flow_noisy_input_var", "flow_loss", "lora_wgrad", "lora_wgrad_tc", "attn_delta",
          "attn_fwd", "attn_bwd", "grad_finalize", "adamw_tables", "fused_adamw", "require_cuda", "ln_modulate_fwd_pair", "ln_modulate_bwd_pair",
          "qk_norm_rope_fwd_pair", "qk_norm_rope_bwd_pair", "attn_delta_pair"]


def install(lib_module):
    """Monkey-patch the emulation over `qflux_b200.lib`; returns a callable that restores the real bindings."""
    saved = {n: getattr(lib_module, n) for n in _NAMES}
    g = globals()
    for n in _NAMES:
        setattr(lib_module, n, g[n])

    def restore():
        for n, f in saved.items():
            setattr(lib_module, n, f)
    return restore
