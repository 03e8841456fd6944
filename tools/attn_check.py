"""GPU check of the joint attention forward / backward (qfx_attn_fwd, qfx_attn_bwd) per row, at the mask and tile edges the
training step reaches, against

  (a) an fp64 reference computed per sample from the kernel's bf16 inputs: masked softmax attention with lse restated in log2,
      and fp64 autograd of it with the same mask and zero dO on padding query rows (positions >= kv_len[b], as the training step
      passes them).  The same operation in bf16 eager on the device (SDPA with the same boolean mask, and its autograd) sets the
      scale of "close": err_kernel <= C * err_eager + FLOOR (relative L2 against fp64) in every (b, h, query row) of O and dQ and
      every (b, h, key row) of dK and dV; lse within LSE_TOL (log2 units) of fp64 in every row;
  (b) exact facts: masked keys (>= kv_len, or inside [txt_len, split)) get exactly zero dK and dV; a query tile of only padding rows
      gets O = 0 and lse = 0; the backward ADDS into dQ (prefilled here) and leaves the rows >= kv_len as the caller set them;
      forward O / lse and backward dK / dV are bit-identical across two launches (dQ is reduced with atomics and is not);
  (c) sentinels: columns outside the output slice, rows past the row groups, and the tail of over-allocated lse / dQ / dK / dV
      buffers past the last (b, h) slab keep their pattern;
  (d) tests/emu_lib.py on CPU copies (small cases): per row within the same bf16-eager scale (the kernel rounds P to bf16 and
      uses an online softmax, the emulation does neither).  Rows the kernel defines and the emulation does not are excluded by
      name: padding query tiles, where the kernel writes zeros and lse = 0.

Text-padding rows (queries in [txt_len, split)) are queries too: their outputs are checked like any other row.  Each case
returns a dict of measurements plus `fail`, the list of violated checks (each names the tensor and its (b, h, row)).  Run
stand-alone: `python tools/attn_check.py [case ...]` (one subprocess per case).
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from harness import ROOT, main  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from glue_check import Checks, _mk  # noqa: E402
from gemm_tile_check import SENT_F32, is_sent, sentinel  # noqa: E402

BF, F64 = torch.bfloat16, torch.float64
LOG2E = 1.4426950408889634
# err_kernel <= C * err_eager + FLOOR per row, relative L2 against fp64 (ratios measured on an H100: see the commit message that
# introduced this file).  dQ and dK reach about 4.5x bf16 SDPA's row error: the kernel rounds dS to bf16 before both contractions
# (tests/emu_lib.py, which does the same, shows the same ratio).  The emulation is held to 2 C: kernel and emulation are each
# within C of fp64.
C_ROW = {"O": 1.5, "dQ": 6.0, "dK": 6.0, "dV": 1.5}
FLOOR_ROW = 1e-3
LSE_TOL = 1e-4
PADC, PADR = 64, 3
DEV = "cuda"


# ============================================================================ fp64 references (device-agnostic; checked on CPU too)
def key_mask(B, S, split, kv_len=None, txt_len=None, device="cpu"):
    """[B, S] valid keys: < kv_len[b] and outside the text padding [txt_len[b], split)"""
    pos = torch.arange(S, device=device)[None]
    m = torch.ones(B, S, dtype=torch.bool, device=device)
    if kv_len is not None:
        m &= pos < kv_len.to(device)[:, None]
    if txt_len is not None:
        m &= ~((pos >= txt_len.to(device)[:, None]) & (pos < split))
    return m


def padding_tile_rows(B, S, split, kv_len, device="cpu"):
    """[B, S] query rows of the forward's padding tiles (128-row tiles starting at or past both kv_len[b] and split)"""
    if kv_len is None:
        return torch.zeros(B, S, dtype=torch.bool, device=device)
    q0 = (torch.arange(S, device=device) // 128 * 128)[None]
    return (q0 >= kv_len.to(device)[:, None]) & (q0 >= split)


def attn_ref(Q, K, V, mask, scale, dO=None, dt=F64):
    """per sample in dtype dt: O [B,H,S,128], lse (log2) [B,H,S] and, with dO, autograd's (dQ, dK, dV)"""
    B = Q.shape[0]
    O, L, G = [], [], []
    for b in range(B):
        q, k, v = (t[b].to(dt).requires_grad_(dO is not None) for t in (Q, K, V))
        s = (q @ k.transpose(-1, -2) * scale).masked_fill(~mask[b][None, None, :], float("-inf"))
        o = torch.softmax(s, -1) @ v
        O.append(o.detach())
        L.append(torch.logsumexp(s, -1).detach() * LOG2E)
        if dO is not None:
            g = dO[b].to(dt)
            dq, dk, dv = torch.autograd.grad(o, (q, k, v), g)
            # the size of dS = P (dP - delta) before the cancellation inside the bracket: the scale dQ / dK rows are measured on
            p = torch.softmax(s, -1).detach()
            a = p * (g.abs() @ v.detach().abs().transpose(-1, -2) + (g * o.detach()).abs().sum(-1, keepdim=True)) * scale
            G.append((dq, dk, dv, (a @ k.detach().abs()).norm(dim=-1), (a.transpose(-1, -2) @ q.detach().abs()).norm(dim=-1)))
    out = dict(O=torch.stack(O), lse=torch.stack(L))
    if dO is not None:
        out.update({n: torch.stack([g[i] for g in G]) for i, n in enumerate(("dQ", "dK", "dV", "dQ_mag", "dK_mag"))})
    return out


def attn_eager(Q, K, V, mask, scale, dO=None):
    """bf16 SDPA with the same boolean mask (and its autograd), per sample"""
    O, G = [], []
    for b in range(Q.shape[0]):
        q, k, v = (t[b:b + 1].detach().clone().requires_grad_(dO is not None) for t in (Q, K, V))
        o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask[b][None, None, None, :], scale=scale)
        O.append(o.detach()[0])
        if dO is not None:
            G.append(torch.autograd.grad(o, (q, k, v), dO[b:b + 1]))
    out = dict(O=torch.stack(O))
    if dO is not None:
        out.update(dQ=torch.cat([g[0] for g in G]), dK=torch.cat([g[1] for g in G]), dV=torch.cat([g[2] for g in G]))
    return out


# ============================================================================ checks
def _rowerr(x, ref, den=None):
    """per-row L2 error relative to the reference row (or to den, a [B, H, S] scale)"""
    ref = ref.double()
    return (x.double() - ref).norm(dim=-1) / (ref.norm(dim=-1) if den is None else den).clamp_min(1e-300)


def _rows(c, name, k, e, ref, sel, C, den=None):
    """per (b, h, row) of [B, H, S, 128] tensors over the rows in sel [B, S]: err_k <= C * err_e + FLOOR_ROW.  dQ / dK rows are
    measured against the size of their terms (den), since dP - delta cancels in rows that attend to few keys"""
    rk, re_ = _rowerr(k, ref, den), _rowerr(e, ref, den)
    s = sel[:, None, :].expand_as(rk)
    if not bool(s.any()):
        return
    c.res[f"{name}_row_worst_k_e"] = [rk[s].max().item(), re_[s].max().item()]
    c.res[f"{name}_row_ratio_max"] = (rk / re_.clamp_min(1e-300))[s].max().item()
    nkt = -(-rk.shape[-1] // 128)  # worst kernel error of each 128-row tile, over (b, h)
    c.res[f"{name}_tile_worst"] = [rk.masked_fill(~s, 0).amax((0, 1))[128 * t:128 * (t + 1)].max().item() for t in range(nkt)]
    bad = ~(rk <= C * re_ + FLOOR_ROW) & s
    for b, h, r in bad.nonzero().tolist()[:3]:
        c.fail.append(f"{name} (b{b}, h{h}, row {r}): kernel {rk[b, h, r].item():.3e} vs bf16 eager {re_[b, h, r].item():.3e}")


def _exact_zero(c, name, t, sel):
    z = t[sel[:, None, :].expand(t.shape[:3])]
    ok = z == 0
    if not bool(ok.all()):
        idx = (~(t == 0).all(-1) & sel[:, None, :]).nonzero().tolist()[:3]
        c.fail.append(f"{name}: {int((~ok).sum())} elements not exactly zero, first (b, h, row) {idx}")


def _o_headmajor(ot, oi, B, H, S, split):
    return torch.cat([ot.reshape(B, split, H, 128), oi.reshape(B, S - split, H, 128)], 1).permute(0, 2, 1, 3)


def run(c, B, H, S, split, txt=None, kv=None, seed=0, emu_check=True, k_tile_gain=None):
    """one forward + backward at (B, H, S, split) with per-sample txt_len / kv_len lists (None: no such mask)"""
    from qflux_b200 import lib
    dev = DEV
    scale = 128 ** -0.5
    Q, K, V = (_mk(B, H, S, 128, seed=seed + i, device=dev) for i in range(3))
    if k_tile_gain is not None:  # sample 1: logits grow tile by tile, so the running maximum rescales at every key tile
        g = torch.tensor(k_tile_gain, device=dev).repeat_interleave(128)[:S]
        K[1] = (K[1].float() * g[None, :, None]).to(BF)
        Q[1] = (Q[1].float() * 2).to(BF)
    kv_len = None if kv is None else torch.tensor(kv, dtype=torch.int32, device=dev)
    txt_len = None if txt is None else torch.tensor(txt, dtype=torch.int32, device=dev)
    mask = key_mask(B, S, split, kv_len, txt_len, dev)
    padq = padding_tile_rows(B, S, split, kv_len, dev)
    qvalid = torch.ones(B, S, dtype=torch.bool, device=dev) if kv is None else torch.arange(S, device=dev)[None] < kv_len[:, None]
    D = H * 128
    n = B * H * S

    def fwd():
        f0, f1 = sentinel(B * split + PADR, D + 2 * PADC, device=dev), sentinel(B * (S - split) + PADR, D + 2 * PADC, device=dev)
        lse_full = torch.full((n + 64,), SENT_F32, device=dev)
        ot, oi = f0[:B * split, PADC:PADC + D], f1[:B * (S - split), PADC:PADC + D]
        lib.attn_fwd(Q, K, V, ot, oi, split, lse_full[:n].view(B, H, S), kv_len, txt_len=txt_len)
        return f0, f1, lse_full
    f0, f1, lse_full = fwd()
    g0, g1, lse_full2 = fwd()
    O = _o_headmajor(f0[:B * split, PADC:PADC + D], f1[:B * (S - split), PADC:PADC + D], B, H, S, split)
    lse = lse_full[:n].view(B, H, S)
    c.check(bool(torch.equal(f0.view(torch.int16), g0.view(torch.int16)) and torch.equal(f1.view(torch.int16), g1.view(torch.int16))
                 and torch.equal(lse_full, lse_full2)), "forward: O / lse differ between two launches")
    for nm, fb, rows in (("O_txt", f0, B * split), ("O_img", f1, B * (S - split))):
        inner = torch.zeros_like(fb, dtype=torch.bool)
        inner[:rows, PADC:PADC + D] = True
        c.check(bool(is_sent(fb)[~inner].all()), f"{nm}: written outside its rows / columns")
    c.check(bool((lse_full[n:] == SENT_F32).all()), "lse: written past the last (b, h) slab")
    # ---- backward: zero dO on padding query rows, delta from the kernel's O (as the training step forms it)
    dO = _mk(B, H, S, 128, seed=seed + 5, device=dev)
    dO = dO * qvalid[:, None, :, None].to(BF)
    delta = (dO.float() * O.float()).sum(-1).contiguous()
    dq_full = torch.full((n * 128 + 256,), SENT_F32, device=dev)
    pre = _mk(B, H, S, 128, seed=seed + 6, scale=0.5, dtype=torch.float32, device=dev)
    dq_full[:n * 128] = pre.flatten()
    dk_full, dv_full = sentinel(n * 128 + 256, device=dev), sentinel(n * 128 + 256, device=dev)
    view = lambda t: t[:n * 128].view(B, H, S, 128)
    lib.attn_bwd(Q, K, V, dO, lse, delta, view(dq_full), view(dk_full), view(dv_full), kv_len, txt_len=txt_len, split=split)
    dk2, dv2 = sentinel(n * 128 + 256, device=dev), sentinel(n * 128 + 256, device=dev)
    dq2 = torch.zeros(n * 128, device=dev)
    lib.attn_bwd(Q, K, V, dO, lse, delta, dq2.view(B, H, S, 128), view(dk2), view(dv2), kv_len, txt_len=txt_len, split=split)
    if dev == "cuda":
        torch.cuda.synchronize()
    dQ = view(dq_full).double() - pre.double()
    dK, dV = view(dk_full), view(dv_full)
    c.check(bool(torch.equal(dk_full.view(torch.int16), dk2.view(torch.int16)) and torch.equal(dv_full.view(torch.int16), dv2.view(torch.int16))),
            "backward: dK / dV differ between two launches")
    c.check(bool((dq_full[n * 128:] == SENT_F32).all()), "dQ: written past the last (b, h) slab")
    c.check(bool(is_sent(dk_full[n * 128:]).all() and is_sent(dv_full[n * 128:]).all()), "dK / dV: written past the last (b, h) slab")
    c.check(not bool(is_sent(dk_full[:n * 128]).any() or is_sent(dv_full[:n * 128]).any()), "dK / dV: rows left unwritten")
    # ---- references
    ref = attn_ref(Q, K, V, mask, scale, dO)
    eag = attn_eager(Q, K, V, mask, scale, dO)
    fsel = ~padq
    _rows(c, "O", O, eag["O"], ref["O"], fsel, C_ROW["O"])
    dl = (lse.double() - ref["lse"]).abs()
    c.res["lse_max_abs_err"] = dl[fsel[:, None, :].expand_as(dl)].max().item()
    for b, h, r in (~(dl <= LSE_TOL) & fsel[:, None, :]).nonzero().tolist()[:3]:
        c.fail.append(f"lse (b{b}, h{h}, row {r}): {lse[b, h, r].item():.6f} vs fp64 {ref['lse'][b, h, r].item():.6f}")
    _exact_zero(c, "O of padding query tiles", O, padq)
    c.check(bool((lse[padq[:, None, :].expand_as(lse)] == 0).all()), "lse of padding query tiles is not 0")
    _rows(c, "dQ", dQ, eag["dQ"], ref["dQ"], qvalid, C_ROW["dQ"], ref["dQ_mag"])
    c.check(bool((view(dq_full)[~qvalid[:, None, :].expand(B, H, S)] == pre[~qvalid[:, None, :].expand(B, H, S)]).all()),
            "dQ rows >= kv_len changed (dO is zero there)")
    _rows(c, "dK", dK, eag["dK"], ref["dK"], mask, C_ROW["dK"], ref["dK_mag"])
    _rows(c, "dV", dV, eag["dV"], ref["dV"], mask, C_ROW["dV"])
    _exact_zero(c, "dK of masked keys", dK, ~mask)
    _exact_zero(c, "dV of masked keys", dV, ~mask)
    c.res["masked_keys"] = int((~mask).sum())
    c.res["padding_tile_rows"] = int(padq.sum())
    if emu_check:
        _vs_emu(c, Q, K, V, dO, lse, delta, pre, O, dQ, dK, dV, eag, ref, split, kv_len, txt_len, scale, mask, padq, qvalid)
    return c


def _vs_emu(c, Q, K, V, dO, lse, delta, pre, O, dQ, dK, dV, eag, ref, split, kv_len, txt_len, scale, mask, padq, qvalid):
    import emu_lib as emu
    B, H, S, _ = Q.shape
    cpu = lambda t: None if t is None else t.cpu()
    ot, oi = torch.empty(B * split, H * 128, dtype=BF), torch.empty(B * (S - split), H * 128, dtype=BF)
    le = torch.empty(B, H, S)
    emu.attn_fwd(cpu(Q), cpu(K), cpu(V), ot, oi, split, le, kv_len=cpu(kv_len), scale=scale, txt_len=cpu(txt_len))
    Oe = _o_headmajor(ot, oi, B, H, S, split)
    sel = (~padq).cpu()
    e_ref = _rowerr(eag["O"], ref["O"]).cpu()
    for name, k, e, er, s in (("O", O.cpu(), Oe, e_ref, sel),):
        d = _rowerr(k, e.double())
        ss = s[:, None, :].expand_as(d)
        c.res[f"emu_{name}_row_worst_over_eager"] = (d / er.clamp_min(1e-300))[ss].max().item()
        c.check(bool((d <= 2 * (C_ROW[name] * er + FLOOR_ROW))[ss].all()), f"emu_{name}: rows beyond the bf16-eager scale")
    dl = (lse.cpu().double() - le.double()).abs()
    c.check(bool((dl <= LSE_TOL)[sel[:, None, :].expand_as(dl)].all()), "emu_lse: beyond LSE_TOL outside the padding tiles")
    dqe = pre.cpu().clone()
    dke, dve = torch.empty(B, H, S, 128, dtype=BF), torch.empty(B, H, S, 128, dtype=BF)
    emu.attn_bwd(cpu(Q), cpu(K), cpu(V), cpu(dO), cpu(lse), cpu(delta), dqe, dke, dve, kv_len=cpu(kv_len), scale=scale, txt_len=cpu(txt_len),
                 split=split)
    dqe = dqe.double() - pre.cpu().double()
    for name, k, e, s in (("dQ", dQ, dqe, qvalid.cpu()), ("dK", dK, dke, mask.cpu()), ("dV", dV, dve, mask.cpu())):
        den = ref.get(name + "_mag")
        d = _rowerr(k.cpu(), e.double(), None if den is None else den.cpu())
        er = _rowerr(eag[name], ref[name], den).cpu()
        ss = s[:, None, :].expand_as(d)
        c.res[f"emu_{name}_row_worst_over_eager"] = (d / er.clamp_min(1e-300))[ss].max().item()
        c.check(bool((d <= 2 * (C_ROW[name] * er + FLOOR_ROW))[ss].all()), f"emu_{name}: rows beyond the bf16-eager scale")
    c.check(bool((dke[~mask.cpu()[:, None, :].expand(B, H, S)] == 0).all() and (dve[~mask.cpu()[:, None, :].expand(B, H, S)] == 0).all()),
            "emu: masked keys do not get zero dK / dV")


def case(B, H, S, split, txt=None, kv=None, **kw):
    return lambda: run(Checks(), B, H, S, split, txt, kv, **kw).out()


CASES = {}
# text mask alone (Qwen single resolution with a prompt mask): split on and next to the 64 / 128 key-tile edges
for _sp in (1, 63, 64, 127, 128, 129):
    CASES[f"txt_split{_sp}"] = case(4, 2, 383, _sp, txt=[1, max(1, _sp - 1), _sp, max(1, _sp // 2)])
# one fully masked 128-key tile (txt_len <= split - 128) at split 352, and one, two and three of them at split 513
CASES["txt_split352"] = case(4, 2, 639, 352, txt=[40, 1, 351, 352])
CASES["txt_split513"] = case(4, 2, 767, 513, txt=[300, 200, 100, 512])
# kv_len alone: split + 1, 64k, 64k - 1, 64k + 1, 128k, S, with S one above and one below a 128 boundary
CASES["kv_S385"] = case(6, 2, 385, 129, kv=[130, 192, 191, 193, 256, 385])
CASES["kv_S383"] = case(6, 2, 383, 129, kv=[130, 320, 319, 321, 256, 383])
# both masks
CASES["both_S639_split352"] = case(4, 2, 639, 352, txt=[40, 129, 351, 1], kv=[353, 448, 513, 639])
CASES["both_S641_split352"] = case(4, 2, 641, 352, txt=[352, 40, 100, 223], kv=[641, 577, 575, 512])
for _sp in (63, 64, 127, 128):
    CASES[f"both_S257_split{_sp}"] = case(4, 2, 257, _sp, txt=[1, _sp - 1, _sp, max(1, _sp // 2)], kv=[_sp + 1, 192, 193, 257])
CASES["h24_both"] = case(2, 24, 257, 64, txt=[40, 64], kv=[200, 257])
# sample 0: the only valid keys are in the last key tile (empty prompt); sample 1: logits grow at every key tile
CASES["rescale_last_tile"] = case(2, 2, 500, 384, txt=[0, 384], k_tile_gain=[1.0, 2.0, 3.0, 4.0])
# the benchmark shape with a 40-token prompt: the backward's inactive key tile [128, 256) at the real size
CASES["full_B4_H24_S2400_txt40"] = case(4, 24, 2400, 352, txt=[40, 40, 40, 40], emu_check=False)

if __name__ == "__main__":
    main(CASES, os.path.abspath(__file__), "attn_check.log")
