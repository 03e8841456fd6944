"""Every LoRA gradient tensor of the fused training step against an fp64 oracle, one tensor at a time.

A pooled relative L2 over all LoRA tensors is set by the largest ones (the `lora_B` of an embedder can carry 90 % of the norm), so a
wrong or missing small tensor — an A-side gradient, a modulation site of one block, one q|k|v slot — hides under it.  Here every
case runs the oracle three times on the same bf16-rounded weights:
  * in fp64 (`.double()` on the module, fp64 inputs) — the reference.  A few points of the oracle stay fp32 by definition: the
    timestep sinusoid (`t.float()`, fp32 frequencies), the Qwen RoPE table and its complex multiply (`x.float()`), the FLUX RoPE
    cos / sin tables and their `x.float()` product, the fp32 variance of diffusers' RMSNorm, and the `.float()` of the prediction
    in the Qwen loss.  Each costs ~1e-7 relative, four orders below the bounds here;
  * in bf16 eager — the yardstick: what the reference trainer itself computes (on the device with the SDPA backends of
    `eager_sdpa`);
  * on the fused model, on three paths: (a) `compute_loss(...).backward()` read from `param.grad`, (b) the no-autograd `train_step`
    read from the fp32 accumulator (`lora_grad_views()`, max_grad_norm = 0: nothing clipped), (c) the module-forward autograd bridge
    (`dit(...)` under grad mode with the loss `pred.pow(2).mean()`; dense batches only).
For every LoRA parameter n:  rel_n = |g_n - g64_n| / |g64_n|,  eager_n the same for bf16 eager; it passes when
rel_n <= 1.5 eager_n + 2e-3 and rel_n <= 3e-2.  Where the fp64 gradient is exactly zero (the oracle never reaches the tensor: e.g.
the text MLP of the last Qwen block, whose output is discarded) the fused gradient must be exactly zero.
Two invariants ride along: the views of `lora_grad_views()` tile the flat accumulator G32 exactly (no overlap, no gap), and after a
`train_step` with one `FusedLoraAdamW` step the padding of every LoRA site (A_pad rows past the rank, B_pad columns past the rank,
both factors of slots without an adapter) is still exactly zero — the fused GEMMs read it as part of the LoRA k-block.

The same functions run on CPU with tests/emu_lib.py installed over `qflux_b200.lib` (host wiring: offsets, slots, per-sample loops)
and on an H100 with the real kernels (`CASES`, run by tests/test_lora_grad_parity.py and stand-alone through harness.main)."""
import contextlib
import copy
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from harness import main  # noqa: E402

import torch  # noqa: E402

F64, BF = torch.float64, torch.bfloat16
RATIO, FLOOR, CAP = 1.5, 2e-3, 3e-2

# every LoRA-capable Linear of a Qwen double block (_DOUBLE_LINEARS), both AdaLN modulation linears and both input embedders
QWEN_ALL = ("attn.to_q", "attn.to_k", "attn.to_v", "attn.add_q_proj", "attn.add_k_proj", "attn.add_v_proj", "attn.to_out.0",
            "attn.to_add_out", "img_mlp.net.0.proj", "txt_mlp.net.0.proj", "img_mlp.net.2", "txt_mlp.net.2", "img_mod.1", "txt_mod.1",
            "img_in", "txt_in")
QWEN_SUBSET = ("attn.to_k", "attn.add_v_proj", "attn.to_add_out", "img_mlp.net.2", "txt_mod.1", "txt_in")
# every LoRA-capable Linear of FLUX: double-block linears and AdaLN linears, single-block q / k / v, proj_mlp, proj_out and AdaLN
# linear, both input embedders
FLUX_ALL = (r"(x_embedder|context_embedder"
            r"|transformer_blocks\.[0-9]+\.(attn\.(to_[qkv]|add_[qkv]_proj|to_out\.0|to_add_out)|ff(_context)?\.net\.(0\.proj|2)"
            r"|norm1(_context)?\.linear)"
            r"|single_transformer_blocks\.[0-9]+\.(attn\.to_[qkv]|proj_mlp|proj_out|norm\.linear))")


def eager_sdpa():
    """Attention backends the bf16-eager oracle may use on the device: flash, memory-efficient and math — not cuDNN attention.
    With torch 2.11 / CUDA 12.8 on an H100, F.scaled_dot_product_attention picks cuDNN attention for the oracle's bf16 calls, and
    its backward is wrong for the FLUX oracle: in a process that never loads this project's library, the LoRA gradients of both
    embedders and every double block of the tiny FLUX case came out 2e4-2e5 times too large (and different from run to run, so it
    reads memory it should not), while the single blocks were fine.  At full width (1 double + 1 single block, S = 2560) the same
    backward ended in an illegal memory access.  Forcing cuDNN attention alone reproduces the wrong gradients; with each of the
    other three backends forced, the same gradients agree with the bf16 run on the host to the same ~2e-2 of fp64."""
    from torch.nn.attention import SDPBackend, sdpa_kernel
    return sdpa_kernel([SDPBackend.FLASH_ATTENTION, SDPBackend.EFFICIENT_ATTENTION, SDPBackend.MATH])


def _flux_yaml_targets():
    from model_check import FLUX_YAML_TARGETS
    return FLUX_YAML_TARGETS


def _dev():
    return torch.device("cuda" if torch.cuda.is_available() else "cpu")


def _nontrivial_norms_(orc, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in orc.named_parameters():
            if n.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.02)
            elif p.ndim == 1:
                p.copy_(1 + torch.randn(p.shape, generator=g) * 0.1)


def _round_bf16_(orc):
    """Every parameter rounded to bf16 once: the fp64 oracle, the bf16 oracle and the fused model share identical weights."""
    with torch.no_grad():
        for p in orc.parameters():
            p.copy_(p.bfloat16().float())
    return orc


def _fused(cls, cfg, dev):
    return cls(cfg) if dev.type == "cuda" else cls(cfg, device="cpu", _host_only=True)


def _load(m, orc, dev):
    missing, unexpected = m.load_state_dict({k: v.to(dev) for k, v in orc.state_dict().items()}, strict=True)
    assert not missing and not unexpected, (missing, unexpected)


def qwen_pair(dev, H=2, L=2, J=128, r=4, targets=QWEN_ALL, w_std=0.05):
    """(fp32 oracle on the host, fused model on `dev`), LoRA alpha = 2r, lora_B ~ N(0, 0.05^2)."""
    from oracle import mmdit_oracle as mo
    from qflux_b200.qwen_model import QwenB200Config, QwenImageB200
    orc = mo.init_synthetic_(mo.QwenImageOracle(mo.QwenConfig(num_layers=L, attention_head_dim=128, num_attention_heads=H,
                                                              joint_attention_dim=J)), std=w_std)
    _nontrivial_norms_(orc, 99)
    mo.add_lora_adapter(orc, r=r, alpha=2 * r, target_modules=targets, b_std=0.05)
    _round_bf16_(orc)
    m = _fused(QwenImageB200, QwenB200Config(num_layers=L, num_attention_heads=H, joint_attention_dim=J), dev)
    m.add_adapter(r, 2 * r, target_modules=targets)
    _load(m, orc, dev)
    return orc, m


def flux_pair(dev, H=2, L=2, Ls=2, J=64, Pp=64, r=4, targets=FLUX_ALL):
    from oracle import mmdit_oracle as mo
    from qflux_b200.flux_model import FluxB200, FluxB200Config
    kw = dict(num_layers=L, num_single_layers=Ls, attention_head_dim=128, num_attention_heads=H, joint_attention_dim=J,
              pooled_projection_dim=Pp, guidance_embeds=True)
    orc = mo.init_synthetic_(mo.FluxOracle(mo.FluxConfig(**kw)), std=0.05 if H < 8 else 0.02)
    _nontrivial_norms_(orc, 98)
    mo.add_lora_adapter(orc, r=r, alpha=2 * r, target_modules=targets, b_std=0.05)
    _round_bf16_(orc)
    m = _fused(FluxB200, FluxB200Config(**kw), dev)
    m.add_adapter(r, 2 * r, target_modules=targets)
    _load(m, orc, dev)
    return orc, m


# ------------------------------------------------------------------------------------------------------------ comparison
def _hp(t):
    """Loss arithmetic of an oracle output: fp32 for a bf16 run (what the trainer does), the output's own dtype for fp64."""
    return t.to(torch.promote_types(t.dtype, torch.float32))


def oracle_grads(orc, dtype, dev, loss_fn):
    """LoRA gradients (fp64 on the host; None where autograd never reached the tensor) of `loss_fn(oracle copy in dtype, dtype, dev)`;
    a bf16 run on the device uses the attention backends of `eager_sdpa`."""
    o = copy.deepcopy(orc).to(dev, dtype)
    with eager_sdpa() if dev.type == "cuda" and dtype == BF else contextlib.nullcontext():
        loss_fn(o, dtype, dev).backward()
    g = {n: (None if p.grad is None else p.grad.detach().to("cpu", F64)) for n, p in o.named_parameters() if p.requires_grad}
    del o
    if dev.type == "cuda":
        torch.cuda.empty_cache()
    return g


def per_tensor(got, g64, g16):
    """Per-tensor comparison of fused gradients `got` with the fp64 gradients `g64`, scaled by the bf16-eager gradients `g16`.
    Returns dict(rows=[...], fail=[...], pooled, pooled_eager, worst_ratio)."""
    fail = []
    if set(got) != set(g64):
        fail.append(f"parameter names differ: {sorted(set(got) ^ set(g64))[:6]}")
    den = math.sqrt(sum(float((v ** 2).sum()) for v in g64.values() if v is not None)) or 1.0
    rows, num, num16, worst = [], 0.0, 0.0, 0.0
    for n in sorted(set(got) & set(g64)):
        ref, g = (None if g64[n] is None else g64[n].to("cpu", F64)), got[n].to("cpu", F64)
        e16 = g16.get(n)
        if ref is None or not bool(ref.abs().max() > 0):
            mx = float(g.abs().max())
            rows.append(dict(name=n, rel=mx, eager=None, ratio=None, share=0.0, zero=True))
            if mx != 0.0 or not math.isfinite(mx):
                fail.append(f"{n}: the fp64 gradient is exactly zero, the fused one has max |g| = {mx:.3e}")
            num += float((g ** 2).sum())
            continue
        e16 = torch.zeros_like(ref) if e16 is None else e16.to("cpu", F64)
        nr = float(ref.norm())
        rel, eager = float((g - ref).norm()) / nr, float((e16 - ref).norm()) / nr
        num += float(((g - ref) ** 2).sum())
        num16 += float(((e16 - ref) ** 2).sum())
        ratio = rel / max(eager, 1e-30)
        bound = min(RATIO * eager + FLOOR, CAP)
        rows.append(dict(name=n, rel=rel, eager=eager, ratio=ratio, share=nr / den, zero=False))
        if not rel <= bound:  # (NaN fails)
            fail.append(f"{n}: rel {rel:.3e} > {bound:.3e} (bf16 eager {eager:.3e}, share {nr / den:.4f})")
        worst = max(worst, ratio) if math.isfinite(ratio) else float("inf")
    return dict(rows=rows, fail=fail, pooled=math.sqrt(num) / den, pooled_eager=math.sqrt(num16) / den, worst_ratio=worst)


def format_table(title, rep):
    lines = [f"{title}: pooled {rep['pooled']:.3e} (bf16 eager {rep['pooled_eager']:.3e}), worst ratio {rep['worst_ratio']:.2f}",
             f"  {'tensor':<62} {'rel':>9} {'eager':>9} {'ratio':>6} {'share':>7}"]
    for r in rep["rows"]:
        if r["zero"]:
            lines.append(f"  {r['name']:<62} {r['rel']:>9.2e} {'(fp64 gradient exactly zero)':>24}")
        else:
            lines.append(f"  {r['name']:<62} {r['rel']:>9.2e} {r['eager']:>9.2e} {r['ratio']:>6.2f} {r['share']:>7.4f}")
    return "\n".join(lines)


# ------------------------------------------------------------------------------------------------------------ invariants
def tiling_fail(m):
    """The views of `lora_grad_views()` cover G32 exactly once: contiguous, inside G32, no overlap, no gap, one per parameter."""
    views, G = m.lora_grad_views(), m.G32
    fail = []
    params = dict(m.named_parameters())
    if set(views) != set(params):
        fail.append(f"views and parameters differ: {sorted(set(views) ^ set(params))[:6]}")
    spans = []
    for n, v in views.items():
        if n in params and tuple(v.shape) != tuple(params[n].shape):
            fail.append(f"{n}: view shape {tuple(v.shape)} != parameter shape {tuple(params[n].shape)}")
        if not v.is_contiguous() or v.untyped_storage().data_ptr() != G.untyped_storage().data_ptr():
            fail.append(f"{n}: not a contiguous view of G32")
        spans.append((v.storage_offset() - G.storage_offset(), v.numel(), n))
    spans.sort()
    end, prev = 0, None
    for off, size, n in spans:
        if off < end:
            fail.append(f"{n} [{off}, {off + size}) overlaps {prev}")
        elif off > end:
            fail.append(f"gap [{end}, {off}) before {n}")
        end, prev = max(end, off + size), n
    if end != G.numel():
        fail.append(f"the views end at {end}, G32 has {G.numel()} elements")
    return fail


def padding_fail(m):
    """Every padded LoRA buffer is exactly zero outside the adapter's rank and in slots without an adapter."""
    fail, r, PAD = [], m.lora_rank, 64
    seen = set()
    for key, site in m.sites.items():
        if id(site) in seen:
            continue
        seen.add(id(site))
        d_out = site.B_pad.shape[0] // site.n
        if bool(site.B_pad[:, r:].ne(0).any()):
            fail.append(f"site {key}: B_pad[:, {r}:] is not zero")
        for slot in range(site.n):
            a = site.A_pad[slot * PAD + (r if slot in site.members else 0):(slot + 1) * PAD]
            if bool(a.ne(0).any()):
                fail.append(f"site {key} slot {slot}: A_pad padding rows are not zero")
            if slot not in site.members and bool(site.B_pad[slot * d_out:(slot + 1) * d_out].ne(0).any()):
                fail.append(f"site {key} slot {slot} (no adapter): B_pad rows are not zero")
    return fail


# ------------------------------------------------------------------------------------------------------------ the three paths
def run_paths(orc, m, step, emb, kw, oracle_step, oracle_fwd=None, fused_fwd=None, keep=False):
    """Oracle (fp64, bf16) and fused gradients on paths (a) autograd, (b) train_step, (c) module forward (when `oracle_fwd` /
    `fused_fwd` are given), the tiling invariant, then one FusedLoraAdamW step and the padding invariant.  The oracle loss
    functions take (oracle, dtype, device)."""
    from qflux_b200.optim import FusedLoraAdamW
    dev = m.dev
    ref = {dt: oracle_grads(orc, dt, dev, oracle_step) for dt in (F64, BF)}
    out = dict(fail=[], paths={})
    step.compute_loss(emb, **kw).backward()
    got = {"autograd": {n: p.grad.to("cpu", F64) for n, p in m.named_parameters()}}
    out["fail"] += ["tiling: " + f for f in tiling_fail(m)]
    for p in m.parameters():
        p.grad = None
    step.train_step(emb, **kw)
    got["train_step"] = {n: v.to("cpu", F64) for n, v in m.lora_grad_views().items()}
    refs = {"autograd": ref, "train_step": ref}
    if oracle_fwd is not None:
        refs["module_forward"] = {dt: oracle_grads(orc, dt, dev, oracle_fwd) for dt in (F64, BF)}
        for p in m.parameters():
            p.grad = None
        fused_fwd(m).backward()
        got["module_forward"] = {n: p.grad.to("cpu", F64) for n, p in m.named_parameters()}
        for p in m.parameters():
            p.grad = None
    opt = FusedLoraAdamW(m, lr=1e-2, weight_decay=0.1)
    step.train_step(emb, opt, **kw)
    out["fail"] += ["padding: " + f for f in padding_fail(m)]
    for path, g in got.items():
        rep = per_tensor(g, refs[path][F64], refs[path][BF])
        out["paths"][path] = rep
        out["fail"] += [f"{path}: {f}" for f in rep["fail"]]
        if keep:
            rep["grads"] = (g, refs[path][F64], refs[path][BF])
    out["worst_ratio"] = max(r["worst_ratio"] for r in out["paths"].values())
    return out


def _to(x, dev, dt=None):
    return x.to(dev) if dt is None else x.to(dev, dt)


# ------------------------------------------------------------------------------------------------------------ Qwen
def qwen_case(H=2, L=2, J=128, r=4, targets=QWEN_ALL, B=3, hw=4, T=24, shapes=None, keep=False, dev=None):
    """Shared-resolution Qwen-Image-Edit step (`shapes`: one list of latent shapes shared by the batch, target first — three
    entries for Edit-Plus), plus the module forward."""
    from oracle import mmdit_oracle as mo
    from qflux_b200.train_step import QwenImageEditStep
    dev = dev or _dev()
    orc, m = qwen_pair(dev, H, L, J, r, targets)
    shapes = shapes or [(1, hw, hw), (1, hw, hw)]
    lt, lc = shapes[0][1] * shapes[0][2], sum(h * w for _, h, w in shapes[1:])
    g = torch.Generator().manual_seed(0)
    rn = lambda *s: torch.randn(*s, generator=g).bfloat16()
    x = dict(image_latents=rn(B, lt, 64), control_latents=rn(B, lc, 64), prompt_embeds=rn(B, T, J) * 3,
             prompt_embeds_mask=torch.ones(B, T, dtype=torch.int64), img_shapes=[shapes] * B, noise=rn(B, lt, 64),
             u=torch.tensor([0.5, 0.25, 0.125, 0.75][:B]))  # sigma .5 / .75 / .875 / .25: exact in bf16
    t_fwd = torch.tensor([0.625, 0.25, 0.875, 0.5][:B])

    def oracle_step(o, dt, dev=dev):
        xd = {k: (_to(v, dev, dt) if k in ("image_latents", "control_latents", "prompt_embeds", "noise") else
                  _to(v, dev) if k == "prompt_embeds_mask" else v) for k, v in x.items()}
        return mo.qwen_compute_loss(o, **xd)[0]

    packed = torch.cat([x["image_latents"], x["control_latents"]], 1)
    fkw = dict(encoder_hidden_states_mask=_to(x["prompt_embeds_mask"], dev), img_shapes=x["img_shapes"], txt_seq_lens=[T] * B)

    def oracle_fwd(o, dt, dev=dev):
        p = o(hidden_states=_to(packed, dev, dt), timestep=_to(t_fwd, dev), encoder_hidden_states=_to(x["prompt_embeds"], dev, dt),
              **fkw)[0]
        return _hp(p).pow(2).mean()

    def fused_fwd(mm):
        return mm(hidden_states=_to(packed, dev), timestep=_to(t_fwd, dev), encoder_hidden_states=_to(x["prompt_embeds"], dev),
                  **fkw)[0].float().pow(2).mean()

    emb = {k: x[k] for k in ("image_latents", "control_latents", "prompt_embeds", "img_shapes")}
    step = QwenImageEditStep(m, max_grad_norm=0.0, use_cuda_graph=False)
    return run_paths(orc, m, step, emb, dict(noise=x["noise"], u=x["u"]), oracle_step, oracle_fwd, fused_fwd, keep)


def qwen_multires_case(targets=QWEN_ALL, r=4, keep=False, dev=None):
    """Pad-to-max multi-resolution batch (per-sample RoPE, text and image key masks, AttentionMask loss) against one un-padded
    oracle run per sample."""
    from qflux_b200.train_step import QwenImageEditStep
    dev = dev or _dev()
    orc, m = qwen_pair(dev, 2, 2, 128, r, targets)
    g = torch.Generator().manual_seed(11)
    rn = lambda *s: torch.randn(*s, generator=g).bfloat16()
    shapes = [[(1, 4, 4), (1, 4, 4)], [(1, 2, 4), (1, 2, 4)], [(1, 4, 2), (1, 4, 2)]]
    lt = [sh[0][1] * sh[0][2] for sh in shapes]
    B, T, txt, Lt = 3, 8, [8, 5, 6], max(lt)
    x0, ctrl, pe, noise = rn(B, Lt, 64), rn(B, Lt, 64), rn(B, T, 128) * 3, rn(B, Lt, 64)
    mask = torch.zeros(B, T, dtype=torch.int64)
    for b in range(B):
        x0[b, lt[b]:] = 0; ctrl[b, lt[b]:] = 0; noise[b, lt[b]:] = 0; pe[b, txt[b]:] = 0; mask[b, :txt[b]] = 1
    u = torch.tensor([0.5, 0.25, 0.75])
    sig = (1000 - (u * 1000).long()).float() / 1000

    def oracle_step(o, dt, dev=dev):
        total = 0.0
        for b in range(B):
            n = lt[b]
            noisy = (1 - sig[b].item()) * x0[b, :n].to(dt) + sig[b].item() * noise[b, :n].to(dt)
            packed = torch.cat([noisy, ctrl[b, :n].to(dt)], 0)[None].to(dev)
            p = o(hidden_states=packed, timestep=_to(sig[b:b + 1], dev), encoder_hidden_states=_to(pe[b:b + 1, :txt[b]], dev, dt),
                  encoder_hidden_states_mask=_to(mask[b:b + 1, :txt[b]], dev), img_shapes=[shapes[b]], txt_seq_lens=[txt[b]])[0][0, :n]
            p = _hp(p)
            total = total + ((p - _to(noise[b, :n].to(p.dtype) - x0[b, :n].to(p.dtype), dev)) ** 2).mean(-1).sum()
        return total / (sum(lt) + 1e-12)

    step = QwenImageEditStep(m, "attention_mask", max_grad_norm=0.0, use_cuda_graph=False)
    emb = dict(image_latents=x0, control_latents=ctrl, prompt_embeds=pe, prompt_embeds_mask=mask, img_shapes=shapes)
    return run_paths(orc, m, step, emb, dict(noise=noise, u=u), oracle_step, keep=keep)


# ------------------------------------------------------------------------------------------------------------ FLUX
def flux_case(targets=FLUX_ALL, r=8, H=2, L=2, Ls=2, J=64, Pp=64, B=2, hw=8, T=24, keep=False, dev=None):
    """FLUX-Kontext shared-resolution step (2 double + 2 single blocks by default), plus the module forward."""
    from oracle import mmdit_oracle as mo
    from qflux_b200.train_step import FluxKontextStep
    dev = dev or _dev()
    orc, m = flux_pair(dev, H, L, Ls, J, Pp, r, targets)
    g = torch.Generator().manual_seed(3)
    rn = lambda *s: torch.randn(*s, generator=g).bfloat16()
    n = hw * hw
    x0, ctrl, pooled, pe, noise = rn(B, n, 64), rn(B, n, 64), rn(B, Pp), rn(B, T, J), rn(B, n, 64)
    text_ids = torch.zeros(T, 3)
    img_ids, ctrl_ids = FluxKontextStep.latent_image_ids(hw, hw, "cpu", 0.0), FluxKontextStep.latent_image_ids(hw, hw, "cpu", 1.0)
    t = torch.tensor([0.5, 0.25, 0.125, 0.0625][:B])  # t * 1000 exact in bf16 (the model multiplies in bf16)
    t_fwd = torch.tensor([0.25, 0.0625, 0.5, 0.125][:B])

    def oracle_step(o, dt, dev=dev):
        return mo.flux_compute_loss_shared(o, _to(x0, dev, dt), _to(ctrl, dev, dt), _to(pooled, dev, dt), _to(pe, dev, dt),
                                           _to(text_ids, dev), _to(img_ids, dev), _to(ctrl_ids, dev), noise=_to(noise, dev, dt),
                                           t=_to(t, dev, dt))[0]

    packed = torch.cat([x0, ctrl], 1)
    ids = torch.cat([img_ids, ctrl_ids], 0)

    def oracle_fwd(o, dt, dev=dev):
        p = o(hidden_states=_to(packed, dev, dt), encoder_hidden_states=_to(pe, dev, dt), pooled_projections=_to(pooled, dev, dt),
              timestep=_to(t_fwd, dev), img_ids=_to(ids, dev), txt_ids=_to(text_ids, dev), guidance=torch.ones(B, device=dev))[0]
        return _hp(p).pow(2).mean()

    def fused_fwd(mm):
        return mm(hidden_states=_to(packed, dev), encoder_hidden_states=_to(pe, dev), pooled_projections=_to(pooled, dev),
                  timestep=_to(t_fwd, dev), img_ids=_to(ids, dev), txt_ids=_to(text_ids, dev),
                  guidance=torch.ones(B, device=dev))[0].float().pow(2).mean()

    emb = dict(image_latents=x0, control_latents=ctrl, pooled_prompt_embeds=pooled, prompt_embeds=pe, text_ids=text_ids,
               image_ids=img_ids, control_ids=ctrl_ids)
    step = FluxKontextStep(m, max_grad_norm=0.0, use_cuda_graph=False)
    return run_paths(orc, m, step, emb, dict(noise=noise, t=t), oracle_step, oracle_fwd, fused_fwd, keep)


def flux_multires_case(targets=FLUX_ALL, r=8, keep=False, dev=None):
    """FLUX pad-to-max multi-resolution recipe (per-sample ids / RoPE, key mask, masked loss) against one un-padded oracle run
    per sample."""
    from qflux_b200.train_step import FluxKontextStep
    dev = dev or _dev()
    orc, m = flux_pair(dev, 2, 2, 2, 64, 64, r, targets)
    g = torch.Generator().manual_seed(21)
    rn = lambda *s: torch.randn(*s, generator=g).bfloat16()
    shapes = [[(1, 6, 6), (1, 6, 6)], [(1, 4, 6), (1, 6, 4)], [(1, 6, 4), (1, 4, 4), (1, 4, 6)]]
    B, T = 3, 24
    lt = [sh[0][1] * sh[0][2] for sh in shapes]
    lc = [sum(h * w for (_, h, w) in sh[1:]) for sh in shapes]
    x0, ctrl, noise = rn(B, max(lt), 64), rn(B, max(lc), 64), rn(B, max(lt), 64)
    for b in range(B):
        x0[b, lt[b]:] = 0; noise[b, lt[b]:] = 0; ctrl[b, lc[b]:] = 0
    pe, pooled, t = rn(B, T, 64), rn(B, 64), torch.tensor([0.5, 0.25, 0.125])
    text_ids = torch.zeros(T, 3)

    def oracle_step(o, dt, dev=dev):
        total = 0.0
        for b in range(B):
            ids = [FluxKontextStep.latent_image_ids(shapes[b][0][1], shapes[b][0][2], "cpu", 0.0)]
            ids += [FluxKontextStep.latent_image_ids(h, w, "cpu", float(j + 1)) for j, (_, h, w) in enumerate(shapes[b][1:])]
            noisy = ((1 - t[b]) * x0[b, :lt[b]].float() + t[b] * noise[b, :lt[b]].float()).bfloat16()  # the trainer's bf16 x_t
            packed = torch.cat([noisy.to(dt), ctrl[b, :lc[b]].to(dt)], 0)[None].to(dev)
            p = o(hidden_states=packed, encoder_hidden_states=_to(pe[b:b + 1], dev, dt), pooled_projections=_to(pooled[b:b + 1], dev, dt),
                  timestep=_to(t[b:b + 1], dev), img_ids=_to(torch.cat(ids, 0), dev), txt_ids=_to(text_ids, dev),
                  guidance=torch.ones(1, device=dev))[0][0, :lt[b]]
            p = _hp(p)
            total = total + ((p - _to(noise[b, :lt[b]].to(p.dtype) - x0[b, :lt[b]].to(p.dtype), dev)) ** 2).mean(-1).sum()
        return total / (sum(lt) + 1e-12)

    step = FluxKontextStep(m, "attention_mask", max_grad_norm=0.0, use_cuda_graph=False)
    emb = dict(image_latents=x0, control_latents=ctrl, pooled_prompt_embeds=pooled, prompt_embeds=pe, text_ids=text_ids, img_shapes=shapes)
    return run_paths(orc, m, step, emb, dict(noise=noise, t=t), oracle_step, keep=keep)


# ------------------------------------------------------------------------------------------------------------ cases
# the tiny cases (also run on CPU with emulated kernels) and the full-width ones, which reach what the tiny configs never do:
# qfx_lora_wgrad_tc at real M with split CTAs, qfx_mod_grad at D = 3072, the 6-problem grouped GEMMs and split-K
TINY = {
    "qwen_all_r4_b3": lambda **k: qwen_case(r=4, B=3, **k),
    "qwen_all_r64": lambda **k: qwen_case(r=64, B=2, **k),
    "qwen_subset_r16": lambda **k: qwen_case(r=16, B=2, targets=QWEN_SUBSET, **k),
    "qwen_mod_embed_r4": lambda **k: qwen_case(r=4, B=2, targets=("to_q", "img_mod.1", "txt_mod.1", "img_in", "txt_in"), **k),
    "qwen_multires": lambda **k: qwen_multires_case(**k),
    "qwen_edit_plus_3img": lambda **k: qwen_case(r=4, B=2, T=16, shapes=[(1, 4, 4), (1, 4, 6), (1, 2, 4)], **k),
    "flux_all": lambda **k: flux_case(**k),
    "flux_yaml_targets": lambda **k: flux_case(targets=_flux_yaml_targets(), **k),
    "flux_multires": lambda **k: flux_multires_case(**k),
}
FULL_WIDTH = {
    "qwen_full_width_1blk": lambda **k: qwen_case(H=24, L=1, J=3584, r=16, B=2, hw=32, T=352, **k),
    "flux_full_width_1p1": lambda **k: flux_case(H=24, L=1, Ls=1, J=4096, Pp=768, r=16, B=1, hw=32, T=512, **k),
}


def _summary(res):
    """JSON-sized result: per path the pooled error, the worst ratio and the failures (the per-tensor rows stay in the table)."""
    return dict(fail=res["fail"], worst_ratio=res["worst_ratio"],
                paths={p: dict(pooled=r["pooled"], pooled_eager=r["pooled_eager"], worst_ratio=r["worst_ratio"])
                       for p, r in res["paths"].items()})


def _gpu_case(fn):
    def run():
        res = fn()
        for p, rep in res["paths"].items():
            print(format_table(p, rep), file=sys.stderr)
        return _summary(res)
    return run


CASES = {name: _gpu_case(fn) for name, fn in {**TINY, **FULL_WIDTH}.items()}

if __name__ == "__main__":
    main(CASES, os.path.abspath(__file__), "lora_grad_check.log")
