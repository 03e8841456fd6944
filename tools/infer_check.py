"""The no-grad forward and the sampling loops at full depth against the block-streamed fp64 oracle (oracle/streamed.py), and validation
between training steps bit for bit.

The no-grad forward is what a validation round runs (the reference trainers' `sampling_from_embeddings` under
`torch.inference_mode()`, here `qflux_b200/sampler.py`).  It launches the training forward's kernels, but its host side is its own: two
ping-pong activation buffers, one saved-tensor dict per block kind shared by every block, an LRU of at most three inference workspaces
and a `GraphCache` of its CUDA graphs.  Models and batches come from bench.py's helpers (`CONFIGS`, `build_model`, `build_flux`,
`make_batch`, adapters with lora_B ~ N(0, 0.02^2)).  Each case runs in its own process (harness.main).

A. Forward vs fp64 (`forward_check`).  The module forward under `torch.no_grad()` three times (eager, capture, replay); the replay's
   output is compared with the streamed oracle on the fused model's own weights, in fp64 (the truth) and in bf16 (the eager reference,
   on `lora_grad_check.eager_sdpa`'s attention backends), one sample at a time (`OracleModule`):
     * per sample, over the target tokens:            rel_fused <= 1.25 rel_bf16 + 1e-3   (depth_check's PRED_RATIO / PRED_FLOOR);
     * per 128-row band of each sample's image rows (target and controls, so the tiles that straddle the target / control boundary are
       in it; the last band may be short):           rel_fused <= BAND_RATIO rel_bf16 + BAND_FLOOR; the worst band of each sample is
       reported;
     * the replay equals the eager forward, and the no-grad prediction equals the grad-enabled call's (`ModelFn`, i.e.
       `_forward_impl(train=True)` on the training workspace) bit for bit: the same kernels at the same shapes, no atomics in the
       forward, so any difference would mean the inference workspace layout changes a result;
     * padded rows of a multi-resolution batch come back exactly zero.
B. Sampling loops (`sampler_check`, the 832x576 cases): `sample_qwen` / `sample_flux` with true CFG and a negative prompt of another
   length for SAMPLER_STEPS steps, against the same loop driven by the streamed oracle in fp64 and in bf16 behind the module signature
   (`OracleModule`, bf16 in / bf16 out like a bf16 model, FLUX's timestep and guidance rounded as `t * 1000` in bf16).  Per sample, the
   final latents: rel_fused <= SAMPLER_RATIO rel_bf16 + SAMPLER_FLOOR.  On the device the inference GraphCache must have captured the
   loop's two shapes (a captured graph replays at once and on every later step), so the replayed path is what was compared.
C. Validation between training steps (`validation_case`), under `torch.use_deterministic_algorithms(True)`, CUDA graphs on,
   `FusedLoraAdamW`: model A runs 3 steps, a validation round under `torch.inference_mode()` (4 samples, each with its own (T, Limg)
   and a CFG negative prompt of another length: 8 forward shapes against 3 cached workspaces, so every round evicts workspaces and
   records graphs again), the same round again, the round with `use_cuda_graph_inference = False`, then 3 more steps.  Model B, built
   from the same seed, runs the same 6 steps and no round.  Required: the losses, G32, every LoRA parameter and both AdamW moments are
   bit-identical after step 6; the training step's graph is the same object before and after the rounds; the three rounds are
   bit-identical.

Errors are relative L2 against fp64.  The same code runs on the host at tiny depth and width with tests/emu_lib.py in place of the
kernels (tests/test_inference_parity.py); on an H100 it is run by that test's GPU cases and stand-alone
(`python tools/infer_check.py [case ...]`)."""
import contextlib
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from harness import main, rel_l2  # noqa: E402

import torch  # noqa: E402

import bench  # noqa: E402
import depth_check as dc  # noqa: E402
import lora_grad_check as lg  # noqa: E402

F64, BF = torch.float64, torch.bfloat16
PRED_RATIO, PRED_FLOOR = dc.PRED_RATIO, dc.PRED_FLOOR
BAND = 128
# Measured on an H100 80GB HBM3 at 700 W: the worst band of every sample of every case has rel_fused / rel_bf16 <= 1.023 (bands at
# about 2e-2 from fp64), and the sampled latents 0.96-1.003 (1.4e-2 to 5.1e-2 from fp64); the constants keep depth_check's form.
BAND_RATIO, BAND_FLOOR = 1.25, 1e-3
SAMPLER_RATIO, SAMPLER_FLOOR = 1.25, 1e-3
SAMPLER_STEPS = 3
SIGMA = (0.75, 0.25, 0.5)          # Qwen: exact in bf16
T_FLUX = (0.5, 0.25, 0.125)        # FLUX: t and t * 1000 exact in bf16
GUIDANCE = 3.5
H832, W832 = 36, 52                # 832 x 576 px: 52 x 36 = 1872 latent patches per image
QWEN_T, QWEN_T_NEG = 352, 64
FLUX_T, FLUX_T_NEG = 512, 256
CFG_QWEN, CFG_FLUX = 4.0, 2.5
ADAMW = dict(lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, max_grad_norm=1.0)
STEP_U = (0.5, 0.25, 0.75, 0.125, 0.625, 0.375)  # one sigma (Qwen) / t (FLUX) per training step, exact in bf16


def _bits(t):
    return t.detach().contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32 if t.element_size() == 4 else torch.int64)


def same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(_bits(a).cpu(), _bits(b).cpu())


# ------------------------------------------------------------------------------------------------------------ oracle behind the module
class OracleModule:
    """A (streamed) oracle behind the fused module's forward signature in `dtype`, one sample at a time: model_check.sampler_tiny's
    F32 wrapper made dtype-generic.  `predict(**kw)` returns each sample's output rows in the oracle dtype (a multi-resolution sample's
    valid rows only); calling it returns a bf16 [B, Limg, C] prediction with padded rows zero, like a bf16 model."""

    def __init__(self, net, dtype, device):
        self.net, self.dtype, self.device = net, dtype, torch.device(device)

    def _cast(self, v):
        return v.to(self.device, self.dtype) if torch.is_tensor(v) and v.is_floating_point() else (
            v.to(self.device) if torch.is_tensor(v) else v)

    def predict(self, **kw):
        flux = "pooled_projections" in kw
        if flux:  # a bf16 FLUX model multiplies timestep / guidance by 1000 in bf16 (transformer_flux.py:707-710)
            for k in ("timestep", "guidance"):
                if kw.get(k) is not None:
                    kw[k] = (kw[k].to(BF) * 1000).float() / 1000
        hs, enc = kw["hidden_states"], kw["encoder_hidden_states"]
        shapes, mask = kw.get("img_shapes"), kw.get("encoder_hidden_states_mask")
        outs = []
        for b in range(hs.shape[0]):
            n, txt = hs.shape[1], enc.shape[1]
            one = {k: v for k, v in kw.items() if k in ("img_ids", "txt_ids")}
            if shapes is not None:
                sh = shapes[b] if isinstance(shapes[0][0], (list, tuple)) else shapes
                sh = [tuple(s) for s in sh]
                n = sum(f * h * w for f, h, w in sh)
                if mask is not None:
                    txt = int(mask[b].sum())
                    one["encoder_hidden_states_mask"] = mask[b:b + 1, :txt]
                one.update(img_shapes=[sh], txt_seq_lens=[txt])
            one.update(hidden_states=hs[b:b + 1, :n], encoder_hidden_states=enc[b:b + 1, :txt], timestep=kw["timestep"][b:b + 1])
            for k in ("pooled_projections", "guidance"):
                if kw.get(k) is not None:
                    one[k] = kw[k][b:b + 1]
            one = {k: self._cast(v) for k, v in one.items()}
            with torch.no_grad(), lg.eager_sdpa() if self.device.type == "cuda" and self.dtype == BF else contextlib.nullcontext():
                outs.append(self.net(**one)[0][0])
        return outs

    def __call__(self, **kw):
        hs = kw["hidden_states"]
        outs = self.predict(**kw)
        res = torch.zeros(hs.shape[0], hs.shape[1], outs[0].shape[-1], device=self.device, dtype=BF)
        for b, o in enumerate(outs):
            res[b, :o.shape[0]] = o.to(BF)
        return (res,)


def _oracle(m, dtype, dev):
    from oracle import streamed
    return OracleModule(streamed.streamed_oracle(m, dtype, dev), dtype, dev)


def _drop_inference_state(m, dev):
    """Frees the training workspace, every inference workspace and every inference graph (before the oracle runs)."""
    m.set_activation_memory_limit(None)
    m._infer_graphs.clear()
    m._infer_ws.clear()
    m._ws = m._ws_key = None
    dc._free(dev)


def _timed(res, tag, dev, fn):
    dc._peak_reset(dev)
    t0 = time.time()
    out = fn()
    dc._sync(dev)
    res.setdefault("seconds", {})[tag] = round(time.time() - t0, 1)
    res.setdefault("peak_gb", {})[tag] = dc._peak_gb(dev)
    return out


# ------------------------------------------------------------------------------------------------------------ A. forward vs fp64
def forward_check(m, kw, n_target, n_rows, dev, res, fail, corrupt=None):
    """kw: the module forward's kwargs; n_target / n_rows: per sample, its target tokens and its valid image rows (target + controls).
    corrupt = (sample, band, factor): scales one band of the fused prediction before the comparison (to show that the check sees it)."""
    B = len(n_rows)

    def fused():
        with torch.no_grad():
            outs = [m(**kw)[0] for _ in range(3)]  # eager, capture, replay
        with torch.enable_grad():
            grad_path = m(**kw)[0].detach()
        return outs, grad_path
    (eager, _, pred), grad_path = _timed(res, "fused", dev, fused)
    res["graphs_captured"] = m._infer_graphs.captured()
    if dev.type == "cuda" and res["graphs_captured"] != 1:
        fail.append(f"the compared forward was not a graph replay ({res['graphs_captured']} graphs captured)")
    res["replay_equals_eager"] = same_bits(pred, eager)
    res["nograd_equals_grad_enabled"] = same_bits(pred, grad_path)
    if not res["replay_equals_eager"]:
        fail.append(f"replay vs eager forward: max |diff| {float((pred.float() - eager.float()).abs().max()):.3e}")
    if not res["nograd_equals_grad_enabled"]:
        fail.append(f"no-grad vs grad-enabled forward: max |diff| {float((pred.float() - grad_path.float()).abs().max()):.3e}")
    pred = pred.to("cpu", F64)
    pad = max(float(pred[b, n_rows[b]:].abs().max()) if n_rows[b] < pred.shape[1] else 0.0 for b in range(B))
    res["padded_rows_max_abs"] = pad
    if pad != 0.0:
        fail.append(f"padded rows: max |pred| {pad!r}, not zero")
    if corrupt is not None:
        b, k, f = corrupt
        pred[b, k * BAND:(k + 1) * BAND] *= f
    del eager, grad_path
    _drop_inference_state(m, dev)

    ref = {}
    for dt, tag in ((F64, "oracle_fp64"), (BF, "oracle_bf16")):
        def run():
            o = _oracle(m, dt, dev)
            out = [p.to("cpu", F64) for p in o.predict(**kw)]
            del o
            dc._free(dev)
            return out
        ref[dt] = _timed(res, tag, dev, run)
    p64, p16 = ref[F64], ref[BF]
    res["samples"] = []
    for b in range(B):
        nt, nr = n_target[b], n_rows[b]
        e_f, e_16 = rel_l2(pred[b, :nt], p64[b][:nt]), rel_l2(p16[b][:nt], p64[b][:nt])
        row = dict(rel_fused=e_f, rel_bf16=e_16, ratio=round(e_f / max(e_16, 1e-30), 3))
        if not e_f <= PRED_RATIO * e_16 + PRED_FLOOR:
            fail.append(f"sample {b}: rel {e_f:.3e} (bf16 eager {e_16:.3e})")
        worst = None
        for k in range((nr + BAND - 1) // BAND):
            sl = slice(k * BAND, min((k + 1) * BAND, nr))
            bf, b16 = rel_l2(pred[b, sl], p64[b][sl]), rel_l2(p16[b][sl], p64[b][sl])
            if not bf <= BAND_RATIO * b16 + BAND_FLOOR:
                fail.append(f"sample {b} band {k}: rel {bf:.3e} (bf16 eager {b16:.3e})")
            if worst is None or bf / max(b16, 1e-30) > worst["ratio"]:
                worst = dict(band=k, rows=[sl.start, sl.stop], rel_fused=bf, rel_bf16=b16, ratio=round(bf / max(b16, 1e-30), 3))
        row["bands"], row["worst_band"] = (nr + BAND - 1) // BAND, worst
        res["samples"].append(row)


# ------------------------------------------------------------------------------------------------------------ B. sampling loops
def sampler_check(m, emb, family, dev, res, fail):
    from qflux_b200 import sampler
    run = sampler.sample_qwen if family == "qwen" else sampler.sample_flux
    m._infer_graphs.clear()
    out = {}
    r = res["sampler"] = dict(steps=int(emb["num_inference_steps"]), true_cfg_scale=emb["true_cfg_scale"])
    out["fused"] = _timed(r, "fused", dev, lambda: run(m, emb).to("cpu", F64))
    r["graphs_captured"] = m._infer_graphs.captured()
    if dev.type == "cuda" and r["graphs_captured"] != 2:
        fail.append(f"sampler: {r['graphs_captured']} inference graphs captured, expected 2 (prompt and negative prompt)")
    _drop_inference_state(m, dev)
    for dt, tag in ((F64, "oracle_fp64"), (BF, "oracle_bf16")):
        def go():
            o = _oracle(m, dt, dev)
            x = run(o, emb).to("cpu", F64)
            del o
            dc._free(dev)
            return x
        out[tag] = _timed(r, tag, dev, go)
    r["samples"] = []
    for b in range(out["fused"].shape[0]):
        e_f, e_16 = rel_l2(out["fused"][b], out["oracle_fp64"][b]), rel_l2(out["oracle_bf16"][b], out["oracle_fp64"][b])
        r["samples"].append(dict(rel_fused=e_f, rel_bf16=e_16, ratio=round(e_f / max(e_16, 1e-30), 3)))
        if not e_f <= SAMPLER_RATIO * e_16 + SAMPLER_FLOOR:
            fail.append(f"sampler sample {b}: rel {e_f:.3e} (bf16 eager {e_16:.3e})")


def _rn(g, *s):
    return torch.randn(*s, generator=g)


def sampler_batch(family, B, hw, T, T_neg, J, Pp=None, steps=SAMPLER_STEPS, seed=17):
    """Initial noise, control latents and prompt / negative prompt embeddings of a true-CFG sampling loop at latent-patch shape hw."""
    from qflux_b200.train_step import FluxKontextStep
    g = torch.Generator().manual_seed(seed)
    h, w = hw
    L = h * w
    e = dict(latents=_rn(g, B, L, 64).to(BF), control_latents=_rn(g, B, L, 64).to(BF), num_inference_steps=steps)
    if family == "qwen":
        e.update(prompt_embeds=(_rn(g, B, T, J) * 3).to(BF), prompt_embeds_mask=torch.ones(B, T, dtype=torch.int64),
                 negative_prompt_embeds=(_rn(g, B, T_neg, J) * 3).to(BF), negative_prompt_embeds_mask=torch.ones(B, T_neg, dtype=torch.int64),
                 img_shapes=[[(1, h, w), (1, h, w)]] * B, true_cfg_scale=CFG_QWEN)
    else:
        e.update(latent_ids=FluxKontextStep.latent_image_ids(h, w, "cpu", 0.0), control_ids=FluxKontextStep.latent_image_ids(h, w, "cpu", 1.0),
                 pooled_prompt_embeds=_rn(g, B, Pp).to(BF), prompt_embeds=_rn(g, B, T, J).to(BF), text_ids=torch.zeros(T, 3),
                 negative_pooled_prompt_embeds=_rn(g, B, Pp).to(BF), negative_prompt_embeds=_rn(g, B, T_neg, J).to(BF),
                 negative_text_ids=torch.zeros(T_neg, 3), guidance=GUIDANCE, true_cfg_scale=CFG_FLUX)
    return e


# ------------------------------------------------------------------------------------------------------------ A + B: one case
def run_case(config, tiny=None, cfg_update=None, hw=None, B=None, T=None, T_neg=None, sampling=False, corrupt=None, dev=None):
    """config: a bench.CONFIGS name; hw: (h, w) latent patches of every image (default: the config's); B / T: batch and prompt length
    (default: the config's); sampling: also run part B with a negative prompt of T_neg tokens; tiny / cfg_update: reduced model / config
    entries (host wiring test); corrupt: see forward_check."""
    dev = dev or lg._dev()
    t_start = time.time()
    cfg = dict(bench.CONFIGS[config], **(cfg_update or {}))
    if B is not None:
        cfg["B"] = B
    if T is not None:
        cfg["T"] = T
    if hw is not None:
        cfg["imgs"] = [(1, hw[0], hw[1])] * len(cfg["imgs"])
    B, qwen, multires = cfg["B"], cfg["model"] == "qwen", config == "qwen_multires"
    torch.manual_seed(1234)  # bench.py's rank-0 seed, set before the model and the batch are made
    m = dc.build(cfg, dev, tiny)
    emb = bench.make_batch(cfg, config, host=False)
    n_blocks = m.L + (0 if qwen else m.Ls)
    res, fail = dict(config=config, B=B, T=cfg["T"], blocks=n_blocks, r=cfg["r"], device=dc._device(dev)), []
    g = torch.Generator().manual_seed(7)
    x0, ctrl, pe = emb["image_latents"].to(BF), emb["control_latents"].to(BF), emb["prompt_embeds"].to(BF)
    noise = _rn(g, *x0.shape).to(BF)
    on = lambda t: t.to(dev)
    if multires:
        shapes = emb["img_shapes"]
        n_target = [sh[0][1] * sh[0][2] for sh in shapes]
        n_rows = [sum(f * h * w for f, h, w in sh) for sh in shapes]
        Lmax = max(n_rows)
        hs = torch.zeros(B, Lmax, 64, dtype=BF)
        sig = torch.tensor(SIGMA[:B])
        for b in range(B):
            n = n_target[b]
            noisy = ((1 - sig[b]) * x0[b, :n].float() + sig[b] * noise[b, :n].float()).to(BF)
            hs[b, :n_rows[b]] = torch.cat([noisy, ctrl[b, :n_rows[b] - n]])
        kw = dict(hidden_states=on(hs), timestep=on(sig), encoder_hidden_states=on(pe), encoder_hidden_states_mask=on(emb["prompt_embeds_mask"]),
                  img_shapes=shapes, txt_seq_lens=[cfg["T"]] * B)
    else:
        n = x0.shape[1]
        n_target, n_rows = [n] * B, [n + ctrl.shape[1]] * B
        s = torch.tensor(SIGMA[:B] if qwen else T_FLUX[:B])
        noisy = ((1 - s[:, None, None]) * x0.float() + s[:, None, None] * noise.float()).to(BF)
        hs = on(torch.cat([noisy, ctrl], 1))
        if qwen:
            kw = dict(hidden_states=hs, timestep=on(s), encoder_hidden_states=on(pe),
                      encoder_hidden_states_mask=on(torch.ones(B, cfg["T"], dtype=torch.int64)), img_shapes=emb["img_shapes"],
                      txt_seq_lens=[cfg["T"]] * B)
        else:
            from qflux_b200.train_step import FluxKontextStep
            h, w = cfg["imgs"][0][1:]
            ids = torch.cat([FluxKontextStep.latent_image_ids(h, w, "cpu", 0.0), FluxKontextStep.latent_image_ids(h, w, "cpu", 1.0)])
            kw = dict(hidden_states=hs, timestep=on(s), encoder_hidden_states=on(pe), pooled_projections=on(emb["pooled_prompt_embeds"].to(BF)),
                      img_ids=on(ids), txt_ids=on(emb["text_ids"]), guidance=on(torch.full((B,), GUIDANCE)))
    res["target_tokens"], res["image_rows"] = n_target, n_rows
    forward_check(m, kw, n_target, n_rows, dev, res, fail, corrupt)
    del kw, hs
    if sampling:
        J = m.J
        e = sampler_batch("qwen" if qwen else "flux", B, cfg["imgs"][0][1:], cfg["T"], T_neg, J, getattr(m.config, "pooled_projection_dim", None))
        sampler_check(m, e, "qwen" if qwen else "flux", dev, res, fail)
    res["seconds"]["total"] = round(time.time() - t_start, 1)
    res["fail"] = fail
    return res


# ------------------------------------------------------------------------------------------------------------ C. validation rounds
class _Poisoned:
    """The module with every activation buffer of every inference workspace (the `_fixed_entries` buffers and the saved dicts; not the
    per-shape tables rope / kv_len / txt_len / bands) filled with NaN before each call: a forward that reads an activation it did not
    write in the same call turns its output into NaN.  Host memory with emulated kernels only."""

    def __init__(self, m, names):
        assert m.dev.type != "cuda", "NaN-poisoning runs on host memory with emulated kernels only"
        self.m, self.names, self.device = m, names, m.device

    def poison(self):
        for ws in self.m._infer_ws.values():
            for n in self.names:
                t = ws["loraT"].get(n[1]) if isinstance(n, tuple) else ws.get(n)
                if torch.is_tensor(t) and t.is_floating_point():
                    t.fill_(float("nan"))
            for kind in ("dbl", "sgl"):
                for d in ws.get(kind, ()):
                    for t in d.values():
                        t.fill_(float("nan"))

    def __call__(self, **kw):
        self.poison()
        return self.m(**kw)


def _record_fixed_names(m):
    """Collect the names `_fixed_entries` hands to every workspace the model allocates from now on."""
    names = set()
    orig = m._fixed_entries

    def rec(*a, **k):
        pre, post = orig(*a, **k)
        names.update(n for n, _, _ in pre + post)
        return pre, post
    m._fixed_entries = rec
    return names


def validation_round(m, spec, family, J, Pp, dit=None):
    """One validation round: one B = 1 sampling loop per (hw, T, T_neg) of `spec`, under torch.inference_mode().  Returns the latents."""
    from qflux_b200 import sampler
    run = sampler.sample_qwen if family == "qwen" else sampler.sample_flux
    outs = []
    with torch.inference_mode():
        for i, (hw, T, T_neg) in enumerate(spec):
            outs.append(run(dit or m, sampler_batch(family, 1, hw, T, T_neg, J, Pp, seed=100 + i)).clone())
    return [o.cpu() for o in outs]


def _train_state(m, opt, losses):
    return dict(losses=torch.stack([l.reshape(()) for l in losses]).cpu(), G32=m.G32.cpu().clone(),
                lora={n: p.detach().cpu().clone() for n, p in m.named_parameters()},
                exp_avg=opt.exp_avg.cpu().clone(), exp_avg_sq=opt.exp_avg_sq.cpu().clone())


def validation_case(config, spec, tiny=None, cfg_update=None, poison=False, nudge=None, dev=None):
    """config: a bench.CONFIGS name (its model and training batch); spec: the round's samples [(hw, T, T_neg)]; poison: the second
    round runs through `_Poisoned` (host only); nudge: a LoRA parameter name whose first element model B gets one ulp larger (to show
    that the check sees it)."""
    from qflux_b200.optim import FusedLoraAdamW
    from qflux_b200.train_step import FluxKontextStep, QwenImageEditStep
    dev = dev or lg._dev()
    t_start = time.time()
    cfg = dict(bench.CONFIGS[config], **(cfg_update or {}))
    qwen = cfg["model"] == "qwen"
    family = "qwen" if qwen else "flux"
    shapes = {(T, hw[0] * hw[1] * 2) for hw, T, Tn in spec} | {(Tn, hw[0] * hw[1] * 2) for hw, T, Tn in spec}
    res, fail = dict(config=config, B=cfg["B"], round_samples=len(spec), round_shapes=len(shapes), device=dc._device(dev)), []
    det0 = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        states = {}
        for model in ("A", "B"):
            torch.manual_seed(1234)
            m = dc.build(cfg, dev, tiny)
            emb = bench.make_batch(cfg, config, host=False)
            if model == "B" and nudge is not None:
                p = dict(m.named_parameters())[nudge].data
                first = (0,) * p.ndim
                p[first] = (p[first].reshape(1).clone().view(torch.int16) + 1).view(BF)[0]  # the next bf16 value up
            names = _record_fixed_names(m)
            J, Pp = m.J, getattr(m.config, "pooled_projection_dim", None)
            opt = FusedLoraAdamW(m, **ADAMW)
            step = (QwenImageEditStep if qwen else FluxKontextStep)(m, "mse", max_grad_norm=ADAMW["max_grad_norm"])
            g = torch.Generator().manual_seed(7)
            noises = [_rn(g, *emb["image_latents"].shape).to(BF) for _ in range(6)]
            u = lambda i: torch.tensor([STEP_U[(i + b) % 6] for b in range(cfg["B"])])
            losses = []

            def train(i):
                kw = dict(noise=noises[i], u=u(i)) if qwen else dict(noise=noises[i], t=u(i))
                losses.append(step.train_step(emb, opt, **kw))
            tag = lambda s: f"{model}_{s}"
            _timed(res, tag("steps_1_3"), dev, lambda: [train(i) for i in range(3)])
            if model == "A":
                graphs = [e["graph"] for e in step._graphs.entries.values() if isinstance(e, dict)]
                r1 = _timed(res, "round_1", dev, lambda: validation_round(m, spec, family, J, Pp))
                res["infer_graphs_after_round"] = m._infer_graphs.captured()
                res["infer_workspaces_after_round"] = len(m._infer_ws)
                dit2 = _Poisoned(m, names) if poison else None
                r2 = _timed(res, "round_2", dev, lambda: validation_round(m, spec, family, J, Pp, dit2))
                m.use_cuda_graph_inference = False
                r3 = _timed(res, "round_no_graphs", dev, lambda: validation_round(m, spec, family, J, Pp))
                m.use_cuda_graph_inference = True
                res["round_repeat_identical"] = all(same_bits(a, b) for a, b in zip(r1, r2))
                res["round_graphs_vs_eager_identical"] = all(same_bits(a, b) for a, b in zip(r1, r3))
                res["round_finite"] = all(bool(torch.isfinite(o.float()).all()) for o in r1 + r2 + r3)
                if not res["round_repeat_identical"]:
                    fail.append("validation: the repeated round differs from the first" + (" (NaN-poisoned workspaces)" if poison else ""))
                if not res["round_graphs_vs_eager_identical"]:
                    fail.append("validation: the round with CUDA graphs differs from the round without")
                if not res["round_finite"]:
                    fail.append("validation: a round's latents are not finite")
            _timed(res, tag("steps_4_6"), dev, lambda: [train(i) for i in range(3, 6)])
            if model == "A" and dev.type == "cuda":
                after = [e["graph"] for e in step._graphs.entries.values() if isinstance(e, dict)]
                res["train_graph_kept"] = len(graphs) == 1 and len(after) == 1 and after[0] is graphs[0]
                if not res["train_graph_kept"]:
                    fail.append(f"validation: the training step's graph was recorded again ({len(graphs)} before, {len(after)} after)")
            states[model] = _train_state(m, opt, losses)
            del m, opt, step, emb, losses
            dc._free(dev)
        a, b = states["A"], states["B"]
        diff = [k for k in ("losses", "G32", "exp_avg", "exp_avg_sq") if not same_bits(a[k], b[k])]
        diff += [n for n in a["lora"] if not same_bits(a["lora"][n], b["lora"][n])]
        res["state_identical"] = not diff
        res["losses"] = a["losses"].tolist()
        res["lora_tensors"] = len(a["lora"])
        if diff:
            fail.append(f"validation: training state after step 6 differs from the run without a round: {len(diff)} tensors, first {diff[:3]}")
    finally:
        torch.use_deterministic_algorithms(det0)
    res["seconds"]["total"] = round(time.time() - t_start, 1)
    res["fail"] = fail
    return res


QWEN_ROUND = [((H832, W832), 352, 64), ((W832, H832), 200, 96), ((32, 32), 128, 40), ((24, 40), 300, 77)]
FLUX_ROUND = [((H832, W832), 512, 256), ((W832, H832), 384, 128), ((32, 32), 512, 64), ((24, 40), 200, 300)]


# ------------------------------------------------------------------------------------------------------------ cases
def qwen_edit(**k):
    """Qwen-Image-Edit, 60 blocks, the benchmark shape: B = 1, T = 352, target + control 32 x 32 patches (512^2), r = 16.
    H100 80GB HBM3, 700 W: prediction fused 2.106e-2, bf16 eager 2.104e-2 (ratio 1.001); worst of 16 bands 1.019 (band 13).
    fp64 oracle 12.8 s, peak 44.1 GB; fused with the grad-enabled forward's training workspace 50.7 GB."""
    return run_case("qwen_edit", **k)


def qwen_edit_832x576(**k):
    """Qwen-Image-Edit, 60 blocks, the reference configs' 832 x 576 training size: B = 2, r = 16, 52 x 36 = 1872 patches per image, so a
    sample's 3744 image rows are no multiple of 64, 128 or 256.  The prompt has T = 352 tokens (the benchmark's) and the sampling loop's
    negative prompt T = 64, a short negative prompt that makes the two CFG shapes differ.
    H100 80GB HBM3, 700 W: prediction per sample fused / bf16 eager 2.064e-2 / 2.063e-2 and 2.245e-2 / 2.252e-2 (ratios 1.001, 0.997);
    worst of 30 bands 1.013 and 1.008.  Sampling (3 steps, true CFG 4.0): latents 5.11e-2 / 5.09e-2 and 5.09e-2 / 5.11e-2 (1.003,
    0.995).  The streamed fp64 forward of the two samples (S = 4096) takes 16.6 s at 48.7 GB peak, the fp64 sampling loop 33.5 s;
    the fused forwards peak at 74.4 GB, with the training workspace of the grad-enabled call (B = 2, S = 4096)."""
    return run_case("qwen_edit", **{**dict(B=2, hw=(H832, W832), T=QWEN_T, T_neg=QWEN_T_NEG, sampling=True), **k})


def flux_kontext_832x576(**k):
    """FLUX-Kontext, 19 double + 38 single blocks, YAML target set (every block Linear, the AdaLN linears and x_embedder) at r = 32,
    guidance 3.5, B = 2, T = 512, 832 x 576 (1872 patches per image); the sampling loop's negative prompt has T = 256.
    H100 80GB HBM3, 700 W: prediction per sample fused / bf16 eager 1.877e-2 / 1.919e-2 and 1.924e-2 / 1.960e-2 (0.978, 0.982);
    worst of 30 bands 0.991 and 0.999.  Sampling (3 steps, true CFG 2.5): latents 1.52e-2 / 1.54e-2 and 1.41e-2 / 1.47e-2 (0.988,
    0.961).  fp64 forward (S = 4256) 15.3 s at 35.6 GB peak, fp64 sampling loop 34.6 s; fused peak 72.0 GB."""
    return run_case("flux_kontext", **{**dict(B=2, hw=(H832, W832), T=FLUX_T, T_neg=FLUX_T_NEG, sampling=True), **k})


def qwen_plus(**k):
    """Qwen-Image-Edit-2509: target + 2 controls (frame offsets 0, 1, 2), T = 448, B = 1.
    H100 80GB HBM3, 700 W: prediction fused 2.095e-2, bf16 eager 2.092e-2 (1.002); worst of 24 bands 1.019 (band 0)."""
    return run_case("qwen_plus_sharded", **k)


def qwen_multires(**k):
    """Qwen-Image-Edit multi-resolution, bench.py's batch: one 512^2 and one 320^2 sample padded to the longer, through the module
    forward with per-sample img_shapes and the prompt mask; the padded rows must come back exactly zero.
    H100 80GB HBM3, 700 W: prediction fused / bf16 eager 2.118e-2 / 2.105e-2 and 2.317e-2 / 2.299e-2 (1.006, 1.008); worst of 16
    and 7 bands 1.020 and 1.023; padded rows exactly zero."""
    return run_case("qwen_multires", **k)


def validation_qwen_edit(**k):
    """Validation between training steps, Qwen-Image-Edit at the benchmark's training shape, 4 round samples: 832 x 576, 576 x 832,
    512^2 and 384 x 640, prompt / negative prompt lengths 352 / 64, 200 / 96, 128 / 40 and 300 / 77.
    H100 80GB HBM3, 700 W: everything bit-identical, 8 inference graphs and 3 workspaces held after a round.  One round (3 steps x
    2 CFG calls x 4 samples) 4.0 s with graphs (3.9 s repeated), 2.6 s without (each shape meets only 3 calls, so capturing does not
    pay off here); peak 50.6 GB after the training steps, 56.4 GB after the rounds."""
    return validation_case("qwen_edit", **{"spec": QWEN_ROUND, **k})


def validation_flux_kontext(**k):
    """Validation between training steps, FLUX-Kontext (YAML targets, B = 2) at the benchmark's training shape, 4 round samples: 832 x
    576, 576 x 832, 512^2 and 384 x 640, prompt / negative prompt lengths 512 / 256, 384 / 128, 512 / 64 and 200 / 300.
    H100 80GB HBM3, 700 W: everything bit-identical, 8 inference graphs and 3 workspaces held after a round.  One round 4.2 s with
    graphs, 2.9 s without; peak 52.9 GB after the training steps, 62.1 GB after the rounds."""
    return validation_case("flux_kontext", **{"spec": FLUX_ROUND, **k})


CASES = {f.__name__: f for f in (qwen_edit, qwen_edit_832x576, flux_kontext_832x576, qwen_plus, qwen_multires,
                                  validation_qwen_edit, validation_flux_kontext)}

if __name__ == "__main__":
    main(CASES, os.path.abspath(__file__), "infer_check.log", timeout=1800)
