"""GPU checks of sharded NF4 / FP8 frozen weights (`shard_frozen_weights()` of an NF4- or FP8-resident model, sharding.ShardedCodes),
one subprocess per case:

    python tools/sharded_quant_check.py [case ...]

  qwen_nf4 / qwen_fp8 / flux_nf4 / flux_fp8
      two processes sharing one GPU (gloo group, peer gather through CUDA IPC), reduced-depth full-width models (Qwen-Image-Edit
      4 blocks; FLUX-Kontext 2 double + 3 single blocks, YAML targets), under torch.use_deterministic_algorithms(True).  On each
      rank, against an unsharded model of the same format held in the same process, on the rank's own batch:
        * the eager fused step: loss, prediction and the whole flat LoRA gradient bit for bit;
        * the step through the CUDA-graph cache: the entry is a captured graph (not "warm"), no capture warning, and every replay
          equals the eager step bit for bit;
        * three train_step()s with FusedLoraAdamW (gradients exchanged between the ranks): losses and LoRA weights bit for bit;
        * Qwen: the no-grad forward of the sampler, eager and replayed, bit for bit.
"""
import os
import socket
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "qwen-image-finetune_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import harness  # noqa: E402

WORLD = 2


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _cfg(family):
    import bench
    if family == "qwen":
        return "qwen_edit", dict(bench.CONFIGS["qwen_edit"], B=1, blocks=4)
    return "flux_kontext", dict(bench.CONFIGS["flux_kontext"], B=1, nd=2, ns=3)


def build(family, fmt, cfg):
    import fp8_check
    import nf4_check
    return nf4_check.build(family, cfg) if fmt == "nf4" else fp8_check.build(family, cfg)


def rank_batch(family, name, cfg, rank):
    """The bench batch of `name` with noise and timestep of this rank (every rank trains on its own data)."""
    import torch
    import nf4_check
    b = nf4_check._fixed(nf4_check.device_batch(cfg, name), family)
    g = torch.Generator(device="cuda").manual_seed(100 + rank)
    b["noise"] = torch.randn(b["image_latents"].shape, device="cuda", generator=g).bfloat16()
    t = 0.25 + 0.5 * rank / WORLD
    if family == "qwen":
        b["u"] = torch.tensor([t] * b["image_latents"].shape[0])
    else:
        b["timestep"] = torch.full((b["image_latents"].shape[0],), t, device="cuda", dtype=torch.bfloat16)
    return b


def _args(step, family, b):
    return step._prepare(b, b["noise"], b["u"] if family == "qwen" else b["timestep"])


def _bits(a, b):
    import torch
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def _same(x, y):
    return x[0] == y[0] and _bits(x[1], y[1]) and _bits(x[2], y[2])


def _lora(m):
    import torch
    return torch.cat([p.detach().float().reshape(-1) for _, p in sorted(m._lora_params.items())])


def _worker(rank, family, fmt, port, out):
    import warnings
    import torch
    import torch.distributed as dist
    import nf4_check
    from qflux_b200.optim import FusedLoraAdamW
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.cuda.set_device(0)  # both ranks share the one GPU
    torch.use_deterministic_algorithms(True)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=WORLD)
    try:
        name, cfg = _cfg(family)
        u, s = build(family, fmt, cfg), build(family, fmt, cfg)
        store = sum(t.numel() * t.element_size() for v in list(s._nf4_store.values()) + list(s._fp8_store.values())
                    for t in (v if isinstance(v, tuple) else (v,)))
        s.shard_frozen_weights(gather="peer")
        rings = [r for r in (s._sharded, s._sharded_s) if r is not None]
        res = dict(rank=rank, gather=[r.gather for r in rings], store_bytes=store,
                   shard_bytes=sum(r.shard.numel() for r in rings), stage_bytes=sum(r.stage.numel() for r in rings))
        b = rank_batch(family, name, cfg, rank)
        # eager step
        ref = nf4_check._one_step(u, family, b)
        got = nf4_check._one_step(s, family, b)
        res["eager_equal"] = _same(ref, got)
        # graph-cache step: warm (eager), capture + replay, replay
        step = nf4_check._step(s, family)
        args = _args(step, family, b)
        outs = []
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            for _ in range(3):
                outs.append((float(step._graphs.run(s, step._run, args, tag=False)), s._ws["pred"].clone(), s.G32.clone()))
        res["capture_warnings"] = [str(w.message) for w in caught]
        res["graph_entries"] = [e if isinstance(e, str) else "graph" for e in step._graphs.entries.values()]
        res["graph_failed"] = step._graphs.failed
        res["replays_equal"] = all(_same(o, ref) for o in outs)
        # no-grad forward of the sampler (Qwen)
        if family == "qwen":
            x = torch.cat([b["noise"], b["control_latents"]], 1)
            ts = torch.full((1,), 0.5, device="cuda")
            kw = dict(hidden_states=x, encoder_hidden_states=b["prompt_embeds"], timestep=ts, img_shapes=b["img_shapes"])
            with torch.no_grad():
                f_ref = u(**kw)[0].clone()
                f_got = [s(**kw)[0].clone() for _ in range(3)]
            res["forward_equal"] = all(_bits(f, f_ref) for f in f_got)
            res["forward_graphs"] = s._infer_graphs.captured()
        # three train_steps with gradient exchange, unsharded then sharded (each model exchanges with its twin on the other rank)
        traj = {}
        for tag, m in (("unsharded", u), ("sharded", s)):
            st = nf4_check._step(m, family)
            opt = FusedLoraAdamW(m, lr=1e-3)
            losses = [float(st.train_step(b, opt, b["noise"], b["u"] if family == "qwen" else b["timestep"])) for _ in range(3)]
            traj[tag] = (losses, _lora(m).cpu(), st._graphs.captured())
        res["trajectory_losses"] = traj["sharded"][0]
        res["trajectory_equal"] = traj["sharded"][0] == traj["unsharded"][0] and _bits(traj["sharded"][1], traj["unsharded"][1])
        res["trajectory_graphs"] = traj["sharded"][2]
        u.close()
        s.close()
        torch.save(res, f"{out}.{rank}")
    finally:
        dist.destroy_process_group()


def _case(family, fmt):
    import torch
    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as d:
        out = os.path.join(d, "res")
        mp.spawn(_worker, args=(family, fmt, _free_port(), out), nprocs=WORLD, join=True)
        res = [torch.load(f"{out}.{r}") for r in range(WORLD)]
    for r in res:
        print(r)
        assert r["gather"] == ["peer"] * len(r["gather"]), r
        assert 1 / WORLD <= r["shard_bytes"] / r["store_bytes"] <= 1 / WORLD + 0.01, r
        assert r["eager_equal"], r
        assert not r["capture_warnings"] and not r["graph_failed"] and r["graph_entries"] == ["graph"], r
        assert r["replays_equal"], r
        assert r.get("forward_equal", True) and r.get("forward_graphs", 1) == 1, r
        assert r["trajectory_equal"] and r["trajectory_graphs"] >= 1, r
    assert res[0]["trajectory_losses"] != res[1]["trajectory_losses"], "the ranks train on different batches"
    return dict(gpu=torch.cuda.get_device_name(0), store_mb=round(res[0]["store_bytes"] / 2 ** 20, 1),
                shard_mb=[round(r["shard_bytes"] / 2 ** 20, 1) for r in res], stage_mb=round(res[0]["stage_bytes"] / 2 ** 20, 1),
                losses=[r["trajectory_losses"] for r in res])


CASES = dict(qwen_nf4=lambda: _case("qwen", "nf4"), qwen_fp8=lambda: _case("qwen", "fp8"),
             flux_nf4=lambda: _case("flux", "nf4"), flux_fp8=lambda: _case("flux", "fp8"))

if __name__ == "__main__":
    if len(sys.argv) == 2 and sys.argv[1] in CASES:  # one case in this process (tests/test_sharded_quantized.py)
        print(CASES[sys.argv[1]]())
    else:
        harness.main(CASES, os.path.abspath(__file__), "sharded_quant_check.log")
