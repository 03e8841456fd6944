"""Cost of sharded NF4 / FP8 frozen weights, two processes sharing one GPU (gloo group, peer gather through CUDA IPC):

    python tools/sharded_quant_bench.py [out.json]

Prints one JSON object (and writes it to out.json when given):
  * card: the GPU's name and power limit, read in the same call;
  * resident: per rank, the frozen block bytes of Qwen-Image-Edit at full depth (60 blocks), exact from the allocation sizes:
    unsharded codes, this rank's shard, the staging slots and the bf16 ring slots;
  * fill: one double-block fill at full width, timed by rank 0 alone (rank 1 waits on the host): expansion from resident codes
    against gather + expansion from the shards, and the no-grad forward of one bf16 double block at Qwen-Image-Edit B = 1 (the
    difference of a 6- and a 2-block forward, over 4).  Both ranks are on one GPU, so the "peer" pull is a copy within one HBM,
    not an NVLink transfer;
  * step: full-depth Qwen-Image-Edit B = 1 fused training step (forward + loss + backward through the CUDA-graph cache), both ranks
    stepping at once on one GPU, unsharded against sharded, NF4 and FP8, each rank's training workspace capped at 12 GiB (the same
    recompute plan for both layouts).  The two processes time-share the GPU: these are not multi-GPU figures.
CUDA events; 3 warm-up calls (capture included) and the median of the timed ones.
"""
import json
import os
import socket
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "qwen-image-finetune_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

WORLD = 2
ACTIVATION_LIMIT = 12 << 30  # per rank: two full-depth models and their workspaces share one 80 GB card


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else f"nvidia-smi failed: {q.stderr.strip()}"


def _median_ms(fn, iters, warmup=3):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2]


def _bytes(rings, attr):
    return sum(getattr(r, attr).numel() * getattr(r, attr).element_size() for r in rings if r is not None)


def _store_bytes(m):
    return sum(t.numel() * t.element_size() for v in list(m._nf4_store.values()) + list(m._fp8_store.values())
               for t in (v if isinstance(v, tuple) else (v,)))


def _flush():
    """Return the memory of the models the caller has dropped to the device (the other rank needs it too)."""
    import gc
    import torch
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _fill_times(rank, cfg):
    """rank 0 times one double-block fill of each ring kind and one bf16 double-block forward; rank 1 only takes part in the
    collectives."""
    import torch
    import torch.distributed as dist
    import fp8_check
    import nf4_check
    import sharded_quant_check as sqc
    out = {}
    small = dict(cfg, blocks=4)
    for fmt in ("nf4", "fp8"):
        u, s = sqc.build("qwen", fmt, small), sqc.build("qwen", fmt, small)
        s.shard_frozen_weights(gather="peer")
        dist.barrier()
        if rank == 0:
            for tag, ring in (("resident_expand", u._expand_rings[0]), ("gather_expand", s._sharded)):
                k = [0]

                def fill():
                    k[0] += 1
                    ring._fill(k[0] & 1, k[0] % ring.L)
                out[f"{fmt}_{tag}_ms"] = round(_median_ms(fill, 20), 3)
            out[f"{fmt}_code_bytes_per_block"] = _store_bytes(u) // u.L
        dist.barrier()
        u.close()
        s.close()
        del u, s
        _flush()
    if rank == 0:  # a bf16 double block's no-grad forward: (6-block forward - 2-block forward) / 4, graph-replayed
        b = nf4_check._fixed(nf4_check.device_batch(cfg, "qwen_edit"), "qwen")
        x = torch.cat([b["noise"], b["control_latents"]], 1)
        ts = torch.full((1,), 0.5, device="cuda")
        fwd = {}
        for n in (2, 6):
            m = fp8_check.build("qwen", dict(cfg, blocks=n), fp8=False)
            with torch.no_grad():
                fwd[n] = _median_ms(lambda: m(hidden_states=x, encoder_hidden_states=b["prompt_embeds"], timestep=ts,
                                              img_shapes=b["img_shapes"]), 20)
            del m
            _flush()
        out["bf16_block_forward_ms"] = round((fwd[6] - fwd[2]) / 4, 3)
    dist.barrier()
    return out


def _step_times(rank, cfg):
    import torch
    import torch.distributed as dist
    import nf4_check
    import sharded_quant_check as sqc
    b = sqc.rank_batch("qwen", "qwen_edit", cfg, rank)
    out, resident = {}, {}
    for fmt in ("nf4", "fp8"):
        for sharded in (False, True):
            for r in range(WORLD):  # one rank at a time: the random fill's temporaries are as large as a code stack
                if r == rank:
                    m = sqc.build("qwen", fmt, cfg)
                    _flush()
                dist.barrier()
            store = _store_bytes(m)
            if sharded:
                m.shard_frozen_weights(gather="peer")
            rings = [r for r in m._expand_rings if r is not None]
            tag = f"{fmt}_{'sharded' if sharded else 'unsharded'}"
            resident[tag] = dict(codes_gb=round((_bytes(rings, "shard") if sharded else store) / 1e9, 3),
                                 staging_gb=round(_bytes(rings, "stage") / 1e9, 3) if sharded else 0.0,
                                 bf16_slots_gb=round(_bytes(rings, "gbuf") / 1e9, 3))
            m.set_activation_memory_limit(ACTIVATION_LIMIT)
            step = nf4_check._step(m, "qwen")
            args = step._prepare(b, b["noise"], b["u"])
            dist.barrier()
            out[tag + "_ms"] = round(_median_ms(lambda: step._graphs.run(m, step._run, args, tag=False), 5), 2)
            out[tag + "_graphs"] = step._graphs.captured()
            out[tag + "_recomputed_blocks"] = len(m.activation_plan.recompute)
            dist.barrier()
            m.close()
            del step, args, m, rings
            _flush()
    return out, resident


def _worker(rank, port, out):
    import torch
    import torch.distributed as dist
    import bench
    torch.cuda.set_device(0)  # both ranks share the one GPU
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=WORLD)
    try:
        cfg = dict(bench.CONFIGS["qwen_edit"], B=1)
        res = dict(rank=rank, fill=_fill_times(rank, cfg))
        res["step"], res["resident"] = _step_times(rank, cfg)
        torch.save(res, f"{out}.{rank}")
    finally:
        dist.destroy_process_group()


def main():
    import torch
    import torch.multiprocessing as mp
    card = _card()
    with tempfile.TemporaryDirectory() as d:
        out = os.path.join(d, "res")
        mp.spawn(_worker, args=(_free_port(), out), nprocs=WORLD, join=True)
        res = [torch.load(f"{out}.{r}") for r in range(WORLD)]
    result = dict(card=card, torch_gpu=torch.cuda.get_device_name(0), world=WORLD, shared_gpu=True,
                  workload="Qwen-Image-Edit LoRA r=16, 512x512, B=1, 60 blocks (fill: 4-block model of the same width)",
                  resident_per_rank=res[0]["resident"], fill=res[0]["fill"], step_ms=[r["step"] for r in res])
    print(json.dumps(result))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
