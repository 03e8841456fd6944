"""What the bit-reproducible data-parallel gradient sum costs (qfx_dp_reduce_det and sharding.GradExchange).

    python tools/dp_reduce_bench.py            (prints one JSON line; needs a GPU, refuses to run without one)

kernel      qfx_dp_reduce_det over W = 2, 4, 8 local fp32 source buffers into a separate destination, at the flat LoRA-gradient sizes of
            Qwen-Image-Edit r = 16 (23,592,960 elements) and FLUX-Kontext with the YAML targets at r = 32 (171,935,744): ms per call from
            CUDA events over ITERS launches after WARMUP, bytes moved ((W + 1) * 4 * n: every source read once, the destination written
            once) over that time, and that rate as a share of the H100 SXM data sheet's 3.35 TB/s.  On one GPU the sources are local, so
            this is the HBM cost of the reduce-scatter's kernel, not an NVLink number.
exchange    with >= 2 GPUs, one process per GPU (NCCL group): GradExchange.all_reduce against dist.all_reduce on the same FLUX-sized
            buffer, and a full-depth FLUX-Kontext B = 2 training step (bench.py's model and batch, FusedLoraAdamW, flag on) with each of
            the two exchanges.  With one GPU these numbers are reported as "not measured".
The card's name and power limit are read in the same run.
"""
import json
import os
import socket
import subprocess
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "qwen-image-finetune_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

SIZES = {"qwen_edit_r16": 23_592_960, "flux_kontext_yaml_r32": 171_935_744}
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet (700 W card)
WARMUP, ITERS, STEPS = 5, 50, 5


def _gpu():
    import torch
    try:
        pl = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the number is still valid; say why the power limit is missing
        pl = f"unavailable ({type(e).__name__})"
    return dict(gpu=torch.cuda.get_device_name(), power_limit=pl)


def _events_ms(fn, iters, warmup):
    import torch
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def kernel():
    import torch
    from qflux_b200 import lib
    out = {}
    for name, n in SIZES.items():
        for w in (2, 4, 8):
            srcs = [torch.randn(n, device="cuda") for _ in range(w)]
            dst = torch.empty(n, device="cuda")
            ms = _events_ms(lambda: lib.dp_reduce_det(srcs, dst), ITERS, WARMUP)
            nbytes = (w + 1) * 4 * n
            out[f"{name}_W{w}"] = dict(elements=n, ms=round(ms, 4), bytes=nbytes, tb_per_s=round(nbytes / ms / 1e9, 3),
                                       share_of_3_35_tb_s=round(nbytes / ms / 1e9 / (HBM_BYTES_PER_S / 1e12), 3))
            del srcs, dst
            torch.cuda.empty_cache()
    return out


class _Flat:
    """The part of a model GradExchange uses: the flat gradient and its device."""

    def __init__(self, n, dev):
        import torch
        self.dev, self.G32 = dev, torch.randn(n, device=dev)
        self._grad_exchange = None


def _exchange_worker(rank, world, port, out):
    import datetime
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    torch.use_deterministic_algorithms(True)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("nccl", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300),
                            device_id=torch.device("cuda", rank))
    try:
        from qflux_b200.sharding import GradExchange
        dev = torch.device("cuda", rank)
        n = SIZES["flux_kontext_yaml_r32"]
        flat = _Flat(n, dev)
        ex = GradExchange.for_model(flat)
        res = dict(world=world, exchange_ms=_events_ms(ex.all_reduce, 20, 3),
                   nccl_all_reduce_ms=_events_ms(lambda: dist.all_reduce(flat.G32), 20, 3))
        ex.close()
        del flat
        torch.cuda.empty_cache()
        res.update(_flux_step_with_each_exchange(dev))
        if rank == 0:
            with open(out, "w") as f:
                json.dump(res, f)
    finally:
        dist.destroy_process_group()


def _flux_step_with_each_exchange(dev):
    import torch
    import bench
    from qflux_b200.optim import FusedLoraAdamW
    from qflux_b200.train_step import FluxKontextStep
    cfg = bench.CONFIGS["flux_kontext"]
    torch.manual_seed(0)
    m = bench.build_flux(dev, cfg, 1.0)
    host = bench.make_batch(cfg, "flux_kontext", host=True)
    step, opt = FluxKontextStep(m, "mse", max_grad_norm=1.0), FusedLoraAdamW(m, lr=1e-4)
    res = {}
    for name, exchange in (("peer_fixed_order", None), ("nccl", False)):
        if exchange is False:
            m.close()
        m._grad_exchange = exchange  # False: GradExchange.for_model declines and _sync_and_step runs dist.all_reduce
        ms = _events_ms(lambda: step.train_step(host, opt), STEPS, 3)
        res[f"flux_kontext_b2_step_ms_{name}"] = round(ms, 2)
    return res


def exchange():
    import torch
    import torch.multiprocessing as mp
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        return dict(exchange="not measured (one GPU)", nccl_all_reduce="not measured (one GPU)", flux_kontext_b2_step="not measured (one GPU)")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    out = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"dp_reduce_bench_{os.getpid()}.json")
    mp.spawn(_exchange_worker, args=(world, port, out), nprocs=world, join=True)
    with open(out) as f:
        return json.load(f)


if __name__ == "__main__":
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("dp_reduce_bench: needs a CUDA device (nothing is estimated without one)")
    print(json.dumps(dict(**_gpu(), kernel=kernel(), exchange=exchange())))
