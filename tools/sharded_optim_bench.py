"""Replicated vs sharded optimizer state (optim.py shard_state=True), per data-parallel rank: optimizer state bytes, peak memory,
step time (exchange + optimizer) and exchange time, for FusedLoraAdamW and FusedLoraProdigy over the LoRA tables of FLUX-Kontext with
the YAML targets at r = 32 and r = 128 (tools/sharded_optim_check.py members(); the frozen model is not built: two full-depth FLUX
models do not fit one GPU, and the optimizer reads only the flat gradient and the LoRA tensors).

Two processes share one GPU through a gloo group, as two ranks of one host; torch.use_deterministic_algorithms(True), so both modes use
the peer-memory exchange (replicated: sharding.GradExchange.all_reduce; sharded: its reduce-scatter, the norm and Prodigy partial
gathers and the weight all-gather).  Device events; 3 warm-up and 5 timed steps per mode, the two modes alternating step by step in one
process.  This is the two-process-on-one-GPU case: both ranks' kernels and copies share one GPU's SMs and HBM, so it is not a number for
2 separate GPUs.  Prints the result as JSON, and also writes it to the path given.

  python tools/sharded_optim_bench.py [out.json]
"""
import datetime
import json
import os
import socket
import subprocess
import sys
import tempfile

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, ROOT, os.path.join(ROOT, "qwen-image-finetune_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

WARMUP, STEPS = 3, 5


class LoraTables:
    """What the fused optimizers read from a model: the LoRA factors, their flat fp32 gradient, the device."""

    def __init__(self, r):
        import sharded_optim_check as chk
        chk.R, chk.RP = r, 64 * -(-r // 64)
        torch.manual_seed(0)
        ms, n = chk.members()
        self.pairs = [(ms[i][0], ms[i + 1][0], ms[i][1], ms[i + 1][1]) for i in range(0, len(ms), 2)]
        self.G32 = torch.zeros(n, device="cuda")
        self.dev = torch.device("cuda", torch.cuda.current_device())
        self._grad_exchange = None

    def _all_members(self):
        for k, (a, b, ga, gb) in enumerate(self.pairs):
            yield f"m{k}", torch.nn.Parameter(a, requires_grad=False), torch.nn.Parameter(b, requires_grad=False), ga, gb, a.shape[1], b.shape[0]

    def parameters(self):
        for a, b, _, _ in self.pairs:
            yield torch.nn.Parameter(a, requires_grad=False)
            yield torch.nn.Parameter(b, requires_grad=False)

    def close(self):
        if self._grad_exchange:
            self._grad_exchange.close()
        self._grad_exchange = None


def _state_bytes(opt):
    keys = ("exp_avg", "exp_avg_sq", "s", "p0", "state1", "state2", "absmax1", "absmax2", "s1_32", "s2_32")
    return sum(getattr(opt, k).numel() * getattr(opt, k).element_size() for k in keys if hasattr(opt, k))


def _worker(rank, world, port, out):
    torch.cuda.set_device(0)
    torch.use_deterministic_algorithms(True)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=600))
    from qflux_b200.optim import FusedLoraAdamW, FusedLoraProdigy
    from qflux_b200.sharding import GradExchange
    rows = []
    for r in (32, 128):
        for name, cls, kw in (("AdamW", FusedLoraAdamW, dict(lr=1e-4)), ("Prodigy", FusedLoraProdigy, dict(lr=1.0))):
            model = LoraTables(r)
            g = torch.randn(model.G32.numel(), device="cuda", generator=torch.Generator("cuda").manual_seed(rank)) * 1e-4
            res = {}
            for mode in ("replicated", "sharded"):
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                opt = cls(model, shard_state=(mode == "sharded"), **kw)
                res[mode] = dict(opt=opt, state_bytes=_state_bytes(opt), step_ms=[], exchange_ms=[], base=base)
            for it in range(WARMUP + STEPS):
                for mode in ("replicated", "sharded"):
                    opt, rec = res[mode]["opt"], res[mode]
                    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
                    model.G32.copy_(g)
                    torch.cuda.reset_peak_memory_stats()
                    ev[0].record()
                    if mode == "replicated":
                        GradExchange.for_model(model).all_reduce()
                        ev[1].record()
                        opt.step(grad_divisor=world)
                    else:  # the exchange alone, then the whole sharded step
                        opt._exchange.reduce_scatter()
                        opt._exchange.gather_weights()
                        ev[1].record()
                        model.G32.copy_(g)
                        opt.step(grad_divisor=world)
                    ev[2].record()
                    torch.cuda.synchronize()
                    if it >= WARMUP:
                        rec["exchange_ms"].append(ev[0].elapsed_time(ev[1]))
                        rec["step_ms"].append(ev[1].elapsed_time(ev[2]) + (ev[0].elapsed_time(ev[1]) if mode == "replicated" else 0.0))
                        rec["peak_gb"] = torch.cuda.max_memory_allocated() / 1e9
            row = dict(lora=f"FLUX-Kontext YAML r={r}", optimizer=name, rank=rank, grad_elements=model.G32.numel())
            for mode, rec in res.items():
                med = lambda xs: sorted(xs)[len(xs) // 2]
                row[mode] = dict(state_gb=rec["state_bytes"] / 1e9, peak_gb=round(rec["peak_gb"], 3), step_ms=round(med(rec["step_ms"]), 3),
                                 exchange_ms=round(med(rec["exchange_ms"]), 3))
            rows.append(row)
            for rec in res.values():
                del rec["opt"]
            model.close()
            del model, res, g
            torch.cuda.empty_cache()
    torch.save(rows, f"{out}.{rank}")
    dist.destroy_process_group()


def main():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    with tempfile.TemporaryDirectory() as tmp:  # the ranks hand their rows back through files here
        ranks = os.path.join(tmp, "rows")
        mp.spawn(_worker, args=(2, port, ranks), nprocs=2, join=True)
        rows = [row for r in range(2) for row in torch.load(f"{ranks}.{r}")]
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    res = dict(gpu=smi.strip(), case="two processes (ranks) sharing one GPU, peer-memory exchange", warmup=WARMUP, timed_steps=STEPS,
               rows=rows)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
