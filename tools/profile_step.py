"""Run a few fused training steps at full width but reduced depth — a target for profiler captures.
Kernel SHARES per block are depth-independent; absolute step numbers from this script are NOT bench values."""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "qwen-image-finetune_b200"))
import torch  # noqa: E402

import bench  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--layers", type=int, default=2)
ap.add_argument("--steps", type=int, default=2)
ap.add_argument("--events", action="store_true", help="print a per-phase CUDA-event breakdown instead")
a = ap.parse_args()
from qflux_b200.train_step import QwenImageEditStep  # noqa: E402

dev = torch.device("cuda", 0)
m = bench.build_model(dev, a.layers)
step = QwenImageEditStep(m)
opt = torch.optim.AdamW(list(m.parameters()), lr=1e-4, foreach=True)
C = bench.CFG
B, L, T, hw = C["B"], C["hw"] ** 2, C["T"], C["hw"]
x = dict(image_latents=torch.randn(B, L, 64, device=dev).bfloat16(), control_latents=torch.randn(B, L, 64, device=dev).bfloat16(),
         prompt_embeds=(torch.randn(B, T, C["joint"], device=dev) * 3).bfloat16(), img_shapes=[[(1, hw, hw), (1, hw, hw)]] * B)
for _ in range(a.steps):
    step.train_step(x, opt)
torch.cuda.synchronize()
if a.events:
    args = step._prepare(x, None, None)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    e = [ev() for _ in range(4)]
    e[0].record()
    packed = torch.empty(B, 2 * L, 64, device=dev, dtype=torch.bfloat16)
    from qflux_b200 import lib
    lib.flow_noisy_input(args[0], args[4], args[1], args[5], packed)
    pred = m._forward_impl(packed, args[2], args[5], args[3], train=True)
    e[1].record()
    ws = m._ws
    lib.flow_loss(pred, args[0], args[4], args[6], args[7], ws["loss"], ws["dpred"])
    m.G32.zero_()
    m._backward_impl(ws["dpred"])
    e[2].record()
    m.finalize_grads(1, 1.0)
    opt.step()
    e[3].record()
    torch.cuda.synchronize()
    print(f"layers={a.layers} fwd {e[0].elapsed_time(e[1]):.3f} ms  bwd {e[1].elapsed_time(e[2]):.3f} ms  opt {e[2].elapsed_time(e[3]):.3f} ms")
print("done")
