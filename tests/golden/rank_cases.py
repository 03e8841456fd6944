"""Reference-golden cases at LoRA ranks other than 4 (tests/golden/ref_rank_golden_*.pt, written by make_ref_rank_golden.py with
make_ref_model_golden.py's reference run): ranks between the powers of two and above 64, where the fused path pads the rank to two 64-wide k-blocks.
Nothing here imports /root/reference.

The r = 96 case holds several MB of fp32 LoRA gradients, more than one golden file may hold, so a case's gradients may be spread
over several files: every file maps case name -> a part of that case, and `load` merges the parts."""
import io
import os

import torch

import ref_common as rc

# one block of each kind keeps the files of the r = 96 / 128 gradients small; the CUDA glue kernels need D = 2 heads x 128 at least
QWEN_HD128_1BLK = dict(rc.QWEN_HD128, num_layers=1)
FLUX_HD128_1P1 = dict(rc.FLUX_HD128, num_layers=1, num_single_layers=1)

RANK_CASES = {
    "qwen_hd128_r24": dict(kind="qwen", cfg=rc.QWEN_HD128, r=24, alpha=16, targets=rc.DEFAULT_TARGETS, B=2, T=24,
                           shapes=[(1, 4, 4), (1, 4, 4)], seed=41),
    "qwen_hd128_r128": dict(kind="qwen", cfg=QWEN_HD128_1BLK, r=128, alpha=128, targets=rc.DEFAULT_TARGETS, B=2, T=24,
                            shapes=[(1, 4, 4), (1, 4, 4)], seed=42),
    # BASELINE config 3's target set, x_embedder included: its 64-channel dA runs in rank chunks of 64 + 32
    "flux_hd128_yaml_r96": dict(kind="flux", cfg=FLUX_HD128_1P1, r=96, alpha=48, targets=rc.FLUX_YAML_TARGETS, B=2, T=8, hw=(4, 4),
                                seed=43),
}


def _nbytes(o) -> int:
    buf = io.BytesIO()
    torch.save(o, buf)
    return len(buf.getvalue())


def save(cases: dict, directory: str, stem: str) -> list:
    """One file per part: a case's fields without its gradients, then its gradients in name order, each part < GOLDEN_PART_BYTES."""
    parts = []
    for name, c in cases.items():
        c = rc._compact(c)
        grads = c.pop("grads")
        cur = dict(c, grads={})
        for k in sorted(grads):
            if cur["grads"] and _nbytes(cur) + _nbytes(grads[k]) > rc.GOLDEN_PART_BYTES:
                parts.append({name: cur})
                cur = {"grads": {}}
            cur["grads"][k] = grads[k]
        assert _nbytes(cur) < rc.GOLDEN_PART_BYTES, f"{name}: one part is too large"
        parts.append({name: cur})
    for f in os.listdir(directory):
        if f.startswith(stem + "_") and f.endswith(".pt"):
            os.remove(os.path.join(directory, f))
    paths = []
    for i, part in enumerate(parts):
        paths.append(os.path.join(directory, f"{stem}_{i}.pt"))
        torch.save(part, paths[-1])
    return paths


def load(directory: str, stem: str) -> dict:
    out = {}
    for f in sorted((f for f in os.listdir(directory) if f.startswith(stem + "_") and f.endswith(".pt")),
                    key=lambda f: int(f[len(stem) + 1:-3])):
        for name, part in torch.load(os.path.join(directory, f), weights_only=False).items():
            c = out.setdefault(name, {"grads": {}})
            c["grads"].update(part.pop("grads"))
            c.update(part)
    assert out, f"no {stem}_*.pt in {directory}"
    return out
