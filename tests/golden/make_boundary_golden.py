"""Generate tests/golden/boundary_golden.pt by running the REFERENCE's OWN code (needs the reference checkout at /root/reference):

    python tests/golden/make_boundary_golden.py

Stored: (1) `QwenEmbedRope(theta=10000, axes_dim=[16, 56, 56], scale_rope=True)` outputs for two image-shape lists; (2) per scheduler config
and (steps, image_seq_len): `calculate_shift`, the timesteps of `BaseTrainer.prepare_predict_timesteps`, the scheduler's sigmas and one
`scheduler.step` on seeded inputs; (3) a cache directory written by `EmbeddingCacheManager.save_cache_embedding` (file bytes) and what
the reference's `load_cache` + `pad_to_max_shape` make of it.  tests/test_reference_trainer_boundary.py compares the fused code with these.
"""
import contextlib
import io
import os
import sys
import tempfile
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests", "shims"))
import stub_importer  # noqa: E402

stub_importer.install()
sys.path.insert(0, "/root/reference/src")

from diffusers.schedulers.scheduling_flow_match_euler_discrete import FlowMatchEulerDiscreteScheduler  # noqa: E402  (tests/shims)
from qflux.data.cache_manager import EmbeddingCacheManager  # noqa: E402
from qflux.models.transformer_qwenimage import QwenEmbedRope  # noqa: E402
from qflux.trainer.base_trainer import BaseTrainer  # noqa: E402
from qflux.utils.sampling import calculate_shift  # noqa: E402
from qflux.utils.tools import pad_to_max_shape  # noqa: E402

ROPE_CASES = [([(1, 4, 4), (1, 4, 4)], 7), ([(1, 4, 6), (1, 4, 6), (1, 2, 8)], 11)]
SCHED = dict(
    qwen=dict(num_train_timesteps=1000, shift=1.0, use_dynamic_shifting=True, base_shift=0.5, max_shift=0.9, base_image_seq_len=256,
              max_image_seq_len=8192, shift_terminal=0.02),
    flux=dict(num_train_timesteps=1000, shift=3.0, use_dynamic_shifting=True, base_shift=0.5, max_shift=1.15, base_image_seq_len=256,
              max_image_seq_len=4096))
SCHED_POINTS = [(20, 1024), (8, 4096), (50, 400)]
CACHE_SIZES = [(128, 128), (64, 128), (128, 96)]  # pixel H, W of the three cached samples


def rope():
    r = QwenEmbedRope(theta=10000, axes_dim=[16, 56, 56], scale_rope=True)
    return [dict(shapes=s, T=T, vid=v.clone(), txt=t.clone()) for s, T in ROPE_CASES for v, t in [r([s], [T], device=torch.device("cpu"))]]


def schedules():
    out = []
    g = torch.Generator().manual_seed(11)
    for name, conf in SCHED.items():
        for steps, seq in SCHED_POINTS:
            tr = types.SimpleNamespace(sampling_scheduler=FlowMatchEulerDiscreteScheduler(**conf), scheduler=None, dit=torch.nn.Linear(1, 1))
            with contextlib.redirect_stdout(io.StringIO()):  # the reference prints the shift arguments
                ts, n = BaseTrainer.prepare_predict_timesteps(tr, steps, seq)
            x, v = torch.randn(2, 8, 64, generator=g).bfloat16(), torch.randn(2, 8, 64, generator=g).bfloat16()
            tr.sampling_scheduler.set_begin_index(0)
            want = tr.sampling_scheduler.step(v, ts[0], x, return_dict=False)[0]
            out.append(dict(config=name, conf=dict(conf), steps=steps, seq=seq, n=n, timesteps=ts.cpu().clone(), sigmas=tr.sampling_scheduler.sigmas.cpu().clone(),
                            shift=calculate_shift(seq, conf["base_image_seq_len"], conf["max_image_seq_len"], conf["base_shift"], conf["max_shift"]),
                            x=x, v=v, euler=want))
    return out


def cache():
    with tempfile.TemporaryDirectory() as d:
        mgr = EmbeddingCacheManager(d)
        g = torch.Generator().manual_seed(5)
        hashes = []
        for i, (H, W) in enumerate(CACHE_SIZES):
            L, T = (H // 16) * (W // 16), 6 + 5 * i
            data = dict(image_latents=torch.randn(L, 64, generator=g), control_latents=torch.randn(L, 64, generator=g),
                        prompt_embeds=torch.randn(T, 48, generator=g))
            fh = dict(main_hash=f"m{i:03d}", image_hash=f"i{i:03d}", control_hash=f"c{i:03d}", prompt_hash=f"p{i:03d}")
            mgr.save_cache_embedding(data, dict(image_latents="image_hash", control_latents="control_hash", prompt_embeds="prompt_hash"), fh,
                                     img_shapes=[[3, H, W], [3, H, W]])
            hashes.append(fh)
        files = {}
        for dp, _, fs in os.walk(d):
            for f in fs:
                p = os.path.join(dp, f)
                files[os.path.relpath(p, d)] = open(p, "rb").read()
        theirs = [mgr.load_cache({"file_hashes": fh}) for fh in hashes]  # the reference's reader, one sample at a time
        want = {k: pad_to_max_shape([t[k] for t in theirs]) for k in ("image_latents", "control_latents", "prompt_embeds")}
    return dict(files=files, sizes=CACHE_SIZES, want=want)


if __name__ == "__main__":
    path = os.path.join(HERE, "boundary_golden.pt")
    torch.save(dict(rope=rope(), schedules=schedules(), cache=cache()), path)
    print(path, os.path.getsize(path), "bytes")
