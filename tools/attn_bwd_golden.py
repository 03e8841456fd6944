"""Bit-level goldens of the joint attention backward: SHA-256 of dK and dV from qfx_attn_bwd, of dK, dV and dQ from
qfx_attn_bwd_det, and of three deterministic FusedLoraAdamW training steps, recorded on one device model and kept in
tests/golden/attn_bwd_bits.json.  A change to the backward's schedule must leave every one of them unchanged: dK and dV keep each
element's operation order (ascending 16-query chunks, head-dim k-steps in order, the same bf16 rounding points for P and dS).

    python tools/attn_bwd_golden.py [--out F]  record on cuda:0 and write the JSON (to F instead, with --out)
    python tools/attn_bwd_golden.py --check    recompute on cuda:0 and compare with the JSON (exit 1 on a mismatch)

Kernel inputs (Q, K, V, dO, delta, kv_len, txt_len) are drawn on the CPU from a per-case seed and copied to the device; lse comes
from qfx_attn_fwd on those inputs.  dO is zero on query rows >= kv_len[b], as the training step passes it.  The training-step
hashes are tools/determinism_check.py's three-step runs of a 2-block, full-width Qwen-Image-Edit model with a ragged prompt mask.
"""
import hashlib
import json
import os
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "qwen-image-finetune_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, "tests", "golden", "attn_bwd_bits.json")

# (name, B, H, S, split, txt_len per sample or None, kv_len per sample or None)
CASES = [
    ("flagship_B1", 1, 24, 2400, 352, [352], None),
    ("B4_txt40", 4, 24, 2400, 352, [40] * 4, None),
    # txt_len on and next to the 64 / 128 key-tile edges, S one below and one above a 128 boundary
    ("txt_edges_S383", 6, 2, 383, 129, [63, 64, 65, 127, 128, 129], None),
    ("txt_edges_S641", 6, 2, 641, 129, [63, 64, 65, 127, 128, 129], None),
    # kv_len on and next to the tile edges: the query tiles past kv_len are padding and skipped
    ("kv_edges_S385", 6, 2, 385, 385, None, [63, 64, 65, 127, 128, 129]),
    ("kv_edges_S639", 6, 2, 639, 639, None, [63, 64, 65, 127, 128, 129]),
    # key tile [128, 256) fully inside the text padding (txt_len 40 < split - 128), a padding query tile past kv_len
    ("masked_key_tile_pad_query_tile", 2, 2, 639, 352, [40, 100], [639, 450]),
]
STEP_CASES = [("step_qwen_edit_B1", 1, [200]), ("step_qwen_edit_B2", 2, [352, 200])]


def case_inputs(case):
    """CPU tensors of one case, from its own seed: Q, K, V, dO (bf16 [B,H,S,128]), delta (fp32 [B,H,S]), kv_len, txt_len"""
    import torch
    name, B, H, S, split, txt, kv = case
    g = torch.Generator().manual_seed(int.from_bytes(hashlib.sha256(name.encode()).digest()[:4], "little"))
    Q, K, V, dO = (torch.randn(B, H, S, 128, generator=g).bfloat16() for _ in range(4))
    kv_len = None if kv is None else torch.tensor(kv, dtype=torch.int32)
    txt_len = None if txt is None else torch.tensor(txt, dtype=torch.int32)
    if kv_len is not None:
        dO = dO * (torch.arange(S)[None] < kv_len[:, None])[:, None, :, None].bfloat16()
    delta = torch.randn(B, H, S, generator=g) * 0.1
    return Q, K, V, dO, delta, kv_len, txt_len


def sha(*ts):
    import torch
    h = hashlib.sha256()
    for t in ts:
        if t is not None:
            h.update(t.detach().contiguous().view(-1).view(torch.uint8).cpu().numpy().tobytes())
    return h.hexdigest()


def inputs_sha(case):
    return sha(*case_inputs(case))


def kernel_case(case):
    import torch
    from qflux_b200 import lib
    name, B, H, S, split, txt, kv = case
    Q, K, V, dO, delta, kv_len, txt_len = (None if t is None else t.cuda() for t in case_inputs(case))
    ot = torch.empty(B * split, H * 128, device="cuda", dtype=torch.bfloat16)
    oi = torch.empty(B * (S - split), H * 128, device="cuda", dtype=torch.bfloat16)
    lse = torch.empty(B, H, S, device="cuda")
    lib.attn_fwd(Q, K, V, ot, oi, split, lse, kv_len, txt_len=txt_len)
    out = {}
    for tag, fn in (("atomic", lib.attn_bwd), ("det", lib.attn_bwd_det)):
        dQ = torch.zeros(B, H, S, 128, device="cuda")
        dK, dV = torch.full_like(Q, 7.0), torch.full_like(Q, 7.0)
        fn(Q, K, V, dO, lse, delta, dQ, dK, dV, kv_len, txt_len=txt_len, split=split)
        torch.cuda.synchronize()
        out[f"{tag}_dK"], out[f"{tag}_dV"] = sha(dK), sha(dV)
        if tag == "det":
            out["det_dQ"] = sha(dQ)
    return out


def step_case(B, txt):
    import torch
    import determinism_check
    import nf4_check
    full = nf4_check.device_batch

    def with_mask(cfg, name):  # bench's qwen_edit batch carries no prompt mask: an all-ones one, made ragged by _three_steps
        return dict(full(cfg, name), prompt_embeds_mask=torch.ones(cfg["B"], cfg["T"], dtype=torch.int64, device="cuda"))
    nf4_check.device_batch = with_mask
    r = determinism_check._three_steps("qwen", "qwen_edit", txt=txt, B=B, blocks=2)
    return dict(loss_sha=r["loss_sha"], g32_sha=r["g32_sha"], lora_sha=r["lora_sha"])


def device():
    import torch
    p = torch.cuda.get_device_properties(0)
    return dict(name=p.name, sm_count=p.multi_processor_count)


def record():
    import subprocess
    res = dict(device=device(), cases={}, steps={})
    for case in CASES:
        res["cases"][case[0]] = dict(B=case[1], H=case[2], S=case[3], split=case[4], txt_len=case[5], kv_len=case[6],
                                     inputs_sha=inputs_sha(case), **kernel_case(case))
    for name, B, txt in STEP_CASES:
        # each step case in a process of its own: the deterministic flag and the model's workspaces start fresh
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--step", name], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"{name} failed:\n{r.stderr[-3000:]}")
        res["steps"][name] = dict(B=B, txt_len=txt, **json.loads(r.stdout.strip().splitlines()[-1]))
    return res


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "--step":
        _, B, txt = next(c for c in STEP_CASES if c[0] == sys.argv[2])
        print(json.dumps(step_case(B, txt)))
    elif "--check" in sys.argv:
        with open(GOLDEN) as f:
            want = json.load(f)
        got = record()
        bad = [(k, n) for k in ("cases", "steps") for n in want[k] if want[k][n] != got[k][n]]
        print(json.dumps(dict(device=got["device"], golden_device=want["device"], mismatches=bad)))
        sys.exit(1 if bad else 0)
    else:
        out = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else GOLDEN
        res = record()
        with open(out, "w") as f:
            json.dump(res, f, indent=1)
            f.write("\n")
        print(json.dumps(res["device"]))
