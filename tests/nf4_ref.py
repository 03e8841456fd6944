"""TEST INFRASTRUCTURE ONLY — the bitsandbytes 4-bit (NF4) side of the NF4 tests, restated in plain PyTorch:

  * `quantize_nf4` writes one Linear's state-dict entries exactly as `Linear4bit._save_to_state_dict` / `QuantState.as_dict(packed=True)`
    do (bitsandbytes/nn/modules.py, bitsandbytes/functional.py quantize_4bit, quantize_blockwise, create_dynamic_map), nested
    (`compress_statistics=True`) or not, with uint8 or another storage dtype for the packed bytes;
  * `dequantize_4bit` is bitsandbytes' dequantization of those entries (dequantize_blockwise for a nested absmax, then the NF4
    lookup times absmax, fp32 product, bf16 result) — written independently of qflux_b200.nf4, which it checks;
  * `nf4_dequant` emulates the `qflux_b200.lib.nf4_dequant` entry point for `-m "not gpu"` runs (see emu_lib.py).
"""
from __future__ import annotations

import json

import torch

import emu_lib

NF4 = [-1.0, -0.6961928009986877, -0.5250730514526367, -0.39491748809814453, -0.28444138169288635, -0.18477343022823334,
       -0.09105003625154495, 0.0, 0.07958029955625534, 0.16093020141124725, 0.24611230194568634, 0.33791524171829224,
       0.44070982933044434, 0.5626170039176941, 0.7229568362236023, 1.0]


def create_dynamic_map(signed=True, max_exponent_bits=7, total_bits=8):
    data, non_sign_bits = [], total_bits - 1
    for i in range(max_exponent_bits):
        items = int(2 ** (i + non_sign_bits - max_exponent_bits) + 1 if signed else 2 ** (i + non_sign_bits - max_exponent_bits + 1) + 1)
        b = torch.linspace(0.1, 1, items)
        means = (b[:-1] + b[1:]) / 2.0
        data += ((10 ** (-(max_exponent_bits - 1) + i)) * means).tolist()
        if signed:
            data += (-(10 ** (-(max_exponent_bits - 1) + i)) * means).tolist()
    data += [0, 1.0]
    data += [0] * (2 ** total_bits - len(data))
    return torch.tensor(sorted(data), dtype=torch.float32)


def _nearest(x, table):
    return (x[:, None] - table[None, :]).abs().argmin(1)


def _quantize_blockwise(x, code, blocksize):
    n = x.numel()
    blocks = x.reshape(-1)
    pad = (-n) % blocksize
    xb = torch.cat([blocks, blocks.new_zeros(pad)]).view(-1, blocksize)
    absmax = xb.abs().amax(1)
    q = _nearest((xb / absmax.clamp_min(1e-30)[:, None]).reshape(-1)[:n], code)
    return q.to(torch.uint8), absmax


def quantize_nf4(W, blocksize=64, nested=False, storage=torch.uint8, nested_blocksize=256):
    """{suffix: tensor} of one quantized Linear weight: "" (packed bytes [n/2, 1] viewed as `storage`), ".absmax", ".quant_map",
    [".nested_absmax", ".nested_quant_map"], ".quant_state.bitsandbytes__nf4"."""
    W = W.float().cpu()
    table = torch.tensor(NF4)
    codes, absmax = _quantize_blockwise(W, table, blocksize)
    packed = ((codes[0::2] << 4) | codes[1::2]).to(torch.uint8).view(-1, 1)
    meta = dict(quant_type="nf4", blocksize=blocksize, dtype="bfloat16", shape=list(W.shape))
    out = {"": packed.view(-1).view(storage).view(-1, 1), ".quant_map": table.clone()}
    if nested:
        offset = absmax.mean()
        code2 = create_dynamic_map()
        q2, absmax2 = _quantize_blockwise(absmax - offset, code2, nested_blocksize)
        out.update({".absmax": q2, ".nested_absmax": absmax2, ".nested_quant_map": code2})
        meta.update(nested_blocksize=nested_blocksize, nested_offset=offset.item(), nested_dtype="float32")
    else:
        out[".absmax"] = absmax
    out[".quant_state.bitsandbytes__nf4"] = torch.tensor(list(json.dumps(meta).encode("utf-8")), dtype=torch.uint8)
    return out


def dequantize_4bit(entries: dict, prefix: str) -> torch.Tensor:
    """bf16 [out, in] from the serialized entries of `<prefix>` (= "<mod>.weight")."""
    meta = json.loads(bytes(entries[prefix + ".quant_state.bitsandbytes__nf4"].tolist()).decode())
    absmax = entries[prefix + ".absmax"]
    if prefix + ".nested_absmax" in entries:
        nbs = meta["nested_blocksize"]
        a = torch.empty(absmax.numel(), dtype=torch.float32)
        code2, am2 = entries[prefix + ".nested_quant_map"], entries[prefix + ".nested_absmax"]
        for j in range(absmax.numel()):  # dequantize_blockwise, then += offset: two fp32 roundings
            a[j] = code2[int(absmax[j])] * am2[j // nbs]
        absmax = a + torch.tensor(meta["nested_offset"], dtype=torch.float32)
    raw = entries[prefix].contiguous().view(torch.uint8).reshape(-1)
    n = raw.numel() * 2
    nib = torch.empty(n, dtype=torch.long)
    nib[0::2], nib[1::2] = (raw >> 4).long(), (raw & 15).long()
    w = torch.tensor(NF4)[nib] * absmax.float().repeat_interleave(meta["blocksize"])[:n]
    return w.to(torch.bfloat16).view(meta["shape"])


def to_nf4_state_dict(sd: dict, select, blocksize=64, nested=False, storage=torch.uint8, key=lambda k: k):
    """sd with every 2-D `.weight` whose module `select(name)` accepts replaced by its NF4 entries; `key` renames the module prefix
    (e.g. adds `.base_layer.` or `transformer.`)."""
    out = {}
    for k, v in sd.items():
        if k.endswith(".weight") and v.ndim == 2 and ".lora_" not in k and select(k[: -len(".weight")].replace(".base_layer", "")):
            for suf, t in quantize_nf4(v, blocksize, nested, storage).items():
                out[key(k) + suf] = t
        else:
            out[key(k)] = v
    return out


def nf4_dequant(segments):
    for codes, absmax, out, bs in segments:
        c = codes.reshape(-1)
        nib = torch.stack(((c >> 4), (c & 15)), -1).reshape(-1).long()
        out.copy_((torch.tensor(NF4)[nib] * absmax.reshape(-1).repeat_interleave(bs)).to(torch.bfloat16).view(out.shape))


def install(lib_module):
    """emu_lib.install plus the NF4 entry point; returns the restore callable."""
    restore_emu = emu_lib.install(lib_module)
    saved = lib_module.nf4_dequant
    lib_module.nf4_dequant = nf4_dequant

    def restore():
        lib_module.nf4_dequant = saved
        restore_emu()
    return restore
