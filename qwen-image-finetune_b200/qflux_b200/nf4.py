"""4-bit NF4 base checkpoints (bitsandbytes `Linear4bit`): the serialized form, its parsing, and the exact dequantization rule.

A bitsandbytes 4-bit Linear used for training dequantizes its weight to bf16 and runs a plain bf16 matmul
(bitsandbytes/autograd/_functions.py MatMul4Bit.forward: `F.dequantize_4bit(B, quant_state).to(A.dtype)`), so an NF4 base model
computes exactly what the bf16 model computes with the dequantized weights.  The only new arithmetic is the dequantization,
restated here from bitsandbytes/functional.py `dequantize_4bit` / `dequantize_blockwise` and csrc/kernels.cu `kDequantizeBlockwise`:

  * element:  w[i] = bf16_rn(NF4[nibble_i] * absmax[i // blocksize]), fp32 product; element 2k is the HIGH nibble of byte k;
  * nested absmax (`compress_statistics=True`):  absmax = fp32(nested_quant_map[absmax_u8[j]] * nested_absmax[j // nested_blocksize])
    then `+ nested_offset` — two separate fp32 roundings (no FMA); done once at load time on the host.

Serialized form (`Linear4bit._save_to_state_dict` + `QuantState.as_dict(packed=True)`), per quantized module `<mod>`:
  `<mod>.weight` packed bytes [n/2, 1] (any storage dtype: the raw bytes count), `<mod>.weight.absmax`, `<mod>.weight.quant_map`,
  optionally `<mod>.weight.nested_absmax` / `<mod>.weight.nested_quant_map`, and `<mod>.weight.quant_state.bitsandbytes__nf4`:
  a uint8 tensor holding JSON {quant_type, blocksize, dtype, shape[, nested_blocksize, nested_offset, nested_dtype]}.
The format is detected per weight tensor: nothing here assumes which modules a checkpoint quantized.
"""
from __future__ import annotations

import json
from typing import NamedTuple

import torch

from .lib import QfxError

# bitsandbytes' built-in NF4 code book (functional.py get_4bit_type("nf4"); the CUDA kernel's dDequantizeNF4 constants)
NF4_TABLE = torch.tensor([-1.0, -0.6961928009986877, -0.5250730514526367, -0.39491748809814453, -0.28444138169288635,
                          -0.18477343022823334, -0.09105003625154495, 0.0, 0.07958029955625534, 0.16093020141124725,
                          0.24611230194568634, 0.33791524171829224, 0.44070982933044434, 0.5626170039176941, 0.7229568362236023,
                          1.0], dtype=torch.float32)
_QS = ".quant_state.bitsandbytes__"
_AUX = ("absmax", "quant_map", "nested_absmax", "nested_quant_map")


class Nf4Weight(NamedTuple):
    """One NF4 matrix as the fused path stores it: codes uint8 [n/2] (row-major [out, in], two elements per byte), fp32 absmax
    [n/blocksize] with any nested quantization folded in."""
    codes: torch.Tensor
    absmax: torch.Tensor
    shape: tuple
    blocksize: int


def _raw_bytes(t: torch.Tensor) -> torch.Tensor:
    return t.detach().contiguous().view(torch.uint8).reshape(-1)


def _fold_nested(absmax_u8, nested_absmax, nested_quant_map, nested_blocksize, nested_offset):
    """dequantize_blockwise(absmax, state2) + offset, with the product and the sum rounded to fp32 separately."""
    n = absmax_u8.numel()
    scale = nested_absmax.float().reshape(-1).repeat_interleave(int(nested_blocksize))[:n]
    prod = nested_quant_map.float().reshape(-1)[absmax_u8.reshape(-1).long()] * scale
    return prod + torch.tensor(float(nested_offset), dtype=torch.float32)


def split_state_dict(sd: dict):
    """(plain, quant): the state dict without the bitsandbytes 4-bit entries, and {"<mod>.weight": Nf4Weight} for every NF4 matrix.
    Refuses what the fused path cannot reproduce exactly: fp4, LLM.int8 (`SCB`), a non-bf16 compute dtype, an unknown code book,
    a blocksize that does not divide in_features."""
    bad = [k for k in sd if k.endswith((".SCB", ".weight_format"))]
    if bad:
        raise QfxError(f"`{bad[0]}`: bitsandbytes int8 (LLM.int8, Int8Params) checkpoints are not supported; only 4-bit NF4 base "
                       f"checkpoints load (or a bf16 checkpoint)")
    quant, skip = {}, set()
    for k, v in sd.items():
        if _QS not in k:
            continue
        wkey, qtype = k.split(_QS)
        if qtype != "nf4":
            raise QfxError(f"`{wkey}`: bitsandbytes 4-bit quant_type {qtype!r} is not supported; only 'nf4' base checkpoints load")
        meta = json.loads(bytes(_raw_bytes(v).tolist()).decode("utf-8"))
        shape, bs = tuple(int(s) for s in meta["shape"]), int(meta["blocksize"])
        mod = wkey.rsplit(".", 1)[0]
        if meta.get("quant_type", "nf4") != "nf4":
            raise QfxError(f"`{mod}`: quant_type {meta['quant_type']!r} is not supported; only 'nf4' base checkpoints load")
        if meta.get("dtype", "bfloat16") not in ("bfloat16", "float32"):
            raise QfxError(f"`{mod}`: NF4 compute dtype {meta['dtype']!r}: the fused path reproduces bitsandbytes' dequantization "
                           f"to bf16 (or fp32) only")
        if len(shape) != 2 or shape[1] % bs:
            raise QfxError(f"`{mod}`: NF4 blocksize {bs} does not divide in_features {shape[-1]} (shape {shape}); the fused "
                           f"layout keeps every quantization block inside one row")
        if bs % 32:
            raise QfxError(f"`{mod}`: NF4 blocksize {bs}: the dequantization kernel takes multiples of 32")
        aux = {a: sd.get(f"{wkey}.{a}") for a in _AUX}
        for a in ("absmax", "quant_map"):
            if aux[a] is None:
                raise QfxError(f"`{mod}`: NF4 weight without `{wkey}.{a}`")
        if not torch.equal(aux["quant_map"].float().reshape(-1).cpu(), NF4_TABLE):
            raise QfxError(f"`{wkey}.quant_map` is not bitsandbytes' NF4 code book (the bitsandbytes kernels ignore a stored map, "
                           f"so its dequantization cannot be reproduced from it)")
        if aux["nested_absmax"] is not None:
            absmax = _fold_nested(aux["absmax"].cpu(), aux["nested_absmax"].cpu(), aux["nested_quant_map"].cpu(),
                                  meta["nested_blocksize"], meta["nested_offset"])
        else:
            absmax = aux["absmax"].float().reshape(-1).cpu()
        n = shape[0] * shape[1]
        codes = _raw_bytes(sd[wkey])
        if codes.numel() * 2 != n or absmax.numel() * bs != n:
            raise QfxError(f"`{mod}`: {codes.numel()} code bytes / {absmax.numel()} absmax values do not match shape {shape} at "
                           f"blocksize {bs}")
        quant[wkey] = Nf4Weight(codes, absmax.contiguous(), shape, bs)
        skip.update([k, wkey] + [f"{wkey}.{a}" for a in _AUX])
    plain = {k: v for k, v in sd.items() if k not in skip}
    return plain, quant


def dequantize(q: Nf4Weight) -> torch.Tensor:
    """bf16 [out, in] on the host: bitsandbytes' `dequantize_4bit` of q, bit for bit."""
    c = q.codes.cpu()
    idx = torch.stack((c >> 4, c & 15), dim=-1).reshape(-1).long()
    w = NF4_TABLE[idx] * q.absmax.cpu().repeat_interleave(q.blocksize)
    return w.to(torch.bfloat16).view(q.shape)
