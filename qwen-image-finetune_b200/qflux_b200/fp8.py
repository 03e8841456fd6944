"""float8-e4m3fn base checkpoints without scales (e.g. `camenduru/flux1-kontext-dev_fp8_e4m3fn_diffusers`): the two forms their
block matrices arrive in, and the check that keeps an FP8-resident model exact.

Every finite e4m3fn value converts to bf16 exactly, so a model that keeps these matrices as e4m3fn bytes and expands them block by
block (qfx_fp8_expand) computes exactly what the bf16 model computes with the upcast weights.  A matrix arrives either

  * as `float8_e4m3fn`, read straight from the checkpoint's safetensors, or
  * as bf16, the form diffusers' `from_pretrained(torch_dtype=bfloat16)` upcasts it to: accepted when every element round-trips
    bf16 -> e4m3fn -> bf16 bit for bit (so -0 stays -0 and nothing saturates).

Anything else would change the model's numerics and is refused: a genuine bf16 matrix, NaN codes (0x7f / 0xff), other dtypes.
"""
from __future__ import annotations

import torch

from .lib import QfxError

E4M3 = torch.float8_e4m3fn


def as_e4m3(key: str, v: torch.Tensor, device=None) -> torch.Tensor:
    """The e4m3fn codes of block matrix `key` (on `device`), from either accepted form; raises QfxError naming `key` and the first
    value that is not an exact finite e4m3fn value."""
    v = v.detach().to(device)
    if v.dtype == E4M3:
        nan = (v.view(torch.uint8) & 0x7F) == 0x7F
        if bool(nan.any()):
            i = int(nan.reshape(-1).nonzero()[0])
            raise QfxError(f"`{key}`: element {i} is the float8-e4m3fn NaN code 0x{int(v.view(torch.uint8).reshape(-1)[i]):02x}; "
                           f"an FP8 base checkpoint holds finite weights only")
        return v
    if v.dtype != torch.bfloat16:
        raise QfxError(f"`{key}` arrives as {v.dtype}: an FP8-resident model (frozen_weights='fp8') takes block matrices as "
                       f"float8_e4m3fn or as their exact bf16 upcast")
    codes = v.to(E4M3)
    # a bf16 NaN converts to the NaN code and back to the same bits: the round trip alone would let it through
    bad = (codes.to(torch.bfloat16).view(torch.int16) != v.view(torch.int16)) | v.isnan()
    if bool(bad.any()):
        i = int(bad.reshape(-1).nonzero()[0])
        raise QfxError(f"`{key}`: element {i} = {float(v.reshape(-1)[i])!r} (bf16) is not a float8-e4m3fn value, so this is not "
                       f"the upcast of an FP8 checkpoint; construct the model with frozen_weights='bf16' for a bf16 checkpoint")
    return codes
