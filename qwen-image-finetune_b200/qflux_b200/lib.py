"""ctypes binding of libqfx_b200.so (include/qfx.h).  Fails loudly when the library or a CUDA device is missing."""
from __future__ import annotations

import ctypes as C
import os

import torch  # noqa: F401  (loads libcudart.so.12 into the process before our library)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libqfx_b200.so")

if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing — build it with `python -c 'import __graft_entry__ as g; g.build()'` "
        "(there is no CPU / eager fallback for the CUDA hot path)")

_lib = C.CDLL(LIB_PATH)
_lib.qfx_last_error.restype = C.c_char_p
_lib.qfx_version.restype = C.c_int


class QfxError(RuntimeError):
    pass


LAUNCHES = 0  # kernels of THIS library launched so far (bench.py reports the per-step delta as gpu_launches)
_KERNELS_PER_CALL = {"qfx_grad_finalize": 2, "qfx_attn_bwd_det": 2, "qfx_lora_wgrad_tc_det": 2, "qfx_lora_wgrad_det": 2,
                     "qfx_mod_grad_det": 2, "qfx_flow_loss_det": 2, "qfx_grad_finalize_det": 3, "qfx_fused_adamw_det": 3,
                     "qfx_fused_prodigy": 5, "qfx_fused_adam8bit": 3}


def check(rc: int, what: str):
    global LAUNCHES
    LAUNCHES += _KERNELS_PER_CALL.get(what, 1)
    if rc != 0:
        raise QfxError(f"{what} failed (rc={rc}): {_lib.qfx_last_error().decode()}")


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise QfxError("qflux_b200 ops need CUDA tensors (no CPU fallback)")


def ptr(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def cur_stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---------------------------------------------------------------------------------------------------- GEMM
EPI_BIAS, EPI_GELU, EPI_RESID_GATE, EPI_DGELU, EPI_ADD, EPI_ATTN_DO = 0, 1, 2, 3, 4, 5


class GemmProblem(C.Structure):
    _fields_ = [
        ("A", C.c_void_p), ("lda", C.c_int64),
        ("B", C.c_void_p), ("ldb", C.c_int64),
        ("M", C.c_int),
        ("A2", C.c_void_p), ("lda2", C.c_int64),
        ("B2", C.c_void_p), ("ldb2", C.c_int64),
        ("kb2", C.c_int), ("a2_col0", C.c_int),
        ("bias", C.c_void_p),
        ("out", C.c_void_p), ("ldo", C.c_int64),
        ("out2", C.c_void_p), ("ldo2", C.c_int64),
        ("resid", C.c_void_p), ("ldr", C.c_int64),
        ("gate", C.c_void_p), ("ldg", C.c_int64), ("rows_per_batch", C.c_int),
        ("aux", C.c_void_p), ("ldaux", C.c_int64),
        ("row_tiles", C.c_void_p), ("n_row_tiles", C.c_int),
        ("delta", C.c_void_p), ("attn_S", C.c_int), ("attn_H", C.c_int), ("s_offset", C.c_int),
    ]


_lib.qfx_gemm_bf16.argtypes = [C.POINTER(GemmProblem), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int,
                               C.c_int, C.c_void_p]
_lib.qfx_gemm_bf16.restype = C.c_int


def _dp(t):
    return 0 if t is None else t.data_ptr()


def _ld(t):
    return 0 if t is None else t.stride(0)


class RowBands:
    """Which rows of a pad-to-max row group a ragged GEMM computes: `tiles` = device int32 start rows of the disjoint 256-row bands
    that cover every valid row; `dead` = device int32 [n_dead, 2] row ranges outside the bands (zero-filled before the GEMM)."""

    def __init__(self, tiles, dead, device):
        self.n, self.n_dead = len(tiles), len(dead)
        self.tiles = torch.tensor(tiles, dtype=torch.int32, device=device)
        self.dead = torch.tensor(dead, dtype=torch.int32, device=device).reshape(-1, 2) if dead else None
        self.host_tiles, self.host_dead = list(tiles), [tuple(d) for d in dead]

    @staticmethod
    def plan(valid, rows_per_sample, band=256):
        """valid[b] = valid rows of sample b (sample b owns rows [b*R, (b+1)*R)).  Returns (band start rows, dead ranges) or None when
        nothing can be skipped.  Bands never overlap: an interval whose last band would run into the next interval is merged with it."""
        R, M = rows_per_sample, rows_per_sample * len(valid)
        iv = []
        for b, v in enumerate(valid):
            if v > 0:
                lo, hi = b * R, b * R + int(v)
                if iv and iv[-1][1] >= lo:
                    iv[-1][1] = hi
                else:
                    iv.append([lo, hi])
        tiles, dead, cur = [], [], 0
        i = 0
        while i < len(iv):
            lo, hi = iv[i]
            while True:
                end = lo + -(-(hi - lo) // band) * band
                if i + 1 < len(iv) and iv[i + 1][0] < end:  # the last band would cross into the next interval: treat the gap as valid
                    hi = iv[i + 1][1]
                    i += 1
                else:
                    break
            if lo > cur:
                dead.append((cur, lo))
            tiles += list(range(lo, end, band))
            cur = min(end, M)
            i += 1
        if cur < M:
            dead.append((cur, M))
        return (tiles, dead) if dead else None


def gemm_problem(A, B, out, *, A2=None, B2=None, kb2=0, a2_col0=0, bias=None, out2=None, resid=None, gate=None,
                 rows_per_batch=0, aux=None, row_bands=None, delta=None, s_offset=0) -> GemmProblem:
    """delta (fp32 [B, H, S]) + s_offset select the EPI_ATTN_DO outputs: `out` is then the head-major dO_joint [B, H, S, 128]."""
    require_cuda(A, B, out, A2, B2, bias, out2, resid, gate, aux, delta)
    for t in (A, B, A2, B2, out2, resid, gate, aux) + (() if delta is not None else (out,)):
        assert t is None or (t.dtype == torch.bfloat16 and t.dim() == 2 and t.stride(1) == 1), "bf16 row-major 2-D expected"
    p = GemmProblem(_dp(A), _ld(A), _dp(B), _ld(B), A.shape[0], _dp(A2), _ld(A2), _dp(B2), _ld(B2), kb2, a2_col0,
                    _dp(bias), _dp(out), _ld(out), _dp(out2), _ld(out2), _dp(resid), _ld(resid), _dp(gate), _ld(gate),
                    rows_per_batch, _dp(aux), _ld(aux), 0 if row_bands is None else row_bands.tiles.data_ptr(),
                    0 if row_bands is None else row_bands.n, _dp(delta), 0, 0, s_offset)
    if delta is not None:  # out = dO_joint [B, H, S, 128] (contiguous), delta [B, H, S]
        assert out.dim() == 4 and out.is_contiguous() and out.shape[3] == 128 and tuple(delta.shape) == tuple(out.shape[:3]) and row_bands is None
        p.ldo, p.attn_S, p.attn_H = 0, out.shape[2], out.shape[1]
    p.bands, p.outs = row_bands, (out, out2)  # kept alive / used by gemm() for the zero fill
    return p


_zero_rows = None


def zero_rows(out, ncols, ranges, n_ranges):
    global _zero_rows
    if _zero_rows is None:
        _zero_rows = _sig("qfx_zero_rows", C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_int, C.c_void_p)
    check(_zero_rows(ptr(out), out.stride(0), ncols, ptr(ranges), n_ranges, cur_stream()), "qfx_zero_rows")


def gemm(problems, N, K, *, trans_b=False, epilogue=EPI_BIAS, alpha=1.0, lora_group_n=0, block_n=0):
    for p in problems:  # ragged row groups: the rows outside the computed bands become zeros
        b = getattr(p, "bands", None)
        if b is not None and b.n_dead:
            for o in p.outs:
                if o is not None:
                    zero_rows(o, N, b.dead, b.n_dead)
    arr = (GemmProblem * len(problems))(*problems)
    check(_lib.qfx_gemm_bf16(arr, len(problems), N, K, int(trans_b), epilogue, float(alpha), lora_group_n, block_n,
                             cur_stream()), "qfx_gemm_bf16")


# ---------------------------------------------------------------------------------------------------- elementwise
def _sig(name, *argtypes):
    f = getattr(_lib, name)
    f.argtypes = list(argtypes)
    f.restype = C.c_int
    return f


_vp, _i, _i64, _f = C.c_void_p, C.c_int, C.c_int64, C.c_float
_ln_fwd = _sig("qfx_ln_modulate_fwd", _vp, _i64, _vp, _i64, _vp, _vp, _i64, _i, _vp, _vp, _i, _i, _f, _vp)
_ln_bwd = _sig("qfx_ln_modulate_bwd", _vp, _i64, _vp, _i64, _vp, _vp, _vp, _i64, _i, _vp, _i64, _vp, _i64, _vp, _i64, _vp,
               _i64, _i, _i, _vp)
_mod_grad = _sig("qfx_mod_grad", _vp, _i64, _vp, _i64, _vp, _vp, _i, _vp, _vp, _i64, _i, _i, _vp)
_gate_mul = _sig("qfx_gate_mul", _vp, _i64, _vp, _i64, _i, _vp, _i64, _i, _i, _vp)
_rms_rows = _sig("qfx_rmsnorm_rows", _vp, _i64, _vp, _vp, _i64, _i, _i, _f, _vp)
_qknr_fwd = _sig("qfx_qk_norm_rope_fwd", _vp, _i64, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _i, _vp)
_qknr_bwd = _sig("qfx_qk_norm_rope_bwd", _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i64, _vp, _i64, _i, _i, _i, _i, _i, _f, _i,
                 _vp)
_gemv = _sig("qfx_gemv_act", _vp, _i64, _vp, _i64, _vp, _vp, _i64, _i, _i, _i, _i, _vp)
_tsin = _sig("qfx_timestep_sinusoid", _vp, _f, _vp, _i, _i, _vp)
_noisy = _sig("qfx_flow_noisy_input", _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp)
_floss = _sig("qfx_flow_loss", _vp, _vp, _vp, _vp, _f, _f, _vp, _vp, _i, _i, _i, _i, _vp)
_wgrad = _sig("qfx_lora_wgrad", _vp, _i64, _vp, _i64, _vp, _i64, _i64, _i, _i, _i, _vp)
_delta = _sig("qfx_attn_delta", _vp, _i64, _vp, _i64, _vp, _vp, _i, _i, _i, _i, _i, _vp)
_attn_bwd = _sig("qfx_attn_bwd", _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _vp)
_gfin = _sig("qfx_grad_finalize", _vp, _i64, _f, _f, _vp, _vp, _vp)
_attn_fwd = _sig("qfx_attn_fwd", _vp, _vp, _vp, _vp, _i64, _i, _vp, _i64, _i, _i, _vp, _vp, _vp, _i, _i, _i, _f, _vp)


_ln_fwd2 = _sig("qfx_ln_modulate_fwd_pair", _vp, _i64, _vp, _i64, _vp, _vp, _i64, _i, _vp, _vp, _i, _i, _f, _i, _vp, _vp, _i, _vp)
_ln_bwd2 = _sig("qfx_ln_modulate_bwd_pair", _vp, _i64, _vp, _i64, _vp, _vp, _vp, _i64, _i, _vp, _i64, _vp, _i64, _vp, _i64, _vp,
                _i64, _i, _i, _i, _vp, _vp, _i, _vp)
_qknr_fwd2 = _sig("qfx_qk_norm_rope_fwd_pair", _vp, _i64, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _i, _i, _vp, _vp,
                  _i, _i, _vp)
_qknr_bwd2 = _sig("qfx_qk_norm_rope_bwd_pair", _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i64, _vp, _i64, _i, _i, _i, _i, _i, _f, _i, _i,
                  _vp, _vp, _i, _i, _i, _vp)
_delta2 = _sig("qfx_attn_delta_pair", _vp, _i64, _vp, _i64, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp)


# ---- stream-pair launches: rows [0, split) of a stream-major buffer are group 0 (text), rows [split, M) group 1 (image); g0 / g1 carry
# the per-stream operands.  One launch instead of two (the text launch alone is too small to fill 148 SMs).
def ln_modulate_fwd_pair(x, y, g0, g1, split, mean=None, rstd=None, eps=1e-6):
    """g = (shift, scale, rows_per_batch)"""
    require_cuda(x, y, g0[0], g0[1], g1[0], g1[1])
    assert g0[0].stride(0) == g0[1].stride(0) == g1[0].stride(0) == g1[1].stride(0)
    check(_ln_fwd2(ptr(x), x.stride(0), ptr(y), y.stride(0), ptr(g0[0]), ptr(g0[1]), g0[0].stride(0), g0[2], ptr(mean), ptr(rstd),
                   x.shape[0], x.shape[1], eps, split, ptr(g1[0]), ptr(g1[1]), g1[2], cur_stream()), "qfx_ln_modulate_fwd_pair")


def ln_modulate_bwd_pair(dy, x, mean, rstd, g0, g1, split, dx, dres=None, dx_gated=None):
    """g = (scale, rows_per_batch, gate or None); the gates (both or neither) produce dx_gated = dx * gate"""
    require_cuda(dy, x, mean, rstd, g0[0], g1[0], dx)
    assert g0[0].stride(0) == g1[0].stride(0) and (g0[2] is None) == (g1[2] is None) == (dx_gated is None)
    assert g0[2] is None or g0[2].stride(0) == g1[2].stride(0)
    check(_ln_bwd2(ptr(dy), dy.stride(0), ptr(x), x.stride(0), ptr(mean), ptr(rstd), ptr(g0[0]), g0[0].stride(0), g0[1], ptr(dres),
                   _ld(dres), ptr(dx), dx.stride(0), ptr(g0[2]), _ld(g0[2]), ptr(dx_gated), _ld(dx_gated), x.shape[0], x.shape[1], split,
                   ptr(g1[0]), ptr(g1[2]), g1[1], cur_stream()), "qfx_ln_modulate_bwd_pair")


def qk_norm_rope_fwd_pair(qkv, g0, g1, split, rope, Q, K, V, eps=1e-6, round_mid=True):
    """g = (wq, wk, tokens_per_sample, s_offset)"""
    require_cuda(qkv, g0[0], g0[1], g1[0], g1[1], rope, Q, K, V)
    B, H, S, _ = Q.shape
    bstride = 0 if rope.dim() == 3 else S
    check(_qknr_fwd2(ptr(qkv), qkv.stride(0), ptr(g0[0]), ptr(g0[1]), ptr(rope), bstride, ptr(Q), ptr(K), ptr(V), qkv.shape[0], g0[2],
                     g0[3], S, H, eps, int(round_mid), split, ptr(g1[0]), ptr(g1[1]), g1[2], g1[3], cur_stream()),
          "qfx_qk_norm_rope_fwd_pair")


def qk_norm_rope_bwd_pair(dQ, dK, dV, qkv, g0, g1, split, rope, dqkv, eps=1e-6, round_mid=True, clear_dq=False):
    """clear_dq: dQ (the fp32 accumulator of the attention backward) is zeroed as it is read."""
    require_cuda(dQ, dK, dV, qkv, g0[0], g0[1], g1[0], g1[1], rope, dqkv)
    B, H, S, _ = dK.shape
    bstride = 0 if rope.dim() == 3 else S
    check(_qknr_bwd2(ptr(dQ), ptr(dK), ptr(dV), ptr(qkv), qkv.stride(0), ptr(g0[0]), ptr(g0[1]), ptr(rope), bstride, ptr(dqkv),
                     dqkv.stride(0), qkv.shape[0], g0[2], g0[3], S, H, eps, int(round_mid), split, ptr(g1[0]), ptr(g1[1]), g1[2], g1[3],
                     int(clear_dq), cur_stream()), "qfx_qk_norm_rope_bwd_pair")


def attn_delta_pair(O, dO, delta, g0, g1, split, dO_joint=None):
    """g = (tokens_per_sample, s_offset)"""
    require_cuda(O, dO, delta, dO_joint)
    B, H, S = delta.shape
    check(_delta2(ptr(O), O.stride(0), ptr(dO), dO.stride(0), ptr(delta), ptr(dO_joint), O.shape[0], g0[0], g0[1], S, H, split, g1[0],
                  g1[1], cur_stream()), "qfx_attn_delta_pair")


def ln_modulate_fwd(x, y, shift, scale, rows_per_batch, mean=None, rstd=None, eps=1e-6):
    """shift/scale: [B, D] views (row stride = stride(0)) of the modulation tensor."""
    require_cuda(x, y, shift, scale)
    assert shift.stride(0) == scale.stride(0)
    check(_ln_fwd(ptr(x), x.stride(0), ptr(y), y.stride(0), ptr(shift), ptr(scale), shift.stride(0), rows_per_batch,
                  ptr(mean), ptr(rstd), x.shape[0], x.shape[1], eps, cur_stream()), "qfx_ln_modulate_fwd")


def ln_modulate_bwd(dy, x, mean, rstd, scale, rows_per_batch, dx, dres=None, gate=None, dx_gated=None):
    require_cuda(dy, x, mean, rstd, scale, dx)
    check(_ln_bwd(ptr(dy), dy.stride(0), ptr(x), x.stride(0), ptr(mean), ptr(rstd), ptr(scale), scale.stride(0),
                  rows_per_batch, ptr(dres), _ld(dres), ptr(dx), dx.stride(0), ptr(gate), _ld(gate), ptr(dx_gated),
                  _ld(dx_gated), x.shape[0], x.shape[1], cur_stream()), "qfx_ln_modulate_bwd")


def mod_grad(g, rows_per_batch, sum_out=None, m=None, prod_out=None, mean=None, rstd=None):
    """Modulation-vector gradients, accumulated (+=) into fp32 [B, D] views: sum_out += sum_t g ; prod_out += sum_t g * m',
    m' = bf16((m - mean) * rstd) when the row statistics are given (d scale), else m itself (d gate)."""
    require_cuda(g, m, sum_out, prod_out, mean, rstd)
    o = sum_out if sum_out is not None else prod_out
    assert o.dtype == torch.float32 and (sum_out is None or prod_out is None or sum_out.stride(0) == prod_out.stride(0))
    check(_mod_grad(ptr(g), g.stride(0), ptr(m), _ld(m), ptr(mean), ptr(rstd), rows_per_batch, ptr(sum_out), ptr(prod_out),
                    o.stride(0), g.shape[0], g.shape[1], cur_stream()), "qfx_mod_grad")


def gate_mul(a, gate, rows_per_batch, out):
    require_cuda(a, gate, out)
    check(_gate_mul(ptr(a), a.stride(0), ptr(gate), gate.stride(0), rows_per_batch, ptr(out), out.stride(0), a.shape[0],
                    a.shape[1], cur_stream()), "qfx_gate_mul")


_add = _sig("qfx_add_bf16", _vp, _vp, _vp, _i64, _vp)


def add_bf16(a, b, out):
    require_cuda(a, b, out)
    assert a.is_contiguous() and b.is_contiguous() and out.is_contiguous()
    check(_add(ptr(a), ptr(b), ptr(out), a.numel(), cur_stream()), "qfx_add_bf16")


def rmsnorm_rows(x, w, y, eps=1e-6):
    require_cuda(x, w, y)
    check(_rms_rows(ptr(x), x.stride(0), ptr(w), ptr(y), y.stride(0), x.shape[0], x.shape[1], eps, cur_stream()),
          "qfx_rmsnorm_rows")


def qk_norm_rope_fwd(qkv, wq, wk, rope, Q, K, V, tokens_per_sample, s_offset, eps=1e-6, round_mid=True):
    """qkv [tokens, 3*H*128]; rope fp32 [S,64,2] (shared) or [B,S,64,2]; Q/K/V [B,H,S,128]."""
    require_cuda(qkv, wq, wk, rope, Q, K, V)
    B, H, S, _ = Q.shape
    bstride = 0 if rope.dim() == 3 else S
    check(_qknr_fwd(ptr(qkv), qkv.stride(0), ptr(wq), ptr(wk), ptr(rope), bstride, ptr(Q), ptr(K), ptr(V), qkv.shape[0],
                    tokens_per_sample, s_offset, S, H, eps, int(round_mid), cur_stream()), "qfx_qk_norm_rope_fwd")


def qk_norm_rope_bwd(dQ, dK, dV, qkv, wq, wk, rope, dqkv, tokens_per_sample, s_offset, eps=1e-6, round_mid=True):
    require_cuda(dQ, dK, dV, qkv, wq, wk, rope, dqkv)
    B, H, S, _ = dK.shape
    bstride = 0 if rope.dim() == 3 else S
    check(_qknr_bwd(ptr(dQ), ptr(dK), ptr(dV), ptr(qkv), qkv.stride(0), ptr(wq), ptr(wk), ptr(rope), bstride, ptr(dqkv),
                    dqkv.stride(0), qkv.shape[0], tokens_per_sample, s_offset, S, H, eps, int(round_mid), cur_stream()),
          "qfx_qk_norm_rope_bwd")


def gemv_act(x, W, bias, y, act=0):
    """y[b, :] = act_in(x[b]) @ W^T + bias ; act: 0 none, 1 SiLU.  x [B<=8, K], W [N, K]."""
    require_cuda(x, W, bias, y)
    check(_gemv(ptr(x), x.stride(0), ptr(W), W.stride(0), ptr(bias), ptr(y), y.stride(0), x.shape[0], W.shape[0], W.shape[1],
                act, cur_stream()), "qfx_gemv_act")


def timestep_sinusoid(t_f32, scale, out):
    require_cuda(t_f32, out)
    check(_tsin(ptr(t_f32), scale, ptr(out), out.shape[0], out.shape[1], cur_stream()), "qfx_timestep_sinusoid")


def flow_noisy_input(x0, noise, control, sigma_f32, packed):
    require_cuda(x0, noise, control, sigma_f32, packed)
    B, L, Cc = x0.shape
    check(_noisy(ptr(x0), ptr(noise), ptr(control), ptr(sigma_f32), ptr(packed), B, L, control.shape[1], Cc, cur_stream()),
          "qfx_flow_noisy_input")


_noisy_var = _sig("qfx_flow_noisy_input_var", _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp)


def flow_noisy_input_var(x0, noise, control, sigma_f32, Lt, Lc, packed):
    """per-sample lengths Lt/Lc (int32 [B]): packed[b] = [noisy target | control | 0]."""
    require_cuda(x0, noise, control, sigma_f32, Lt, Lc, packed)
    B, Ltmax, Cc = x0.shape
    check(_noisy_var(ptr(x0), ptr(noise), ptr(control), ptr(sigma_f32), ptr(Lt), ptr(Lc), ptr(packed), B, Ltmax, control.shape[1],
                     packed.shape[1], Cc, cur_stream()), "qfx_flow_noisy_input_var")


def flow_loss(pred, x0, noise, w, norm, loss, dpred=None, grad_scale=1.0):
    require_cuda(pred, x0, noise, w, loss, dpred)
    B, L, Cc = x0.shape
    check(_floss(ptr(pred), ptr(x0), ptr(noise), ptr(w), norm, grad_scale, ptr(loss), ptr(dpred), B, L, pred.shape[1], Cc,
                 cur_stream()), "qfx_flow_loss")


class AdamWTensor(C.Structure):
    _fields_ = [("param", C.c_void_p), ("grad_offset", C.c_int64), ("numel", C.c_int), ("cols", C.c_int), ("ld", C.c_int64)]


ADAMW_CHUNK = 4096
_adamw = _sig("qfx_fused_adamw", _vp, _vp, _i, _vp, _i64, _vp, _vp, _vp, _f, _f, _f, _f, _f, _f, _f, _i, _vp)


def adamw_tables(members, device):
    """members: iterable of (param tensor [rows, cols] bf16 with unit column stride, grad offset).  Returns the device tables
    (tensor descriptors as a uint8 tensor, chunk list int32 [n, 2]) qfx_fused_adamw walks."""
    members = list(members)
    arr = (AdamWTensor * len(members))()
    chunks = []
    for i, (p, off) in enumerate(members):
        assert p.dtype == torch.bfloat16 and p.dim() == 2 and p.stride(1) == 1
        arr[i] = AdamWTensor(p.data_ptr(), off, p.numel(), p.shape[1], p.stride(0))
        chunks += [(i, e) for e in range(0, p.numel(), ADAMW_CHUNK)]
    raw = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).clone().to(device)
    return raw, torch.tensor(chunks, dtype=torch.int32).to(device)


def fused_adamw(tables, grad, exp_avg, exp_avg_sq, sumsq, pre_scale, max_norm, lr, beta1, beta2, eps, weight_decay, step):
    """Clip (global L2 norm of grad * pre_scale) + AdamW on every tensor of `tables` in place; fp32 grad / moments."""
    raw, chunks = tables
    require_cuda(raw, chunks, grad, exp_avg, exp_avg_sq, sumsq)
    check(_adamw(ptr(raw), ptr(chunks), chunks.shape[0], ptr(grad), grad.numel(), ptr(exp_avg), ptr(exp_avg_sq), ptr(sumsq),
                 float(pre_scale), float(max_norm), float(lr), float(beta1), float(beta2), float(eps), float(weight_decay),
                 int(step), cur_stream()), "qfx_fused_adamw")


# Prodigy (qfx.h qfx_fused_prodigy): the device scalars' slots, and the scratch rule restated (the C side refuses less).
PRODIGY_SCALARS = 8
PRODIGY_D, PRODIGY_D_MAX, PRODIGY_D_NUM, PRODIGY_K, PRODIGY_DLR, PRODIGY_SKIPPED, PRODIGY_D_DEN, PRODIGY_D_HAT = range(8)
_d = C.c_double
_prodigy = _sig("qfx_fused_prodigy", _vp, _vp, _i, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _f, _f, _d, _d, _d, _d, _d, _d,
                _i, _i, _i, _d, _d, _d, _vp)


def prodigy_scratch_floats(tables):
    return DET_NORM_PARTIALS + 4 * tables[1].shape[0]


def fused_prodigy(tables, grad, exp_avg, exp_avg_sq, s, p0, scalars, sumsq, scratch, pre_scale, max_norm, lr, beta1, beta2, beta3, eps,
                  weight_decay, decouple, use_bias_correction, safeguard_warmup, d0, d_coef, growth_rate):
    """Clip + one Prodigy step on every tensor of `tables` in place (qfx.h); fp32 grad / m / v / s, bf16 p0, fp64 scalars, lr > 0."""
    raw, chunks = tables
    require_cuda(raw, chunks, grad, exp_avg, exp_avg_sq, s, p0, scalars, sumsq, scratch)
    assert p0.dtype == torch.bfloat16 and scalars.dtype == torch.float64 and scalars.numel() == PRODIGY_SCALARS
    check(_prodigy(ptr(raw), ptr(chunks), chunks.shape[0], ptr(grad), grad.numel(), ptr(exp_avg), ptr(exp_avg_sq), ptr(s), ptr(p0),
                   ptr(scalars), ptr(sumsq), *_scratch(scratch), float(pre_scale), float(max_norm), float(lr), float(beta1), float(beta2),
                   float(beta3), float(eps), float(weight_decay), int(bool(decouple)), int(bool(use_bias_correction)),
                   int(bool(safeguard_warmup)), float(d0), float(d_coef), float(growth_rate), cur_stream()), "qfx_fused_prodigy")


# 8-bit Adam (qfx.h qfx_fused_adam8bit)
ADAM8BIT_BLOCK = 256
_adam8bit = _sig("qfx_fused_adam8bit", _vp, _vp, _i, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _f, _f, _f, _f, _f,
                 _f, _f, _i, _i, _vp)


def dynamic_map(signed: bool):
    """bitsandbytes' `functional.create_dynamic_map(signed)` with its defaults (7 exponent bits, 8 bits): 256 sorted fp32 values,
    built the way bitsandbytes builds them (fp32 linspace means, scaled in Python floats)."""
    data = []
    for i in range(7):
        items = 2 ** i + 1 if signed else 2 ** (i + 1) + 1
        b = torch.linspace(0.1, 1, items, dtype=torch.float32)
        means = (b[:-1] + b[1:]) / 2.0
        data += ((10 ** (-6 + i)) * means).tolist()
        if signed:
            data += (-(10 ** (-6 + i)) * means).tolist()
    data += [0, 1.0]
    return torch.tensor(sorted(data), dtype=torch.float32)


def adam8bit_layout(members, min_8bit_size):
    """Per tensor of `members` ((param, grad offset) pairs, as adamw_tables takes them): the offset of its absmax blocks (numel >=
    min_8bit_size) or of its fp32 states (smaller tensors), in member order.  Returns (offsets, absmax values, fp32 state elements)."""
    offsets, n_absmax, n_small = [], 0, 0
    for p, _ in members:
        n = p.numel()
        if n >= min_8bit_size:
            offsets.append(n_absmax)
            n_absmax += -(-n // ADAM8BIT_BLOCK)
        else:
            offsets.append(n_small)
            n_small += n
    return offsets, n_absmax, n_small


def fused_adam8bit(tables, state_offsets, grad, state1, state2, absmax1, absmax2, s1_32, s2_32, qmap1, qmap2, sumsq, scratch, pre_scale,
                   max_norm, lr, beta1, beta2, eps, weight_decay, step, min_8bit_size):
    """Clip + one bitsandbytes Adam8bit step on every tensor of `tables` in place (qfx.h): fp32 grad, uint8 codes [n_grad], fp32 absmax
    and small-tensor states at `state_offsets` (int64 device tensor, adam8bit_layout), fp32 maps [256]."""
    raw, chunks = tables
    require_cuda(raw, chunks, state_offsets, grad, state1, state2, absmax1, absmax2, s1_32, s2_32, qmap1, qmap2, sumsq, scratch)
    assert state1.dtype == state2.dtype == torch.uint8 and state_offsets.dtype == torch.int64 and qmap1.numel() == qmap2.numel() == 256
    check(_adam8bit(ptr(raw), ptr(chunks), chunks.shape[0], ptr(state_offsets), ptr(grad), grad.numel(), ptr(state1), ptr(state2),
                    ptr(absmax1), ptr(absmax2), ptr(s1_32), ptr(s2_32), ptr(qmap1), ptr(qmap2), ptr(sumsq), *_scratch(scratch),
                    float(pre_scale), float(max_norm), float(lr), float(beta1), float(beta2), float(eps), float(weight_decay), int(step),
                    int(min_8bit_size), cur_stream()), "qfx_fused_adam8bit")


# Sharded optimizer state (qfx.h "slice forms"; optim.py shard_state=True).  `chunk_range` = (c0, c1) selects entries [c0, c1) of the
# tables' chunk list (sharding.SlicePlan); the state arrays hold the flat-gradient range starting at `state_base`.
_sumsq_det = _sig("qfx_sumsq_det", _vp, _i64, _f, _vp, _vp, _i64, _vp)
_adamw_slice = _sig("qfx_fused_adamw_slice", _vp, _vp, _i, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _f, _f, _f, _f, _f, _f, _f, _i, _vp)
_adam8bit_slice = _sig("qfx_fused_adam8bit_slice", _vp, _vp, _i, _vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                       _f, _f, _f, _f, _f, _f, _f, _i, _i, _vp)
_prodigy_a = _sig("qfx_prodigy_slice_partials", _vp, _vp, _i, _i, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _f, _f,
                  _d, _d, _d, _d, _d, _i, _i, _i, _d, _vp)
_prodigy_b = _sig("qfx_prodigy_slice_update", _vp, _vp, _i, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _i, _d, _d, _d, _d, _d, _d, _i, _i, _d,
                  _d, _d, _vp)
_pack = _sig("qfx_lora_pack", _vp, _vp, _i, _i64, _i64, _vp, _vp)
_unpack = _sig("qfx_lora_unpack", _vp, _vp, _i, _i64, _i64, _vp, _vp)
_KERNELS_PER_CALL.update({"qfx_sumsq_det": 2, "qfx_prodigy_slice_update": 2})


def _sub_chunks(tables, chunk_range):
    """(tensor table pointer, pointer to chunk c0, number of chunks) of a chunk range."""
    raw, chunks = tables
    c0, c1 = chunk_range
    assert 0 <= c0 <= c1 <= chunks.shape[0]
    return ptr(raw), C.c_void_p(chunks.data_ptr() + 8 * c0), c1 - c0


def sumsq_det(x, pre_scale, out, *, scratch):
    """out[0] = ||x * pre_scale||^2 (fp32, x contiguous, any length), summed in a fixed order."""
    require_cuda(x, out, scratch)
    assert x.dtype == torch.float32 and x.is_contiguous()
    check(_sumsq_det(ptr(x), x.numel(), float(pre_scale), ptr(out), *_scratch(scratch), cur_stream()), "qfx_sumsq_det")


def _state(t, n):
    assert t.is_contiguous() and t.numel() >= n
    return ptr(t)


def fused_adamw_slice(tables, chunk_range, state_base, grad, exp_avg, exp_avg_sq, sumsq, pre_scale, max_norm, lr, beta1, beta2, eps,
                      weight_decay, step):
    """fused_adamw on the chunks of `chunk_range`, with moments of the slice only and the clip from the given sumsq."""
    require_cuda(grad, exp_avg, exp_avg_sq, sumsq)
    n = exp_avg.numel()
    check(_adamw_slice(*_sub_chunks(tables, chunk_range), ptr(grad), grad.numel(), int(state_base), n, _state(exp_avg, n),
                       _state(exp_avg_sq, n), ptr(sumsq), float(pre_scale), float(max_norm), float(lr), float(beta1), float(beta2),
                       float(eps), float(weight_decay), int(step), cur_stream()), "qfx_fused_adamw_slice")


def fused_adam8bit_slice(tables, chunk_range, state_base, state_offsets, grad, state1, state2, absmax1, absmax2, s1_32, s2_32, qmap1,
                         qmap2, sumsq, pre_scale, max_norm, lr, beta1, beta2, eps, weight_decay, step, min_8bit_size):
    """fused_adam8bit on the chunks of `chunk_range`: codes of the slice, the slice's absmax / fp32 states at its own `state_offsets`."""
    require_cuda(state_offsets, grad, state1, state2, absmax1, absmax2, s1_32, s2_32, qmap1, qmap2, sumsq)
    assert state1.dtype == state2.dtype == torch.uint8 and state_offsets.dtype == torch.int64 and qmap1.numel() == qmap2.numel() == 256
    n = state1.numel()
    check(_adam8bit_slice(*_sub_chunks(tables, chunk_range), ptr(state_offsets), ptr(grad), grad.numel(), int(state_base), n,
                          _state(state1, n), _state(state2, n), ptr(absmax1), ptr(absmax2), ptr(s1_32), ptr(s2_32), ptr(qmap1), ptr(qmap2),
                          ptr(sumsq), float(pre_scale), float(max_norm), float(lr), float(beta1), float(beta2), float(eps),
                          float(weight_decay), int(step), int(min_8bit_size), cur_stream()), "qfx_fused_adam8bit_slice")


def prodigy_slice_partials(tables, chunk_range, state_base, grad, exp_avg, exp_avg_sq, s, p0, scalars, sumsq, part, pre_scale, max_norm,
                           lr, beta1, beta2, beta3, weight_decay, decouple, use_bias_correction, safeguard_warmup, d0):
    """Pass A of fused_prodigy on the slice; its chunks' fp64 partials go to part[2 c], part[2 c + 1] (c = the chunk's index in the
    full table; part holds 2 x every chunk)."""
    require_cuda(grad, exp_avg, exp_avg_sq, s, p0, scalars, sumsq, part)
    assert p0.dtype == torch.bfloat16 and scalars.dtype == part.dtype == torch.float64 and part.is_contiguous()
    n = exp_avg.numel()
    check(_prodigy_a(*_sub_chunks(tables, chunk_range), int(chunk_range[0]), ptr(grad), grad.numel(), int(state_base), n,
                     _state(exp_avg, n), _state(exp_avg_sq, n), _state(s, n), _state(p0, n), ptr(scalars), ptr(sumsq), ptr(part),
                     part.numel() // 2, float(pre_scale), float(max_norm), float(lr), float(beta1), float(beta2), float(beta3),
                     float(weight_decay), int(bool(decouple)), int(bool(use_bias_correction)), int(bool(safeguard_warmup)), float(d0),
                     cur_stream()), "qfx_prodigy_slice_partials")


def prodigy_slice_update(tables, chunk_range, state_base, n_grad, exp_avg, exp_avg_sq, scalars, part, lr, beta1, beta2, beta3, eps,
                         weight_decay, decouple, use_bias_correction, d0, d_coef, growth_rate):
    """The scalar update of fused_prodigy from every chunk's partials in `part`, then pass B on the slice."""
    require_cuda(exp_avg, exp_avg_sq, scalars, part)
    assert scalars.dtype == part.dtype == torch.float64 and scalars.numel() == PRODIGY_SCALARS
    n = exp_avg.numel()
    check(_prodigy_b(*_sub_chunks(tables, chunk_range), int(n_grad), int(state_base), n, _state(exp_avg, n), _state(exp_avg_sq, n),
                     ptr(scalars), ptr(part), part.numel() // 2, float(lr), float(beta1), float(beta2), float(beta3), float(eps),
                     float(weight_decay), int(bool(decouple)), int(bool(use_bias_correction)), float(d0), float(d_coef), float(growth_rate),
                     cur_stream()), "qfx_prodigy_slice_update")


def lora_pack(tables, chunk_range, g_lo, g_hi, flat):
    """flat[fi - g_lo] = the LoRA weight at flat-gradient offset fi, for fi in [g_lo, g_hi) within the chunks of `chunk_range`."""
    require_cuda(flat)
    assert flat.dtype == torch.bfloat16 and flat.is_contiguous() and flat.numel() >= g_hi - g_lo
    check(_pack(*_sub_chunks(tables, chunk_range), int(g_lo), int(g_hi), ptr(flat), cur_stream()), "qfx_lora_pack")


def lora_unpack(tables, chunk_range, g_lo, g_hi, flat):
    """The inverse of lora_pack: the LoRA weights at offsets [g_lo, g_hi) within the chunks of `chunk_range` = flat[fi - g_lo]."""
    require_cuda(flat)
    assert flat.dtype == torch.bfloat16 and flat.is_contiguous() and flat.numel() >= g_hi - g_lo
    check(_unpack(*_sub_chunks(tables, chunk_range), int(g_lo), int(g_hi), ptr(flat), cur_stream()), "qfx_lora_unpack")


def lora_wgrad(P, Q, G, gs_i, gs_j, r):
    """G[i*gs_i + j*gs_j] += sum_m P[m,i] Q[m,j], j < r.  G fp32."""
    require_cuda(P, Q, G)
    check(_wgrad(ptr(P), P.stride(0), ptr(Q), Q.stride(0), ptr(G), gs_i, gs_j, P.shape[0], P.shape[1], r, cur_stream()),
          "qfx_lora_wgrad")


_wgrad_tc = _sig("qfx_lora_wgrad_tc", _vp, _i64, _i, _vp, _i64, _i, _i, _i, _i, C.POINTER(C.c_void_p), _i64, _i64, _i, _vp)


def lora_wgrad_tc(A, B, G_list, gs_i, gs_j, r, mode=0, Dg=0):
    """wgmma LoRA weight gradient: G_g += A^T B_g over rows, r <= 128.  A [M, Na], B [M, Rp*G] bf16 with Rp = 64 * ceil(r / 64), group
    g's columns [g*Rp, g*Rp + r); G_list: fp32 tensors (one per group).  mode 0: all A columns pair with every group; mode 1: A columns
    [g*Dg, (g+1)*Dg) pair with group g only."""
    require_cuda(A, B, *G_list)
    n = len(G_list)
    arr = (C.c_void_p * n)(*[g.data_ptr() for g in G_list])
    check(_wgrad_tc(ptr(A), A.stride(0), A.shape[1], ptr(B), B.stride(0), n, A.shape[0], mode, Dg, arr, gs_i, gs_j, r,
                    cur_stream()), "qfx_lora_wgrad_tc")


def attn_delta(O, dO, delta, tokens_per_sample, s_offset, dO_joint=None):
    """delta[b,h,s] = sum_d O*dO for token-major O/dO rows; optionally scatters dO into the joint [B,H,S,128] layout."""
    require_cuda(O, dO, delta, dO_joint)
    B, H, S = delta.shape
    check(_delta(ptr(O), O.stride(0), ptr(dO), dO.stride(0), ptr(delta), ptr(dO_joint), O.shape[0], tokens_per_sample,
                 s_offset, S, H, cur_stream()), "qfx_attn_delta")


def attn_bwd(Q, K, V, dO, lse, delta, dQ_accum, dK, dV, kv_len=None, scale=None, txt_len=None, split=0):
    """All [B,H,S,128]; dQ_accum fp32 and zeroed by the caller; lse/delta [B,H,S] fp32."""
    require_cuda(Q, K, V, dO, lse, delta, dQ_accum, dK, dV, kv_len, txt_len)
    B, H, S, d = Q.shape
    assert d == 128 and dQ_accum.dtype == torch.float32
    scale = scale if scale is not None else d ** -0.5
    check(_attn_bwd(ptr(Q), ptr(K), ptr(V), ptr(dO), ptr(lse), ptr(delta), ptr(dQ_accum), ptr(dK), ptr(dV), ptr(kv_len),
                    ptr(txt_len), split, B, H, S, scale, cur_stream()), "qfx_attn_bwd")


def grad_finalize(g_f32, pre_scale, max_norm, sumsq, out_bf16):
    require_cuda(g_f32, sumsq, out_bf16)
    check(_gfin(ptr(g_f32), g_f32.numel(), pre_scale, max_norm, ptr(sumsq), ptr(out_bf16), cur_stream()), "qfx_grad_finalize")


def attn_fwd(Q, K, V, out_txt, out_img, split, lse=None, kv_len=None, scale=None, txt_len=None):
    """Q/K/V [B,H,S,128]; rows s<split of sample b -> out_txt[b*split + s], others -> out_img[b*(S-split) + s-split]."""
    require_cuda(Q, K, V, out_txt, out_img, lse, kv_len, txt_len)
    B, H, S, d = Q.shape
    assert d == 128 and Q.is_contiguous() and K.is_contiguous() and V.is_contiguous()
    scale = scale if scale is not None else d ** -0.5
    check(_attn_fwd(ptr(Q), ptr(K), ptr(V), ptr(out_txt), _ld(out_txt), split, ptr(out_img), _ld(out_img), S - split, split,
                    ptr(lse), ptr(kv_len), ptr(txt_len), B, H, S, scale, cur_stream()), "qfx_attn_fwd")


# ---------------------------------------------------------------------------------------------------- deterministic variants
# Picked by the model under torch.use_deterministic_algorithms(True): the same operations without floating-point atomics (qfx.h).
# The reductions take caller-owned fp32 scratch; the det_scratch_* rules below restate qfx.h's size rules (the C side refuses less).
DET_WGRAD_CTAS, DET_MODGRAD_CTAS, DET_LOSS_PARTIALS, DET_NORM_PARTIALS = 264, 528, 296, 592


def _cdiv(a, b):
    return -(-a // b)


def det_scratch_wgrad_tc(M, Na, ng, r):
    """fp32 scratch of qfx_lora_wgrad_tc_det; ng = 1 for mode 1, else the number of groups.  The split count does not depend on r,
    so for r > 64 (two 64-wide rank chunks per group, each its own CTA) the rule is the same: splits x Na x ng x r floats."""
    splits = max(1, min(_cdiv(M, 256), _cdiv(DET_WGRAD_CTAS, Na // 128)))
    rows = _cdiv(_cdiv(M, splits), 64) * 64
    return _cdiv(M, rows) * Na * ng * r


def det_scratch_wgrad(M, Dp, r):
    rows = _cdiv(_cdiv(M, _cdiv(M, 512)), 64) * 64
    return _cdiv(M, rows) * Dp * r


def det_scratch_mod_grad(M, rows_per_batch, D):
    B = M // rows_per_batch
    cb = _cdiv(D, 256)
    splits = max(1, min(_cdiv(rows_per_batch, 32), _cdiv(DET_MODGRAD_CTAS, cb * B)))
    return splits * 2 * B * D


def _scratch(t):
    assert t.dtype == torch.float32 and t.is_contiguous()
    return ptr(t), t.numel()


_attn_bwd_det = _sig("qfx_attn_bwd_det", _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _vp)
_wgrad_tc_det = _sig("qfx_lora_wgrad_tc_det", _vp, _i64, _i, _vp, _i64, _i, _i, _i, _i, C.POINTER(C.c_void_p), _i64, _i64, _i, _vp,
                     _i64, _vp)
_wgrad_det = _sig("qfx_lora_wgrad_det", _vp, _i64, _vp, _i64, _vp, _i64, _i64, _i, _i, _i, _vp, _i64, _vp)
_mod_grad_det = _sig("qfx_mod_grad_det", _vp, _i64, _vp, _i64, _vp, _vp, _i, _vp, _vp, _i64, _i, _i, _vp, _i64, _vp)
_floss_det = _sig("qfx_flow_loss_det", _vp, _vp, _vp, _vp, _f, _f, _vp, _vp, _i, _i, _i, _i, _vp, _i64, _vp)
_gfin_det = _sig("qfx_grad_finalize_det", _vp, _i64, _f, _f, _vp, _vp, _vp, _i64, _vp)
_adamw_det = _sig("qfx_fused_adamw_det", _vp, _vp, _i, _vp, _i64, _vp, _vp, _vp, _f, _f, _f, _f, _f, _f, _f, _i, _vp, _i64, _vp)


def attn_bwd_det(Q, K, V, dO, lse, delta, dQ_accum, dK, dV, kv_len=None, scale=None, txt_len=None, split=0):
    """attn_bwd without atomics: dQ_accum (prefilled by the caller) receives every element once."""
    require_cuda(Q, K, V, dO, lse, delta, dQ_accum, dK, dV, kv_len, txt_len)
    B, H, S, d = Q.shape
    assert d == 128 and dQ_accum.dtype == torch.float32
    scale = scale if scale is not None else d ** -0.5
    check(_attn_bwd_det(ptr(Q), ptr(K), ptr(V), ptr(dO), ptr(lse), ptr(delta), ptr(dQ_accum), ptr(dK), ptr(dV), ptr(kv_len),
                        ptr(txt_len), split, B, H, S, scale, cur_stream()), "qfx_attn_bwd_det")


def lora_wgrad_tc_det(A, B, G_list, gs_i, gs_j, r, mode=0, Dg=0, *, scratch):
    require_cuda(A, B, scratch, *G_list)
    n = len(G_list)
    arr = (C.c_void_p * n)(*[g.data_ptr() for g in G_list])
    check(_wgrad_tc_det(ptr(A), A.stride(0), A.shape[1], ptr(B), B.stride(0), n, A.shape[0], mode, Dg, arr, gs_i, gs_j, r,
                        *_scratch(scratch), cur_stream()), "qfx_lora_wgrad_tc_det")


def lora_wgrad_det(P, Q, G, gs_i, gs_j, r, *, scratch):
    require_cuda(P, Q, G, scratch)
    check(_wgrad_det(ptr(P), P.stride(0), ptr(Q), Q.stride(0), ptr(G), gs_i, gs_j, P.shape[0], P.shape[1], r, *_scratch(scratch),
                     cur_stream()), "qfx_lora_wgrad_det")


def mod_grad_det(g, rows_per_batch, sum_out=None, m=None, prod_out=None, mean=None, rstd=None, *, scratch):
    require_cuda(g, m, sum_out, prod_out, mean, rstd, scratch)
    o = sum_out if sum_out is not None else prod_out
    assert o.dtype == torch.float32 and (sum_out is None or prod_out is None or sum_out.stride(0) == prod_out.stride(0))
    check(_mod_grad_det(ptr(g), g.stride(0), ptr(m), _ld(m), ptr(mean), ptr(rstd), rows_per_batch, ptr(sum_out), ptr(prod_out),
                        o.stride(0), g.shape[0], g.shape[1], *_scratch(scratch), cur_stream()), "qfx_mod_grad_det")


def flow_loss_det(pred, x0, noise, w, norm, loss, dpred=None, grad_scale=1.0, *, scratch):
    require_cuda(pred, x0, noise, w, loss, dpred, scratch)
    B, L, Cc = x0.shape
    check(_floss_det(ptr(pred), ptr(x0), ptr(noise), ptr(w), norm, grad_scale, ptr(loss), ptr(dpred), B, L, pred.shape[1], Cc,
                     *_scratch(scratch), cur_stream()), "qfx_flow_loss_det")


def grad_finalize_det(g_f32, pre_scale, max_norm, sumsq, out_bf16, *, scratch):
    require_cuda(g_f32, sumsq, out_bf16, scratch)
    check(_gfin_det(ptr(g_f32), g_f32.numel(), pre_scale, max_norm, ptr(sumsq), ptr(out_bf16), *_scratch(scratch), cur_stream()),
          "qfx_grad_finalize_det")


def fused_adamw_det(tables, grad, exp_avg, exp_avg_sq, sumsq, pre_scale, max_norm, lr, beta1, beta2, eps, weight_decay, step, *,
                    scratch):
    raw, chunks = tables
    require_cuda(raw, chunks, grad, exp_avg, exp_avg_sq, sumsq, scratch)
    check(_adamw_det(ptr(raw), ptr(chunks), chunks.shape[0], ptr(grad), grad.numel(), ptr(exp_avg), ptr(exp_avg_sq), ptr(sumsq),
                     float(pre_scale), float(max_norm), float(lr), float(beta1), float(beta2), float(eps), float(weight_decay),
                     int(step), *_scratch(scratch), cur_stream()), "qfx_fused_adamw_det")


# ---------------------------------------------------------------------------------------------------- NF4 frozen weights (nf4.py)
class Nf4Segment(C.Structure):
    _fields_ = [("codes", C.c_void_p), ("absmax", C.c_void_p), ("out", C.c_void_p), ("n", C.c_int64), ("blocksize", C.c_int)]


NF4_MAX_SEGMENTS = 8
_nf4 = _sig("qfx_nf4_dequant", C.POINTER(Nf4Segment), _i, _vp)


def nf4_dequant(segments):
    """segments: [(codes uint8 [n/2], absmax fp32 [n/blocksize], out bf16 [n], blocksize)], contiguous; ONE launch fills every out."""
    arr = (Nf4Segment * len(segments))()
    for i, (codes, absmax, out, bs) in enumerate(segments):
        require_cuda(codes, absmax, out)
        n = out.numel()
        assert codes.dtype == torch.uint8 and absmax.dtype == torch.float32 and out.dtype == torch.bfloat16
        assert codes.is_contiguous() and absmax.is_contiguous() and out.is_contiguous()
        assert codes.numel() * 2 == n and absmax.numel() * bs == n
        arr[i] = Nf4Segment(codes.data_ptr(), absmax.data_ptr(), out.data_ptr(), n, bs)
    check(_nf4(arr, len(segments), cur_stream()), "qfx_nf4_dequant")


# ---------------------------------------------------------------------------------------------------- FP8 frozen weights (fp8.py)
class Fp8Segment(C.Structure):
    _fields_ = [("codes", C.c_void_p), ("out", C.c_void_p), ("n", C.c_int64)]


FP8_MAX_SEGMENTS = 8
_fp8 = _sig("qfx_fp8_expand", C.POINTER(Fp8Segment), _i, _vp)


def fp8_expand(segments):
    """segments: [(codes float8_e4m3fn or uint8 [n], out bf16 [n])], contiguous; ONE launch fills every out with bf16(codes),
    exact for every finite code."""
    arr = (Fp8Segment * len(segments))()
    for i, (codes, out) in enumerate(segments):
        require_cuda(codes, out)
        assert codes.dtype in (torch.float8_e4m3fn, torch.uint8) and out.dtype == torch.bfloat16
        assert codes.is_contiguous() and out.is_contiguous() and codes.numel() == out.numel()
        arr[i] = Fp8Segment(codes.data_ptr(), out.data_ptr(), out.numel())
    check(_fp8(arr, len(segments), cur_stream()), "qfx_fp8_expand")


# ---------------------------------------------------------------------------------------------------- peer memory (sharding.py)
PEER_HANDLE_BYTES = 64
for _f in ("qfx_peer_alloc", "qfx_peer_free", "qfx_peer_open", "qfx_peer_close", "qfx_peer_copy_async"):
    getattr(_lib, _f).restype = C.c_int
_lib.qfx_peer_alloc.argtypes = [C.c_int64, C.POINTER(C.c_void_p), C.c_char_p]
_lib.qfx_peer_free.argtypes = [C.c_void_p]
_lib.qfx_peer_open.argtypes = [C.c_char_p, C.POINTER(C.c_void_p)]
_lib.qfx_peer_close.argtypes = [C.c_void_p]
_lib.qfx_peer_copy_async.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]


def _rc(rc: int, what: str):  # like check(), but these are not kernel launches
    if rc != 0:
        raise QfxError(f"{what} failed (rc={rc}): {_lib.qfx_last_error().decode()}")


class PeerBuffer:
    """A device allocation other ranks of the node can map (CUDA IPC).  `.tensor(dtype, shape)` views it as a torch tensor."""

    def __init__(self, nbytes: int, device):
        self.nbytes, self.device = int(nbytes), torch.device(device)
        p, h = C.c_void_p(), C.create_string_buffer(PEER_HANDLE_BYTES)
        with torch.cuda.device(self.device):
            _rc(_lib.qfx_peer_alloc(self.nbytes, C.byref(p), h), "qfx_peer_alloc")
        self.ptr, self.handle = p.value, h.raw

    @property
    def __cuda_array_interface__(self):
        return dict(shape=(self.nbytes,), typestr="|u1", data=(self.ptr, False), version=2)

    def tensor(self, dtype, shape):
        return torch.as_tensor(self, device=self.device).view(dtype).view(shape)

    def free(self):
        if self.ptr:
            _rc(_lib.qfx_peer_free(C.c_void_p(self.ptr)), "qfx_peer_free")
            self.ptr = 0


def peer_open(handle: bytes, device) -> int:
    p = C.c_void_p()
    with torch.cuda.device(device):
        _rc(_lib.qfx_peer_open(handle, C.byref(p)), "qfx_peer_open")
    return p.value


def peer_close(p: int):
    _rc(_lib.qfx_peer_close(C.c_void_p(p)), "qfx_peer_close")


def peer_copy_async(dst_ptr: int, src_ptr: int, nbytes: int, stream=None):
    s = cur_stream() if stream is None else C.c_void_p(stream.cuda_stream)
    _rc(_lib.qfx_peer_copy_async(C.c_void_p(dst_ptr), C.c_void_p(src_ptr), int(nbytes), s), "qfx_peer_copy_async")


# ---------------------------------------------------------------------------------------------------- data-parallel sum (sharding.py)
MAX_RANKS = 8
_dp_reduce = _sig("qfx_dp_reduce_det", C.POINTER(C.c_void_p), _i, _vp, _i64, _vp)


def dp_reduce_det(srcs, dst):
    """dst = ((+0 + srcs[0]) + srcs[1]) + ... elementwise in fp32, in list order, bit-reproducible.  srcs: fp32 tensors of dst's
    numel, or raw device pointers to that many floats (peer mappings); dst may be one of them, but may not otherwise overlap one."""
    require_cuda(dst)
    assert dst.dtype == torch.float32 and dst.is_contiguous() and 1 <= len(srcs) <= MAX_RANKS
    ptrs = (C.c_void_p * len(srcs))()
    for i, s in enumerate(srcs):
        if torch.is_tensor(s):
            require_cuda(s)
            assert s.dtype == torch.float32 and s.is_contiguous() and s.numel() == dst.numel()
            s = s.data_ptr()
        ptrs[i] = s
    check(_dp_reduce(ptrs, len(srcs), ptr(dst), dst.numel(), cur_stream()), "qfx_dp_reduce_det")
