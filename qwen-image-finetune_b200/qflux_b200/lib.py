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
_KERNELS_PER_CALL = {"qfx_grad_finalize": 2}


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


def lora_wgrad(P, Q, G, gs_i, gs_j, r):
    """G[i*gs_i + j*gs_j] += sum_m P[m,i] Q[m,j], j < r.  G fp32."""
    require_cuda(P, Q, G)
    check(_wgrad(ptr(P), P.stride(0), ptr(Q), Q.stride(0), ptr(G), gs_i, gs_j, P.shape[0], P.shape[1], r, cur_stream()),
          "qfx_lora_wgrad")


_wgrad_tc = _sig("qfx_lora_wgrad_tc", _vp, _i64, _i, _vp, _i64, _i, _i, _i, _i, C.POINTER(C.c_void_p), _i64, _i64, _i, _vp)


def lora_wgrad_tc(A, B, G_list, gs_i, gs_j, r, mode=0, Dg=0):
    """wgmma LoRA weight gradient: G_g += A^T B_g over rows.  A [M, Na], B [M, 64*G] bf16; G_list: fp32 tensors (one per
    group).  mode 0: all A columns pair with every group; mode 1: A columns [g*Dg, (g+1)*Dg) pair with group g only."""
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
