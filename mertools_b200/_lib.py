"""ctypes binding of libmer_b200.so (the C ABI declared in include/mer_b200.h).

PyTorch is used by callers for device memory and streams only; tensors cross this boundary as
raw device pointers.  There is NO fallback: if the shared library is missing or the device is
not sm_90a (H100), the first call raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libmer_b200.so")

MER_EPI_GELU = 1
MER_EPI_ROUND_TF32 = 2
MER_EPI_SPLIT_BF16 = 4
MER_EPI_GELU_LIBM = 8
MER_GEMM_TF32 = 0
MER_GEMM_BF16X3 = 1
MER_GEMM_F16 = 2
MER_EPI_OUT_F16 = 16
MER_EPI_QUICK_GELU = 64
MER_EPI_RELU = 128
MER_EPI_GELU_TANH = 256
MER_LN_OUT_F16 = 8
MER_ATT_QKV_F16 = 32
MER_LN_ROUND_TF32 = 1
MER_LN_ACC_INIT = 2
MER_LN_ACC_ADD = 4
MER_LN_GELU = 16
MER_LN_SPLIT_F16 = 32
MER_LN_PAD = 64


class MerError(RuntimeError):
    pass


class MerGemmEpilogue(C.Structure):
    _fields_ = [
        ("bias", C.c_void_p), ("res", C.c_void_p), ("out", C.c_void_p),
        ("out_bstride", C.c_longlong), ("out_row0", C.c_longlong),
        ("res_bstride", C.c_longlong), ("res_row0", C.c_longlong),
        ("ld_out", C.c_int), ("ld_res", C.c_int), ("flags", C.c_int), ("split_off", C.c_int),
        ("vt", C.c_void_p), ("vt_ld", C.c_longlong), ("vt_col0", C.c_int),
    ]


class MerGemmDesc(C.Structure):
    _fields_ = [
        ("A", C.c_void_p), ("W", C.c_void_p),
        ("rows_per_batch", C.c_int), ("a_rows_dim", C.c_int), ("batches", C.c_int),
        ("N", C.c_int), ("K_inner", C.c_int), ("taps", C.c_int), ("P", C.c_int),
        ("a_phase_stride", C.c_longlong), ("a_row_stride", C.c_longlong),
        ("a_batch_stride", C.c_longlong), ("force_block_n", C.c_int), ("mode", C.c_int),
        ("cluster", C.c_int), ("a_row0", C.c_int), ("a_cols", C.c_int), ("a_col_group", C.c_int),
        ("ep", MerGemmEpilogue),
    ]


_lib = None


def lib() -> C.CDLL:
    """Load the shared library (once).  Raises MerError when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise MerError(
                f"{LIB_PATH} not found: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(no CPU fallback exists for the mertools_b200 hot path)")
        _lib = C.CDLL(LIB_PATH)
        _lib.mer_last_error.restype = C.c_char_p
        _declare(_lib)
    return _lib


def _declare(l):
    vp, i32, i64, f32 = C.c_void_p, C.c_int, C.c_longlong, C.c_float
    sig = {
        "mer_abi_version": [],
        "mer_check_device": [],
        "mer_gemm": [C.POINTER(MerGemmDesc), vp],
        "mer_layernorm": [vp, vp, vp, vp, vp, vp, i64, i32, f32, i32, vp],
        "mer_round_tf32": [vp, i64, vp],
        "mer_split_bf16": [vp, vp, i64, i32, vp],
        "mer_attention": [vp, vp, i64, vp, vp, i32, i64, i32, i32, i32, vp],
        "mer_xlnet_attention": [vp, vp, i64, vp, i64, vp, vp, vp, vp, vp, vp, f32, vp, vp, i32, i64, i32, i32, i32, vp],
    }
    for name, args in sig.items():
        fn = getattr(l, name)
        fn.argtypes = args
        fn.restype = C.c_int
    # optional (later-added) entry points are declared by the modules that use them


def declare(name, args, restype=C.c_int):
    fn = getattr(lib(), name)
    fn.argtypes = args
    fn.restype = restype
    return fn


def check(rc: int):
    if rc != 0:
        raise MerError(f"libmer_b200 error {rc}: {lib().mer_last_error().decode(errors='replace')}")


def ptr(t):
    """Device pointer of a torch tensor (or None)."""
    if t is None:
        return None
    return C.c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---- thin python wrappers of the kernel-level entry points (used by tests and the encoders) ----
def gemm(A, W, out, *, bias=None, res=None, gelu=False, round_out=False, split_out=False,
         mode=MER_GEMM_TF32, rows_per_batch=None, batches=1, a_rows_dim=None, K_inner=None, taps=1, P=1,
         a_phase_stride=0, a_row_stride=None, a_batch_stride=0,
         out_bstride=0, out_row0=0, res_bstride=0, res_row0=0,
         ld_out=None, ld_res=None, force_block_n=0, cluster=0, vt=None, vt_col0=0, gelu_libm=False,
         f16_out=False, a_row0=0, a_cols=0, a_col_group=0, relu=False, gelu_tanh=False, quick_gelu=False):
    """out = epilogue(A @ W.T).  A, W: fp32 CUDA tensors of LOGICAL shape [rows, K] / [N, K] (holding
    tf32-rounded fp32, or split bf16 hi|lo bytes when mode is BF16X3; fp16 tensors when mode is F16);
    see MerGemmDesc in mer_b200.h.  a_phase_stride defaults to K_inner when P == 1; a nonzero value is passed through
    (the tensor map's phase dimension then has the stride a caller's own descriptor would give it)."""
    N, K = W.shape
    d = MerGemmDesc()
    d.A, d.W = A.data_ptr(), W.data_ptr()
    d.taps, d.P = taps, P
    d.K_inner = K_inner if K_inner is not None else K // taps
    assert d.K_inner * taps == K
    d.rows_per_batch = rows_per_batch if rows_per_batch is not None else A.shape[0]
    d.a_rows_dim = a_rows_dim if a_rows_dim is not None else d.rows_per_batch
    d.batches = batches
    d.N = N
    d.a_phase_stride = a_phase_stride if (P > 1 or a_phase_stride) else d.K_inner
    d.a_row_stride = a_row_stride if a_row_stride is not None else K
    d.a_batch_stride = a_batch_stride if batches > 1 else d.a_row_stride * d.a_rows_dim
    d.force_block_n = force_block_n
    d.mode = mode
    d.cluster = cluster
    d.a_row0, d.a_cols, d.a_col_group = a_row0, a_cols, a_col_group
    d.ep.bias = bias.data_ptr() if bias is not None else None
    d.ep.res = res.data_ptr() if res is not None else None
    d.ep.out = out.data_ptr()
    d.ep.out_bstride, d.ep.out_row0 = out_bstride, out_row0
    d.ep.res_bstride, d.ep.res_row0 = res_bstride, res_row0
    d.ep.ld_out = ld_out if ld_out is not None else N
    d.ep.ld_res = ld_res if ld_res is not None else N
    d.ep.flags = ((MER_EPI_GELU if gelu else 0) | (MER_EPI_ROUND_TF32 if round_out else 0)
                  | (MER_EPI_SPLIT_BF16 if split_out else 0) | (MER_EPI_GELU_LIBM if gelu_libm else 0)
                  | (MER_EPI_OUT_F16 if f16_out else 0) | (MER_EPI_RELU if relu else 0)
                  | (MER_EPI_GELU_TANH if gelu_tanh else 0) | (MER_EPI_QUICK_GELU if quick_gelu else 0))
    d.ep.split_off = N
    if vt is not None:
        d.ep.vt, d.ep.vt_ld, d.ep.vt_col0 = vt.data_ptr(), vt.shape[1], vt_col0
    check(lib().mer_gemm(C.byref(d), stream_ptr()))
    return out


gemm_tf32 = gemm


def gemm_epilogue_launches():
    """(register, TMA) epilogue launches of mer_gemm so far in this process (MER_GEMM_EPI_TMA=0 forces the first)."""
    f = lib().mer_gemm_epilogue_launches
    f.restype, f.argtypes = C.c_longlong, [C.c_int]
    return int(f(0)), int(f(1))


def layernorm(x, gamma, beta, y, *, eps, y_split=None, acc=None, flags=0):
    rows = x.numel() // x.shape[-1]
    check(lib().mer_layernorm(ptr(x), ptr(gamma), ptr(beta), ptr(y), ptr(y_split), ptr(acc), rows,
                              x.shape[-1], eps, flags, stream_ptr()))
    return y


def split_bf16(x):
    """fp32 [rows, K] CUDA tensor -> same-shape fp32-typed tensor whose bytes are split rows
    (128-byte groups of 32 bf16 hi | 32 bf16 lo; see mer_b200.h)."""
    import torch
    x = x.contiguous()
    out = torch.empty_like(x)
    check(lib().mer_split_bf16(ptr(x), ptr(out), x.numel() // x.shape[-1], x.shape[-1], stream_ptr()))
    return out


def unsplit_bf16(xs):
    """Inverse of split_bf16 (for tests): hi + lo as fp32."""
    import torch
    K = xs.shape[-1]
    b = xs.contiguous().view(torch.bfloat16).view(*xs.shape[:-1], K // 32, 2, 32).float()
    return (b[..., 0, :] + b[..., 1, :]).reshape(*xs.shape[:-1], K)


def round_tf32_(x):
    check(lib().mer_round_tf32(ptr(x), x.numel(), stream_ptr()))
    return x


def attention(qkv, ctx, cu_seqlens, max_seqlen, heads, round_out=False, vt=None, f16_out=False, split_out=False):
    """vt: optional V^T [heads*64, ld] (enables the tf32 V^T kernel of attention_f16.cu for max_seqlen <= 253).  fp16
    qkv / vt select the fp16-operand V^T kernel (max_seqlen <= 505); its ctx is fp16 for an fp16 ctx tensor, else fp32
    (plain, round_out = tf32-rounded, split_out = bf16 hi | lo rows)."""
    import torch
    if qkv.dtype == torch.float16:
        assert vt is not None and vt.dtype == torch.float16
        if ctx.dtype == torch.float16:
            out_fl = MER_EPI_OUT_F16
        else:
            assert ctx.dtype == torch.float32
            out_fl = MER_EPI_SPLIT_BF16 if split_out else (MER_EPI_ROUND_TF32 if round_out else 0)
        check(lib().mer_attention(ptr(qkv), ptr(vt), vt.shape[1], ptr(ctx), ptr(cu_seqlens),
                                  cu_seqlens.numel() - 1, qkv.shape[0], max_seqlen, heads,
                                  out_fl | MER_ATT_QKV_F16, stream_ptr()))
        return ctx
    check(lib().mer_attention(ptr(qkv), ptr(vt), vt.shape[1] if vt is not None else 0, ptr(ctx),
                              ptr(cu_seqlens), cu_seqlens.numel() - 1, qkv.shape[0], max_seqlen, heads,
                              MER_EPI_OUT_F16 if f16_out else
                              (MER_EPI_SPLIT_BF16 if split_out else (MER_EPI_ROUND_TF32 if round_out else 0)),
                              stream_ptr()))
    return ctx


def last_error() -> str:
    return lib().mer_last_error().decode(errors="replace")


def launch_count() -> int:
    f = lib().mer_launch_count
    f.restype, f.argtypes = C.c_longlong, []
    return int(f())


def segment_reduce(x, begins, ends, out, *, dim, mean=False, n_seg=None):
    """out[s] = sum | mean of the rows x[begins[s] : ends[s]] (begins / ends: int32 CUDA tensors)."""
    f = declare("mer_segment_reduce", [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                       C.c_void_p])
    check(f(ptr(x), ptr(begins), ptr(ends), begins.numel() if n_seg is None else n_seg, dim, 1 if mean else 0,
            ptr(out), stream_ptr()))
    return out


def wave_normalize(x, out, *, batch, n_samples, ld_in, ld_out):
    f = declare("mer_wave_normalize", [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_longlong, C.c_longlong,
                                       C.c_void_p])
    check(f(ptr(x), ptr(out), batch, n_samples, ld_in, ld_out, stream_ptr()))
    return out


def hubert_conv0_workspace_bytes(batch):
    f = lib().mer_hubert_conv0_workspace_bytes
    f.restype, f.argtypes = C.c_longlong, [C.c_int]
    return int(f(batch))


def hubert_conv0(model, wave, out, *, batch, n_samples, ld_wave, out_bstride, frames=None, f16_out=False,
                 workspace=None, workspace_bytes=None):
    """mer_hubert_conv0 on a MerHubertModel (ctypes struct, encoders.py).  out: split-bf16 rows in an fp32-typed tensor,
    or fp16 rows (f16_out); frames: optional int32 CUDA tensor of per-clip frame counts; workspace: a CUDA tensor
    (default: a fresh one of mer_hubert_conv0_workspace_bytes(batch))."""
    import torch
    if workspace is None:
        workspace = torch.empty(max(hubert_conv0_workspace_bytes(batch), 16), dtype=torch.uint8, device=wave.device)
    f = declare("mer_hubert_conv0", [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_longlong, C.c_void_p, C.c_int,
                                     C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong, C.c_void_p])
    check(f(C.byref(model), ptr(wave), batch, n_samples, ld_wave, ptr(frames),
            MER_EPI_OUT_F16 if f16_out else MER_EPI_SPLIT_BF16, ptr(out), out_bstride, ptr(workspace),
            workspace.numel() * workspace.element_size() if workspace_bytes is None else workspace_bytes,
            stream_ptr()))
    return out


def wavlm_gate(x, w, b, c, gate, *, tokens, heads):
    f = declare("mer_wavlm_gate", [C.c_void_p, C.c_longlong, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p])
    check(f(ptr(x), tokens, heads, ptr(w), ptr(b), ptr(c), ptr(gate), stream_ptr()))
    return gate


def biased_attention(qkv, bias, rowscale, ctx, *, batch, T, heads, round_out=False):
    f = declare("mer_biased_attention", [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                         C.c_int, C.c_void_p])
    check(f(ptr(qkv), ptr(bias), ptr(rowscale), batch, T, heads, ptr(ctx), 1 if round_out else 0, stream_ptr()))
    return ctx


def small_attention(q, k, v, out, *, ld_q, ld_k, ld_v, ld_out, batch, heads, nq, nk, causal=False):
    """q / k / v / out may be views into wider buffers: their data pointers carry the column offset."""
    f = declare("mer_small_attention", [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                        C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p])
    check(f(ptr(q), ld_q, ptr(k), ld_k, ptr(v), ld_v, batch, heads, nq, nk, 1 if causal else 0, ptr(out), ld_out,
            stream_ptr()))
    return out


def swiglu(x, out, *, rows, hidden, round_out=False):
    f = declare("mer_swiglu", [C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_void_p])
    check(f(ptr(x), ptr(out), rows, hidden, 1 if round_out else 0, stream_ptr()))
    return out


def videomae_patchify(frames, mean, std, out, *, n_clips):
    """frames: uint8 CUDA tensor [n_clips * 16, 224, 224, 3] (BGR); mean / std: three host floats each (RGB)."""
    f = declare("mer_videomae_patchify", [C.c_void_p, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_void_p,
                                          C.c_void_p])
    check(f(ptr(frames), n_clips, (C.c_float * 3)(*mean), (C.c_float * 3)(*std), ptr(out), stream_ptr()))
    return out
