"""Kernel-level parity of the wgmma GEMM (gemm.cu) over its descriptor space, and its host validation.

GPU tests (marked gpu) run gemm_kernel<BLOCK_N, MODE> directly on operands that the mode represents exactly (fp16
values, tf32-rounded fp32, split bf16 pairs), so a float64 product of the same values measures the kernel alone:
- every instantiation {128, 256} x {TF32, BF16X3, F16} on ragged row counts, one-stage K, K whose stage count is no
  multiple of the smem ring depth, K = 3072 / 4096, several tiles per CTA and the automatic width choice;
- the convolution and batch forms of the A map (strided HuBERT conv, zero-padded conv, block-diagonal positional
  conv, ViT patch embedding);
- every epilogue flag combination mer_gemm accepts, against the kernel's own plain output (bit-exact formats,
  residual, in-place residual, V^T) and against float64 activations;
- schedule invariance, fp16 subnormal operands and the two operand converters, bit for bit.
Every output carries guard rows / columns prefilled with NaN (0x7E00 for fp16) that must survive every call.

CPU tests (unmarked) call mer_gemm with fake, never-dereferenced addresses on a machine without a CUDA driver:
validation runs before any CUDA call, so a refused descriptor stops with its `mer_gemm:` message and an accepted one
at the tensor-map encode.  Both halves are driven by one table of epilogue flag combinations (COMBOS)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from mertools_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F16, TF32, BF16X3 = L.MER_GEMM_F16, L.MER_GEMM_TF32, L.MER_GEMM_BF16X3
MODE_NAME = {F16: "f16", TF32: "tf32", BF16X3: "bf16x3"}
STAGE_K = {F16: 64, TF32: 32, BF16X3: 32}      # K elements of one pipeline stage
RING_K = {F16: 320, TF32: 800, BF16X3: 800}    # 5 / 25 stages: no multiple of the 6- (BLOCK_N 128) or 4-deep (256) ring
INSTANTIATIONS = [(bn, m) for bn in (128, 256) for m in (TF32, BF16X3, F16)]
NAN32, NAN16 = 0x7FC00000, 0x7E00

# Normalised error bar, e = max |out - ref| / (|A| |W|^T + |bias| + |res|).  F16 and TF32 products are exact, so only
# the fp32 accumulation contributes (truncating adds of the tensor-core accumulator, ~K/8 of them at 2^-23 of a partial
# sum that is itself ~sqrt(K) smaller than the denominator: <= 2^-20 at K = 4096; measured <= 1.2e-6 on an H100
# 80GB HBM3 at 700 W).
# BF16X3 also drops lo(a) lo(w), |lo| <= 2^-8 |x|: up to 2^-16 per product.  At K = 32 few products average it out and
# it measured 5.3e-6, within 4x of the bar, so plain BF16X3 cases are also held to the three products the kernel does
# compute (hi hi + lo hi + hi lo, float64): that leaves the accumulation error alone, under the same bar with margin.
BAR = 2.0 ** -16


# ---------------------------------------------------------------------------------------------------------------------
# epilogue flag combinations: one table for the CPU refusal test and the GPU epilogue test
ACTS = {"none": 0, "gelu": L.MER_EPI_GELU, "libm": L.MER_EPI_GELU | L.MER_EPI_GELU_LIBM,
        "quick": L.MER_EPI_QUICK_GELU, "relu": L.MER_EPI_RELU, "tanh": L.MER_EPI_GELU_TANH}
FMTS = {"fp32": 0, "tf32": L.MER_EPI_ROUND_TF32, "split": L.MER_EPI_SPLIT_BF16, "f16": L.MER_EPI_OUT_F16}
COMBOS = [(a, f, r, v) for a in ACTS for f in FMTS for r in (False, True) for v in (False, True)]
FMT_MODE = {"fp32": F16, "tf32": TF32, "split": BF16X3, "f16": F16}  # the arithmetic mode each output format feeds


def _accepted(act, fmt, res, vt):
    """The combinations include/mer_b200.h documents as supported."""
    if res and vt:
        return False
    if fmt == "f16" and res or fmt == "split" and (res or vt):
        return False
    if act in ("gelu", "libm"):
        return not vt and (not res or (act == "gelu" and fmt == "fp32"))
    if act == "quick":
        return fmt != "split" and not res and not vt
    if act == "relu":
        return fmt in ("fp32", "f16") and not vt and not (res and fmt != "fp32")
    if act == "tanh":
        return fmt in ("fp32", "f16") and not res and not vt
    return True


ACCEPTED = [c for c in COMBOS if _accepted(*c)]
REFUSED = [c for c in COMBOS if not _accepted(*c)]


def test_combination_table_is_a_partition():
    assert len(COMBOS) == len(set(COMBOS)) == 6 * 4 * 2 * 2
    assert sorted(ACCEPTED + REFUSED) == sorted(COMBOS) and not set(ACCEPTED) & set(REFUSED)
    assert len(ACCEPTED) == 26


# ---------------------------------------------------------------------------------------------------------------------
# CPU: host validation of mer_gemm_launch
def _cpu_lib():
    if torch.cuda.is_available():
        pytest.skip("fake device addresses are only safe where no CUDA driver can launch anything")
    if not os.path.exists(L.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    dll = L.lib()
    dll.mer_last_error.restype = C.c_char_p
    return dll


def _fake_desc(flags, mode, res=False, vt=False, vt_col0=128, out_off=0, res_off=0, bias_off=0):
    base = 0x7F0000000000  # never dereferenced
    d = L.MerGemmDesc()
    d.A, d.W = base, base + (1 << 20)
    d.rows_per_batch = d.a_rows_dim = 64
    d.batches, d.N, d.K_inner, d.taps, d.P = 1, 256, 64, 1, 1
    d.a_phase_stride = d.a_row_stride = 64
    d.a_batch_stride = 64 * 64
    d.mode = mode
    d.ep.bias = base + (2 << 20) + bias_off
    d.ep.out = base + (3 << 20) + out_off
    d.ep.res = base + (4 << 20) + res_off if res else None
    d.ep.ld_out = d.ep.ld_res = 256
    d.ep.flags = flags
    d.ep.vt_col0 = vt_col0
    if vt:
        d.ep.vt, d.ep.vt_ld = base + (5 << 20), 64
    return d


def _host_verdict(dll, d):
    rc = dll.mer_gemm(C.byref(d), None)
    msg = dll.mer_last_error().decode()
    assert rc != 0  # nothing can run here
    if "cuTensorMapEncodeTiled entry point unavailable" in msg:
        return "accepted", msg
    assert msg.startswith("mer_gemm:"), msg
    return "refused", msg


def test_host_validation_follows_the_combination_table():
    dll = _cpu_lib()
    for act, fmt, res, vt in COMBOS:
        d = _fake_desc(ACTS[act] | FMTS[fmt], FMT_MODE[fmt], res=res, vt=vt)
        verdict, msg = _host_verdict(dll, d)
        assert verdict == ("accepted" if _accepted(act, fmt, res, vt) else "refused"), (act, fmt, res, vt, msg)


def test_host_validation_refuses_silently_mishandled_descriptors():
    dll = _cpu_lib()
    refused = {
        # vt_col0 odd (column vt_col0 would go to out), negative (vt rows past N - vt_col0), >= N (no V^T at all)
        "vt_col0 odd": _fake_desc(0, F16, vt=True, vt_col0=129),
        "vt_col0 negative": _fake_desc(0, F16, vt=True, vt_col0=-128),
        "vt_col0 = N": _fake_desc(0, F16, vt=True, vt_col0=256),
        "vt_col0 > N": _fake_desc(L.MER_EPI_OUT_F16, F16, vt=True, vt_col0=1000),
        # MER_EPI_GELU_LIBM without MER_EPI_GELU used to be ignored
        "libm alone": _fake_desc(L.MER_EPI_GELU_LIBM, F16),
        "libm + quick": _fake_desc(L.MER_EPI_GELU_LIBM | L.MER_EPI_QUICK_GELU, F16),
        "libm + relu": _fake_desc(L.MER_EPI_GELU_LIBM | L.MER_EPI_RELU, F16),
        "libm + residual": _fake_desc(L.MER_EPI_GELU_LIBM, F16, res=True),
        # tf32 | split used to write the split output
        "tf32 + split": _fake_desc(L.MER_EPI_ROUND_TF32 | L.MER_EPI_SPLIT_BF16, BF16X3),
        "gelu + tf32 + split": _fake_desc(L.MER_EPI_GELU | L.MER_EPI_ROUND_TF32 | L.MER_EPI_SPLIT_BF16, BF16X3),
        # float2 / fp16-pair epilogue accesses used to fault on the device
        "fp32 out 4-byte aligned": _fake_desc(0, F16, out_off=4),
        "split out 4-byte aligned": _fake_desc(L.MER_EPI_SPLIT_BF16, BF16X3, out_off=4),
        "fp16 out 2-byte aligned": _fake_desc(L.MER_EPI_OUT_F16, F16, out_off=2),
        "res 4-byte aligned": _fake_desc(0, F16, res=True, res_off=4),
        "bias 4-byte aligned": _fake_desc(0, F16, bias_off=4),
    }
    for name, d in refused.items():
        verdict, msg = _host_verdict(dll, d)
        assert verdict == "refused", (name, msg)
    accepted = {
        "vt_col0 = 0": _fake_desc(0, F16, vt=True, vt_col0=0),
        "vt_col0 = N - 2": _fake_desc(L.MER_EPI_ROUND_TF32, TF32, vt=True, vt_col0=254),
        "vt_col0 ignored without vt": _fake_desc(0, F16, vt_col0=-7),
        "fp16 out 4-byte aligned": _fake_desc(L.MER_EPI_OUT_F16, F16, out_off=4),
        "res 8-byte aligned": _fake_desc(0, F16, res=True, res_off=8),
        "libm with gelu": _fake_desc(L.MER_EPI_GELU | L.MER_EPI_GELU_LIBM, TF32),
    }
    for name, d in accepted.items():
        verdict, msg = _host_verdict(dll, d)
        assert verdict == "accepted", (name, msg)


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers
def _variants():
    f = L.lib().mer_gemm_variant_launches
    f.restype, f.argtypes = C.c_longlong, [C.c_int] * 4
    return {(bn, m): int(f(bn, m, 1, 0)) for bn, m in INSTANTIATIONS}


def _gemm(expect, A, W, out, **kw):
    """L.gemm that asserts which instantiation (BLOCK_N, mode) ran: exactly one launch of exactly that kernel."""
    before = _variants()
    L.gemm(A, W, out, mode=expect[1], **kw)
    torch.cuda.synchronize()
    after = _variants()
    launched = {k: after[k] - before[k] for k in after if after[k] != before[k]}
    assert launched == {expect: 1}, (expect, launched)
    return out


def _sentinel(shape, dtype, dev):
    if dtype == torch.float16:
        return torch.full(shape, NAN16, dtype=torch.int16, device=dev).view(torch.float16)
    return torch.full(shape, NAN32, dtype=torch.int32, device=dev).view(torch.float32)


def _bits(x):
    return x.view(torch.int16 if x.dtype == torch.float16 else torch.int32)


def _check_guards(buf, written, split=False):
    """Every element the descriptor writes is finite; every other element (guard rows / columns, skipped rows) still
    holds its sentinel bits."""
    sent = NAN16 if buf.dtype == torch.float16 else NAN32
    assert bool((_bits(buf)[~written] == sent).all()), "a guard / skipped element was written"
    vals = buf[written]
    if split:  # each fp32 slot of a split row holds two bf16 values
        vals = vals.view(torch.bfloat16)
    assert bool(torch.isfinite(vals.float()).all()), "a written element is not finite"


def _mask(rows, cols, shape, dev):
    m = torch.zeros(shape, dtype=torch.bool, device=dev)
    m[rows, cols] = True
    return m


def _operand(mode, rows, K, gen, dev, scale=True):
    """(kernel operand, the float64 values it holds).  Rows are scaled by 2^[-4, 4] so that small-magnitude rows exist:
    the normalised error sees an error there that max-ref would hide."""
    x = torch.randn(rows, K, generator=gen, device=dev)
    if scale:
        x = x * torch.exp2(torch.randint(-4, 5, (rows, 1), generator=gen, device=dev).float())
    if mode == F16:
        x = x.half()
        return x, x.double()
    if mode == TF32:
        L.round_tf32_(x)
        return x, x.double()
    s = L.split_bf16(x)
    return s, L.unsplit_bf16(s).double()


def _lo64(s):
    """The lo halves of a split operand, float64."""
    K = s.shape[-1]
    return s.contiguous().view(torch.bfloat16).view(-1, K // 32, 2, 32)[:, :, 1].reshape(-1, K).double()


def _nerr(out, ref, den):
    return float(((out.double() - ref).abs() / den).max())


def _report(name, expect, e, bar=BAR):
    print(f"{name:<52s} gemm_kernel<{expect[0]}, {MODE_NAME[expect[1]]:>6s}>  e = {e:.2e}  (bar {bar:.1e})")
    assert e < bar, (name, e, bar)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: instantiations, tails, pipeline depth, persistence
def _plain_case(dev, gen, expect, M, K, N, force, name, ld_pad=8):
    mode = expect[1]
    a, a64 = _operand(mode, M, K, gen, dev)
    w, w64 = _operand(mode, N, K, gen, dev)
    bias = torch.randn(N, generator=gen, device=dev)
    ld = N + ld_pad
    out = _sentinel((M + 1, ld), torch.float32, dev)
    _gemm(expect, a, w, out, bias=bias, ld_out=ld, force_block_n=force)
    _check_guards(out, _mask(slice(0, M), slice(0, N), out.shape, dev))
    b64 = bias.double()
    ref = torch.addmm(b64, a64, w64.T)
    den = torch.addmm(b64.abs(), a64.abs(), w64.abs().T)
    _report(f"{name} M={M} K={K} N={N}", expect, _nerr(out[:M, :N], ref, den))
    if mode == BF16X3:  # without the lo * lo product the kernel leaves out
        ref -= _lo64(a) @ _lo64(w).T
        _report(f"{name} M={M} K={K} N={N} (three products)", expect, _nerr(out[:M, :N], ref, den))


@pytest.mark.gpu
@pytest.mark.parametrize("block_n,mode", INSTANTIATIONS, ids=[f"{bn}-{MODE_NAME[m]}" for bn, m in INSTANTIATIONS])
def test_gemm_instantiation_vs_float64(cuda, block_n, mode):
    gen = torch.Generator(device=cuda).manual_seed(block_n + 10 * mode)
    expect = (block_n, mode)
    # single row, rows only in consumer warpgroup 0, a full tile half, ragged tiles; one stage and an odd stage count
    for M in (1, 63, 64, 65, 129, 300):
        for K in (STAGE_K[mode], RING_K[mode]):
            _plain_case(cuda, gen, expect, M, K, 256, block_n, "tails")
    for K in (3072, 4096):
        _plain_case(cuda, gen, expect, 300, K, 512, block_n, "deep K")
    # >= 3 tiles per CTA on 132 SMs (798 tiles at 128, 399 at 256): the smem ring's stage / phase carry across tiles
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    M, N = 17000, 768
    assert (M + 127) // 128 * (N // block_n) >= 3 * sms
    _plain_case(cuda, gen, expect, M, RING_K[mode], N, block_n, "persistent")
    # automatic width: 256 when 256-wide tiles fill the machine, 128 when N cannot take them
    if block_n == 256:
        _plain_case(cuda, gen, expect, 40000, RING_K[mode], 2304, 0, "auto width")
    else:
        _plain_case(cuda, gen, expect, 40000, RING_K[mode], 384, 0, "auto width (N % 256 != 0)")


# ---------------------------------------------------------------------------------------------------------------------
# GPU: convolution and batch forms of the A map
@pytest.mark.gpu
@pytest.mark.parametrize("mode", [F16, BF16X3], ids=["f16", "bf16x3"])
def test_gemm_strided_conv_vs_conv1d(cuda, mode):
    """HuBERT conv1..6: Conv1d(k, stride 2) over time-major [B, T_pad, C] activations as a (taps = k, P = 2) GEMM; odd T,
    NaN in the padding rows beyond T; output packed (out_bstride = T_out) and padded (T_out + 3 rows per clip)."""
    gen = torch.Generator(device=cuda).manual_seed(21 + mode)
    B, T, T_pad, C, N = 3, 301, 306, 128, 256
    for k in (2, 3):
        T_out = (T - k) // 2 + 1
        x = torch.full((B, T_pad, C), float("nan"), device=cuda)
        xv, xv64 = _operand(mode if mode == F16 else TF32, B * T, C, gen, cuda)
        x[:, :T] = xv.float().view(B, T, C)
        wt = torch.randn(N, C, k, generator=gen, device=cuda) * 0.1
        if mode == F16:
            x16, wt = x.half(), wt.half().float()
            a, x64 = x16, x16.double()
            w = wt.permute(0, 2, 1).reshape(N, k * C).half()
            w64 = w.double()
        else:
            a = L.split_bf16(x.view(B * T_pad, C))
            x64 = L.unsplit_bf16(a).double().view(B, T_pad, C)
            w = L.split_bf16(wt.permute(0, 2, 1).reshape(N, k * C).contiguous())
            w64 = L.unsplit_bf16(w).double()
        wc = w64.view(N, k, C).permute(0, 2, 1)  # the conv weight the GEMM holds, [N, C, k]
        bias = torch.randn(N, generator=gen, device=cuda)
        xin = x64[:, :T].transpose(1, 2)
        ref = F.conv1d(xin, wc, bias.double(), stride=2).transpose(1, 2)
        den = F.conv1d(xin.abs(), wc.abs(), bias.double().abs(), stride=2).transpose(1, 2)
        for bstride in (T_out, T_out + 3):
            out = _sentinel((B * bstride + 1, N), torch.float32, cuda)
            _gemm((128, mode), a, w, out, bias=bias, rows_per_batch=T_out, batches=B, a_rows_dim=T_pad // 2,
                  K_inner=C, taps=k, P=2, a_phase_stride=C, a_row_stride=2 * C, a_batch_stride=T_pad * C,
                  out_bstride=bstride)
            rows = torch.cat([torch.arange(T_out, device=cuda) + b * bstride for b in range(B)])
            _check_guards(out, _mask(rows[:, None], slice(None), out.shape, cuda))
            got = out[rows].view(B, T_out, N)
            _report(f"strided conv k={k} P=2 out_bstride={bstride}", (128, mode), _nerr(got, ref, den))


@pytest.mark.gpu
def test_gemm_zero_padded_conv_vs_conv1d(cuda):
    """Conv1d(k = 19, padding 9) as a 19-tap GEMM with a_row0 = -9: rows outside [0, T) of a clip read as zero, never
    as the neighbouring clip's rows."""
    gen = torch.Generator(device=cuda).manual_seed(22)
    B, T, C, N, k = 3, 150, 64, 256, 19
    x = torch.randn(B, T, C, generator=gen, device=cuda).half()
    wt = (torch.randn(N, C, k, generator=gen, device=cuda) * 0.1).half()
    w = wt.permute(0, 2, 1).reshape(N, k * C).contiguous()
    bias = torch.randn(N, generator=gen, device=cuda)
    out = _sentinel((B * T + 1, N + 8), torch.float32, cuda)
    _gemm((128, F16), x.view(B * T, C), w, out, bias=bias, rows_per_batch=T, batches=B, a_rows_dim=T, K_inner=C,
          taps=k, P=1, a_row_stride=C, a_batch_stride=T * C, a_row0=-9, out_bstride=T, ld_out=N + 8)
    _check_guards(out, _mask(slice(0, B * T), slice(0, N), out.shape, cuda))
    xin = x.double().transpose(1, 2)
    ref = F.conv1d(xin, wt.double(), bias.double(), padding=9).transpose(1, 2)
    den = F.conv1d(xin.abs(), wt.double().abs(), bias.double().abs(), padding=9).transpose(1, 2)
    _report("padded conv taps=19 a_row0=-9", (128, F16), _nerr(out[:B * T, :N].view(B, T, N), ref, den))


@pytest.mark.gpu
@pytest.mark.parametrize("hidden", [768, 1024])
def test_gemm_block_diagonal_pos_conv_vs_grouped_conv1d(cuda, hidden):
    """The positional conv (16 groups, k = 128, padding 64, last frame dropped) as one fp16 GEMM over windowed
    block-diagonal weights: a_col_group windows, 128 taps from a_row0 = -64, force_block_n = 256 (the product's
    descriptor)."""
    from mertools_b200.encoders import block_diagonal_pos_conv_weight
    gen = torch.Generator(device=cuda).manual_seed(hidden)
    gch = hidden // 16
    window = 320 if gch == 48 else 256
    B, T, taps = 3, 150, 128
    wt = (torch.randn(hidden, gch, taps, generator=gen, device=cuda) * 0.05).half()
    x = torch.randn(B, T, hidden, generator=gen, device=cuda).half()
    w = torch.from_numpy(block_diagonal_pos_conv_weight(wt.float().cpu().numpy(), window=window, group=gch))
    w = w.to(cuda).half()
    bias = torch.randn(hidden, generator=gen, device=cuda)
    out = _sentinel((B * T + 1, hidden), torch.float32, cuda)
    _gemm((256, F16), x.view(B * T, hidden), w, out, bias=bias, rows_per_batch=T, batches=B, a_rows_dim=T,
          K_inner=window, taps=taps, P=1, a_phase_stride=hidden, a_row_stride=hidden, a_batch_stride=T * hidden,
          a_row0=-64, a_cols=hidden, a_col_group=gch, force_block_n=256, out_bstride=T)
    _check_guards(out, _mask(slice(0, B * T), slice(None), out.shape, cuda))
    xin = x.double().transpose(1, 2)
    ref = F.conv1d(xin, wt.double(), bias.double(), padding=64, groups=16)[..., :-1].transpose(1, 2)
    den = F.conv1d(xin.abs(), wt.double().abs(), bias.double().abs(), padding=64, groups=16)[..., :-1].transpose(1, 2)
    _report(f"block-diagonal pos conv hidden={hidden}", (256, F16), _nerr(out[:B * T].view(B, T, hidden), ref, den))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [TF32, F16], ids=["tf32", "f16"])
def test_gemm_patch_embed_batches_vs_float64(cuda, mode):
    """ViT patch embedding: batches = frames of 196 patches, written from row 1 of each 197-row frame (the class row is
    skipped), plus position embeddings broadcast to every frame through res_bstride = 0."""
    gen = torch.Generator(device=cuda).manual_seed(23)
    frames, P_, D = 5, 196, 768
    a, a64 = _operand(mode, frames * P_, D, gen, cuda)
    w, w64 = _operand(mode, D, D, gen, cuda)
    bias = torch.randn(D, generator=gen, device=cuda)
    pos = torch.randn(P_ + 1, D, generator=gen, device=cuda)  # one guard row
    out = _sentinel((frames * 197 + 1, D), torch.float32, cuda)
    _gemm((128, mode), a, w, out, bias=bias, res=pos, rows_per_batch=P_, batches=frames, a_rows_dim=P_,
          a_batch_stride=P_ * D, out_bstride=197, out_row0=1, res_bstride=0)
    rows = torch.cat([torch.arange(1, 197, device=cuda) + f * 197 for f in range(frames)])
    _check_guards(out, _mask(rows[:, None], slice(None), out.shape, cuda))
    p64 = pos[:P_].double().repeat(frames, 1)
    ref = torch.addmm(bias.double(), a64, w64.T) + p64
    den = torch.addmm(bias.double().abs(), a64.abs(), w64.abs().T) + p64.abs()
    _report("patch embed out_row0=1 res_bstride=0", (128, mode), _nerr(out[rows], ref, den))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: epilogues
def _tf32(x):
    """cvt.rna.tf32.f32 (ties away from zero) in integer arithmetic."""
    return ((x.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


def _split(x):
    """(hi, lo) with hi = bf16_rn(x), lo = bf16_rn(x - hi)."""
    hi = x.to(torch.bfloat16)
    return hi, (x - hi.float()).to(torch.bfloat16)


def _half_sat(x):
    return x.clamp(-65504.0, 65504.0).half()


def _unpack_split(buf, M, N):
    b = buf[:M, :N].contiguous().view(torch.bfloat16).view(M, N // 32, 2, 32)
    return b[:, :, 0].reshape(M, N), b[:, :, 1].reshape(M, N)


def _act64(act, x):
    if act in ("gelu", "libm"):
        return 0.5 * x * (1.0 + torch.erf(x / 2.0 ** 0.5))
    if act == "quick":
        return x * torch.sigmoid(1.702 * x)
    if act == "tanh":
        return 0.5 * x * (1.0 + torch.tanh(0.79788456 * x * (1.0 + 0.044715 * x * x)))
    raise AssertionError(act)


# Activation bars on |act(x) - act64(x)| / max(1, |x|), x = the kernel's own fp32 pre-activation:
# - gelu (12-op polynomial): Abramowitz-Stegun 7.1.26 is within 1.5e-7 of erf, ex2.approx / rcp.approx add ~2^-22
#   each to the 1 - erf term, scaled by |x| / 2, plus the final rounding: <= 4e-7.
# - libm (libdevice erff, <= 2 ulp): a few fp32 roundings of x / 2 (1 + erf): <= 3e-7.
# - quick (x sigmoid(1.702 x), ex2.approx / rcp.approx): the 1.702 log2(e) product rounded to fp32 shifts the
#   exponent argument by up to 2^-24 |1.702 x log2 e|, which at |x| = 23 is ~6e-7 of the sigmoid: <= 1e-6.
# - tanh (BLOOM): include/mer_b200.h promises <= 1e-6 on [-20, 20].
# Measured (H100 80GB HBM3, 700 W): gelu 1.7e-7, libm 1.2e-7, quick 1.6e-7, tanh 9.5e-8.
ACT_BAR = {"gelu": 4e-7, "libm": 3e-7, "quick": 1e-6, "tanh": 1e-6}


@pytest.mark.gpu
@pytest.mark.parametrize("block_n,mode", INSTANTIATIONS, ids=[f"{bn}-{MODE_NAME[m]}" for bn, m in INSTANTIATIONS])
def test_gemm_epilogue_combinations(cuda, block_n, mode):
    """Every accepted epilogue combination, checked against the same instantiation's plain fp32 output (same operands
    and bias, no activation): output formats, residual and V^T bit for bit, activations against float64."""
    gen = torch.Generator(device=cuda).manual_seed(31 + block_n + mode)
    expect = (block_n, mode)
    M, K, N = 300, 64, 2304  # the last row tile has 44 rows: consumer warpgroup 1 owns none
    ld = N + 8
    a, _ = _operand(mode, M, K, gen, cuda, scale=False)
    w, _ = _operand(mode, N, K, gen, cuda, scale=False)
    # distinct per column, spanning [-20, 20] around the ~N(0, 8) product; the last four columns saturate fp16
    bias = torch.linspace(-20.0, 20.0, N, device=cuda) + torch.rand(N, generator=gen, device=cuda) * 1e-2
    bias[-4:] = torch.tensor([7e4, -7e4, 65519.0, -1e6], device=cuda)
    res = torch.randn(M + 1, ld, generator=gen, device=cuda) * 4.0  # one guard row
    rows_cols = _mask(slice(0, M), slice(0, N), (M + 1, ld), cuda)

    def run(act, fmt, res_t=None, out=None, vt=None, vt_col0=0):
        dtype = torch.float16 if fmt == "f16" else torch.float32
        out = _sentinel((M + 1, ld), dtype, cuda) if out is None else out
        kw = dict(bias=bias, ld_out=ld, ld_res=ld, force_block_n=block_n, res=res_t, vt=vt, vt_col0=vt_col0,
                  gelu=act in ("gelu", "libm"), gelu_libm=act == "libm", quick_gelu=act == "quick",
                  relu=act == "relu", gelu_tanh=act == "tanh", round_out=fmt == "tf32", split_out=fmt == "split",
                  f16_out=fmt == "f16")
        _gemm(expect, a, w, out, **kw)
        return out

    def same(x, y):
        return torch.equal(_bits(x.contiguous()), _bits(y.contiguous()))

    plain = run("none", "fp32")
    _check_guards(plain, rows_cols)
    x = plain[:M, :N]
    x64 = x.double()
    by_act = {"none": x}
    for act, fmt, has_res, has_vt in ACCEPTED:
        if fmt != "fp32" or has_res or has_vt or act == "none":
            continue
        out = run(act, "fp32")
        _check_guards(out, rows_cols)
        by_act[act] = out[:M, :N]
        if act == "relu":
            assert same(by_act[act], x.clamp(min=0.0)), "relu"
            print("epilogue relu  fp32: bit-exact clamp of the plain output")
            continue
        err = float(((by_act[act].double() - _act64(act, x64)).abs() / x64.abs().clamp(min=1.0)).max())
        print(f"epilogue {act:<5s} fp32: max |act - act64| / max(1, |x|) = {err:.2e}  (bar {ACT_BAR[act]:.0e})")
        assert err < ACT_BAR[act], (act, err)

    checked = 0
    for act, fmt, has_res, has_vt in ACCEPTED:
        p = by_act[act]
        tag = f"{act}/{fmt}/{'res' if has_res else '-'}/{'vt' if has_vt else '-'}"
        if has_vt:
            for c0 in (0, 128, 1536):
                dtype = torch.float16 if fmt == "f16" else torch.float32
                vt = _sentinel((N - c0 + 1, M + 8), dtype, cuda)  # one guard row, eight guard columns
                out = run(act, fmt, vt=vt, vt_col0=c0)
                full = {"fp32": p, "tf32": _tf32(p), "f16": _half_sat(p)}[fmt]
                _check_guards(out, _mask(slice(0, M), slice(0, c0), out.shape, cuda))
                _check_guards(vt, _mask(slice(0, N - c0), slice(0, M), vt.shape, cuda))
                assert same(out[:M, :c0], full[:, :c0]), (tag, c0)
                assert same(vt[:N - c0, :M], full[:, c0:].T), (tag, c0)
            checked += 1
            continue
        if has_res:
            out = run(act, fmt, res_t=res)
            r = res[:M, :N]
            want = {"none": x + r, "gelu": p + r, "relu": (x + r).clamp(min=0.0)}[act]
            if fmt == "tf32":
                want = _tf32(want)
            _check_guards(out, rows_cols)
            assert same(out[:M, :N], want), tag
            inplace = res.clone()
            run(act, fmt, res_t=inplace, out=inplace)
            assert same(inplace[:M, :N], out[:M, :N]), tag + " in place"
            assert same(inplace[M:], res[M:]) and same(inplace[:M, N:], res[:M, N:]), tag + " in-place guards"
            checked += 1
            continue
        out = run(act, fmt)
        _check_guards(out, rows_cols, split=fmt == "split")
        if fmt == "fp32":
            assert same(out[:M, :N], p), tag
        elif fmt == "tf32":
            assert same(out[:M, :N], _tf32(p)), tag
        elif fmt == "f16":
            assert same(out[:M, :N], _half_sat(p)), tag
            if act == "none":  # saturation, never inf
                assert out[:M, N - 4].eq(65504).all() and out[:M, N - 3].eq(-65504).all(), "fp16 saturation"
                assert out[:M, N - 1].eq(-65504).all(), "fp16 saturation"
        else:
            hi, lo = _unpack_split(out, M, N)
            want_hi, want_lo = _split(p)
            assert same(hi, want_hi) and same(lo, want_lo), tag
        checked += 1
    assert checked == len(ACCEPTED)
    print(f"gemm_kernel<{block_n}, {MODE_NAME[mode]}>: {checked} accepted epilogue combinations bit-exact")


# ---------------------------------------------------------------------------------------------------------------------
# GPU: schedule invariance and fp16 subnormals
def _late_row_tiles(M, N, K, mode, block_n, sms):
    """Row tiles that the persistent loop runs as the 3rd or later tile of every CTA that touches them, starting at a
    smem ring (slot, phase) other than the (0, 0) a CTA's first tile starts at: [(row tile, tile index in its CTA,
    start slot, start phase)].  Tile t = row tile * n_tiles + column block runs on CTA t % grid as its (t // grid)-th
    tile; a CTA's i-th tile starts after i * stages_per_tile ring steps."""
    n_tiles, row_tiles = N // block_n, (M + 127) // 128
    grid = min(sms, row_tiles * n_tiles)
    ring = 4 if block_n == 256 else 6
    stages = K // STAGE_K[mode]
    picked = []
    for r in range(row_tiles - 1, -1, -1):
        idx = {(r * n_tiles + j) // grid for j in range(n_tiles)}
        starts = {((i * stages) % ring, (i * stages // ring) & 1) for i in idx}
        if min(idx) >= 2 and (0, 0) not in starts:
            picked.append((r, sorted(idx), sorted(starts)))
        if len(picked) == 2:
            break
    return picked


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [TF32, BF16X3, F16], ids=["tf32", "bf16x3", "f16"])
def test_gemm_schedule_invariance(cuda, mode):
    """Each output element accumulates the same wgmma k-steps in the same order whatever the tile width or the number
    of tiles a CTA runs before it, so the fp32 results are bit-identical: BLOCK_N 128 against 256, and a row tile run
    alone (one tile per CTA, ring slot 0, phase 0) against the same rows computed late in a persistent run."""
    gen = torch.Generator(device=cuda).manual_seed(41 + mode)
    M, N = 17000, 768
    K = 49 * STAGE_K[mode]  # 49 stages: no multiple of either ring depth, so later tiles start at other slots
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    a, _ = _operand(mode, M, K, gen, cuda)
    w, _ = _operand(mode, N, K, gen, cuda)
    bias = torch.randn(N, generator=gen, device=cuda)
    outs = {}
    for bn in (128, 256):  # one guard row each
        outs[bn] = _gemm((bn, mode), a, w, _sentinel((M + 1, N), torch.float32, cuda), bias=bias, force_block_n=bn)
        _check_guards(outs[bn], _mask(slice(0, M), slice(None), outs[bn].shape, cuda))
        late = _late_row_tiles(M, N, K, mode, bn, sms)
        assert late, f"no row tile runs late at BLOCK_N {bn}"
        for r, idx, starts in late:
            r0, r1 = 128 * r, min(M, 128 * (r + 1))
            rows = r1 - r0
            one = _gemm((bn, mode), a[r0:r1], w, _sentinel((rows + 1, N), torch.float32, cuda), bias=bias,
                        force_block_n=bn)
            _check_guards(one, _mask(slice(0, rows), slice(None), one.shape, cuda))
            assert torch.equal(_bits(one[:rows]), _bits(outs[bn][r0:r1])), ("one tile per CTA vs late tile", bn, r)
            print(f"schedule invariance {MODE_NAME[mode]} K={K} BLOCK_N {bn}: rows [{r0}, {r1}) alone == the same rows "
                  f"as tile {idx} of their CTAs (ring slot, phase {starts}), bit for bit")
    assert torch.equal(_bits(outs[128]), _bits(outs[256])), "BLOCK_N 128 vs 256"
    print(f"schedule invariance {MODE_NAME[mode]} K={K}: BLOCK_N 128 == 256, bit for bit")


@pytest.mark.gpu
def test_gemm_f16_subnormal_operands(cuda):
    """fp16 subnormals (|x| < 2^-14) in A, in W and in both contribute exactly: the products are fp32 normals."""
    gen = torch.Generator(device=cuda).manual_seed(51)
    M, K, N = 300, 256, 256
    sub = lambda r: (torch.randint(-1023, 1024, (r, K), generator=gen, device=cuda).double() * 2.0 ** -24).half()  # noqa: E731
    nrm = lambda r: torch.randn(r, K, generator=gen, device=cuda).half()  # noqa: E731
    for name, a, w in (("A subnormal", sub(M), nrm(N)), ("W subnormal", nrm(M), sub(N)), ("both", sub(M), sub(N))):
        assert bool((a.float().abs() < 2.0 ** -14).all() or (w.float().abs() < 2.0 ** -14).all())
        out = _sentinel((M + 1, N), torch.float32, cuda)
        _gemm((128, F16), a, w, out)
        _check_guards(out, _mask(slice(0, M), slice(None), out.shape, cuda))
        a64, w64 = a.double(), w.double()
        _report(f"fp16 subnormals: {name}", (128, F16), _nerr(out[:M], a64 @ w64.T, a64.abs() @ w64.abs().T))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the operand converters the GEMM tests rely on
def _bf16_rn_bits(u):
    """fp32 bits (uint32 numpy) -> bf16 bits, round to nearest even."""
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


@pytest.mark.gpu
def test_round_tf32_is_ties_away(cuda):
    rng = np.random.default_rng(61)
    n = 1 << 20
    u = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    exp = (u >> 23) & 0xFF
    u = np.where((exp == 0) | (exp >= 0xFE), u & 0x807FFFFF | (0x7F << 23), u).astype(np.uint32)  # normal, no overflow
    u[: n // 4] = (u[: n // 4] & ~np.uint32(0x1FFF)) | np.uint32(0x1000)  # exact ties, both signs
    u[n // 4: n // 4 + 8] = [0x3F801000, 0xBF801000, 0x3F803000, 0xBF803000, 0x3F800FFF, 0xBF800FFF, 0x3F801001,
                             0xBF801001]
    want = ((u.astype(np.uint64) + 0x1000) & ~np.uint64(0x1FFF)).astype(np.uint32)
    x = torch.from_numpy(u.view(np.int32)).to(cuda).view(torch.float32)
    L.round_tf32_(x)
    torch.cuda.synchronize()
    got = x.view(torch.int32).cpu().numpy().view(np.uint32)
    assert np.array_equal(got, want), int((got != want).sum())
    ties = u[: n // 4]
    print(f"mer_round_tf32: {n} values bit-exact, {len(ties)} exact ties "
          f"({int((ties >> 31).sum())} negative) rounded away from zero")


@pytest.mark.gpu
@pytest.mark.parametrize("K", [32, 3072])
def test_split_bf16_is_hi_lo_round_to_nearest(cuda, K):
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    per_stride = sms * 32 * 256 * 4  # values one grid-stride pass of mer_split_bf16 covers
    rows = per_stride // K + 100  # rows beyond the first pass
    rng = np.random.default_rng(K)
    x = (rng.standard_normal((rows, K)) * np.exp2(rng.integers(-20, 20, (rows, 1)))).astype(np.float32)
    u = x.view(np.uint32)
    u[:16, :16] = (u[:16, :16] & ~np.uint32(0xFFFF)) | np.uint32(0x8000)  # exact ties of the hi rounding
    hi = _bf16_rn_bits(u)
    lo_f = x - (hi.astype(np.uint32) << 16).view(np.float32)  # exact in fp32
    lo = _bf16_rn_bits(lo_f.view(np.uint32))
    s = L.split_bf16(torch.from_numpy(x).to(cuda))
    torch.cuda.synchronize()
    b = s.view(torch.int16).cpu().numpy().view(np.uint16).reshape(rows, K // 32, 2, 32)
    assert np.array_equal(b[:, :, 0].reshape(rows, K), hi)
    assert np.array_equal(b[:, :, 1].reshape(rows, K), lo)
    print(f"mer_split_bf16 K={K}: {rows} rows ({rows * K / per_stride:.2f} grid strides) bit-exact")
