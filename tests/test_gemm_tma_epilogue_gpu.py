"""The two epilogues of gemm_kernel write the same bits.

gemm.cu stores a tile's output either straight from the accumulator registers (the register epilogue) or through
64-row shared-memory slots and TMA stores (the TMA epilogue: fp32, tf32 and fp16 outputs without residual or
activation, wherever the tensor map can express the output exactly).  Both compute the same values, so every
descriptor gives identical outputs with MER_GEMM_EPI_TMA=0 and without it.  Each case below runs both, asserts through
mer_gemm_epilogue_launches which epilogue ran, and compares bit for bit, guard rows / columns (NaN sentinels) included:
- every (BLOCK_N, mode) instantiation with every accepted activation / output-format / residual / V^T combination, on
  ragged row counts and a persistent run (the residual, activation and split-bf16 forms must take the register
  epilogue);
- the batched patch-embedding form (out_bstride, out_row0; with its broadcast residual a register-epilogue form) and a
  strided convolution;
- descriptors the TMA map cannot express exactly, which must take the register epilogue;
- whole ViT, HuBERT and BERT forwards."""
import os

import numpy as np
import pytest
import torch

from mertools_b200 import _lib as L
from test_gemm_gpu import (ACCEPTED, INSTANTIATIONS, MODE_NAME, STAGE_K, _bits, _check_guards, _mask, _operand,
                           _sentinel)

F16, TF32, BF16X3 = L.MER_GEMM_F16, L.MER_GEMM_TF32, L.MER_GEMM_BF16X3
TMA_COMBOS = [c for c in ACCEPTED if c[0] == "none" and c[1] != "split" and not c[2]]  # (act, fmt, res, vt)


_counts = L.gemm_epilogue_launches


def _run(call, tma, launches=1):
    """call() under MER_GEMM_EPI_TMA=0 (tma False) or the default; asserts that its launches took that epilogue."""
    before = _counts()
    old = os.environ.pop("MER_GEMM_EPI_TMA", None)
    if not tma:
        os.environ["MER_GEMM_EPI_TMA"] = "0"
    try:
        out = call()
        torch.cuda.synchronize()
    finally:
        os.environ.pop("MER_GEMM_EPI_TMA", None)
        if old is not None:
            os.environ["MER_GEMM_EPI_TMA"] = old
    after = _counts()
    want = (0, launches) if tma else (launches, 0)
    assert (after[0] - before[0], after[1] - before[1]) == want, ("epilogue launches", tma, before, after)
    return out


def _same(x, y):
    return torch.equal(_bits(x.contiguous()), _bits(y.contiguous()))


def _both(call, launches=1, tma_expected=True):
    """Outputs of call() on both epilogues (each call allocates its own sentinel-filled buffers)."""
    reg = _run(call, tma=False, launches=launches)
    if not tma_expected:  # the descriptor must fall back: the default run takes the register epilogue as well
        before = _counts()
        tma = call()
        torch.cuda.synchronize()
        after = _counts()
        assert (after[0] - before[0], after[1] - before[1]) == (launches, 0), "expected the register epilogue"
        return reg, tma
    return reg, _run(call, tma=True, launches=launches)


def _kw(act, fmt):
    return dict(gelu=act in ("gelu", "libm"), gelu_libm=act == "libm", quick_gelu=act == "quick", relu=act == "relu",
                gelu_tanh=act == "tanh", round_out=fmt == "tf32", split_out=fmt == "split", f16_out=fmt == "f16")


def _combo_case(dev, gen, block_n, mode, M, K, N, combo, vt_col0=0):
    act, fmt, has_res, has_vt = combo
    a, _ = _operand(mode, M, K, gen, dev, scale=False)
    w, _ = _operand(mode, N, K, gen, dev, scale=False)
    bias = torch.linspace(-8.0, 8.0, N, device=dev) + torch.rand(N, generator=gen, device=dev) * 1e-2
    ld = N + 8
    dtype = torch.float16 if fmt == "f16" else torch.float32
    res = torch.randn(M + 1, ld, generator=gen, device=dev) * 4.0 if has_res else None  # one guard row

    def call(inplace=False):
        out = res.clone() if inplace else _sentinel((M + 1, ld), dtype, dev)
        vt = _sentinel((N - vt_col0 + 1, M + 8), dtype, dev) if has_vt else None
        L.gemm(a, w, out, bias=bias, res=out if inplace else res, ld_out=ld, ld_res=ld, force_block_n=block_n,
               mode=mode, vt=vt, vt_col0=vt_col0, **_kw(act, fmt))
        return out, vt

    (o_reg, v_reg), (o_tma, v_tma) = _both(call, tma_expected=combo in TMA_COMBOS)
    tag = (block_n, MODE_NAME[mode], M, K, N, combo, vt_col0)
    assert _same(o_reg, o_tma), tag
    written_cols = slice(0, vt_col0) if has_vt else slice(0, N)
    _check_guards(o_tma, _mask(slice(0, M), written_cols, o_tma.shape, dev), split=fmt == "split")
    if has_vt:
        assert _same(v_reg, v_tma), tag + ("vt",)
        _check_guards(v_tma, _mask(slice(0, N - vt_col0), slice(0, M), v_tma.shape, dev))
    if has_res:
        (i_reg, _), (i_tma, _) = _both(lambda: call(inplace=True), tma_expected=False)
        assert _same(i_reg, i_tma), tag + ("in place",)
        assert _same(i_tma[:M, :N], o_tma[:M, :N]), tag + ("in place",)
        assert _same(i_tma[M:], res[M:]) and _same(i_tma[:M, N:], res[:M, N:]), tag + ("in-place guards",)


@pytest.mark.gpu
@pytest.mark.parametrize("block_n,mode", INSTANTIATIONS, ids=[f"{bn}-{MODE_NAME[m]}" for bn, m in INSTANTIATIONS])
def test_tma_epilogue_combinations_bit_exact(cuda, block_n, mode):
    gen = torch.Generator(device=cuda).manual_seed(71 + block_n + mode)
    N, K = 2304, STAGE_K[mode]
    cases = 0
    for combo in ACCEPTED:
        for M in (1, 63, 64, 65, 129, 300):
            for c0 in ((0, 128, 1536) if combo[3] else (0,)):
                if combo[3] and M not in (65, 300):
                    continue
                _combo_case(cuda, gen, block_n, mode, M, K, N, combo, vt_col0=c0)
                cases += 1
    print(f"gemm_kernel<{block_n}, {MODE_NAME[mode]}>: {len(ACCEPTED)} combinations ({len(TMA_COMBOS)} on the TMA "
          f"epilogue), {cases} cases, default == MER_GEMM_EPI_TMA=0 bit for bit")


@pytest.mark.gpu
@pytest.mark.parametrize("block_n,mode", INSTANTIATIONS, ids=[f"{bn}-{MODE_NAME[m]}" for bn, m in INSTANTIATIONS])
def test_tma_epilogue_persistent_bit_exact(cuda, block_n, mode):
    """17,000 rows x 768 columns: several tiles per CTA, so the slot pairs and their bulk-store groups carry across
    tiles."""
    gen = torch.Generator(device=cuda).manual_seed(81 + block_n + mode)
    for combo in (("none", "fp32", False, False), ("none", "f16", False, False), ("none", "f16", False, True),
                  ("none", "tf32", False, True), ("none", "fp32", True, False)):
        _, fmt, _, _ = combo
        if fmt == "f16" and mode != F16 or fmt == "tf32" and mode == F16:
            continue
        _combo_case(cuda, gen, block_n, mode, 17000, 3 * STAGE_K[mode], 768, combo, vt_col0=512 if combo[3] else 0)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [TF32, F16], ids=["tf32", "f16"])
def test_tma_epilogue_patch_embed_form(cuda, mode):
    """Batches of 196 rows written from row 1 of each 197-row frame: the output map's batch pitch and row offset.  With
    the position rows broadcast to every frame (res_bstride 0), as the ViT runs it, the register epilogue."""
    gen = torch.Generator(device=cuda).manual_seed(91 + mode)
    frames, P_, D = 5, 196, 768
    a, _ = _operand(mode, frames * P_, D, gen, cuda)
    w, _ = _operand(mode, D, D, gen, cuda)
    bias = torch.randn(D, generator=gen, device=cuda)
    pos = torch.randn(P_ + 1, D, generator=gen, device=cuda)

    def call(res):
        out = _sentinel((frames * 197 + 1, D), torch.float32, cuda)
        L.gemm(a, w, out, bias=bias, res=res, mode=mode, rows_per_batch=P_, batches=frames, a_rows_dim=P_,
               a_batch_stride=P_ * D, out_bstride=197, out_row0=1, res_bstride=0)
        return out

    rows = torch.cat([torch.arange(1, 197, device=cuda) + f * 197 for f in range(frames)])
    for res in (None, pos):
        reg, tma = _both(lambda: call(res), tma_expected=res is None)
        _check_guards(tma, _mask(rows[:, None], slice(None), tma.shape, cuda))
        assert _same(reg, tma)


@pytest.mark.gpu
def test_tma_epilogue_strided_conv_form(cuda):
    """HuBERT-style Conv1d(k 3, stride 2) over time-major rows, output packed and with 3 spare rows per clip."""
    gen = torch.Generator(device=cuda).manual_seed(95)
    B, T, T_pad, C, N, k = 3, 301, 306, 128, 256, 3
    T_out = (T - k) // 2 + 1
    x = (torch.randn(B, T_pad, C, generator=gen, device=cuda)).half()
    w = (torch.randn(N, k * C, generator=gen, device=cuda) * 0.1).half()
    bias = torch.randn(N, generator=gen, device=cuda)
    for bstride in (T_out, T_out + 3):
        for flags in (dict(), dict(f16_out=True)):
            dtype = torch.float16 if flags.get("f16_out") else torch.float32

            def call():
                out = _sentinel((B * bstride + 1, N), dtype, cuda)
                L.gemm(x.view(B * T_pad, C), w, out, bias=bias, mode=F16, rows_per_batch=T_out, batches=B,
                       a_rows_dim=T_pad // 2, K_inner=C, taps=k, P=2, a_phase_stride=C, a_row_stride=2 * C,
                       a_batch_stride=T_pad * C, out_bstride=bstride, **flags)
                return out

            reg, tma = _both(call)
            rows = torch.cat([torch.arange(T_out, device=cuda) + b * bstride for b in range(B)])
            _check_guards(tma, _mask(rows[:, None], slice(None), tma.shape, cuda))
            assert _same(reg, tma), (bstride, flags)


@pytest.mark.gpu
def test_tma_epilogue_fallback_descriptors(cuda):
    """Descriptors the TMA maps cannot express take the register epilogue by default and still compute the same
    values as an aligned descriptor on the TMA epilogue."""
    gen = torch.Generator(device=cuda).manual_seed(97)
    M, K, N = 300, 64, 256
    a, _ = _operand(F16, M, K, gen, cuda)
    w, _ = _operand(F16, N, K, gen, cuda)
    bias = torch.randn(N, generator=gen, device=cuda)

    def aligned(f16):
        out = _sentinel((M, N), torch.float16 if f16 else torch.float32, cuda)
        L.gemm(a, w, out, bias=bias, mode=F16, f16_out=f16)
        return out

    ref16, ref32 = _run(lambda: aligned(True), tma=True), _run(lambda: aligned(False), tma=True)

    def f16_pitch():  # fp16 rows of N + 4 elements: a pitch of 8 bytes modulo 16
        out = _sentinel((M + 1, N + 4), torch.float16, cuda)
        L.gemm(a, w, out, bias=bias, mode=F16, f16_out=True, ld_out=N + 4)
        return out

    def base8():  # fp32 output starting 8 bytes into a 16-byte-aligned buffer
        buf = _sentinel((M * N + 4,), torch.float32, cuda)
        L.gemm(a, w, buf[2:2 + M * N].view(M, N), bias=bias, mode=F16)
        return buf

    def vt_col0_mid():  # V^T from column 160: not a multiple of the 64-column fp16 sub-tile
        out = _sentinel((M, N), torch.float16, cuda)
        vt = _sentinel((N - 160, M + 4), torch.float16, cuda)
        L.gemm(a, w, out, bias=bias, mode=F16, f16_out=True, vt=vt, vt_col0=160)
        return out, vt

    reg, dflt = _both(f16_pitch, tma_expected=False)
    assert _same(reg, dflt) and _same(dflt[:M, :N], ref16)
    _check_guards(dflt, _mask(slice(0, M), slice(0, N), dflt.shape, cuda))
    reg, dflt = _both(base8, tma_expected=False)
    assert _same(reg, dflt) and _same(dflt[2:2 + M * N].view(M, N), ref32)
    assert bool((_bits(dflt[:2]) == 0x7FC00000).all() and (_bits(dflt[2 + M * N:]) == 0x7FC00000).all())
    (o_reg, v_reg), (o_dflt, v_dflt) = _both(vt_col0_mid, tma_expected=False)
    assert _same(o_reg, o_dflt) and _same(v_reg, v_dflt)
    assert _same(o_dflt[:, :160], ref16[:, :160]) and _same(v_dflt[:, :M], ref16[:, 160:].T)


@pytest.mark.gpu
def test_tma_epilogue_encoders_bit_identical(cuda):
    """ViT frame features (64 frames), HuBERT and BERT forwards: the same bits on both epilogues."""
    from mertools_b200 import synthetic as S
    from mertools_b200.encoders import BertEncoder, HubertEncoder, VitEncoder

    def both(fn):
        os.environ["MER_GEMM_EPI_TMA"] = "0"
        try:
            reg = fn()
        finally:
            os.environ.pop("MER_GEMM_EPI_TMA", None)
        before = _counts()
        tma = fn()
        torch.cuda.synchronize()
        assert _counts()[1] > before[1], "no launch took the TMA epilogue"
        return reg, tma

    vit = VitEncoder(S.vit_state_dict(seed=0, layers=4), device=cuda)
    frames = torch.from_numpy(S.synth_frames(1, 64, seed=1)[0]).to(cuda)
    reg, tma = both(lambda: vit.frame_features(frames).cpu())
    assert np.array_equal(reg.numpy(), tma.numpy()), "ViT"

    hub = HubertEncoder(S.hubert_state_dict(seed=1, layers=4), device=cuda)
    wav = torch.from_numpy((S.synth_waves(2, 32000, seed=2).astype(np.float64) / 32768.0).astype(np.float32)).to(cuda)
    reg, tma = both(lambda: hub.forward(wav)[0].cpu())
    assert np.array_equal(reg.numpy(), tma.numpy()), "HuBERT"

    bert = BertEncoder(S.bert_state_dict(300, seed=2, layers=4), device=cuda)
    ids = [[2, 17, 250, 99, 42, 7, 3], list(range(5, 60))]
    reg, tma = both(lambda: bert.forward(ids)[0].cpu())
    assert np.array_equal(reg.numpy(), tma.numpy()), "BERT"
    print("ViT / HuBERT / BERT outputs bit-identical on the register and TMA epilogues")
