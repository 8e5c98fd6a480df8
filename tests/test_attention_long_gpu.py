"""GPU parity of the fp16 V^T attention kernel (attention_f16.cu) on sequences of 250 .. 505 tokens (audio rows of up to
10 s = 499 HuBERT frames, extract_audio_huggingface.py:40-50; CLIP L/14's 257 tokens).

Kernel level: ragged batches against a float64 softmax(Q K^T / 8) V of the same fp16 operand values (HF eager
attention, modeling_hubert.py:372-405), at several operand scales and in every ctx format the stacks ask for (fp16 /
fp32 / tf32-rounded fp32 / bf16 hi | lo split rows), element by element under attention_tc_bound
(tests/_kernel_refs.py).  Stack level: a 10 s HuBERT clip and an L/14 frame must no longer launch the mma.sync kernel of attention.cu, and must agree with the MER_ATT_F16_LONG=0 path."""
import os

import numpy as np
import pytest
import torch

import _kernel_refs as R
from mertools_b200 import _lib as L

pytestmark = pytest.mark.gpu
HEADS, HD = 3, 64
# every tile count (1..4), both S halves, every key-range shape: 16..32 steps, odd / empty third ranges, the 505 maximum
LENS = [499, 257, 250, 505, 300, 1, 17, 129, 384, 497, 256, 130, 273, 401, 64, 498]


def _operands(lens, cuda, scale=1.5):
    g = torch.Generator().manual_seed(11)
    tokens = sum(lens)
    qkv = (torch.randn(tokens, 3 * HEADS * HD, generator=g) * scale).to(torch.float16).to(cuda)
    ld = (tokens + 7) // 8 * 8
    vt = torch.zeros(HEADS * HD, ld, dtype=torch.float16, device=cuda)
    vt[:, :tokens] = qkv[:, 2 * HEADS * HD:].T
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    return qkv, vt, torch.tensor(cu, dtype=torch.int32, device=cuda), cu


def _within_bound(out, qkv, cu, fmt):
    """Worst |out - float64| / attention_tc_bound (tests/_kernel_refs.py) for ctx in format fmt."""
    return R.tc_bound_ratio(out.double(), qkv, cu, HEADS, fmt)


def _env(name, value):
    class _Ctx:
        def __enter__(self):
            self.old = os.environ.get(name)
            os.environ[name] = str(value)

        def __exit__(self, *a):
            if self.old is None:
                os.environ.pop(name, None)
            else:
                os.environ[name] = self.old
    return _Ctx()


@pytest.mark.parametrize("scale", [0.25, 1.0, 2.0, 3.0])
def test_long_attention_f16_out_vs_float64(cuda, scale):
    """fp16 ctx at operand scales from flat (0.25: nearly uniform rows) to peaked (3: scores of +-35 before the 1/8)."""
    qkv, vt, cu, cu_l = _operands(LENS, cuda, scale=scale)
    ctx = torch.full((qkv.shape[0], HEADS * HD), float("nan"), dtype=torch.float16, device=cuda)
    L.attention(qkv, ctx, cu, max(LENS), HEADS, vt=vt)
    torch.cuda.synchronize()
    assert torch.isfinite(ctx).all()
    # fp16 P, fp32 sums and the fp16 output rounding
    err = _within_bound(ctx, qkv, cu_l, "f16")
    assert err <= 1.0, err


@pytest.mark.parametrize("mode", ["fp32", "tf32", "split"])
def test_long_attention_fp32_operand_formats(cuda, mode):
    """The TF32 / BF16X3 stacks hand their 254 .. 505-token rows to this kernel and read ctx in their own operand format."""
    qkv, vt, cu, cu_l = _operands(LENS, cuda)
    ctx = torch.full((qkv.shape[0], HEADS * HD), float("nan"), dtype=torch.float32, device=cuda)
    L.attention(qkv, ctx, cu, max(LENS), HEADS, vt=vt, round_out=(mode == "tf32"), split_out=(mode == "split"))
    torch.cuda.synchronize()
    out = L.unsplit_bf16(ctx) if mode == "split" else ctx
    assert torch.isfinite(out).all()
    err = _within_bound(out, qkv, cu_l, mode)
    assert err <= 1.0, err  # fp16 P, fp32 sums and the ctx format's rounding
    if mode == "tf32":
        bits = ctx.view(torch.int32)
        assert int((bits & 0x1FFF).abs().max()) == 0  # low 13 mantissa bits cleared


def test_long_attention_agrees_with_short_kernel(cuda):
    """Sequences both kernels accept (<= 249 tokens): the tiled kernel (MER_ATT_SHORT=0) and the short kernel
    (MER_ATT_SHORT=1) round the same fp16 probabilities in another summation order; both stay under the bound."""
    lens = [197, 249, 5, 128, 129, 200, 33, 64]
    qkv, vt, cu, cu_l = _operands(lens, cuda)
    out = {}
    for short in (0, 1):
        ctx = torch.zeros((qkv.shape[0], HEADS * HD), dtype=torch.float32, device=cuda)
        fn = lambda: L.attention(qkv, ctx, cu, max(lens), HEADS, vt=vt)  # noqa: E731
        with R.env("MER_ATT_SHORT", short):
            _, names = R.attention_kernels(fn)
        assert any(("attention_short_kernel" if short else "attention_vt_kernel<true") in n for n in names), names
        out[short] = ctx
    assert not torch.equal(out[0], out[1])                   # two kernels, two summation orders
    for short in (0, 1):
        assert _within_bound(out[short], qkv, cu_l, "fp32") <= 1.0, short


def test_long_attention_large_scores(cuda):
    """Peaked rows (scores of +-60 before the 1/8 scale): the row maximum is exchanged between four warps."""
    lens = [499, 310]
    qkv, vt, cu, cu_l = _operands(lens, cuda, scale=4.0)
    ctx = torch.zeros((qkv.shape[0], HEADS * HD), dtype=torch.float32, device=cuda)
    L.attention(qkv, ctx, cu, max(lens), HEADS, vt=vt)
    torch.cuda.synchronize()
    assert torch.isfinite(ctx).all()
    assert _within_bound(ctx, qkv, cu_l, "fp32") <= 1.0


@pytest.mark.parametrize("precision", ["f16", "bf16x3"])
def test_ten_second_audio_rows_take_the_long_key_kernel(cuda, precision):
    """A 10 s clip (499 frames) through HubertEncoder in both operand formats: against the oracle, and against the
    round-1 path (MER_ATT_F16_LONG=0: TF32-rounded operands through the mma.sync flash kernel of attention.cu)."""
    from mertools_b200 import synthetic as S
    from mertools_b200.encoders import HubertEncoder
    from oracle import encoders as E
    from oracle import pipeline as P
    layers = 4
    sd = S.hubert_state_dict(seed=1, layers=layers)
    wav = (S.synth_waves(2, 160000, seed=29).astype(np.float64) / 32768.0).astype(np.float32)
    enc = HubertEncoder(sd, device=cuda, stack_precision=precision)
    utt, frames = enc.forward(torch.from_numpy(wav).to(cuda), normalize=True, want_frames=True)
    with _env("MER_ATT_F16_LONG", 0):
        utt0, frames0 = enc.forward(torch.from_numpy(wav).to(cuda), normalize=True, want_frames=True)
    torch.cuda.synchronize()
    assert frames.shape[1] == 499
    iv = torch.from_numpy(np.stack([P.wav2vec2_normalize(w) for w in wav]))
    ref_hs = E.hubert_hidden_states(sd, iv, layers=layers)
    ref = torch.stack(ref_hs)[[-4, -3, -2, -1]].sum(dim=0)
    scale = float(ref.abs().max())
    assert float((frames.cpu() - ref).abs().max()) / scale < 2e-3
    assert float((frames.cpu() - frames0.cpu()).abs().max()) / scale < 2e-3
    assert float((utt.cpu() - ref.mean(dim=1)).abs().max()) / float(ref.mean(dim=1).abs().max()) < 1e-3
