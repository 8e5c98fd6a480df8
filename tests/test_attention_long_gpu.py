"""GPU parity of the fp16 V^T attention kernel (attention_f16.cu) on sequences of 250 .. 505 tokens (audio rows of up to
10 s = 499 HuBERT frames, extract_audio_huggingface.py:40-50; CLIP L/14's 257 tokens).

Kernel level: ragged batches against a float64 softmax(Q K^T / 8) V of the same fp16 operand values (HF eager
attention, modeling_hubert.py:372-405), for every share of FMA-pipe exponentials and every ctx format the stacks ask
for (fp16 / fp32 / tf32-rounded fp32 / bf16 hi | lo split rows).  Stack level: a 10 s HuBERT clip and an L/14 frame
must no longer launch the mma.sync kernel of attention.cu, and must agree with the MER_ATT_F16_LONG=0 path."""
import os

import numpy as np
import pytest
import torch

from mertools_b200 import _lib as L

pytestmark = pytest.mark.gpu
HEADS, HD = 3, 64
# every tile count (1..4), both S halves, every key-range shape: 16..32 steps, odd / empty third ranges, the 505 maximum
LENS = [499, 257, 250, 505, 300, 1, 17, 129, 384, 497, 256, 130, 273, 401, 64, 498]


def _reference(q, k, v, cu):
    out = torch.zeros(q.shape, dtype=torch.float64)
    for s in range(len(cu) - 1):
        a, b = cu[s], cu[s + 1]
        for h in range(HEADS):
            c = slice(h * HD, (h + 1) * HD)
            p = torch.softmax(q[a:b, c] @ k[a:b, c].T / 8.0, dim=-1)
            out[a:b, c] = p @ v[a:b, c]
    return out


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
    host = qkv.double().cpu()
    ref = _reference(host[:, :HEADS * HD], host[:, HEADS * HD:2 * HEADS * HD], host[:, 2 * HEADS * HD:], cu)
    return qkv, vt, torch.tensor(cu, dtype=torch.int32, device=cuda), ref


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


@pytest.mark.parametrize("poly", [0, 1, 2, 3])
def test_long_attention_f16_out_vs_float64(cuda, poly):
    qkv, vt, cu, ref = _operands(LENS, cuda)
    ctx = torch.full((qkv.shape[0], HEADS * HD), float("nan"), dtype=torch.float16, device=cuda)
    with _env("MER_ATT_F16_POLY", poly):
        L.attention(qkv, ctx, cu, max(LENS), HEADS, vt=vt)
    torch.cuda.synchronize()
    out = ctx.double().cpu()
    assert torch.isfinite(out).all()
    # fp16 P (2^-11 relative per probability) and the fp16 output rounding: the bar of the <= 249-token kernel
    assert float((out - ref).abs().max() / ref.abs().max()) < 2e-3


@pytest.mark.parametrize("mode", ["fp32", "tf32", "split"])
def test_long_attention_fp32_operand_formats(cuda, mode):
    """The TF32 / BF16X3 stacks hand their 254 .. 505-token rows to this kernel and read ctx in their own operand format."""
    qkv, vt, cu, ref = _operands(LENS, cuda)
    ctx = torch.full((qkv.shape[0], HEADS * HD), float("nan"), dtype=torch.float32, device=cuda)
    L.attention(qkv, ctx, cu, max(LENS), HEADS, vt=vt, round_out=(mode == "tf32"), split_out=(mode == "split"))
    torch.cuda.synchronize()
    out = (L.unsplit_bf16(ctx) if mode == "split" else ctx).double().cpu()
    assert torch.isfinite(out).all()
    err = float((out - ref).abs().max() / ref.abs().max())
    assert err < 1e-3, err  # no fp16 rounding of the output here: fp16 P only
    if mode == "tf32":
        bits = ctx.view(torch.int32)
        assert int((bits & 0x1FFF).abs().max()) == 0  # low 13 mantissa bits cleared


def test_long_attention_agrees_with_short_kernel(cuda):
    """Sequences both kernels accept (<= 249 tokens): the same fp16 probabilities, another summation order."""
    lens = [197, 249, 5, 128, 129, 200, 33, 64]
    qkv, vt, cu, ref = _operands(lens, cuda)
    a = torch.zeros((qkv.shape[0], HEADS * HD), dtype=torch.float16, device=cuda)
    L.attention(qkv, a, cu, max(lens), HEADS, vt=vt)             # attention_f16.cu
    b = torch.zeros((qkv.shape[0], HEADS * HD), dtype=torch.float32, device=cuda)
    L.attention(qkv, b, cu, max(lens), HEADS, vt=vt)             # fp32 ctx: the long-key kernel
    torch.cuda.synchronize()
    assert float((a.double() - b.double()).abs().max().cpu() / ref.abs().max()) < 1.5e-3
    assert float((b.double().cpu() - ref).abs().max() / ref.abs().max()) < 1e-3


def test_long_attention_large_scores(cuda):
    """Peaked rows (scores of +-60 before the 1/8 scale): the row maximum is exchanged between four warps."""
    lens = [499, 310]
    qkv, vt, cu, ref = _operands(lens, cuda, scale=4.0)
    ctx = torch.zeros((qkv.shape[0], HEADS * HD), dtype=torch.float32, device=cuda)
    L.attention(qkv, ctx, cu, max(lens), HEADS, vt=vt)
    torch.cuda.synchronize()
    out = ctx.double().cpu()
    assert torch.isfinite(out).all()
    assert float((out - ref).abs().max() / ref.abs().max()) < 1e-3


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
