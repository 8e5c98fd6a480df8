"""GPU tests of MER2023's audio extractor (extract/audio_mer2023.py): whole clips of any length with the
hidden_states[-1] readout.

* Kernel level: mer_attention_long against a float64 softmax(Q K^T / 8) V of the same fp16 operand values at 506,
  1,000, 1,249 and 2,999 tokens, and in ragged packs that mix 5 s (249-frame) and 40 s (1,999-frame) rows; rows of up
  to 505 tokens give what mer_attention gives, bit for bit; the refusals.
* Encoder level: the one-layer readout against HF HubertModel / Wav2Vec2Model hidden_states[-1] for the base (post-LN)
  and large (stable-layer-norm) families; the goldens of the unmodified reference extract; a x5 stress checkpoint at
  full depth on the default (fp16) operands; one clip alone against the same clip inside a mixed launch."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from mertools_b200 import _lib as L
from mertools_b200 import synthetic as S
from mertools_b200.extract.audio_mer2023 import LAST, LAST_FOUR, Mer2023AudioExtractor

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
HEADS, HD = 2, 64
LONG_MAX = 4096   # MER_ATT_LONG_MAX


def _rel(a, b):
    a, b = torch.as_tensor(np.asarray(a)).double(), torch.as_tensor(np.asarray(b)).double()
    return float((a - b).abs().max() / b.abs().max())


def _attention_long(qkv, vt, ctx, cu, max_seqlen, flags):
    f = L.declare("mer_attention_long", [C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_int,
                                         C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_void_p])
    L.check(f(L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(ctx), L.ptr(cu), cu.numel() - 1, qkv.shape[0], max_seqlen,
              HEADS, flags, L.stream_ptr()))
    return ctx


def _operands(lens, cuda, scale=1.5, seed=11):
    g = torch.Generator().manual_seed(seed)
    tokens = sum(lens)
    qkv = (torch.randn(tokens, 3 * HEADS * HD, generator=g) * scale).to(torch.float16)
    ld = (tokens + 7) // 8 * 8
    vt = torch.zeros(HEADS * HD, ld, dtype=torch.float16)
    vt[:, :tokens] = qkv[:, 2 * HEADS * HD:].T
    cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    host = qkv.double()
    ref = torch.zeros(tokens, HEADS * HD, dtype=torch.float64)
    for s in range(len(lens)):
        a, b = int(cu[s]), int(cu[s + 1])
        for h in range(HEADS):
            q = host[a:b, h * HD:(h + 1) * HD]
            k = host[a:b, (HEADS + h) * HD:(HEADS + h + 1) * HD]
            v = host[a:b, (2 * HEADS + h) * HD:(2 * HEADS + h + 1) * HD]
            ref[a:b, h * HD:(h + 1) * HD] = torch.softmax(q @ k.T / 8.0, dim=-1) @ v
    return qkv.to(cuda), vt.to(cuda), torch.from_numpy(cu).to(cuda), ref


@pytest.mark.parametrize("lens", [[506], [1000], [1249], [2999], [249, 1999, 249, 1999, 17], [1999, 249, 506, 1249]],
                         ids=["506", "1000", "1249", "2999", "mix5s40s", "mixall"])
@pytest.mark.parametrize("fmt", ["f16", "fp32", "split"])
def test_long_rows_vs_float64(cuda, lens, fmt):
    qkv, vt, cu, ref = _operands(lens, cuda)
    dt = torch.float16 if fmt == "f16" else torch.float32
    ctx = torch.full((qkv.shape[0], HEADS * HD), float("nan"), dtype=dt, device=cuda)
    flags = {"f16": L.MER_EPI_OUT_F16, "fp32": 0, "split": L.MER_EPI_SPLIT_BF16}[fmt]
    _attention_long(qkv, vt, ctx, cu, max(lens), flags)
    torch.cuda.synchronize()
    out = (L.unsplit_bf16(ctx) if fmt == "split" else ctx).double().cpu()
    assert torch.isfinite(out).all()
    err = _rel(out, ref)
    # fp16 P (2^-11 per probability) averaged over up to 2,999 keys; the fp16 output adds its own rounding
    assert err < (2e-3 if fmt == "f16" else 1e-3), err


def test_rows_up_to_505_are_what_mer_attention_computes(cuda):
    lens = [505, 17, 300, 249, 64]
    qkv, vt, cu, _ = _operands(lens, cuda, seed=5)
    for dt in (torch.float16, torch.float32):
        a = torch.zeros((qkv.shape[0], HEADS * HD), dtype=dt, device=cuda)
        b = torch.zeros_like(a)
        L.attention(qkv, a, cu, max(lens), HEADS, vt=vt)
        _attention_long(qkv, vt, b, cu, max(lens), L.MER_EPI_OUT_F16 if dt == torch.float16 else 0)
        torch.cuda.synchronize()
        assert torch.equal(a, b)


def test_long_rows_refusals(cuda):
    qkv, vt, cu, _ = _operands([LONG_MAX + 1], cuda, seed=3)
    ctx = torch.zeros((qkv.shape[0], HEADS * HD), dtype=torch.float16, device=cuda)
    with pytest.raises(L.MerError, match=r"mer_attention_long: max_seqlen 4097 \(1 \.\. min\(MER_ATT_LONG_MAX = 4096"):
        _attention_long(qkv, vt, ctx, cu, LONG_MAX + 1, L.MER_EPI_OUT_F16)
    with pytest.raises(L.MerError, match=r"mer_attention_long: flags 0x20"):
        _attention_long(qkv, vt, ctx, cu, 100, L.MER_ATT_QKV_F16)
    with pytest.raises(L.MerError, match=r"mer_attention_long: V\^T pitch"):
        _attention_long(qkv, vt[:, :qkv.shape[0] - 8], ctx, cu, 100, 0)
    # mer_attention keeps its own bound
    with pytest.raises(L.MerError, match=r"sequences <= 505 tokens \(max_seqlen 506\)"):
        L.attention(qkv, ctx, cu, 506, HEADS, vt=vt)


def _hf_last(sd, wave, layers, large):
    from transformers import HubertConfig, HubertModel
    kw = dict(hidden_size=1024, num_attention_heads=16, intermediate_size=4096, feat_extract_norm="layer",
              do_stable_layer_norm=True, conv_bias=True) if large else {}
    m = HubertModel(HubertConfig(num_hidden_layers=layers, **kw)).eval()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=False)
    from oracle import pipeline as P
    x = torch.from_numpy(P.wav2vec2_normalize(wave))[None]   # Wav2Vec2FeatureExtractor(do_normalize=True)
    with torch.no_grad():
        return m(x, output_hidden_states=True).hidden_states[-1][0].numpy()


@pytest.mark.parametrize("large", [False, True], ids=["base", "large"])
def test_last_layer_readout_vs_hf(cuda, large):
    layers = 4 if large else 12
    sd = S.hubert_state_dict(seed=41, layers=layers, large=large)
    waves = [S.synth_waves(1, n, seed=60 + i)[0].astype(np.float64) / 32768.0
             for i, n in enumerate((48000, 400000, 170000))]   # 3 s, 25 s (1,249 frames), 10.6 s
    ext = Mer2023AudioExtractor(sd, layer_ids=LAST, device=cuda)
    frames = ext.extract_waves(waves, "FRAME")
    utt = ext.extract_waves(waves, "UTTERANCE")
    for w, fr, u in zip(waves, frames, utt):
        ref = _hf_last(sd, w, layers, large)
        assert fr.shape == ref.shape
        # the bars of the audio goldens (tests/test_golden_gpu.py): 1e-3 on the utterance, twice that per frame
        assert _rel(u, ref.mean(axis=0)) < 1e-3, _rel(u, ref.mean(axis=0))
        assert _rel(fr, ref) < 2e-3, _rel(fr, ref)


GOLDEN_MODELS = {"hubert_base": dict(seed=21), "wav2vec2_base": dict(seed=22), "hubert_large": dict(seed=23, large=True)}


@pytest.mark.parametrize("key", list(GOLDEN_MODELS))
def test_goldens(cuda, key):
    z = np.load(os.path.join(G, "mer2023_audio_golden.npz"))
    layers, step, cols = int(z[f"{key}_layers"]), int(z["frame_step"]), int(z["frame_cols"])
    sd = S.hubert_state_dict(layers=layers, **GOLDEN_MODELS[key])
    waves = [S.synth_waves(1, int(n), seed=int(z["seed0"]) + i)[0].astype(np.float64) / 32768.0
             for i, n in enumerate(z["lens"])]
    readouts = [("last", LAST)] + ([("last4", LAST_FOUR)] if f"{key}_last4_utt0" in z else [])
    for tag, layer_ids in readouts:
        ext = Mer2023AudioExtractor(sd, layer_ids=layer_ids, device=cuda)
        levels = ("UTTERANCE", "FRAME") if tag == "last" else ("UTTERANCE",)
        for level in levels:
            got = ext.extract_waves(waves, level)
            for i, g in enumerate(got):
                name = f"{key}_{tag}_{level[:3].lower()}{i}"
                if level == "FRAME":
                    assert g.shape == (int(z[name + "_frames"]), ext.enc.hidden)
                    g = g[::step, :cols]   # the rows and features the fixture keeps
                assert g.shape == z[name].shape, name
                assert _rel(g, z[name]) < (1e-3 if level == "UTTERANCE" else 2e-3), (name, _rel(g, z[name]))


def test_x5_stress_full_depth_default_operands(cuda):
    """12 layers, weights x5, whole 25 s and 40 s clips on the default fp16 stack against the float32 oracle.  The bar
    is 1e-2, not 1e-3: on this checkpoint the emulated hidden_states[-1] error is 4e-3 .. 6e-3 in fp16 and 1.4e-3 ..
    2.3e-3 even in bf16x3 at every clip length from 1 s to 60 s (profiles/mer2023_long_audio_precision_table.json);
    it does not grow with the row length."""
    from oracle import encoders as E
    from oracle import pipeline as P
    sd = S.hubert_state_dict(seed=1, layers=12, scale=5.0)
    waves = [S.synth_waves(1, n, seed=80 + i)[0].astype(np.float64) / 32768.0 for i, n in enumerate((400000, 640000))]
    ext = Mer2023AudioExtractor(sd, layer_ids=LAST, device=cuda)
    assert ext.enc.stack_precision == "f16"
    got = ext.extract_waves(waves, "UTTERANCE")
    for w, g in zip(waves, got):
        iv = torch.from_numpy(P.wav2vec2_normalize(w))[None]
        with torch.no_grad():
            ref = E.hubert_hidden_states(sd, iv, layers=12)[-1][0].numpy().mean(axis=0)
        assert _rel(g, ref) < 1e-2, _rel(g, ref)


def test_packing_invariance(cuda):
    """A 40 s clip alone, and inside one launch with 1 s, 5 s, 12 s and 25 s clips."""
    sd = S.hubert_state_dict(seed=7, layers=4)
    lens = (640000, 16000, 80000, 192000, 400000)
    waves = [S.synth_waves(1, n, seed=90 + i)[0].astype(np.float64) / 32768.0 for i, n in enumerate(lens)]
    ext = Mer2023AudioExtractor(sd, layer_ids=LAST, device=cuda)
    alone = ext.extract_waves(waves[:1], "FRAME")[0]
    mixed = ext.extract_waves(waves, "FRAME")
    assert mixed[0].shape == alone.shape
    # the packed position shifts the key-tile boundaries of attention (the online softmax sums in another order, and
    # the fp16 context rounds accordingly): a last-bit difference, far below the 1e-3 bar
    err = _rel(mixed[0], alone)
    print(f"packing invariance, 40 s clip: {err:.2e}")
    assert err < 2e-4, err
    for w, m in zip(waves[1:], mixed[1:]):
        solo = ext.extract_waves([w], "FRAME")[0]
        assert _rel(m, solo) < 2e-4, _rel(m, solo)
