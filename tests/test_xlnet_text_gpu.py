"""GPU parity of the XLNet branch of the text extractor: mer_xlnet_attention against mer_attention with zero R and
biases (its kernel-level parity with float64 is tests/test_attention_rel_gpu.py); and the whole path —
extract_embedding on the two synthetic checkpoints against the golden of the unmodified reference (1e-3, max-abs /
max-ref and relative L2), a x5 stress copy under the stress-bar rule of test_bench_config_gpu.py, packing invariance and full-width stacks against the torch restatement in fp32."""
import json
import os
import shutil
import types

import numpy as np
import pytest
import torch

from mertools_b200 import _lib as L
from mertools_b200 import synthetic as S
from mertools_b200.extract import xlnet_text as XT

pytestmark = pytest.mark.gpu
HD = 64
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FRAME_STEP = 4  # token-row stride of the golden's FRAME features (make_golden_xlnet.py)
NAMES = {"base": ("chinese-xlnet-base", "chinese"), "large": ("xlnet-large-cased", "english")}


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def _rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def _round(x, f16):
    """Operand values as the kernel reads them: fp16, or tf32 (cvt.rna: round half away on the 13 dropped bits)."""
    if f16:
        return x.half()
    i = x.float().contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def _operands(lens, heads, f16, cuda, seed=0, zero=False, clamp_len=-1):
    g = torch.Generator(device=cuda).manual_seed(seed)
    T, D = sum(lens), heads * HD
    qkv = _round(torch.randn(T, 3 * D, generator=g, device=cuda) * 1.2, f16)
    vt = torch.zeros(D, (T + 7) // 8 * 8, dtype=qkv.dtype, device=cuda)
    vt[:, :T] = qkv[:, 2 * D:].T
    _, rows = XT.rel_table(D, max(lens), clamp_len)
    s = 0.0 if zero else 1.0
    # R in a wider buffer: the kernel reads it through its row pitch
    rbuf = _round(torch.randn(int(rows.max()) + 1, D + 64, generator=g, device=cuda) * 1.2 * s, f16)
    bias = tuple(torch.randn(n, heads, HD, generator=g, device=cuda) * 0.5 * s for n in (1, 1, 1, 2))
    tt = [np.r_[np.zeros(n - 1), 2].astype(np.int32) for n in lens]
    for k, t in enumerate(tt):   # a second segment inside some sentences as well
        t[: len(t) // 3] = k % 2
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=cuda)
    return dict(qkv=qkv, vt=vt, r=rbuf[:, :D], rows=torch.from_numpy(rows).to(cuda), bias=bias,
                types=torch.from_numpy(np.concatenate(tt)).to(cuda), cu=cu, heads=heads, max_len=max(lens))


def _attn(o, with_types, f16, scale=0.125, out=None, flags=None):
    T, D = o["qkv"].shape[0], o["heads"] * HD
    ctx = out if out is not None else torch.full((T, D), float("nan"), device=o["qkv"].device)
    if flags is None:
        flags = L.MER_ATT_QKV_F16 if f16 else 0
    L.check(L.lib().mer_xlnet_attention(
        L.ptr(o["qkv"]), L.ptr(o["vt"]), o["vt"].shape[1], L.ptr(o["r"]), o["r"].stride(0), L.ptr(o["rows"]),
        *(L.ptr(b) for b in o["bias"]), L.ptr(o["types"]) if with_types else None, scale, L.ptr(ctx), L.ptr(o["cu"]),
        o["cu"].numel() - 1, T, o["max_len"], o["heads"], flags, L.stream_ptr()))
    torch.cuda.synchronize()
    return ctx


# P is rounded to the operand format (10 mantissa bits, unit roundoff 2^-11) before P V: |ctx - ref| <= 2^-11 max|V|
# from that rounding, the fp32 scores and ex2.approx add far less; the bar doubles it.
BAR = 2.0 ** -10


@pytest.mark.parametrize("fmt", ["f16", "tf32"])
def test_zero_tables_match_mer_attention(cuda, fmt):
    """R = 0, zero biases, no token types and scale 1/8: softmax(Q K^T / 8) V, what mer_attention computes (its V^T
    kernels: up to 505 tokens in fp16, 253 in tf32)."""
    f16 = fmt == "f16"
    lens = [3, 1, 63, 65, 129, 300] if f16 else [3, 1, 63, 65, 129, 250]
    o = _operands(lens, 12, f16, cuda, seed=7, zero=True)
    got = _attn(o, False, f16)
    ref = torch.full_like(got, float("nan"))
    L.attention(o["qkv"], ref, o["cu"], max(lens), 12, vt=o["vt"])
    torch.cuda.synchronize()
    vmax = float(o["qkv"][:, 2 * 12 * HD:].float().abs().max())
    err = float((got - ref).abs().max())
    print(f"{fmt} zero tables vs mer_attention: {err:.2e} = {err / vmax:.2e} max|V|")
    assert err <= BAR * vmax


# ---- whole path ---------------------------------------------------------------------------------------------------
def _golden(family):
    g = np.load(os.path.join(G, "xlnet_text_golden.npz"))
    return {k[len(family) + 1:]: g[k] for k in g.files if k.startswith(family + "_")}


def _checkpoint(root, family, scale=1.0):
    """The golden's checkpoint as the reference loads it: tools/transformers/<model name>/, with the committed
    tokenizer (and, for "large", the config that makes token_type_ids a tokenizer output)."""
    import transformers as tf
    g = _golden(family)
    kw = dict(S.XLNET_GOLDEN_CFGS[family], vocab_size=int(g["vocab_size"]))
    cfg = tf.XLNetConfig(**kw)
    sd = S.xlnet_state_dict(kw, seed=int(g["seed"]), scale=scale)
    m = tf.XLNetModel(cfg).eval()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    mdir = os.path.join(root, "tools", "transformers", NAMES[family][0])
    m.save_pretrained(mdir)
    shutil.copy(os.path.join(G, "xlnet_tokenizer", "spiece.model"), mdir)
    tcfg = json.load(open(os.path.join(G, "xlnet_tokenizer", "tokenizer_config.json")))
    if g["with_types"]:
        tcfg["model_input_names"] = ["input_ids", "token_type_ids", "attention_mask"]
    json.dump(tcfg, open(os.path.join(mdir, "tokenizer_config.json"), "w"))
    return g, sd, cfg, m


def _run_extract(tmp_path, family, g, level):
    import pandas as pd

    from mertools_b200.extract import text
    name, lang = NAMES[family]
    cfg = types.SimpleNamespace(PATH_TO_PRETRAINED_MODELS=str(tmp_path / "tools"))
    sents = [np.nan if nan else str(s) for s, nan in zip(g["sentences"], g["isnan"])]
    names = [f"sample_{i:05d}" for i in range(len(sents))]
    csv = str(tmp_path / "transcription.csv")
    pd.DataFrame({"name": names, lang: sents}).to_csv(csv, index=False)
    text.extract_embedding(name, csv, str(tmp_path / "features"), level, gpu=0, config=cfg, language=lang)
    d = tmp_path / "features" / f"{name}-{'langeng-' if lang == 'english' else ''}{level[:3]}"
    return [np.load(str(d / f"{n}.npy")) for n in names]


@pytest.mark.parametrize("level", ["UTTERANCE", "FRAME"])
@pytest.mark.parametrize("family", ["base", "large"])
def test_extract_embedding_matches_reference_golden(cuda, tmp_path, family, level):
    g, _, _, _ = _checkpoint(str(tmp_path), family)
    got = _run_extract(tmp_path, family, g, level)
    for i, x in enumerate(got):
        ref = g[f"{level[:3].lower()}{i}"]
        if level == "FRAME":   # the golden keeps every FRAME_STEP-th token row and the full row count
            assert x.shape[0] == int(g[f"fran{i}"]), (i, x.shape, int(g[f"fran{i}"]))
            x = x[::FRAME_STEP]
        assert x.shape == ref.shape, (i, x.shape, ref.shape)
        if not ref.any():
            assert not x.any()
            continue
        assert x.dtype == np.float32, x.dtype
        m, l2 = _rel(x, ref), _rel_l2(x, ref)
        print(f"{family} {level} row {i}: max-rel {m:.2e} rel-L2 {l2:.2e}")
        assert m < 1e-3 and l2 < 1e-3, (i, m, l2)


def _ids_types(g):
    keep = [i for i in range(len(g["sentences"])) if not g["isnan"][i] and len(g[f"ids{i}"]) > 2]
    return [g[f"ids{i}"] for i in keep], ([g[f"types{i}"] for i in keep] if g["with_types"] else None)


@pytest.mark.parametrize("family", ["base", "large"])
def test_stress_checkpoint_x5(cuda, tmp_path, family):
    """Every layer matrix x5: err <= max(1e-3, 4 * 2^13 * |fp32 reference - fp64 reference|)."""
    g, sd, cfg, m = _checkpoint(str(tmp_path), family, scale=5.0)
    ids, tts = _ids_types(g)
    enc = XT.XlnetTextEncoder({k: torch.from_numpy(v) for k, v in sd.items()}, cfg, device=cuda)
    utt, _ = enc.forward(ids, token_types=tts)
    net64 = XT.XlnetNet({k: torch.from_numpy(v) for k, v in sd.items()}, XT.TorchOps(dtype=torch.float64),
                        XT.XlnetDims(cfg))
    worst, noise = 0.0, 0.0
    with torch.no_grad():
        for j, x in enumerate(ids):
            extra = dict(token_type_ids=torch.from_numpy(tts[j])[None]) if tts is not None else {}
            r32 = torch.stack(m(torch.from_numpy(x)[None], output_hidden_states=True, **extra).hidden_states)
            r32 = r32[[-4, -3, -2, -1]].sum(0)[0, :-2].mean(0).numpy()
            r64 = net64.forward(x, [len(x)], tts[j] if tts is not None else None)[:-2].mean(0).numpy()
            noise = max(noise, _rel(r32, r64))
            worst = max(worst, _rel(utt[j].cpu(), r32))
    bar = max(1e-3, 4.0 * 2.0 ** 13 * noise)
    print(f"{family} x5: readout max-rel {worst:.2e}; bar {bar:.2e} (fp32-vs-fp64 {noise:.1e})")
    assert bool(torch.isfinite(utt).all()) and worst < bar


@pytest.mark.parametrize("family", ["base", "large"])
def test_sentence_alone_matches_packed_and_does_not_leak(cuda, tmp_path, family):
    """A sentence alone and inside the packed batch: the LLaMA branch's bars (2e-4 on the UTTERANCE feature, 5e-4
    relative L2 / 1e-3 max on the token rows), except that the UTTERANCE bar of the fp16 path ("base", 768 wide) is one
    fp16 unit roundoff, 2^-11: a sentence's keys sit at other columns of the 8-aligned V^T tile once packed, so the
    fp32 sums of the attention run in another order and single fp16 roundings of ctx and the FFN activation flip; the
    mean of a short sentence's few kept rows (2 for the 4-token one) shows such a flip undiluted (2.6e-4 measured).
    New tokens in the neighbouring sentences leave a sentence's token rows bit-identical."""
    g, sd, cfg, _ = _checkpoint(str(tmp_path), family)
    enc = XT.XlnetTextEncoder({k: torch.from_numpy(v) for k, v in sd.items()}, cfg, device=cuda)
    ids, tts = _ids_types(g)
    utt_bar = 2.0 ** -11 if enc.precision == "f16" else 2e-4
    utt_p, packed = enc.forward(ids, want_tokens=True, token_types=tts)
    packed, utt_p = packed.cpu().clone(), utt_p.cpu()
    o = 0
    for j, x in enumerate(ids):
        utt_a, alone = enc.forward([x], want_tokens=True, token_types=[tts[j]] if tts is not None else None)
        tok = packed[o:o + len(x)]
        d_utt = _rel(utt_a[0], utt_p[j])
        d_l2, d_max = _rel_l2(alone.cpu().numpy(), tok.numpy()), _rel(alone, tok)
        print(f"{family} sentence {j} ({len(x)} tokens): alone vs packed UTT {d_utt:.1e}, rel-L2 {d_l2:.1e}, max {d_max:.1e}")
        assert d_utt <= utt_bar and d_l2 <= 5e-4 and d_max <= 1e-3, (j, d_utt, d_l2, d_max)
        o += len(x)
    rng = np.random.default_rng(1)
    other = [x if j % 2 == 0 else rng.integers(10, int(g["vocab_size"]), len(x)) for j, x in enumerate(ids)]
    _, changed = enc.forward(other, want_tokens=True, token_types=tts)
    changed = changed.cpu()
    o = 0
    for j, x in enumerate(ids):
        if j % 2 == 0:
            assert torch.equal(changed[o:o + len(x)], packed[o:o + len(x)]), j
        o += len(x)


@pytest.mark.parametrize("hidden,heads,act", [(768, 12, "relu"), (1024, 16, "gelu")])
def test_full_width_stack_matches_fp32_restatement(cuda, hidden, heads, act):
    """xlnet-base (768, 12 heads; f16 operands) and xlnet-large (1024, 16 heads; bf16x3) widths at 3 layers, random
    weights, token types on: the CUDA path against the torch restatement in fp32 (TF32 off), 1e-3 max-abs / max-ref and
    relative L2."""
    import transformers as tf
    kw = dict(vocab_size=1000, d_model=hidden, n_head=heads, d_inner=4 * hidden, n_layer=3, ff_activation=act,
              dropout=0.0)
    cfg = tf.XLNetConfig(**kw)
    sd = S.xlnet_state_dict(kw, seed=31)
    rng = np.random.default_rng(3)
    lens = [int(n) for n in rng.integers(3, 130, 12)] + [600]
    ids = [rng.integers(10, 1000, n) for n in lens]
    tts = [np.r_[np.zeros(n - 1), 2].astype(np.int64) for n in lens]
    refs = {}
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for dt in (torch.float32, torch.float64):
            net = XT.XlnetNet({k: torch.from_numpy(v) for k, v in sd.items()}, XT.TorchOps(cuda, dt), XT.XlnetDims(cfg))
            with torch.no_grad():
                refs[dt] = net.forward(np.concatenate(ids), lens, np.concatenate(tts)).cpu()
            del net
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    ref = refs[torch.float32]
    noise = _rel(ref, refs[torch.float64])
    enc = XT.XlnetTextEncoder({k: torch.from_numpy(v) for k, v in sd.items()}, cfg, device=cuda)
    assert enc.precision == ("f16" if hidden == 768 else "bf16x3")
    _, got = enc.forward(ids, want_tokens=True, token_types=tts)
    m, l2 = _rel(got, ref), _rel_l2(got.cpu().numpy(), ref.numpy())
    print(f"{hidden}/{heads} {act} stack ({enc.precision}): max-rel {m:.2e} (fp32-vs-fp64 {noise:.1e}) rel-L2 {l2:.2e}")
    assert bool(torch.isfinite(got).all()) and m < 1e-3 and l2 < 1e-3
