"""GPU parity of the DeBERTa branch of the text extractor: mer_disentangled_attention against mer_attention with zero
tables (its kernel-level parity with float64 is tests/test_attention_rel_gpu.py); and the whole path —
extract_embedding on the two synthetic checkpoints against the golden of the unmodified reference (1e-3, max-abs /
max-ref and relative L2), a x5 stress copy under the stress-bar rule of test_bench_config_gpu.py, packing
invariance (the conv layer included) and full-width stacks against the torch restatement in fp32."""
import ctypes as C
import os
import types

import numpy as np
import pytest
import torch

from mertools_b200 import _lib as L
from mertools_b200 import synthetic as S
from mertools_b200.extract import deberta_text as DT

pytestmark = pytest.mark.gpu
HD = 64
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FRAME_STEP = 4  # token-row stride of the golden's FRAME features (make_golden_deberta.py)
MAPS = {"v1": (False, dict(max_relative_positions=512)),
        "v2": (True, dict(max_relative_positions=512, position_buckets=256))}


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def _rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def _dims(v2, kw):
    import transformers as tf
    base = dict(vocab_size=10, hidden_size=128, num_attention_heads=2, intermediate_size=256, num_hidden_layers=1,
                max_position_embeddings=512, pos_att_type=["c2p", "p2c"], relative_attention=True)
    return DT.DebertaDims((tf.DebertaV2Config if v2 else tf.DebertaConfig)(**dict(base, **kw)))


def _round(x, f16):
    """Operand values as the kernel reads them: fp16, or tf32 (cvt.rna: round half away on the 13 dropped bits)."""
    if f16:
        return x.half()
    i = x.float().contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def _operands(lens, heads, span, f16, cuda, seed=0, zero_tables=False):
    g = torch.Generator(device=cuda).manual_seed(seed)
    T, D = sum(lens), heads * HD
    qkv = _round(torch.randn(T, 3 * D, generator=g, device=cuda) * 1.2, f16)
    vt = torch.zeros(D, (T + 7) // 8 * 8, dtype=qkv.dtype, device=cuda)
    vt[:, :T] = qkv[:, 2 * D:].T
    pos = _round(torch.randn(2 * span, 2 * D, generator=g, device=cuda) * (0.0 if zero_tables else 1.2), f16)
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=cuda)
    return qkv, vt, pos, cu


def _attn(qkv, vt, pos, cu, rows, heads, span, scale, f16, out=None, flags=None, max_len=None):
    fn = L.declare("mer_disentangled_attention", [C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p,
                                                  C.c_longlong, C.c_int, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p,
                                                  C.c_int, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_void_p])
    T, D = qkv.shape[0], heads * HD
    ctx = out if out is not None else torch.full((T, D), float("nan"), device=qkv.device)
    if flags is None:
        flags = L.MER_ATT_QKV_F16 if f16 else 0
    max_len = max_len or int((cu[1:] - cu[:-1]).max())
    L.check(fn(L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(pos), L.ptr(pos[:, D:]), pos.shape[1], span, L.ptr(rows), scale,
               L.ptr(ctx), L.ptr(cu), cu.numel() - 1, T, max_len, heads, flags, L.stream_ptr()))
    torch.cuda.synchronize()
    return ctx


# P is rounded to the operand format (10 mantissa bits, unit roundoff 2^-11) before P V: |ctx - ref| <= 2^-11 max|V|
# from that rounding, the fp32 scores and ex2.approx add far less; the bar doubles it.
BAR = 2.0 ** -10


@pytest.mark.parametrize("fmt", ["f16", "tf32"])
def test_zero_tables_match_mer_attention(cuda, fmt):
    """PK = PQ = 0 and scale 1/8: softmax(Q K^T / 8) V, what mer_attention computes (its V^T kernels: up to 505 tokens
    in fp16, 253 in tf32)."""
    f16 = fmt == "f16"
    lens = [3, 1, 63, 65, 129, 300] if f16 else [3, 1, 63, 65, 129, 250]
    heads, span = 12, 256
    qkv, vt, pos, cu = _operands(lens, heads, span, f16, cuda, seed=7, zero_tables=True)
    rows = torch.from_numpy(DT.rel_rows(_dims(*MAPS["v2"]), max(lens))).to(cuda)
    got = _attn(qkv, vt, pos, cu, rows, heads, span, 0.125, f16)
    ref = torch.full_like(got, float("nan"))
    L.attention(qkv, ref, cu, max(lens), heads, vt=vt)
    torch.cuda.synchronize()
    vmax = float(qkv[:, 2 * heads * HD:].float().abs().max())
    err = float((got - ref).abs().max())
    print(f"{fmt} zero tables vs mer_attention: {err:.2e} = {err / vmax:.2e} max|V|")
    assert err <= BAR * vmax


# ---- whole path ---------------------------------------------------------------------------------------------------
def _golden(family):
    g = np.load(os.path.join(G, "deberta_text_golden.npz"))
    return {k[len(family) + 1:]: g[k] for k in g.files if k.startswith(family + "_")}


def _checkpoint(root, family, scale=1.0):
    """The golden's checkpoint as the reference loads it: tools/transformers/deberta-chinese-large/."""
    import transformers as tf
    g = _golden(family)
    v2 = family == "v2"
    kw = dict(S.DEBERTA_GOLDEN_CFGS[family], vocab_size=int(g["vocab_size"]))
    cfg = (tf.DebertaV2Config if v2 else tf.DebertaConfig)(**kw)
    sd = S.deberta_state_dict(kw, v2, seed=int(g["seed"]), scale=scale)
    m = (tf.DebertaV2Model if v2 else tf.DebertaModel)(cfg).eval()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    mdir = os.path.join(root, "tools", "transformers", "deberta-chinese-large")
    m.save_pretrained(mdir)
    tf.BertTokenizer(os.path.join(G, "text_vocab.txt")).save_pretrained(mdir)
    return g, sd, cfg, m


def _run_extract(tmp_path, g, level):
    import pandas as pd

    from mertools_b200.extract import text
    cfg = types.SimpleNamespace(PATH_TO_PRETRAINED_MODELS=str(tmp_path / "tools"))
    sents = [np.nan if nan else str(s) for s, nan in zip(g["sentences"], g["isnan"])]
    names = [f"sample_{i:05d}" for i in range(len(sents))]
    csv = str(tmp_path / "transcription.csv")
    pd.DataFrame({"name": names, "chinese": sents}).to_csv(csv, index=False)
    text.extract_embedding("deberta-chinese-large", csv, str(tmp_path / "features"), level, gpu=0, config=cfg)
    d = tmp_path / "features" / f"deberta-chinese-large-{level[:3]}"
    return [np.load(str(d / f"{n}.npy")) for n in names]


@pytest.mark.parametrize("level", ["UTTERANCE", "FRAME"])
@pytest.mark.parametrize("family", ["v1", "v2"])
def test_extract_embedding_matches_reference_golden(cuda, tmp_path, family, level):
    g, _, _, _ = _checkpoint(str(tmp_path), family)
    got = _run_extract(tmp_path, g, level)
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


def _ids(g):
    return [g[f"ids{i}"] for i in range(len(g["sentences"])) if not g["isnan"][i] and len(g[f"ids{i}"]) > 2]


@pytest.mark.parametrize("family", ["v1", "v2"])
def test_stress_checkpoint_x5(cuda, tmp_path, family):
    """Every layer matrix x5: err <= max(1e-3, 4 * 2^13 * |fp32 reference - fp64 reference|)."""
    g, sd, cfg, m = _checkpoint(str(tmp_path), family, scale=5.0)
    ids = _ids(g)
    utt, _ = DT.DebertaTextEncoder({k: torch.from_numpy(v) for k, v in sd.items()}, cfg, device=cuda).forward(ids)
    net64 = DT.DebertaNet({k: torch.from_numpy(v) for k, v in sd.items()}, DT.TorchOps(family == "v2", dtype=torch.float64),
                          DT.DebertaDims(cfg))
    worst, noise = 0.0, 0.0
    with torch.no_grad():
        for j, x in enumerate(ids):
            r32 = torch.stack(m(torch.from_numpy(x)[None], output_hidden_states=True).hidden_states)[[-4, -3, -2, -1]]
            r32 = r32.sum(0)[0, 1:-1].mean(0).numpy()
            r64 = net64.forward(x, [len(x)])[1:-1].mean(0).numpy()
            noise = max(noise, _rel(r32, r64))
            worst = max(worst, _rel(utt[j].cpu(), r32))
    bar = max(1e-3, 4.0 * 2.0 ** 13 * noise)
    print(f"{family} x5: readout max-rel {worst:.2e}; bar {bar:.2e} (fp32-vs-fp64 {noise:.1e})")
    assert bool(torch.isfinite(utt).all()) and worst < bar


@pytest.mark.parametrize("family", ["v1", "v2"])
def test_sentence_alone_matches_packed_and_the_conv_does_not_leak(cuda, tmp_path, family):
    """A sentence alone and inside the packed batch: the LLaMA branch's bars (2e-4 on the UTTERANCE feature, 5e-4
    relative L2 / 1e-3 max on the token rows).  New tokens in the neighbouring sentences leave a sentence's token rows
    bit-identical: neither the attention nor (v2) the conv layer's taps cross a sentence boundary."""
    g, sd, cfg, _ = _checkpoint(str(tmp_path), family)
    enc = DT.DebertaTextEncoder({k: torch.from_numpy(v) for k, v in sd.items()}, cfg, device=cuda)
    ids = _ids(g)
    utt_p, packed = enc.forward(ids, want_tokens=True)
    packed, utt_p = packed.cpu().clone(), utt_p.cpu()
    o = 0
    for j, x in enumerate(ids):
        utt_a, alone = enc.forward([x], want_tokens=True)
        tok = packed[o:o + len(x)]
        d_utt = _rel(utt_a[0], utt_p[j])
        d_l2, d_max = _rel_l2(alone.cpu().numpy(), tok.numpy()), _rel(alone, tok)
        print(f"{family} sentence {j} ({len(x)} tokens): alone vs packed UTT {d_utt:.1e}, rel-L2 {d_l2:.1e}, max {d_max:.1e}")
        assert d_utt <= 2e-4 and d_l2 <= 5e-4 and d_max <= 1e-3, (j, d_utt, d_l2, d_max)
        o += len(x)
    rng = np.random.default_rng(1)
    other = [x if j % 2 == 0 else rng.integers(5, int(g["vocab_size"]), len(x)) for j, x in enumerate(ids)]
    _, changed = enc.forward(other, want_tokens=True)
    changed = changed.cpu()
    o = 0
    for j, x in enumerate(ids):
        if j % 2 == 0:
            assert torch.equal(changed[o:o + len(x)], packed[o:o + len(x)]), j
        o += len(x)


@pytest.mark.parametrize("hidden,heads,v2", [(1024, 16, False), (1536, 24, True)])
def test_full_width_stack_matches_fp32_restatement(cuda, hidden, heads, v2):
    """deberta-large (1024, 16 heads, v1) and deberta-v2-xxlarge (1536, 24 heads, buckets 256, conv) widths at 3 layers,
    random weights: the CUDA path (bf16x3 above hidden 768) against the torch restatement in fp32 (TF32 off), 1e-3
    max-abs / max-ref and relative L2.  The stress-bar rule of test_bench_config_gpu.py would allow more here (the fp32
    restatement itself is 2.9e-4 from fp64 at 1536 wide); the split-bf16 products carry ~fp32 accuracy, so 1e-3 holds."""
    import transformers as tf
    kw = dict(vocab_size=1000, hidden_size=hidden, num_attention_heads=heads, intermediate_size=4 * hidden,
              num_hidden_layers=3, max_position_embeddings=512, relative_attention=True, pos_att_type=["c2p", "p2c"],
              position_biased_input=False, type_vocab_size=0, layer_norm_eps=1e-7)
    if v2:
        kw.update(position_buckets=256, norm_rel_ebd="layer_norm", share_att_key=True, conv_kernel_size=3,
                  conv_act="gelu")
    cfg = (tf.DebertaV2Config if v2 else tf.DebertaConfig)(**kw)
    sd = S.deberta_state_dict(kw, v2, seed=31)
    rng = np.random.default_rng(3)
    lens = [int(n) for n in rng.integers(3, 130, 12)] + [600]
    ids = [rng.integers(5, 1000, n) for n in lens]
    refs = {}
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for dt in (torch.float32, torch.float64):
            net = DT.DebertaNet({k: torch.from_numpy(v) for k, v in sd.items()}, DT.TorchOps(v2, cuda, dt),
                                DT.DebertaDims(cfg))
            with torch.no_grad():
                refs[dt] = net.forward(np.concatenate(ids), lens).cpu()
            del net
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    ref = refs[torch.float32]
    noise = _rel(ref, refs[torch.float64])
    enc = DT.DebertaTextEncoder({k: torch.from_numpy(v) for k, v in sd.items()}, cfg, device=cuda)
    assert enc.precision == "bf16x3"
    _, got = enc.forward(ids, want_tokens=True)
    m, l2 = _rel(got, ref), _rel_l2(got.cpu().numpy(), ref.numpy())
    bar = 1e-3
    print(f"{hidden}/{heads} stack: max-rel {m:.2e} (bar {bar:.2e}, fp32-vs-fp64 {noise:.1e}) rel-L2 {l2:.2e}")
    assert bool(torch.isfinite(got).all()) and m < bar and l2 < 1e-3
