"""GPU parity of the ALBERT branch of the text extractor: mer_attention_hd at head_dim 32 and 64 on both operand formats
against float64 (rows of 1 to 512 tokens, 26-column heads zero-padded to 32 at scale 1 / sqrt(26)), its isolation
between packed sentences and NaN guard rows, bit-for-bit agreement with mer_attention at head_dim 64 / scale 1/8;
mer_layernorm at 128 / 384 and at 312 valid columns in 384 (MER_LN_PAD); and the whole path — extract_embedding on the
three synthetic checkpoints against the golden of the unmodified reference (1e-3, max-abs / max-ref and relative L2), a
x5 stress copy under the stress-bar rule of test_bench_config_gpu.py, packing invariance and stacks at the published
widths (xxlarge's 4096 x 64 heads x 16384 at reduced depth) against the torch restatement in fp32."""
import math
import os
import shutil
import types

import numpy as np
import pytest
import torch

import _kernel_refs as R
from mertools_b200 import _lib as L
from mertools_b200 import synthetic as S
from mertools_b200.extract import albert_text as A

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FRAME_STEP = 4
NAMES = {"tiny": ("albert_chinese_tiny", "chinese"), "small": ("albert_chinese_small", "chinese"),
         "base": ("albert-base-v2", "english")}
# a 3-token sentence first: every later sentence starts off a multiple of 8 in the packed buffer
LENS = [3, 1, 2, 63, 64, 65, 130, 300, 512]


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def _rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def _round(x, f16):
    """Operand values as the kernel reads them: fp16, or tf32 (cvt.rna)."""
    if f16:
        return x.half().float()
    b = x.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)


def _operands(lens, heads, hd, valid, f16, cuda, seed=0):
    """qkv [T, 3 heads hd] in the operand format (head columns >= valid zero), vt [heads hd, pitch], cu_seqlens."""
    g = torch.Generator().manual_seed(seed)
    T = sum(lens)
    x = torch.randn(T, 3, heads, hd, generator=g) * 1.5
    x[..., valid:] = 0
    x = _round(x.reshape(T, 3 * heads * hd), f16)
    D = heads * hd
    pitch = (T + 7) // 8 * 8
    vt = torch.zeros(D, pitch)
    vt[:, :T] = x[:, 2 * D:].T
    dt = torch.float16 if f16 else torch.float32
    cu = torch.tensor(np.r_[0, np.cumsum(lens)], dtype=torch.int32, device=cuda)
    return x, x.to(cuda, dt), vt.to(cuda, dt), cu


def _attn_hd(qkv, vt, cu, lens, heads, hd, scale, f16, ctx=None, out_flags=None):
    T = qkv.shape[0]
    if ctx is None:
        ctx = torch.full((T + 3, heads * hd), float("nan"), dtype=torch.float32, device=qkv.device)
    flags = (L.MER_ATT_QKV_F16 if f16 else 0) | (0 if out_flags is None else out_flags)
    f = L.declare("mer_attention_hd", [L.C.c_void_p] * 2 + [L.C.c_longlong, L.C.c_void_p, L.C.c_void_p, L.C.c_int,
                                                            L.C.c_longlong] + [L.C.c_int] * 3
                  + [L.C.c_float, L.C.c_int, L.C.c_void_p])
    L.check(f(L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(ctx), L.ptr(cu), len(lens), T, max(lens), heads, hd, scale,
              flags, L.stream_ptr()))
    torch.cuda.synchronize()
    return ctx


@pytest.mark.parametrize("fmt", ["f16", "tf32"])
@pytest.mark.parametrize("hd,valid", [(32, 26), (32, 32), (64, 64)])
def test_kernel_vs_float64(cuda, hd, valid, fmt):
    f16 = fmt == "f16"
    scale = 1.0 / math.sqrt(valid)
    x, qkv, vt, cu = _operands(LENS, 12, hd, valid, f16, cuda)
    ctx = _attn_hd(qkv, vt, cu, LENS, 12, hd, scale, f16)
    T = sum(LENS)
    got = ctx[:T].cpu()
    cu_l = [0] + np.cumsum(LENS).tolist()
    err = R.tc_bound_ratio(got, x, cu_l, 12, "fp32", hd=hd, scale=float(np.float32(scale)))
    print(f"hd {hd} ({valid} valid) {fmt}: max |err| / bound {err:.2f}")
    assert err <= 1.0                                       # attention_tc_bound, elementwise
    assert torch.isnan(ctx[T:]).all()                       # guard rows after the last token
    pad = got.view(T, 12, hd)[..., valid:]
    assert not pad.any()                                    # zero-padded head columns give exactly zero ctx


@pytest.mark.parametrize("fmt", ["f16", "tf32"])
def test_neighbours_do_not_leak(cuda, fmt):
    f16 = fmt == "f16"
    lens = [5, 70, 9, 200]
    x, qkv, vt, cu = _operands(lens, 12, 32, 26, f16, cuda)
    a = _attn_hd(qkv, vt, cu, lens, 12, 32, 1 / math.sqrt(26), f16)
    x2, qkv2, vt2, _ = _operands(lens, 12, 32, 26, f16, cuda, seed=7)
    o = np.r_[0, np.cumsum(lens)]
    for j in (1, 3):    # sentences 0 and 2 keep their operands, their neighbours change
        qkv[o[j]:o[j + 1]] = qkv2[o[j]:o[j + 1]]
        vt[:, o[j]:o[j + 1]] = vt2[:, o[j]:o[j + 1]]
    b = _attn_hd(qkv, vt, cu, lens, 12, 32, 1 / math.sqrt(26), f16)
    for j in (0, 2):
        assert torch.equal(a[o[j]:o[j + 1]], b[o[j]:o[j + 1]]), j


@pytest.mark.parametrize("fmt,lens", [("f16", [3, 1, 100, 249]), ("f16", [3, 300, 505]), ("tf32", [3, 1, 100, 253])])
def test_head_dim_64_at_one_eighth_equals_mer_attention(cuda, fmt, lens):
    f16 = fmt == "f16"
    x, qkv, vt, cu = _operands(lens, 12, 64, 64, f16, cuda)
    for out in (0, L.MER_EPI_ROUND_TF32, L.MER_EPI_SPLIT_BF16):
        a = _attn_hd(qkv, vt, cu, lens, 12, 64, 0.125, f16, out_flags=out)
        b = torch.full_like(a, float("nan"))
        L.check(L.lib().mer_attention(L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(b), L.ptr(cu), len(lens), sum(lens),
                                      max(lens), 12, out | (L.MER_ATT_QKV_F16 if f16 else 0), L.stream_ptr()))
        torch.cuda.synchronize()
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), out


# ---- LayerNorm ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [128, 384])
def test_layernorm_new_widths_match_torch(cuda, dim):
    g = torch.Generator().manual_seed(dim)
    rows = 1000
    x = (torch.randn(rows, dim, generator=g) * 3 + 1).to(cuda)
    gam, bet = (1 + 0.1 * torch.randn(dim, generator=g)).to(cuda), (0.1 * torch.randn(dim, generator=g)).to(cuda)
    y = torch.empty_like(x)
    y16 = torch.empty(rows, dim, dtype=torch.float16, device=cuda)
    acc = torch.ones_like(x)
    L.layernorm(x, gam, bet, y, eps=1e-12, y_split=y16, acc=acc, flags=L.MER_LN_SPLIT_F16 | L.MER_LN_ACC_ADD)
    ref = torch.nn.functional.layer_norm(x.double(), (dim,), gam.double(), bet.double(), 1e-12)
    assert float((y - ref).abs().max()) < 1e-5
    assert torch.equal(y16, y.half()) and float((acc - 1 - y).abs().max()) < 1e-6


def test_layernorm_padded_rows(cuda):
    g = torch.Generator().manual_seed(3)
    rows, valid, W = 777, 312, 384
    x = torch.randn(rows + 1, W, generator=g).to(cuda) * 2
    x[:, valid:] = torch.randn(rows + 1, W - valid, generator=g).to(cuda) * 100   # garbage in the pad is ignored
    gam, bet = (1 + 0.1 * torch.randn(W, generator=g)).to(cuda), (0.1 * torch.randn(W, generator=g)).to(cuda)
    ref = torch.nn.functional.layer_norm(x[:rows, :valid].double(), (valid,), gam[:valid].double(),
                                         bet[:valid].double(), 1e-12)
    for fl, dt in ((L.MER_LN_SPLIT_F16, torch.float16), (0, torch.float32)):
        y = torch.full((rows + 1, W), float("nan"), device=cuda)
        op = torch.full((rows + 1, W), float("nan"), dtype=dt, device=cuda)
        acc = torch.full((rows + 1, W), 1.0, device=cuda)
        acc[rows] = float("nan")
        L.check(L.lib().mer_layernorm(L.ptr(x), L.ptr(gam), L.ptr(bet), L.ptr(y), L.ptr(op), L.ptr(acc), rows, valid,
                                      1e-12, fl | L.MER_LN_PAD | L.MER_LN_ACC_ADD, L.stream_ptr()))
        torch.cuda.synchronize()
        assert float((y[:rows, :valid] - ref).abs().max()) < 1e-5
        assert not y[:rows, valid:].any() and not acc[:rows, valid:].any()
        ops = op[:rows].float() if fl else L.unsplit_bf16(op[:rows])
        assert not ops[:, valid:].any()
        assert float((acc[:rows, :valid] - 1 - y[:rows, :valid]).abs().max()) < 1e-6
        assert torch.isnan(y[rows]).all() and torch.isnan(acc[rows]).all()    # the guard row is not touched


# ---- whole path ---------------------------------------------------------------------------------------------------
def _golden(family):
    g = np.load(os.path.join(G, "albert_text_golden.npz"))
    return {k[len(family) + 1:]: g[k] for k in g.files if k.startswith(family + "_")}


def _checkpoint(root, family, scale=1.0):
    """The golden's checkpoint as the reference loads it: tools/transformers/<model name>/ with its tokenizer."""
    import transformers as tf
    g = _golden(family)
    kw = dict(S.ALBERT_GOLDEN_CFGS[family], vocab_size=int(g["vocab_size"]))
    cfg = tf.AlbertConfig(**kw)
    sd = S.albert_state_dict(kw, seed=int(g["seed"]), scale=scale)
    m = tf.AlbertModel(cfg).eval()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    mdir = os.path.join(root, "tools", "transformers", NAMES[family][0])
    m.save_pretrained(mdir)
    if family == "base":
        for f in ("spiece.model", "tokenizer_config.json"):
            shutil.copy(os.path.join(G, "albert_tokenizer", f), mdir)
    else:
        tf.BertTokenizer(os.path.join(G, "text_vocab.txt")).save_pretrained(mdir)
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
@pytest.mark.parametrize("family", ["tiny", "small", "base"])
def test_extract_embedding_matches_reference_golden(cuda, tmp_path, family, level):
    g, _, _, _ = _checkpoint(str(tmp_path), family)
    got = _run_extract(tmp_path, family, g, level)
    for i, x in enumerate(got):
        ref = g[f"{level[:3].lower()}{i}"]
        if level == "FRAME":
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
    keep = [i for i in range(len(g["sentences"])) if not g["isnan"][i] and len(g[f"ids{i}"]) > 2]
    return [g[f"ids{i}"] for i in keep]


@pytest.mark.parametrize("family", ["tiny", "small", "base"])
def test_stress_checkpoint_x5(cuda, tmp_path, family):
    """Every layer matrix x5: err <= max(1e-3, 4 * 2^13 * |fp32 reference - fp64 reference|)."""
    g, sd, cfg, m = _checkpoint(str(tmp_path), family, scale=5.0)
    ids = _ids(g)
    enc = A.AlbertTextEncoder({k: torch.from_numpy(v) for k, v in sd.items()}, cfg, device=cuda)
    utt, _ = enc.forward(ids, start=1, end=-1)
    net64 = A.AlbertNet({k: torch.from_numpy(v) for k, v in sd.items()}, A.TorchOps(dtype=torch.float64),
                        A.AlbertDims(cfg))
    H = cfg.hidden_size
    worst, noise = 0.0, 0.0
    with torch.no_grad():
        for j, x in enumerate(ids):
            r32 = torch.stack(m(torch.from_numpy(x)[None], output_hidden_states=True).hidden_states)
            r32 = r32[[-4, -3, -2, -1]].sum(0)[0, 1:-1].mean(0).numpy()
            r64 = net64.forward(x, [len(x)])[1:-1, :H].mean(0).numpy()
            noise = max(noise, _rel(r32, r64))
            worst = max(worst, _rel(utt[j].cpu(), r32))
    bar = max(1e-3, 4.0 * 2.0 ** 13 * noise)
    print(f"{family} x5 ({enc.precision}): readout max-rel {worst:.2e}; bar {bar:.2e} (fp32-vs-fp64 {noise:.1e})")
    assert bool(torch.isfinite(utt).all()) and worst < bar


@pytest.mark.parametrize("family", ["tiny", "small", "base"])
def test_sentence_alone_matches_packed_and_does_not_leak(cuda, tmp_path, family):
    """A sentence alone and inside the packed batch, with the XLNet branch's bars (UTTERANCE 2^-11 on the fp16 path,
    5e-4 relative L2 / 1e-3 max on the token rows); new tokens in the neighbouring sentences leave a sentence's token
    rows bit-identical."""
    g, sd, cfg, _ = _checkpoint(str(tmp_path), family)
    enc = A.AlbertTextEncoder({k: torch.from_numpy(v) for k, v in sd.items()}, cfg, device=cuda)
    ids = _ids(g)
    utt_bar = 2.0 ** -11 if enc.precision == "f16" else 2e-4
    utt_p, packed = enc.forward(ids, start=1, end=-1, want_tokens=True)
    packed, utt_p = packed.cpu().clone(), utt_p.cpu()
    assert packed.shape[1] == cfg.hidden_size
    o = 0
    for j, x in enumerate(ids):
        utt_a, alone = enc.forward([x], start=1, end=-1, want_tokens=True)
        tok = packed[o:o + len(x)]
        d_utt = _rel(utt_a[0], utt_p[j])
        d_l2, d_max = _rel_l2(alone.cpu().numpy(), tok.numpy()), _rel(alone, tok)
        print(f"{family} sentence {j} ({len(x)} tokens): alone vs packed UTT {d_utt:.1e}, rel-L2 {d_l2:.1e}, "
              f"max {d_max:.1e}")
        assert d_utt <= utt_bar and d_l2 <= 5e-4 and d_max <= 1e-3, (j, d_utt, d_l2, d_max)
        o += len(x)
    rng = np.random.default_rng(1)
    other = [x if j % 2 == 0 else rng.integers(10, int(g["vocab_size"]), len(x)) for j, x in enumerate(ids)]
    _, changed = enc.forward(other, start=1, end=-1, want_tokens=True)
    changed = changed.cpu()
    o = 0
    for j, x in enumerate(ids):
        if j % 2 == 0:
            assert torch.equal(changed[o:o + len(x)], packed[o:o + len(x)]), j
        o += len(x)


@pytest.mark.parametrize("name,layers", [("albert_chinese_tiny", 4), ("albert_chinese_small", 6),
                                         ("albert-base-v2", 6), ("albert-large-v2", 4), ("albert-xxlarge-v2", 2)])
def test_full_width_stack_matches_fp32_restatement(cuda, name, layers):
    """The published widths (base, large and xxlarge at reduced depth: fp16 rounding grows with depth, and twelve
    random-weight base layers on the f16 path measured 1.0e-3), random weights, rows up to 512 tokens: the CUDA path
    against the torch restatement in fp32 (TF32 off), 1e-3 max-abs / max-ref and relative L2."""
    import transformers as tf
    kw = dict(S.ALBERT_PUBLISHED_CFGS[name], num_hidden_layers=layers, vocab_size=1000)
    cfg = tf.AlbertConfig(**kw)
    sd = S.albert_state_dict(kw, seed=31)
    rng = np.random.default_rng(3)
    lens = [int(n) for n in rng.integers(3, 130, 12)] + [512]
    ids = [rng.integers(10, 1000, n) for n in lens]
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        net = A.AlbertNet({k: torch.from_numpy(v) for k, v in sd.items()}, A.TorchOps(cuda), A.AlbertDims(cfg))
        with torch.no_grad():
            ref = net.forward(np.concatenate(ids), lens).cpu()[:, :cfg.hidden_size]
        del net
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    enc = A.AlbertTextEncoder({k: torch.from_numpy(v) for k, v in sd.items()}, cfg, device=cuda)
    assert enc.precision == ("f16" if cfg.hidden_size <= 768 else "bf16x3")
    _, got = enc.forward(ids, want_tokens=True)
    m, l2 = _rel(got, ref), _rel_l2(got.cpu().numpy(), ref.numpy())
    print(f"{name} x{layers} stack ({enc.precision}): max-rel {m:.2e} rel-L2 {l2:.2e}")
    assert bool(torch.isfinite(got).all()) and m < 1e-3 and l2 < 1e-3
