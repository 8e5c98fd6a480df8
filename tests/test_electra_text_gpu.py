"""GPU parity of the ELECTRA / hidden-256 branch of the text extractor: mer_layernorm at 256 columns in every flag form
the post-LN stack uses (fp32, split fp16, split bf16, ACC_INIT / ACC_ADD, ROUND_TF32, MER_LN_VER=1, MER_LN_PAD) against
float64; the 128- and 256-wide embeddings (hidden state 0) against float64; every hidden state of mer_bert_forward /
mer_bert_forward_projected on both operand formats against the fp32 restatement (tests/_electra_ref.py); extract_embedding
and MER2023's English word path against the goldens of the unmodified reference (1e-3, max-abs / max-ref and relative
L2); a x5 stress copy; packing invariance; and 12-layer ELECTRA-small / LERT-small stacks."""
import os
import types

import numpy as np
import pytest
import torch

from _electra_ref import electra_hidden_states
from mertools_b200 import _lib as L
from mertools_b200 import synthetic as S
from mertools_b200.encoders import BertEncoder

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FRAME_STEP = 4
NAMES = {"small": ("chinese-electra-180g-small", "chinese"), "base": ("chinese-electra-180g-base", "chinese"),
         "lert_small": ("chinese-lert-small", "chinese"), "eng": ("electra-base-discriminator", "english")}
CFG_OF = {"small": "small", "base": "base", "lert_small": "lert_small", "eng": "base", "words": "base"}


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def _rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def _tf32(x):
    """cvt.rna to tf32 (round to nearest, ties away), as MER_LN_ROUND_TF32 does."""
    b = x.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)


# ---- LayerNorm at 256 -------------------------------------------------------------------------------------------------
def _ln_inputs(cuda, rows=1000, dim=256, seed=256):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(rows, dim, generator=g) * 3 + 1).to(cuda)
    gam, bet = (1 + 0.1 * torch.randn(dim, generator=g)).to(cuda), (0.1 * torch.randn(dim, generator=g)).to(cuda)
    ref = torch.nn.functional.layer_norm(x.double(), (dim,), gam.double(), bet.double(), 1e-12)
    return x, gam, bet, ref


def _ln_forms(x, gam, bet, cuda):
    """Every flag form the post-LN stacks use; returns {form: (y, second output, acc)}."""
    rows, dim = x.shape
    out = {}
    for form, fl in (("fp32", 0), ("split_f16", L.MER_LN_SPLIT_F16), ("split_bf16", 0),
                     ("acc_init", L.MER_LN_ACC_INIT | L.MER_LN_ROUND_TF32), ("acc_add", L.MER_LN_ACC_ADD | L.MER_LN_SPLIT_F16),
                     ("round_tf32", L.MER_LN_ROUND_TF32)):
        y = torch.full((rows + 1, dim), float("nan"), device=cuda)
        ys = None
        if form == "split_f16" or form == "acc_add":
            ys = torch.full((rows + 1, dim), float("nan"), dtype=torch.float16, device=cuda)
        elif form == "split_bf16":
            ys = torch.full((rows + 1, dim), float("nan"), device=cuda)
        acc = torch.full((rows + 1, dim), 1.0, device=cuda) if form.startswith("acc") else None
        L.check(L.lib().mer_layernorm(L.ptr(x), L.ptr(gam), L.ptr(bet), L.ptr(y), L.ptr(ys), L.ptr(acc), rows, dim,
                                      1e-12, fl, L.stream_ptr()))
        torch.cuda.synchronize()
        out[form] = (y, ys, acc)
    return out


@pytest.mark.parametrize("ver", ["2", "1"])
def test_layernorm_256_every_flag_form_against_float64(cuda, monkeypatch, ver):
    if ver == "1":
        monkeypatch.setenv("MER_LN_VER", "1")
    x, gam, bet, ref = _ln_inputs(cuda)
    rows = x.shape[0]
    forms = _ln_forms(x, gam, bet, cuda)
    for form, (y, ys, acc) in forms.items():
        assert torch.isnan(y[rows]).all(), form                       # the guard row is not touched
        yv = y[:rows]
        if form in ("acc_init", "round_tf32"):
            assert torch.equal(yv, _tf32(forms["fp32"][0][:rows])), form
        else:
            err = float((yv - ref).abs().max())
            print(f"v{ver} {form}: max|err| {err:.2e}")
            assert err < 1e-5, (form, err)
        if form in ("split_f16", "acc_add"):
            assert torch.equal(ys[:rows], forms["fp32"][0][:rows].half()), form
        if form == "split_bf16":
            un = L.unsplit_bf16(ys[:rows])
            assert float(((un - yv).abs() / yv.abs().clamp_min(1e-30)).max()) < 2.0 ** -15
        if form == "acc_init":
            assert torch.equal(acc[:rows], forms["fp32"][0][:rows])  # acc takes the value before the tf32 rounding
        if form == "acc_add":
            assert float((acc[:rows] - 1 - forms["fp32"][0][:rows]).abs().max()) < 1e-6
        if acc is not None:
            assert (acc[rows] == 1).all()


def test_layernorm_256_versions_agree_bit_for_bit(cuda, monkeypatch):
    x, gam, bet, _ = _ln_inputs(cuda, rows=4099, seed=7)
    v2 = _ln_forms(x, gam, bet, cuda)
    monkeypatch.setenv("MER_LN_VER", "1")
    v1 = _ln_forms(x, gam, bet, cuda)
    for form in v2:
        for a, b in zip(v2[form], v1[form]):
            if a is not None:
                assert torch.equal(a.view(torch.int16 if a.dtype == torch.float16 else torch.int32),
                                   b.view(torch.int16 if b.dtype == torch.float16 else torch.int32)), form


@pytest.mark.parametrize("valid", [129, 200, 255, 256])
def test_layernorm_256_padded_rows(cuda, valid):
    g = torch.Generator().manual_seed(valid)
    rows, W = 777, 256
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
        assert torch.isnan(y[rows]).all() and torch.isnan(acc[rows]).all()


def test_layernorm_640_refusal_lists_256(cuda):
    x = torch.zeros(4, 640, device=cuda)
    g = torch.ones(640, device=cuda)
    with pytest.raises(L.MerError, match=r"mer_layernorm: dim 640 not supported \(512, 768, 1024, 1280, 1536\) "
                                         r"\(also 128, 384 and 256"):
        L.layernorm(x, g, g, torch.empty_like(x), eps=1e-12)


# ---- encoder ---------------------------------------------------------------------------------------------------------
def _model(family, vocab, seed, layers=None, scale=1.0):
    kw = dict(S.ELECTRA_GOLDEN_CFGS[CFG_OF[family]], vocab_size=vocab)
    if layers is not None:
        kw["num_hidden_layers"] = layers
    ekw = dict(kw, embedding_size=kw["hidden_size"]) if family == "lert_small" else kw
    return kw, S.electra_state_dict(ekw, seed=seed, scale=scale)


def _sentences(vocab, lens, seed=3):
    rng = np.random.default_rng(seed)
    out = []
    for n in lens:
        x = rng.integers(5, vocab, n)
        x[0], x[-1] = 2, 3
        out.append(x)
    return out


# a 3-token sentence first: later sentences start off a multiple of 8; 300 / 512 take the fp16 long-row attention
LENS = [3, 1, 2, 17, 63, 64, 65, 130, 300, 512]


def _restated(sd, ids, kw, dtype=torch.float32):
    with torch.no_grad():
        hs = [electra_hidden_states(sd, x, kw["num_hidden_layers"], kw["num_attention_heads"], dtype=dtype)
              for x in ids]
    return torch.stack([torch.cat([h[i][0] for h in hs]) for i in range(kw["num_hidden_layers"] + 1)])


@pytest.mark.parametrize("family", ["small", "lert_small"])
def test_embedding_at_128_and_256_against_float64(cuda, family):
    """hidden state 0: LayerNorm_256 of the embedding sum (LERT-small), or LayerNorm_128 then the bf16x3 projection
    (ELECTRA-small), against float64."""
    kw, sd = _model(family, 2000, seed=9)
    ids = _sentences(2000, LENS)
    enc = BertEncoder(sd, device=cuda, precision="bf16x3")
    assert enc.hidden == 256 and enc.emb_dim == (128 if family == "small" else 256)
    _, _, hidden, _ = enc.forward(ids, want_tokens=True, return_hidden=True)
    ref = _restated(sd, ids, dict(kw, num_hidden_layers=0), dtype=torch.float64)[0]
    err = _rel(hidden[0], ref)
    print(f"{family} hidden_states[0]: max-abs / max-ref {err:.2e}")
    assert err < (2e-6 if family == "lert_small" else 2e-5)


@pytest.mark.parametrize("precision", ["f16", "bf16x3"])
@pytest.mark.parametrize("family", ["small", "lert_small"])
def test_every_hidden_state_against_restatement(cuda, family, precision):
    kw, sd = _model(family, 2000, seed=11)
    ids = _sentences(2000, LENS)
    enc = BertEncoder(sd, device=cuda, precision=precision)
    _, _, hidden, _ = enc.forward(ids, want_tokens=True, return_hidden=True)
    ref = _restated(sd, ids, kw, dtype=torch.float64)
    assert hidden.shape == ref.shape
    bar = 4e-3 if precision == "f16" else 2e-4
    for i in range(hidden.shape[0]):
        err = _rel(hidden[i], ref[i])
        print(f"{family} {precision} hidden_states[{i}]: max-abs / max-ref {err:.2e}")
        assert err < bar, (i, err)


def test_projection_refusals(cuda):
    _, sd = _model("small", 100, seed=1)
    enc = BertEncoder(sd, device=cuda)
    enc.proj.emb_dim = 64
    with pytest.raises(L.MerError, match="embedding size 64"):
        enc.forward([[2, 5, 3]])
    enc.proj.emb_dim = 128
    enc.proj.proj_w = None
    with pytest.raises(L.MerError, match="null table or weight"):
        enc.forward([[2, 5, 3]])


# ---- whole path against the goldens -------------------------------------------------------------------------------------
def _golden(family):
    g = np.load(os.path.join(G, "electra_text_golden.npz"))
    return {k[len(family) + 1:]: g[k] for k in g.files if k.startswith(family + "_")}


def _checkpoint(root, family, vocab_file="text_vocab.txt"):
    """The golden's checkpoint as the reference loads it: tools/transformers/<model name>/ with its tokenizer."""
    import transformers as tf
    g = _golden(family)
    kw = dict(S.ELECTRA_GOLDEN_CFGS[CFG_OF[family]], vocab_size=int(g["vocab_size"]))
    if family == "lert_small":
        bkw = {k: v for k, v in kw.items() if k != "embedding_size"}
        m = tf.BertModel(tf.BertConfig(**bkw), add_pooling_layer=False)
        sd = S.electra_state_dict(dict(kw, embedding_size=kw["hidden_size"]), int(g["seed"]))
    elif family in ("eng", "words"):
        m = tf.ElectraForPreTraining(tf.ElectraConfig(**kw))
        sd = S.electra_state_dict(kw, int(g["seed"]), pretraining=True)
    else:
        m = tf.ElectraModel(tf.ElectraConfig(**kw))
        sd = S.electra_state_dict(kw, int(g["seed"]))
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=False)
    name = NAMES["eng" if family == "words" else family][0]
    mdir = os.path.join(root, "tools", "transformers", name)
    m.save_pretrained(mdir)
    tf.BertTokenizer(os.path.join(G, vocab_file), do_lower_case=True).save_pretrained(mdir)
    return g


@pytest.mark.parametrize("level", ["UTTERANCE", "FRAME"])
@pytest.mark.parametrize("family", ["small", "base", "lert_small", "eng"])
def test_extract_embedding_matches_reference_golden(cuda, tmp_path, family, level):
    import pandas as pd

    from mertools_b200.extract import text
    g = _checkpoint(str(tmp_path), family)
    name, lang = NAMES[family]
    cfg = types.SimpleNamespace(PATH_TO_PRETRAINED_MODELS=str(tmp_path / "tools"))
    sents = [np.nan if nan else str(s) for s, nan in zip(g["sentences"], g["isnan"])]
    names = [f"sample_{i:05d}" for i in range(len(sents))]
    csv = str(tmp_path / "transcription.csv")
    pd.DataFrame({"name": names, lang: sents}).to_csv(csv, index=False)
    text.extract_embedding(name, csv, str(tmp_path / "features"), level, gpu=0, config=cfg, language=lang)
    d = tmp_path / "features" / f"{name}-{'langeng-' if lang == 'english' else ''}{level[:3]}"
    for i, n in enumerate(names):
        x = np.load(str(d / f"{n}.npy"))
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


@pytest.mark.parametrize("level", ["UTTERANCE", "FRAME"])
def test_english_word_path_matches_reference_golden(cuda, tmp_path, level):
    import pandas as pd

    from mertools_b200.extract import text_english as TE
    g = _checkpoint(str(tmp_path), "words", vocab_file="text_words_vocab.txt")
    name = NAMES["eng"][0]
    csv = str(tmp_path / "trans.csv")
    pd.DataFrame({"name": [str(n) for n in g["names"]], "sentence": [str(s) for s in g["sentences"]]}).to_csv(
        csv, index=False)
    cfg = types.SimpleNamespace(PATH_TO_PRETRAINED_MODELS=str(tmp_path / "tools"))
    TE.extract_bert_embedding_english(name, csv, str(tmp_path / "feat"), level, gpu=0, config=cfg)
    for n in g["names"]:
        x = np.load(str(tmp_path / "feat" / f"{name}-4-{level[:3]}" / f"{n}.npy"))
        ref = g[f"{level[:3].lower()}_{n}"]
        assert x.shape == ref.shape, (n, x.shape, ref.shape)
        m, l2 = _rel(x, ref), _rel_l2(x, ref)
        print(f"words {level} {n}: max-rel {m:.2e} rel-L2 {l2:.2e}")
        assert m < 1e-3 and l2 < 1e-3, (n, m, l2)


@pytest.mark.parametrize("family", ["small", "lert_small"])
def test_stress_checkpoint_x5(cuda, family):
    """Every layer matrix x5: err <= max(1e-3, 4 * 2^13 * |fp32 restatement - fp64 restatement|)."""
    kw, sd = _model(family, 2000, seed=13, scale=5.0)
    ids = _sentences(2000, [3, 17, 64, 130, 300])
    enc = BertEncoder(sd, device=cuda)
    utt, _ = enc.forward(ids, start=1, end=-1)
    r32 = _restated(sd, ids, kw)[-4:].sum(0)
    r64 = _restated(sd, ids, kw, dtype=torch.float64)[-4:].sum(0)
    worst, noise, o = 0.0, 0.0, 0
    for j, x in enumerate(ids):
        a32, a64 = r32[o + 1:o + len(x) - 1].mean(0), r64[o + 1:o + len(x) - 1].mean(0)
        noise = max(noise, _rel(a32, a64))
        worst = max(worst, _rel(utt[j], a32))
        o += len(x)
    bar = max(1e-3, 4.0 * 2.0 ** 13 * noise)
    print(f"{family} x5 ({enc.precision}): readout max-rel {worst:.2e}; bar {bar:.2e} (fp32-vs-fp64 {noise:.1e})")
    assert bool(torch.isfinite(utt).all()) and worst < bar


@pytest.mark.parametrize("precision", ["f16", "bf16x3"])
@pytest.mark.parametrize("family", ["small", "lert_small"])
def test_sentence_alone_matches_packed_and_does_not_leak(cuda, family, precision):
    """A sentence alone and inside the packed batch (UTTERANCE 2^-11 on the fp16 path, 2e-4 on bf16x3; 5e-4 relative L2
    / 1e-3 max on the token rows); new tokens in the neighbouring sentences leave a sentence's token rows bit-identical."""
    _, sd = _model(family, 2000, seed=15)
    enc = BertEncoder(sd, device=cuda, precision=precision)
    ids = _sentences(2000, LENS[3:])
    utt_bar = 2.0 ** -11 if precision == "f16" else 2e-4
    utt_p, packed = enc.forward(ids, start=1, end=-1, want_tokens=True)
    packed, utt_p = packed.cpu().clone(), utt_p.cpu()
    o = 0
    for j, x in enumerate(ids):
        utt_a, alone = enc.forward([x], start=1, end=-1, want_tokens=True)
        tok = packed[o:o + len(x)]
        d_utt = _rel(utt_a[0], utt_p[j])
        d_l2, d_max = _rel_l2(alone.cpu().numpy(), tok.numpy()), _rel(alone, tok)
        print(f"{family} {precision} sentence {j} ({len(x)} tokens): alone vs packed UTT {d_utt:.1e}, "
              f"rel-L2 {d_l2:.1e}, max {d_max:.1e}")
        assert d_utt <= utt_bar and d_l2 <= 5e-4 and d_max <= 1e-3, (j, d_utt, d_l2, d_max)
        o += len(x)
    rng = np.random.default_rng(1)
    other = [x if j % 2 == 0 else rng.integers(10, 2000, len(x)) for j, x in enumerate(ids)]
    _, changed = enc.forward(other, start=1, end=-1, want_tokens=True)
    changed = changed.cpu()
    o = 0
    for j, x in enumerate(ids):
        if j % 2 == 0:
            assert torch.equal(changed[o:o + len(x)], packed[o:o + len(x)]), j
        o += len(x)


@pytest.mark.parametrize("precision", ["f16", "bf16x3"])
@pytest.mark.parametrize("name", ["chinese-electra-180g-small", "chinese-lert-small"])
def test_full_depth_small_stack_matches_fp32_restatement(cuda, name, precision):
    """The published small shapes at their full 12 layers, random weights, rows up to 512 tokens: the CUDA path
    against the fp32 restatement (TF32 off), 1e-3 max-abs / max-ref and relative L2 on the last-four token readout."""
    kw = dict(S.ELECTRA_PUBLISHED_CFGS[name], vocab_size=1000)
    ekw = dict(kw, embedding_size=kw["hidden_size"]) if name == "chinese-lert-small" else kw
    sd = S.electra_state_dict(ekw, seed=31)
    rng = np.random.default_rng(3)
    lens = [int(n) for n in rng.integers(3, 130, 12)] + [512]
    ids = _sentences(1000, lens, seed=5)
    ref = _restated(sd, ids, kw)[-4:].sum(0)
    enc = BertEncoder(sd, device=cuda, precision=precision)
    assert enc.n_layers == 12 and enc.hidden == 256
    _, got = enc.forward(ids, want_tokens=True)
    m, l2 = _rel(got, ref), _rel_l2(got.cpu().numpy(), ref.numpy())
    print(f"{name} x12 stack ({precision}): max-rel {m:.2e} rel-L2 {l2:.2e}")
    assert bool(torch.isfinite(got).all()) and m < 1e-3 and l2 < 1e-3


def test_default_precision_at_hidden_256(cuda, monkeypatch):
    monkeypatch.delenv("MER_TEXT_PRECISION", raising=False)
    _, sd = _model("small", 100, seed=1)
    assert BertEncoder(sd, device=cuda).precision == "bf16x3"
    monkeypatch.setenv("MER_TEXT_PRECISION", "f16")
    assert BertEncoder(sd, device=cuda).precision == "f16"
