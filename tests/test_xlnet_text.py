"""XLNet text branch on CPU: the orchestration (XlnetNet over TorchOps) against HF XLNetModel on every hidden state for
each toggle (activation, clamp_len, token types), the relative-position rows against HF's own position code, the
weight reshapes against HF's einsums, the reference golden (tests/golden/xlnet_text_golden.npz, written by
make_golden_xlnet.py from the unmodified reference extract_embedding), the tokenizer hook that forwards token_type_ids,
the config refusals (before any weight is read) and the C ABI refusals of mer_xlnet_attention (fake, never-dereferenced
addresses)."""
import ctypes as C
import json
import os
import shutil

import numpy as np
import pytest
import torch

from mertools_b200 import _lib as L
from mertools_b200 import synthetic as S
from mertools_b200.extract import xlnet_text as XT

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FRAME_STEP = 4  # token-row stride of the golden's FRAME features (make_golden_xlnet.py)

SMALL = dict(vocab_size=97, d_model=128, n_head=2, d_inner=256, n_layer=4, dropout=0.0)
# (ff_activation, clamp_len, token types): every toggle the path computes
TOGGLES = {
    "relu": ("relu", -1, False),
    "gelu-types": ("gelu", -1, True),
    "gelu-clamp-types": ("gelu", 7, True),
    "relu-clamp": ("relu", 5, False),
}
LENS = (5, 40, 1, 23)


def hf_config(kw):
    import transformers as tf
    return tf.XLNetConfig(**kw)


def hf_model(kw, sd):
    import transformers as tf
    m = tf.XLNetModel(hf_config(kw)).eval()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    return m


def torch_net(kw, sd, dtype=torch.float32):
    return XT.XlnetNet({k: torch.from_numpy(v) for k, v in sd.items()}, XT.TorchOps(dtype=dtype),
                       XT.XlnetDims(hf_config(kw)))


def _types(n):
    """The 4.x XLNetTokenizer's token_type_ids of one sentence: 0 for the text and <sep>, 2 for <cls>."""
    return np.r_[np.zeros(n - 1, np.int64), 2]


@pytest.mark.parametrize("name", sorted(TOGGLES))
def test_orchestration_matches_hf_on_every_hidden_state(name):
    act, clamp, with_types = TOGGLES[name]
    kw = dict(SMALL, ff_activation=act, clamp_len=clamp)
    sd = S.xlnet_state_dict(kw, seed=5)
    m = hf_model(kw, sd)
    rng = np.random.default_rng(0)
    sents = [rng.integers(5, kw["vocab_size"], n) for n in LENS]
    types = [_types(n) for n in LENS]
    net = torch_net(kw, sd)
    with torch.no_grad():
        acc, hs = net.forward(np.concatenate(sents), list(LENS), np.concatenate(types) if with_types else None,
                              return_hidden=True)
    assert len(hs) == kw["n_layer"] + 1
    o = 0
    for ids, tt, n in zip(sents, types, LENS):
        extra = dict(token_type_ids=torch.from_numpy(tt)[None]) if with_types else {}
        with torch.no_grad():
            ref = m(input_ids=torch.from_numpy(ids)[None], attention_mask=torch.ones(1, n, dtype=torch.long),
                    output_hidden_states=True, **extra).hidden_states
        for k, (got, want) in enumerate(zip(hs, ref)):
            err = float((got[o:o + n] - want[0]).abs().max())
            assert err <= 5e-5, (name, n, k, err)
        err = float((acc[o:o + n] - torch.stack(ref)[[-4, -3, -2, -1]].sum(0)[0]).abs().max())
        assert err <= 2e-4, (name, n, err)
        o += n


def test_segment_term_changes_the_result():
    """With token types the segment term is live (a restatement that ignored it would pass the no-types toggles)."""
    kw = dict(SMALL, ff_activation="gelu")
    net = torch_net(kw, S.xlnet_state_dict(kw, seed=5))
    ids = np.random.default_rng(1).integers(5, 97, 12)
    with torch.no_grad():
        a = net.forward(ids, [12])
        b = net.forward(ids, [12], _types(12))
    assert float((a - b).abs().max()) > 1e-4


def _golden_lengths():
    g = np.load(os.path.join(G, "xlnet_text_golden.npz"))
    return sorted({len(g[k]) for k in g.files if "_ids" in k})


@pytest.mark.parametrize("clamp_len", [-1, 9])
def test_rel_table_bit_exact_against_hf_relative_positions(clamp_len):
    """For every golden sentence length n, alone (max_len n) and packed with a longer one (max_len 512): the row our
    table gives the distance i - j equals, bit for bit, the row HF's relative_positional_encoding(n, n) puts at (i, j)
    after rel_shift_bnij."""
    import transformers as tf
    d_model = 128
    m = tf.XLNetModel(tf.XLNetConfig(vocab_size=8, d_model=d_model, n_head=2, d_inner=8, n_layer=1,
                                     clamp_len=clamp_len))
    for n in _golden_lengths():
        pos = m.relative_positional_encoding(n, n, bsz=1)[:, 0]                        # [2n, d_model]
        idx = torch.arange(2 * n, dtype=torch.float32).expand(1, 1, n, 2 * n)
        col = m.layer[0].rel_attn.rel_shift_bnij(idx, klen=n)[0, 0].long()            # [n, n]: HF row of (i, j)
        i = torch.arange(n)
        for max_len in (n, 512):
            table, rows = XT.rel_table(d_model, max_len, clamp_len)
            assert table.dtype == torch.float32 and rows.dtype == np.int32 and rows.shape == (2 * max_len - 1,)
            ours = torch.from_numpy(rows).long()[(i[:, None] - i[None, :]) + max_len - 1]
            assert torch.equal(table[ours].view(torch.int32), pos[col].view(torch.int32)), (n, max_len)


def test_weight_reshapes_match_hf_einsums():
    """q | k | v, o and r as GEMM weights against HF's einsums on the [d_model, heads, 64] parameters: a transposed
    reshape gives different numbers here."""
    d, h = 128, 2
    g = torch.Generator().manual_seed(0)
    p = {f"x.{n}": torch.randn(d, h, 64, generator=g) for n in ("q", "k", "v", "o", "r")}
    x = torch.randn(7, d, generator=g)
    qkv, o, r = XT.proj_weights(dict(p), "x.", d, h)
    for blk, n in enumerate(("q", "k", "v")):
        want = torch.einsum("ih,hnd->ind", x, p[f"x.{n}"]).reshape(7, d)
        assert torch.allclose(x @ qkv[blk * d:(blk + 1) * d].T, want, atol=1e-5), n
    assert torch.allclose(x @ r.T, torch.einsum("ih,hnd->ind", x, p["x.r"]).reshape(7, d), atol=1e-5)
    vec = torch.randn(7, h, 64, generator=g)
    assert torch.allclose(vec.reshape(7, d) @ o.T, torch.einsum("ind,hnd->ih", vec, p["x.o"]), atol=1e-5)


def test_state_dict_prefix_and_heads_are_dropped():
    kw = dict(SMALL, n_layer=1, ff_activation="relu")
    sd = {k: torch.from_numpy(v) for k, v in S.xlnet_state_dict(kw, seed=1).items()}
    lm = {"transformer." + k: v for k, v in sd.items()}
    lm["lm_loss.bias"] = torch.zeros(97)
    a = XT.XlnetNet(sd, XT.TorchOps(), XT.XlnetDims(hf_config(kw)))
    b = XT.XlnetNet(lm, XT.TorchOps(), XT.XlnetDims(hf_config(kw)))
    ids = np.arange(5, 15)
    with torch.no_grad():
        assert torch.equal(a.forward(ids, [10]), b.forward(ids, [10]))


# ---- golden -----------------------------------------------------------------------------------------------------------
def _golden(family):
    g = np.load(os.path.join(G, "xlnet_text_golden.npz"))
    return {k[len(family) + 1:]: g[k] for k in g.files if k.startswith(family + "_")}


def _golden_cfg(family, vocab):
    return dict(S.XLNET_GOLDEN_CFGS[family], vocab_size=vocab)


def _tokenizer(tmp_path, with_types):
    import transformers as tf
    d = tmp_path / ("types" if with_types else "plain")
    d.mkdir()
    shutil.copy(os.path.join(G, "xlnet_tokenizer", "spiece.model"), d)
    cfg = json.load(open(os.path.join(G, "xlnet_tokenizer", "tokenizer_config.json")))
    if with_types:
        cfg["model_input_names"] = ["input_ids", "token_type_ids", "attention_mask"]
    json.dump(cfg, open(d / "tokenizer_config.json", "w"))
    return tf.AutoTokenizer.from_pretrained(str(d), use_fast=False)


@pytest.mark.parametrize("family", ["base", "large"])
def test_golden_token_ids_and_offsets_match_the_tokenizer(tmp_path, family):
    from mertools_b200.extract.text import find_start_end_pos
    g = _golden(family)
    tok = _tokenizer(tmp_path, bool(g["with_types"]))
    assert tok.convert_tokens_to_ids(["<unk>", "<cls>", "<sep>"]) == [0, 3, 4]
    assert (int(g["start"]), int(g["end"])) == find_start_end_pos(tok) == (0, -2)
    for i, s in enumerate(g["sentences"]):
        if g["isnan"][i]:
            continue
        enc = tok(str(s))
        np.testing.assert_array_equal(np.array(enc["input_ids"]), g[f"ids{i}"])
        assert ("token_type_ids" in enc) == bool(g["with_types"])
        if g["with_types"]:
            np.testing.assert_array_equal(np.array(enc["token_type_ids"]), g[f"types{i}"])


@pytest.mark.parametrize("family", ["base", "large"])
def test_orchestration_reproduces_the_reference_golden(family):
    g = _golden(family)
    kw = _golden_cfg(family, int(g["vocab_size"]))
    net = torch_net(kw, S.xlnet_state_dict(kw, seed=int(g["seed"])))
    n_sent = len(g["sentences"])
    rows = [i for i in range(n_sent) if f"ids{i}" in g]
    ids = [g[f"ids{i}"] for i in rows]
    types = np.concatenate([g[f"types{i}"] for i in rows]) if g["with_types"] else None
    assert any(len(x) > 64 for x in ids)   # a sentence crosses two key tiles
    with torch.no_grad():
        acc = net.forward(np.concatenate(ids), [len(x) for x in ids], types).numpy()
    o, j = 0, 0
    for i in range(n_sent):
        if f"ids{i}" not in g:
            assert g["isnan"][i] and not g[f"utt{i}"].any()
            continue
        n = len(ids[j])
        if n <= 2:   # nothing left before <sep> <cls>: the reference's zeros
            assert not g[f"utt{i}"].any() and not g[f"fra{i}"].any()
            o, j = o + n, j + 1
            continue
        frame = acc[o:o + n - 2]
        assert int(g[f"fran{i}"]) == len(frame), (i, int(g[f"fran{i}"]), len(frame))
        want_f, want_u = g[f"fra{i}"], g[f"utt{i}"]   # the golden keeps every FRAME_STEP-th token row
        got_f = frame[::FRAME_STEP]
        assert want_f.dtype == np.float32 and want_f.shape == got_f.shape, (i, want_f.shape, got_f.shape)
        assert np.abs(got_f - want_f).max() <= 5e-5 * max(1.0, np.abs(want_f).max())
        assert np.abs(frame.mean(0) - want_u).max() <= 5e-5 * max(1.0, np.abs(want_u).max())
        o, j = o + n, j + 1


class _NoEncoder:
    hidden = 8


def test_extractor_hook_forwards_token_types_only_when_the_tokenizer_returns_them(tmp_path):
    from mertools_b200.extract.text import TextExtractor
    for with_types in (False, True):
        tok = _tokenizer(tmp_path, with_types)
        ids = XT.XlnetTextExtractor(None, tok, encoder=_NoEncoder()).tokenize("今天天气真好")
        assert list(ids) == tok("今天天气真好")["input_ids"] and ids[-2:] == [4, 3]
        if with_types:
            assert ids.token_types == [0] * (len(ids) - 1) + [2]
        else:
            assert ids.token_types is None
        plain = TextExtractor(None, tok, encoder=_NoEncoder()).tokenize("今天天气真好")
        assert type(plain) is list and plain == list(ids)


# ---- refusals ---------------------------------------------------------------------------------------------------------
class _Untouchable(dict):
    def __getitem__(self, k):
        raise AssertionError("a weight was read")

    pop = get = items = keys = values = __iter__ = __getitem__


BASE = dict(vocab_size=100, d_model=768, n_head=12, d_inner=1536, n_layer=2, ff_activation="gelu")
REFUSED = {
    "attn_type uni": dict(attn_type="uni"),
    "bi_data": dict(bi_data=True),
    "d_head 32": dict(n_head=24),
    "n_head * d_head != d_model": dict(_n_head=10),
    "d_model 128": dict(d_model=128, n_head=2),
    "ff_activation gelu_new": dict(ff_activation="gelu_new"),
    "ff_activation tanh": dict(ff_activation="tanh"),
}


@pytest.mark.parametrize("name", sorted(REFUSED))
def test_unsupported_configs_are_refused_before_any_weight_is_read(name):
    kw = dict(BASE, **REFUSED[name])
    n_head = kw.pop("_n_head", None)
    cfg = hf_config(kw)
    if n_head is not None:   # XLNetConfig itself derives d_head = d_model / n_head; a loaded config may disagree
        cfg.n_head = n_head
    with pytest.raises(ValueError, match="XLNet path"):
        XT.check_xlnet_config(cfg)
    with pytest.raises(ValueError, match="XLNet path"):
        XT.XlnetTextEncoder(_Untouchable(), cfg, device="cpu")


def test_golden_configs_are_accepted():
    for family in ("base", "large"):
        XT.check_xlnet_config(hf_config(_golden_cfg(family, 100)))


def _cpu_lib():
    if torch.cuda.is_available():
        pytest.skip("fake device addresses are only safe where no CUDA driver can launch anything")
    if not os.path.exists(L.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return L.lib()


def _call(dll, **over):
    base = 0x7F0000000000  # never dereferenced
    a = dict(qkv=base, vt=base + (1 << 24), vt_ld=104, r=base + (2 << 24), r_ld=768 * 4, rel_row=base + (3 << 24),
             r_w=base + (4 << 24), r_r=base + (4 << 24) + 3072, r_s=base + (4 << 24) + 6144,
             seg=base + (4 << 24) + 9216, types=base + (5 << 24), scale=0.125, ctx=base + (6 << 24),
             cu=base + (7 << 24), n_seq=2, tokens=100, max_seqlen=60, heads=12,
             flags=L.MER_ATT_QKV_F16 | L.MER_EPI_OUT_F16)
    a.update(over)
    vp, i64 = C.c_void_p, C.c_longlong
    rc = dll.mer_xlnet_attention(vp(a["qkv"]), vp(a["vt"]), i64(a["vt_ld"]), vp(a["r"]), i64(a["r_ld"]),
                                 vp(a["rel_row"]), vp(a["r_w"]), vp(a["r_r"]), vp(a["r_s"]), vp(a["seg"]),
                                 vp(a["types"]), C.c_float(a["scale"]), vp(a["ctx"]), vp(a["cu"]), C.c_int(a["n_seq"]),
                                 i64(a["tokens"]), C.c_int(a["max_seqlen"]), C.c_int(a["heads"]), C.c_int(a["flags"]),
                                 vp(0))
    return rc, dll.mer_last_error().decode()


def test_abi_refusals_of_mer_xlnet_attention():
    dll = _cpu_lib()
    refused = {
        "heads 0": dict(heads=0), "heads 65536": dict(heads=65536),
        "n_seq 0": dict(n_seq=0), "n_seq 65536": dict(n_seq=65536),
        "vt_ld misaligned": dict(vt_ld=108), "vt_ld < tokens": dict(vt_ld=96),
        "tf32 vt_ld misaligned": dict(flags=0, vt_ld=102),
        "null qkv": dict(qkv=None), "null ctx": dict(ctx=None), "null cu": dict(cu=None),
        "null r": dict(r=None), "null rel_row": dict(rel_row=None),
        "null r_w_bias": dict(r_w=None), "null r_r_bias": dict(r_r=None), "null r_s_bias": dict(r_s=None),
        "null seg_embed": dict(seg=None),
        "r_ld < heads * 64": dict(r_ld=704), "r_ld misaligned": dict(r_ld=772),
        "r misaligned": dict(r=0x7F0000000000 + (2 << 24) + 8),
        "r_w_bias misaligned": dict(r_w=0x7F0000000000 + (4 << 24) + 4),
        "max_seqlen 0": dict(max_seqlen=0), "max_seqlen > tokens": dict(max_seqlen=101),
        "two ctx formats": dict(flags=L.MER_EPI_OUT_F16 | L.MER_EPI_SPLIT_BF16), "gelu flag": dict(flags=L.MER_EPI_GELU),
    }
    for name, over in refused.items():
        rc, msg = _call(dll, **over)
        assert rc != 0 and msg.startswith("mer_xlnet_attention:"), (name, rc, msg)
    # accepted arguments get past validation and stop at the first CUDA call (no driver here); NULL token types are
    # the no-segment-term form, not a refusal
    for over in (dict(), dict(types=None), dict(flags=L.MER_EPI_SPLIT_BF16, vt_ld=100), dict(flags=L.MER_EPI_ROUND_TF32)):
        rc, msg = _call(dll, **over)
        assert not msg.startswith("mer_xlnet_attention:"), (over, msg)
