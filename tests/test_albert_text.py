"""CPU checks of the ALBERT branch of the text extractor (mertools_b200/extract/albert_text.py): the torch restatement
against HF AlbertModel on every hidden state (padded and unpadded packing, each golden family's shape), against the
goldens of the unmodified reference, the loader's name handling and its single packed layer, the refused configs (before
any weight is read), the tokenizer chosen per model name, the golden ids, and the argument refusals of
mer_attention_hd (before any launch)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from mertools_b200 import _lib as L
from mertools_b200 import synthetic as S
from mertools_b200.extract import albert_text as A

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FRAME_STEP = 4
FAMILIES = ("tiny", "small", "base")


def _cfg(kw):
    import transformers as tf
    return tf.AlbertConfig(**kw)


def _golden(family):
    g = np.load(os.path.join(G, "albert_text_golden.npz"))
    return {k[len(family) + 1:]: g[k] for k in g.files if k.startswith(family + "_")}


@pytest.mark.parametrize("pad", [True, False])
@pytest.mark.parametrize("family", FAMILIES)
def test_orchestration_matches_hf_on_every_hidden_state(family, pad):
    import transformers as tf
    kw = dict(S.ALBERT_GOLDEN_CFGS[family], vocab_size=300)
    cfg = _cfg(kw)
    sd = S.albert_state_dict(kw, seed=5)
    m = tf.AlbertModel(cfg).eval()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    d = A.AlbertDims(cfg, pad=pad)
    assert (d.hidden_pad, d.khd) == ({"tiny": (384, 32), "small": (384, 32), "base": (768, 64)}[family] if pad
                                     else (cfg.hidden_size, cfg.hidden_size // 12))
    net = A.AlbertNet(sd, A.TorchOps(), d)
    rng = np.random.default_rng(0)
    lens = [7, 70, 1]
    ids = [rng.integers(0, 300, n) for n in lens]
    with torch.no_grad():
        acc, hs = net.forward(np.concatenate(ids), lens, return_hidden=True)
    H, o = cfg.hidden_size, 0
    for x in ids:
        with torch.no_grad():
            ref = m(torch.from_numpy(x)[None], output_hidden_states=True).hidden_states
        assert len(ref) == len(hs) == cfg.num_hidden_layers + 1
        for i, h in enumerate(ref):
            got = hs[i][o:o + len(x)]
            assert float((got[:, :H] - h[0]).abs().max() / h.abs().max()) < 5e-6, (i, family, pad)
            assert not got[:, H:].any()      # the pad columns stay exactly zero
        want = torch.stack(ref)[[-4, -3, -2, -1]].sum(0)[0]
        assert float((acc[o:o + len(x), :H] - want).abs().max() / want.abs().max()) < 5e-6
        o += len(x)


def test_padded_head_packing_is_exact_on_the_weights():
    kw = dict(S.ALBERT_GOLDEN_CFGS["tiny"], vocab_size=50)
    cfg = _cfg(kw)
    sd = A.strip_albert({k: torch.from_numpy(v) for k, v in S.albert_state_dict(kw, seed=1).items()})
    d = A.AlbertDims(cfg)
    p = A.pack_layer(dict(sd), d)
    q = sd[A.LAYER + "attention.query.weight"]
    assert p["qkv"].shape == (3 * 384, 384) and p["o"].shape == (384, 384)
    assert p["up"].shape == (1280, 384) and p["down"].shape == (384, 1280)
    qp = p["qkv"][:384].reshape(12, 32, 384)
    assert torch.equal(qp[:, :26, :312], q.reshape(12, 26, 312)) and not qp[:, 26:].any() and not qp[..., 312:].any()
    op = p["o"].reshape(384, 12, 32)
    assert torch.equal(op[:312, :, :26], sd[A.LAYER + "attention.dense.weight"].reshape(312, 12, 26))
    assert not op[:, :, 26:].any() and not op[312:].any()
    assert not p["b_qkv"].reshape(3, 12, 32)[:, :, 26:].any()
    assert not p["b_up"][1248:].any() and not p["ln1"][0][312:].any()


def test_state_dict_prefix_and_heads_are_dropped_and_the_layer_is_packed_once():
    kw = dict(S.ALBERT_GOLDEN_CFGS["small"], vocab_size=40, num_hidden_layers=5)
    sd = {"albert." + k: torch.from_numpy(v) for k, v in S.albert_state_dict(kw, seed=2).items()}
    sd.update({"predictions.bias": torch.zeros(40), "predictions.decoder.weight": torch.zeros(40, 128),
               "sop_classifier.classifier.weight": torch.zeros(2, 384), "albert.embeddings.position_ids":
               torch.arange(512)[None]})
    kept = A.strip_albert(sd)
    assert not any(k.startswith(("albert.", "predictions.", "sop_classifier.", "pooler.")) for k in kept)
    assert "embeddings.position_ids" not in kept

    class Counting(A.TorchOps):
        n = 0

        def weight(self, t):
            Counting.n += 1
            return super().weight(t)

    ops = Counting()
    net = A.AlbertNet(sd, ops, A.AlbertDims(_cfg(kw)))   # unknown names would fail its "unused weights" assert
    # five GEMM weights, packed once whatever the depth: the embedding mapping and the shared layer's qkv, o, up, down
    assert Counting.n == 5
    assert set(net.layer) == {"qkv", "b_qkv", "o", "b_o", "ln1", "up", "b_up", "down", "b_down", "ln2"}


def test_restatement_reproduces_the_reference_golden():
    for family in FAMILIES:
        g = _golden(family)
        kw = dict(S.ALBERT_GOLDEN_CFGS[family], vocab_size=int(g["vocab_size"]))
        net = A.AlbertNet(S.albert_state_dict(kw, seed=int(g["seed"])), A.TorchOps(), A.AlbertDims(_cfg(kw)))
        H = kw["hidden_size"]
        n_sent = len(g["sentences"])
        rows = [i for i in range(n_sent) if f"ids{i}" in g]
        ids = [g[f"ids{i}"] for i in rows]
        assert any(len(x) > 64 for x in ids)
        with torch.no_grad():
            acc = net.forward(np.concatenate(ids), [len(x) for x in ids]).numpy()[:, :H]
        o, j = 0, 0
        for i in range(n_sent):
            if f"ids{i}" not in g:
                assert g["isnan"][i] and not g[f"utt{i}"].any()
                continue
            n = len(ids[j])
            if n <= 2:
                assert not g[f"utt{i}"].any() and not g[f"fra{i}"].any()
            else:
                frame = acc[o + 1:o + n - 1]
                assert int(g[f"fran{i}"]) == len(frame)
                want_f, want_u = g[f"fra{i}"], g[f"utt{i}"]
                assert want_f.dtype == np.float32 and want_f.shape == frame[::FRAME_STEP].shape
                assert np.abs(frame[::FRAME_STEP] - want_f).max() <= 5e-5 * max(1.0, np.abs(want_f).max()), family
                assert np.abs(frame.mean(0) - want_u).max() <= 5e-5 * max(1.0, np.abs(want_u).max()), family
            o, j = o + n, j + 1


def _tokenizer(family):
    import transformers as tf
    if family == "base":
        return tf.AutoTokenizer.from_pretrained(os.path.join(G, "albert_tokenizer"), use_fast=False)
    return tf.BertTokenizer(os.path.join(G, "text_vocab.txt"))


@pytest.mark.parametrize("family", FAMILIES)
def test_golden_token_ids_and_offsets_match_the_tokenizer(family):
    from mertools_b200.extract.text import find_start_end_pos
    g = _golden(family)
    tok = _tokenizer(family)
    if family == "base":
        assert type(tok).__name__ == "AlbertTokenizer"
        assert tok.convert_tokens_to_ids(["<pad>", "<unk>", "[CLS]", "[SEP]", "[MASK]"]) == [0, 1, 2, 3, 4]
        assert "token_type_ids" not in tok("hello")
    assert (int(g["start"]), int(g["end"])) == find_start_end_pos(tok) == (1, -1)
    for i, s in enumerate(g["sentences"]):
        if not g["isnan"][i]:
            np.testing.assert_array_equal(np.array(tok(str(s))["input_ids"]), g[f"ids{i}"])


@pytest.mark.parametrize("name,cls", [("albert_chinese_tiny", "BertTokenizer"), ("albert_chinese_small", "BertTokenizer"),
                                      ("albert-base-v2", "AutoTokenizer"), ("albert-large-v2", "AutoTokenizer"),
                                      ("albert-xxlarge-v2", "AutoTokenizer")])
def test_tokenizer_chosen_per_model_name(monkeypatch, name, cls):
    import transformers as tf
    seen = []
    for c in ("BertTokenizer", "AutoTokenizer"):
        monkeypatch.setattr(getattr(tf, c), "from_pretrained",
                            classmethod(lambda k, d, c=c, **kw: seen.append((c, d, kw)) or c))
    assert A.albert_tokenizer(name, "/m") == cls
    assert seen == [(cls, "/m", dict(use_fast=False))]


# ---- refusals ---------------------------------------------------------------------------------------------------------
class _Untouchable(dict):
    def __getitem__(self, k):
        raise AssertionError("a weight was read")

    pop = get = items = keys = values = __iter__ = __getitem__


BASE = dict(vocab_size=100, embedding_size=128, hidden_size=768, num_attention_heads=12, intermediate_size=3072,
            num_hidden_layers=2, hidden_act="gelu_new")
REFUSED = {
    "two hidden groups": dict(num_hidden_groups=2),
    "two inner groups": dict(inner_group_num=2),
    "hidden % heads": dict(num_attention_heads=10),
    "head_dim 48": dict(hidden_size=768, num_attention_heads=16),
    "head_dim 128": dict(hidden_size=1024, num_attention_heads=8),
    "hidden_act relu": dict(hidden_act="relu"),
    "hidden_act gelu_fast": dict(hidden_act="gelu_fast"),
    "relative positions": dict(position_embedding_type="relative_key"),
    "embedding_size 96": dict(embedding_size=96),
    "max_position_embeddings 1024": dict(max_position_embeddings=1024),
    "heads x 32 not a multiple of 128": dict(hidden_size=260, num_attention_heads=10, intermediate_size=1040),
    "hidden 2112": dict(hidden_size=2112, num_attention_heads=33),
}


@pytest.mark.parametrize("name", sorted(REFUSED))
def test_unsupported_configs_are_refused_before_any_weight_is_read(name):
    cfg = _cfg(dict(BASE, **REFUSED[name]))
    with pytest.raises(ValueError, match="ALBERT path"):
        A.check_albert_config(cfg)
    with pytest.raises(ValueError, match="ALBERT path"):
        A.AlbertTextEncoder(_Untouchable(), cfg, device="cpu")


def test_published_and_golden_configs_are_accepted():
    for kw in list(S.ALBERT_PUBLISHED_CFGS.values()) + [dict(c, vocab_size=100) for c in S.ALBERT_GOLDEN_CFGS.values()]:
        A.check_albert_config(_cfg(kw))


def test_extract_embedding_dispatches_albert(monkeypatch, tmp_path):
    from mertools_b200.extract import text
    called = []
    monkeypatch.setattr(text, "_albert_extractor", lambda *a: called.append(a) or (_ for _ in ()).throw(StopIteration))
    cfg = _cfg(dict(BASE))
    cfg.save_pretrained(str(tmp_path))
    monkeypatch.setattr("mertools_b200.shard.device_index", lambda g: 0)
    with pytest.raises(StopIteration):
        text.extract_embedding("albert-base-v2", "unused.csv", str(tmp_path / "f"), "UTTERANCE", gpu=0,
                               model_dir=str(tmp_path))
    assert called and called[0][0] == "albert-base-v2"


# ---- mer_attention_hd argument refusals -----------------------------------------------------------------------------
def _cpu_lib():
    if torch.cuda.is_available():
        pytest.skip("fake device addresses are only safe where no CUDA driver can launch anything")
    if not os.path.exists(L.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return L.lib()


def _call(dll, **over):
    base = 0x7F0000000000  # never dereferenced
    a = dict(qkv=base, vt=base + (1 << 24), vt_ld=104, ctx=base + (2 << 24), cu=base + (3 << 24), n_seq=2, tokens=100,
             max_seqlen=60, heads=12, head_dim=32, scale=1 / 26 ** 0.5, flags=L.MER_ATT_QKV_F16 | L.MER_EPI_OUT_F16)
    a.update(over)
    vp, i64, i32 = C.c_void_p, C.c_longlong, C.c_int
    rc = dll.mer_attention_hd(vp(a["qkv"]), vp(a["vt"]), i64(a["vt_ld"]), vp(a["ctx"]), vp(a["cu"]), i32(a["n_seq"]),
                              i64(a["tokens"]), i32(a["max_seqlen"]), i32(a["heads"]), i32(a["head_dim"]),
                              C.c_float(a["scale"]), i32(a["flags"]), vp(0))
    return rc, dll.mer_last_error().decode()


def test_abi_refusals_of_mer_attention_hd():
    dll = _cpu_lib()
    refused = {
        "head_dim 26": dict(head_dim=26), "head_dim 128": dict(head_dim=128), "head_dim 0": dict(head_dim=0),
        "scale 0": dict(scale=0.0), "scale < 0": dict(scale=-0.125), "scale nan": dict(scale=float("nan")),
        "scale inf": dict(scale=float("inf")), "scale 2": dict(scale=2.0),
        "null qkv": dict(qkv=None), "null vt": dict(vt=None), "null ctx": dict(ctx=None), "null cu": dict(cu=None),
        "vt_ld misaligned": dict(vt_ld=108), "vt_ld < tokens": dict(vt_ld=96),
        "tf32 vt_ld misaligned": dict(flags=0, vt_ld=102),
        "max_seqlen 0": dict(max_seqlen=0), "max_seqlen > tokens": dict(max_seqlen=101),
        "max_seqlen 513": dict(max_seqlen=513, tokens=600, vt_ld=600),
        "heads 0": dict(heads=0), "heads 65536": dict(heads=65536), "n_seq 0": dict(n_seq=0),
        "n_seq 65536": dict(n_seq=65536), "gelu flag": dict(flags=L.MER_EPI_GELU),
    }
    for name, over in refused.items():
        rc, msg = _call(dll, **over)
        assert rc != 0 and msg.startswith("mer_attention_hd:"), (name, rc, msg)
    # accepted arguments get past validation and stop at the first CUDA call (no driver here)
    for over in (dict(), dict(head_dim=64, scale=0.125), dict(head_dim=64, scale=0.125, max_seqlen=512, tokens=600,
                                                              vt_ld=600),
                 dict(flags=L.MER_EPI_SPLIT_BF16, vt_ld=100), dict(flags=L.MER_EPI_ROUND_TF32)):
        rc, msg = _call(dll, **over)
        assert not msg.startswith("mer_attention_hd:"), (over, msg)
