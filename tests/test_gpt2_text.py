"""CPU checks of the GPT-2 family of the LayerNorm-decoder text branch (mertools_b200/extract/ln_decoder_text.py): the
orchestration with a torch fp32 backend against HF GPT2Model (every hidden state, with and without token types) and
against the goldens of the unmodified reference extract_embedding (tests/golden/make_golden_gpt2.py), the streaming
loader (Conv1D transpose, prefixes, dropped buffers and lm_head, shards), the configs the path refuses, the tokenizer
choice by model name and the token-type hook."""
import json
import os

import numpy as np
import pytest
import torch

from mertools_b200 import synthetic as S
from mertools_b200.extract import common
from mertools_b200.extract import ln_decoder_text as LD
from mertools_b200.extract import text

transformers = pytest.importorskip("transformers")
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAMES = list(S.GPT2_GOLDEN_CFGS)
GOLDEN = {"gpt2-chinese-cluecorpussmall": "gpt2_chinese_text_golden.npz",
          "wenzhong2-gpt2-chinese": "wenzhong_text_golden.npz"}
SMALL = dict(vocab=300, hidden=256, heads=4, ffn=1024, layers=3, max_pos=256)


def _cfg(c, **kw):
    base = dict(vocab_size=c["vocab"], n_positions=c["max_pos"], n_embd=c["hidden"], n_layer=c["layers"],
                n_head=c["heads"], n_inner=c["ffn"])
    base.update(kw)
    return transformers.GPT2Config(**base)


def _sd(c, seed=29, scale=1.0):
    return S.gpt2_state_dict(seed=seed, vocab=c["vocab"], hidden=c["hidden"], ffn=c["ffn"], layers=c["layers"],
                             max_pos=c["max_pos"], scale=scale)


def _as_loaded(sd):
    """A GPT2Model state dict as load_ln_decoder_weights names and lays it out (fp32 here)."""
    return {LD._strip(k, "gpt2"): (torch.from_numpy(v).T.contiguous() if k.endswith(LD.GPT2_CONV1D)
                                   else torch.from_numpy(v)) for k, v in sd.items()}


def _hf(sd, cfg):
    m = transformers.GPT2Model(cfg).eval()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    return m


def _net(sd, cfg, dtype=torch.float32):
    fam, layers, heads, _, _, eps, max_pos = LD.net_dims(cfg)
    assert fam == "gpt2"
    return LD.LnDecoderNet(_as_loaded(sd), LD.TorchOps(dtype=dtype), fam, layers, heads, eps, max_pos)


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / np.abs(b).max())


@pytest.mark.parametrize("with_types", [False, True])
@pytest.mark.parametrize("heads", [4, 2])   # head_dim 64 and 128
def test_torch_orchestration_matches_hf_every_hidden_state(heads, with_types):
    """Three sentences packed (one crosses 64 tokens): positions restart, no attention across them.  GPT2Model's
    hidden_states are h[0] = wte[ids] + wpe[pos] (+ wte[token_type_ids]), the block outputs, and
    last_hidden_state = ln_f(h[L]) in place of h[L] (transformers 5's output capture ties the last entry)."""
    c = dict(SMALL, heads=heads)
    sd, cfg = _sd(c), _cfg(c)
    m = _hf(sd, cfg)
    rng = np.random.default_rng(0)
    sents = [rng.integers(4, c["vocab"], n) for n in (37, 70, 1)]
    types = [rng.integers(0, 3, len(s)) for s in sents] if with_types else None
    with torch.no_grad():
        acc, hs = _net(sd, cfg).forward(np.concatenate(sents), [len(s) for s in sents], return_hidden=True,
                                        token_types=np.concatenate(types) if with_types else None)
        o = 0
        for j, s in enumerate(sents):
            kw = dict(token_type_ids=torch.from_numpy(types[j])[None]) if with_types else {}
            out = m(torch.from_numpy(s)[None], output_hidden_states=True, **kw)
            ref = out.hidden_states
            assert len(ref) == len(hs) == c["layers"] + 1
            for i, (r, h) in enumerate(zip(ref, hs)):
                assert _rel(h[o:o + len(s)], r[0]) < 2e-5, (i, _rel(h[o:o + len(s)], r[0]))
            assert torch.equal(ref[-1], out.last_hidden_state)
            assert _rel(acc[o:o + len(s)], torch.stack(ref)[[-4, -3, -2, -1]].sum(0)[0]) < 2e-5
            o += len(s)


def test_head_dim_96_restatement_matches_hf():
    """Wenzhong's head_dim: hidden 768 over 8 heads."""
    c = dict(SMALL, hidden=768, heads=8, ffn=3072)
    sd, cfg = _sd(c), _cfg(c)
    x = np.random.default_rng(1).integers(4, c["vocab"], 80)
    with torch.no_grad():
        ref = torch.stack(_hf(sd, cfg)(torch.from_numpy(x)[None], output_hidden_states=True).hidden_states)
        acc = _net(sd, cfg).forward(x, [len(x)])
    assert _rel(acc, ref[[-4, -3, -2, -1]].sum(0)[0]) < 2e-5


def _golden(name):
    return np.load(os.path.join(G, GOLDEN[name]))


def _install_tokenizer(name, dest):
    """The committed tokenizer fixture of ``name`` (as make_golden_gpt2.install_tokenizer writes it)."""
    import gzip
    import shutil
    os.makedirs(dest, exist_ok=True)
    if name == "gpt2-chinese-cluecorpussmall":
        shutil.copyfile(os.path.join(G, "text_vocab.txt"), os.path.join(dest, "vocab.txt"))
    else:
        for f in ("vocab.json", "merges.txt"):
            with gzip.open(os.path.join(G, "opt_tokenizer", f + ".gz"), "rb") as a, open(os.path.join(dest, f), "wb") as b:
                b.write(a.read())
    with open(os.path.join(G, "gpt2_tokenizer_configs.json")) as f:
        cfg = json.load(f)[name]
    with open(os.path.join(dest, "tokenizer_config.json"), "w") as f:
        json.dump(cfg, f)


@pytest.mark.parametrize("name,probe,cls", [("gpt2-chinese-cluecorpussmall", (1, -1), "BertTokenizer"),
                                            ("wenzhong2-gpt2-chinese", (0, None), "GPT2Tokenizer")])
def test_tokenizer_fixture_probe_ids_and_types(tmp_path, name, probe, cls):
    """The tokenizer extract_embedding loads for each name reproduces the golden's ids, and the token-type hook attaches
    the BertTokenizer's (all-zero) token_type_ids and nothing for GPT2Tokenizer."""
    d = str(tmp_path / "tok")
    _install_tokenizer(name, d)
    g, tok = _golden(name), text._gpt2_tokenizer(name, d)
    assert type(tok).__name__ == cls
    assert text.find_start_end_pos(tok) == probe == (int(g["start"]), None if int(g["end"]) == 0 else int(g["end"]))
    ext = text.TokenTypeTextExtractor(None, tok, encoder=_NoEncoder())
    for i, (s, nan) in enumerate(zip(g["sentences"], g["isnan"])):
        if nan:
            continue
        ids = ext.tokenize(str(s))
        assert list(ids) == g[f"ids{i}"].tolist(), i
        if cls == "BertTokenizer":
            assert ids.token_types == g[f"types{i}"].tolist() == [0] * len(ids)
        else:
            assert ids.token_types is None and f"types{i}" not in g.files
    lens = [len(g[f"ids{i}"]) for i in range(len(g["sentences"])) if not g["isnan"][i]]
    assert max(lens) > 64 and min(lens) <= 3


class _NoEncoder:
    hidden = 8


@pytest.mark.parametrize("name,want", [("wenzhong2-gpt2-chinese", "GPT2Tokenizer"),
                                       ("gpt2-chinese-cluecorpussmall", "AutoTokenizer"),
                                       ("some-other-gpt2", "AutoTokenizer")])
def test_tokenizer_class_by_model_name(monkeypatch, name, want):
    """GPT2Tokenizer(use_fast=False) for wenzhong2-gpt2-chinese (reference :167-169), AutoTokenizer(use_fast=False) for
    every other name (:188-190)."""
    calls = []
    for cls in ("GPT2Tokenizer", "AutoTokenizer"):
        monkeypatch.setattr(getattr(transformers, cls), "from_pretrained",
                            classmethod(lambda k, d, _c=cls, **kw: calls.append((_c, d, kw))))
    text._gpt2_tokenizer(name, "/models/x")
    assert calls == [(want, "/models/x", dict(use_fast=False))]


@pytest.mark.parametrize("which", ["hf", "torch_backend"])
@pytest.mark.parametrize("name", NAMES)
def test_readout_matches_reference_golden(name, which):
    """The golden's features from HF GPT2Model (the oracle) and from LnDecoderNet on the torch backend, with the
    tokenizer's token types where it returns them."""
    g, c = _golden(name), S.GPT2_GOLDEN_CFGS[name]
    sd, cfg = _sd(c, seed=int(g["seed"])), _cfg(c)
    start, end = int(g["start"]), int(g["end"]) or None
    idx = [i for i in range(len(g["sentences"])) if not g["isnan"][i]]
    ids = [g[f"ids{i}"] for i in idx]
    types = [g[f"types{i}"] for i in idx] if f"types{idx[0]}" in g.files else None
    with torch.no_grad():
        if which == "hf":
            m = _hf(sd, cfg)
            rows = []
            for j, x in enumerate(ids):
                kw = dict(token_type_ids=torch.from_numpy(types[j])[None]) if types else {}
                hs = m(torch.from_numpy(x)[None], output_hidden_states=True, **kw).hidden_states
                rows.append(torch.stack(hs)[[-4, -3, -2, -1]].sum(0)[0].numpy())
        else:
            acc = _net(sd, cfg).forward(np.concatenate(ids), [len(x) for x in ids],
                                        token_types=np.concatenate(types) if types else None).numpy()
            cu = np.concatenate([[0], np.cumsum([len(x) for x in ids])])
            rows = [acc[cu[j]:cu[j + 1]] for j in range(len(ids))]
    for j, i in enumerate(idx):
        for level in ("UTTERANCE", "FRAME"):
            ref = g[f"{level[:3].lower()}{i}"]
            got = common.save_feature(None, rows[j][start:end], level, c["hidden"])
            assert got.shape == ref.shape, (which, i, level)
            if not ref.any():   # nothing left after the special tokens: the reference's zeros
                assert not got.any()
                continue
            assert ref.dtype == np.float32 and _rel(got, ref) < 2e-5, (which, i, level, _rel(got, ref))
    nan = [i for i in range(len(g["sentences"])) if g["isnan"][i]]
    assert nan and all(g[f"utt{i}"].dtype == np.float64 and not g[f"utt{i}"].any() for i in nan)


def test_token_type_term_is_pinned_by_the_golden():
    """Without wte[token_type_ids] (wte[0], the [PAD] row, on every token) the gpt2-chinese golden is missed."""
    name = "gpt2-chinese-cluecorpussmall"
    g, c = _golden(name), S.GPT2_GOLDEN_CFGS[name]
    sd = _sd(c, seed=int(g["seed"]))
    assert np.abs(sd["wte.weight"][0]).max() > 0.1
    x = g["ids0"]
    with torch.no_grad():
        acc = _net(sd, _cfg(c)).forward(x, [len(x)]).numpy()
    assert _rel(acc[1:-1].mean(0), g["utt0"]) > 1e-2


def _write_checkpoint(d, sd, fmt, dtype, prefix, shards=3, buffers=False):
    """A sharded checkpoint as save_pretrained writes one (shard files + index.json), keys under ``prefix``, an lm_head
    when there is a prefix (GPT2LMHeadModel), and with ``buffers`` the attn.bias / attn.masked_bias buffers of older
    GPT-2 checkpoints."""
    os.makedirs(d, exist_ok=True)
    tensors = {prefix + k: torch.from_numpy(v).to(dtype) for k, v in sd.items()}
    if prefix:
        tensors["lm_head.weight"] = torch.zeros(SMALL["vocab"], SMALL["hidden"], dtype=dtype)
    if buffers:
        for i in range(SMALL["layers"]):
            tensors[f"{prefix}h.{i}.attn.bias"] = torch.ones(1, 1, 8, 8, dtype=dtype).tril()
            tensors[f"{prefix}h.{i}.attn.masked_bias"] = torch.tensor(-1e4, dtype=dtype)
    keys = sorted(tensors)
    ext = "safetensors" if fmt == "safetensors" else "bin"
    base = "model" if fmt == "safetensors" else "pytorch_model"
    wmap = {}
    for s in range(shards):
        part = {k: tensors[k].contiguous() for k in keys[s::shards]}
        fn = f"{base}-{s + 1:05d}-of-{shards:05d}.{ext}"
        if fmt == "safetensors":
            from safetensors.torch import save_file
            save_file(part, os.path.join(d, fn))
        else:
            torch.save(part, os.path.join(d, fn))
        wmap.update({k: fn for k in part})
    with open(os.path.join(d, f"{base}.{ext}.index.json"), "w") as f:
        json.dump({"metadata": {}, "weight_map": wmap}, f)


@pytest.mark.parametrize("fmt", ["safetensors", "bin"])
@pytest.mark.parametrize("prefix,buffers", [("", False), ("transformer.", True), ("", True)])
def test_streaming_loader_on_sharded_prefixed_checkpoints(tmp_path, prefix, buffers, fmt):
    """GPT2Model / GPT2LMHeadModel (transformer., lm_head) keys, with and without the mask buffers: names stripped,
    lm_head and buffers dropped, Conv1D weights transposed to [out, in]."""
    sd = _sd(SMALL)
    d = str(tmp_path / "ckpt")
    _write_checkpoint(d, sd, fmt, torch.bfloat16, prefix, buffers=buffers)
    got = LD.load_ln_decoder_weights(d, "cpu", "gpt2")
    assert sorted(got) == sorted(sd)
    for k, v in sd.items():
        want = torch.from_numpy(v).to(torch.bfloat16).to(torch.float16)
        if k.endswith(LD.GPT2_CONV1D):
            want = want.T
            assert got[k].shape == (v.shape[1], v.shape[0]), k
        assert got[k].dtype == torch.float16 and got[k].is_contiguous() and torch.equal(got[k], want), k
    c_attn = got["h.0.attn.c_attn.weight"]
    assert c_attn.shape == (3 * SMALL["hidden"], SMALL["hidden"])
    LD.LnDecoderNet(dict(got), LD.TorchOps(), "gpt2", SMALL["layers"], SMALL["heads"], 1e-5, SMALL["max_pos"])


def test_strip_keeps_the_c_attn_bias():
    assert LD._strip("h.3.attn.c_attn.bias", "gpt2") == "h.3.attn.c_attn.bias"
    assert LD._strip("transformer.h.3.attn.bias", "gpt2") is None
    assert LD._strip("h.11.attn.masked_bias", "gpt2") is None
    assert LD._strip("lm_head.weight", "gpt2") is None
    assert LD._strip("transformer.wte.weight", "gpt2") == "wte.weight"


REFUSED = [
    (dict(activation_function="gelu"), "activation_function"),
    (dict(activation_function="relu"), "activation_function"),
    (dict(scale_attn_weights=False), "scale_attn_weights"),
    (dict(scale_attn_by_inverse_layer_idx=True), "scale_attn_by_inverse_layer_idx"),
    (dict(add_cross_attention=True), "add_cross_attention"),
    (dict(n_head=5, n_embd=400), "head_dim"),
    (dict(n_head=8, n_embd=640), "head_dim"),          # head_dim 80
    (dict(n_head=2, n_embd=192), "multiple of 256"),   # head_dim 96
    (dict(n_head=6, n_embd=384), "multiple of 256"),   # head_dim 64
    (dict(n_inner=1000), "n_inner"),
]


@pytest.mark.parametrize("kw,msg", REFUSED)
def test_unsupported_configs_are_rejected(kw, msg):
    LD.check_ln_decoder_config(_cfg(SMALL))
    with pytest.raises(ValueError, match=msg):
        LD.check_ln_decoder_config(_cfg(SMALL, **kw))


def test_accepted_variants():
    """gelu_pytorch_tanh is the same function; reorder_and_upcast_attn only changes the reference's own rounding;
    n_inner None means 4 x hidden."""
    for kw in (dict(activation_function="gelu_pytorch_tanh"), dict(reorder_and_upcast_attn=True), dict(n_inner=None),
               dict(n_head=8, n_embd=768), dict(n_head=2, n_embd=256)):
        LD.check_ln_decoder_config(_cfg(SMALL, **kw))
    assert LD.net_dims(_cfg(SMALL, n_inner=None, layer_norm_epsilon=1e-6)) == ("gpt2", 3, 4, 256, 1024, 1e-6, 256)


@pytest.mark.parametrize("kw,msg", REFUSED)
def test_rejects_before_reading_weights(tmp_path, kw, msg):
    """extract_embedding's GPT-2 branch refuses from the config alone: no weight or tokenizer file exists here."""
    d = tmp_path / "tools" / "transformers" / "m"
    d.mkdir(parents=True)
    _cfg(SMALL, **kw).save_pretrained(str(d))
    with pytest.raises(ValueError, match=msg):
        text._gpt2_extractor("gpt2-chinese-cluecorpussmall", str(d), transformers.AutoConfig.from_pretrained(str(d)),
                             "cpu")


def test_refuses_sentences_longer_than_n_positions():
    net = _net(_sd(dict(SMALL, max_pos=64)), _cfg(dict(SMALL, max_pos=64)))
    with pytest.raises(ValueError, match="max_position_embeddings"):
        net.forward(np.arange(4, 69), [65])


def test_token_types_only_for_gpt2():
    from mertools_b200.extract import xlnet_text
    assert xlnet_text.XlnetTextExtractor is text.TokenTypeTextExtractor and xlnet_text.TokenIds is text.TokenIds
    a, b = text.TokenIds([5, 6, 7]), text.TokenIds([8])
    a.token_types, b.token_types = [0, 0, 1], [1]
    assert text.packed_token_types([a, b]).tolist() == [0, 0, 1, 1]
    assert text.packed_token_types([[5, 6], [7]]) is None
    b.token_types = None
    with pytest.raises(AssertionError, match="some only"):
        text.packed_token_types([a, b])
