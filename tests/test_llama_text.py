"""CPU checks of the LLaMA branch of the text extractor (mertools_b200/extract/llama_text.py): the orchestration with a
torch fp32 backend against HF LlamaModel (every hidden state, both rms_norm_eps values) and against the golden of the
unmodified reference extract_embedding (tests/golden/make_golden_llama.py), the tokenizer probe, the streaming weight
loader on sharded safetensors / .bin checkpoints, and the configs the path refuses."""
import json
import os

import numpy as np
import pytest
import torch

from mertools_b200 import synthetic as S
from mertools_b200.extract import common
from mertools_b200.extract import llama_text as LT

transformers = pytest.importorskip("transformers")
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOK = os.path.join(G, "llama_tokenizer")
C = S.LLAMA_SMALL_CFG


def _cfg(eps=1e-6, **kw):
    return transformers.LlamaConfig(vocab_size=C["vocab"], hidden_size=C["hidden"], num_attention_heads=C["heads"],
                                    intermediate_size=C["ffn"], num_hidden_layers=C["layers"],
                                    max_position_embeddings=C["max_pos"], rms_norm_eps=eps, **kw)


def _hf(sd, cfg):
    m = transformers.LlamaModel(cfg).eval()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    return m


def _net(sd, cfg, dtype=torch.float32):
    return LT.LlamaNet({k: torch.from_numpy(v) for k, v in sd.items()}, LT.TorchOps(dtype=dtype), cfg.num_hidden_layers,
                       cfg.num_attention_heads, cfg.rms_norm_eps, LT.rope_theta(cfg), cfg.max_position_embeddings)


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / np.abs(b).max())


@pytest.mark.parametrize("eps", [1e-6, 1e-5])
def test_torch_orchestration_matches_hf_llama_every_hidden_state(eps):
    """LLaMA-1 (1e-6) and Llama-2 (1e-5) eps; two sentences packed: positions restart, no attention across them."""
    sd, cfg = S.llama_state_dict(seed=3), _cfg(eps)
    m = _hf(sd, cfg)
    rng = np.random.default_rng(0)
    sents = [rng.integers(3, C["vocab"], n) for n in (37, 70)]
    with torch.no_grad():
        acc, hs = _net(sd, cfg).forward(np.concatenate(sents), [len(s) for s in sents], return_hidden=True)
        o = 0
        for s in sents:
            ref = m(torch.from_numpy(s)[None], output_hidden_states=True).hidden_states
            assert len(ref) == len(hs) == C["layers"] + 1
            for i, (r, h) in enumerate(zip(ref, hs)):
                assert _rel(h[o:o + len(s)], r[0]) < 2e-5, (i, _rel(h[o:o + len(s)], r[0]))
            # the readout: raw residual states h[-4..-2], and h[-1] = the final norm's output (last_hidden_state)
            assert torch.equal(ref[-1], m(torch.from_numpy(s)[None]).last_hidden_state)
            assert _rel(acc[o:o + len(s)], torch.stack(ref)[[-4, -3, -2, -1]].sum(0)[0]) < 2e-5
            o += len(s)


def _golden():
    return np.load(os.path.join(G, "llama_text_golden.npz"))


def _tokenizer():
    from transformers import AutoTokenizer
    return AutoTokenizer.from_pretrained(TOK, use_fast=False)


def test_tokenizer_fixture_probe_and_ids():
    from mertools_b200.extract.text import find_start_end_pos
    g, tok = _golden(), _tokenizer()
    assert type(tok).__name__ == "LlamaTokenizer"
    assert find_start_end_pos(tok) == (1, None) == (int(g["start"]), None if int(g["end"]) == 0 else int(g["end"]))
    for i, (s, nan) in enumerate(zip(g["sentences"], g["isnan"])):
        if not nan:
            assert tok(str(s))["input_ids"] == g[f"ids{i}"].tolist(), i


def _features(readout_rows, level):
    return common.save_feature(None, readout_rows[1:], level, C["hidden"])


@pytest.mark.parametrize("which", ["hf", "torch_backend"])
def test_readout_matches_reference_golden(which):
    """The golden's features from HF LlamaModel (the oracle) and from LlamaNet on the torch backend, packed."""
    g = _golden()
    sd, cfg = S.llama_state_dict(seed=int(g["seed"])), _cfg()
    idx = [i for i in range(len(g["sentences"])) if not g["isnan"][i]]
    ids = [g[f"ids{i}"] for i in idx]
    with torch.no_grad():
        if which == "hf":
            m = _hf(sd, cfg)
            rows = [torch.stack(m(torch.from_numpy(x)[None], output_hidden_states=True).hidden_states)[[-4, -3, -2, -1]]
                    .sum(0)[0].numpy() for x in ids]
        else:
            acc = _net(sd, cfg).forward(np.concatenate(ids), [len(x) for x in ids]).numpy()
            cu = np.concatenate([[0], np.cumsum([len(x) for x in ids])])
            rows = [acc[cu[j]:cu[j + 1]] for j in range(len(ids))]
    for j, i in enumerate(idx):
        for level in ("UTTERANCE", "FRAME"):
            ref = g[f"{level[:3].lower()}{i}"]
            got = _features(rows[j], level)
            assert got.shape == ref.shape and _rel(got, ref) < 2e-5, (which, i, level, _rel(got, ref))
    nan = [i for i in range(len(g["sentences"])) if g["isnan"][i]]
    assert nan and all(g[f"utt{i}"].dtype == np.float64 and not g[f"utt{i}"].any() for i in nan)


def _write_checkpoint(d, sd, fmt, dtype, prefix, shards=3):
    """A sharded checkpoint as save_pretrained writes one: shard files + index.json with the weight_map."""
    os.makedirs(d, exist_ok=True)
    names = sorted(sd)
    tensors = {prefix + k: torch.from_numpy(sd[k]).to(dtype) for k in names}
    if prefix:
        tensors["lm_head.weight"] = torch.zeros(C["vocab"], C["hidden"], dtype=dtype)
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
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("prefix", ["", "model."])
def test_streaming_loader_matches_state_dict_rounded_to_fp16(tmp_path, fmt, dtype, prefix):
    sd = S.llama_state_dict(seed=5, layers=3)
    d = str(tmp_path / "ckpt")
    _write_checkpoint(d, sd, fmt, dtype, prefix)
    got = LT.load_llama_weights(d, "cpu")
    assert sorted(got) == sorted(sd)
    for k, v in sd.items():
        assert got[k].dtype == torch.float16
        assert torch.equal(got[k], torch.from_numpy(v).to(dtype).to(torch.float16)), k


def test_streaming_loader_prefers_bin_when_asked(tmp_path):
    sd = S.llama_state_dict(seed=5, layers=3)
    d = str(tmp_path / "ckpt")
    _write_checkpoint(d, sd, "safetensors", torch.float32, "")
    _write_checkpoint(d, {k: v * 0 for k, v in sd.items()}, "bin", torch.float32, "")
    assert float(LT.load_llama_weights(d, "cpu")["norm.weight"].abs().sum()) > 0
    assert float(LT.load_llama_weights(d, "cpu", prefer_bin=True)["norm.weight"].abs().sum()) == 0


@pytest.mark.parametrize("kw,msg", [
    (dict(num_key_value_heads=2), "grouped-query"),
    (dict(rope_scaling={"rope_type": "linear", "factor": 2.0}), "rotary"),
    (dict(attention_bias=True), "bias"),
    (dict(mlp_bias=True), "bias"),
    (dict(hidden_act="gelu"), "hidden_act"),
    (dict(head_dim=64), "head_dim"),
])
def test_unsupported_configs_are_rejected(kw, msg):
    LT.check_llama_config(_cfg())
    with pytest.raises(ValueError, match=msg):
        LT.check_llama_config(_cfg(**kw))


def test_rejects_before_reading_weights(tmp_path):
    """extract_embedding refuses a grouped-query checkpoint from its config alone (no weight file exists here)."""
    from mertools_b200.extract import text
    d = tmp_path / "tools" / "transformers" / "llama-7b-hf"
    d.mkdir(parents=True)
    _cfg(num_key_value_heads=2).save_pretrained(str(d))
    with pytest.raises(ValueError, match="grouped-query"):
        text._llama_extractor("llama-7b-hf", str(d), transformers.AutoConfig.from_pretrained(str(d)), "cpu")


def test_rope_tables_match_hf():
    cfg = _cfg()
    rot = transformers.models.llama.modeling_llama.LlamaRotaryEmbedding(cfg)
    pos = torch.arange(4096)[None]
    cos, sin = rot(torch.zeros(1, dtype=torch.float32), pos)
    c, s = LT.rope_tables(4096, LT.rope_theta(cfg))
    assert torch.equal(cos[0, :, :64], c) and torch.equal(cos[0, :, 64:], c)
    assert torch.equal(sin[0, :, :64], s) and torch.equal(sin[0, :, 64:], s)


def test_activation_budget_per_token():
    """~200 KB of activations per token at the 13 B shape (what the tokens-per-launch choice divides by)."""
    assert 180e3 < LT.activation_bytes_per_token(5120, 13824) < 260e3
