"""CPU checks of the Falcon family of the LN-decoder text branch (mertools_b200/extract/ln_decoder_text.py): the
orchestration with a torch fp32 backend against HF FalconModel (every hidden state) and against the golden of the
unmodified reference extract_embedding (tests/golden/make_golden_falcon.py), the tokenizer fixture, the streaming
loader, the padded QKV / dense / FFN layout of the CUDA backend restated in plain torch, and the configs the path
refuses."""
import json
import os
import types

import numpy as np
import pytest
import torch

from mertools_b200 import synthetic as S
from mertools_b200.extract import common
from mertools_b200.extract import ln_decoder_text as LD
from mertools_b200.extract.llama_text import rope_tables

transformers = pytest.importorskip("transformers")
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
C = S.FALCON_SMALL_CFG


def _cfg(**kw):
    base = dict(vocab_size=C["vocab"], hidden_size=C["hidden"], num_attention_heads=C["heads"], ffn_hidden_size=C["ffn"],
                num_hidden_layers=C["layers"], max_position_embeddings=C["max_pos"], layer_norm_epsilon=1e-5,
                bos_token_id=0, eos_token_id=2, pad_token_id=1)
    base.update(kw)
    return transformers.FalconConfig(**base)


def _sd(seed=43, **kw):
    return S.falcon_state_dict(seed=seed, **kw)


def _hf(sd, cfg):
    m = transformers.FalconModel(cfg).eval()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    return m


def _net(sd, cfg, dtype=torch.float32):
    fam, layers, heads, _, _, eps, max_pos = LD.net_dims(cfg)
    assert fam == "falcon"
    return LD.LnDecoderNet({LD._strip(k, fam): torch.from_numpy(v) for k, v in sd.items()}, LD.TorchOps(dtype=dtype),
                           fam, layers, heads, eps, max_pos, theta=LD.rope_theta(cfg))


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / np.abs(b).max())


def test_torch_orchestration_matches_hf_every_hidden_state():
    """Three sentences packed (one crosses 64 tokens): rotary positions restart, no attention across them.  hidden_states
    is h[0] = E[ids], the layer outputs, and ln_f(h[L])."""
    sd, cfg = _sd(), _cfg()
    m = _hf(sd, cfg)
    rng = np.random.default_rng(0)
    sents = [rng.integers(4, C["vocab"], n) for n in (37, 70, 1)]
    with torch.no_grad():
        acc, hs = _net(sd, cfg).forward(np.concatenate(sents), [len(s) for s in sents], return_hidden=True)
        o = 0
        for s in sents:
            out = m(torch.from_numpy(s)[None], output_hidden_states=True)
            ref = out.hidden_states
            assert len(ref) == len(hs) == C["layers"] + 1
            for i, (r, h) in enumerate(zip(ref, hs)):
                assert _rel(h[o:o + len(s)], r[0]) < 2e-5, (i, _rel(h[o:o + len(s)], r[0]))
            assert _rel(acc[o:o + len(s)], torch.stack(ref)[[-4, -3, -2, -1]].sum(0)[0]) < 2e-5
            o += len(s)


def _golden():
    return np.load(os.path.join(G, "falcon_text_golden.npz"))


def _tokenizer(dest):
    import sys
    from transformers import AutoTokenizer
    sys.path.insert(0, G)
    try:
        from make_golden_falcon import unpack_falcon_tokenizer
    finally:
        sys.path.remove(G)
    unpack_falcon_tokenizer(dest)
    return AutoTokenizer.from_pretrained(dest, use_fast=False)


def test_tokenizer_fixture_probe_and_ids(tmp_path):
    from mertools_b200.extract.text import find_start_end_pos
    g, tok = _golden(), _tokenizer(str(tmp_path / "tok"))
    assert type(tok).__name__ in ("PreTrainedTokenizerFast", "TokenizersBackend")
    assert find_start_end_pos(tok) == (0, None) == (int(g["start"]), None if int(g["end"]) == 0 else int(g["end"]))
    for i, (s, nan) in enumerate(zip(g["sentences"], g["isnan"])):
        if not nan:
            enc = tok(str(s))
            assert enc["input_ids"] == g[f"ids{i}"].tolist(), i
            assert "token_type_ids" not in enc
    lens = [len(g[f"ids{i}"]) for i in range(len(g["sentences"])) if not g["isnan"][i]]
    assert max(lens) > 64 and min(lens) <= 2


@pytest.mark.parametrize("which", ["hf", "torch_backend"])
def test_readout_matches_reference_golden(which):
    """The golden's features from HF FalconModel (the oracle) and from LnDecoderNet on the torch backend."""
    g = _golden()
    sd, cfg = _sd(seed=int(g["seed"])), _cfg()
    start = int(g["start"])
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
            got = common.save_feature(None, rows[j][start:], level, C["hidden"])
            assert got.shape == ref.shape and _rel(got, ref) < 2e-5, (which, i, level, _rel(got, ref))
    nan = [i for i in range(len(g["sentences"])) if g["isnan"][i]]
    assert nan and all(g[f"utt{i}"].dtype == np.float64 and not g[f"utt{i}"].any() for i in nan)


def _padding_ops():
    """The CUDA backend's packing methods, run on the CPU (they only pad, cast to fp16 and move)."""
    ops = LD.CudaOps.__new__(LD.CudaOps)
    ops.device = torch.device("cpu")
    return ops


@pytest.mark.parametrize("hidden,heads,ffn", [(448, 7, 1792), (4544, 71, 512)])
def test_padded_layout_reproduces_hf_split_and_outputs(hidden, heads, ffn):
    """The padded QKV (q | k | zero rows | v, V^T from column vt_col0 on), the zero-row-padded dense / dense_4h_to_h and
    the padded embedding rows give HF's q / k / v split and outputs in plain torch, and leave the pad columns zero."""
    from transformers.models.falcon.modeling_falcon import FalconAttention
    torch.manual_seed(0)
    cfg = _cfg(hidden_size=hidden, num_attention_heads=heads, ffn_hidden_size=ffn)
    att = FalconAttention(cfg, layer_idx=0).eval()
    hd, T, W = 64, 11, (hidden + 127) // 128 * 128
    w_qkv = (torch.randn(hidden + 2 * hd, hidden) * 0.03).half().float()
    ops = _padding_ops()
    packed, vt_col0 = ops.falcon_qkv(w_qkv, heads)
    assert packed.shape[0] % 128 == 0 and packed.shape[0] - vt_col0 == hd
    assert packed.shape[0] == ((heads + 2) * hd + 127) // 128 * 128
    y = torch.zeros(T, W)
    y[:, :hidden] = torch.randn(T, hidden).half().float()
    with torch.no_grad():
        q, k, v = att._split_heads((y[:, :hidden] @ w_qkv.T)[None])
        out = y[:, :hidden] @ packed.float().T              # the GEMM reads the first K = hidden columns of y
    assert torch.equal(out[:, :heads * hd].view(T, heads, hd), q[0])
    assert torch.equal(out[:, heads * hd:(heads + 1) * hd].view(T, 1, hd), k[0])
    assert not out[:, (heads + 1) * hd:vt_col0].any()
    assert torch.equal(out[:, vt_col0:].T.contiguous(), v[0, :, 0].T.contiguous())     # the V^T side output
    w_o = (torch.randn(hidden, hidden) * 0.03).half().float()
    w_down = (torch.randn(hidden, ffn) * 0.03).half().float()
    ctx, h = torch.randn(T, hidden), torch.randn(T, ffn)
    x = torch.zeros(T, W)
    x[:, :hidden] = torch.randn(T, hidden)
    x_ref = x[:, :hidden] + (h @ w_down.T + ctx @ w_o.T)
    p_o, p_down = ops.falcon_out(w_o), ops.falcon_out(w_down)
    assert p_o.shape == (W, hidden) and p_down.shape == (W, ffn)
    x = x + ctx @ p_o.float().T                              # the two residual-epilogue GEMMs, dense first
    x = x + h @ p_down.float().T
    assert not x[:, hidden:].any()
    assert torch.allclose(x[:, :hidden], x_ref, rtol=1e-5, atol=1e-5)
    E = torch.randn(50, hidden)
    pe = ops.falcon_embedding(E)
    assert pe.shape == (50, W) and not pe[:, hidden:].any() and torch.equal(pe[:, :hidden], E.half())


def test_rope_tables_at_head_dim_64_match_falcon_rotary_embedding():
    from transformers.models.falcon.modeling_falcon import FalconRotaryEmbedding
    cfg = _cfg(rope_parameters={"rope_type": "default", "rope_theta": 5000.0})
    emb = FalconRotaryEmbedding(cfg)
    cos, sin = emb(torch.zeros(1, 1, 64), torch.arange(300)[None])
    c, s = rope_tables(300, LD.rope_theta(cfg), 64)
    assert c.shape == (300, 32)
    assert torch.equal(torch.cat([c, c], -1), cos[0]) and torch.equal(torch.cat([s, s], -1), sin[0])
    assert torch.equal(rope_tables(64, 10000.0)[0], rope_tables(64, 10000.0, 128)[0])   # the LLaMA default


def _write_checkpoint(d, sd, fmt, dtype, prefix, shards=3):
    os.makedirs(d, exist_ok=True)
    tensors = {prefix + k: torch.from_numpy(v).to(dtype) for k, v in sd.items()}
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
@pytest.mark.parametrize("prefix", ["", "transformer."])
def test_streaming_loader_on_sharded_prefixed_checkpoints(tmp_path, prefix, fmt, dtype):
    """FalconModel and FalconForCausalLM (transformer., lm_head) keys."""
    sd = _sd(layers=3)
    d = str(tmp_path / "ckpt")
    _write_checkpoint(d, sd, fmt, dtype, prefix)
    got = LD.load_ln_decoder_weights(d, "cpu", "falcon")
    assert sorted(got) == sorted(sd) and not any(k.startswith(("transformer.", "lm_head")) for k in got)
    for k, v in sd.items():
        assert got[k].dtype == torch.float16
        assert torch.equal(got[k], torch.from_numpy(v).to(dtype).to(torch.float16)), k
    LD.LnDecoderNet(dict(got), LD.TorchOps(), "falcon", 3, C["heads"], 1e-5, C["max_pos"])


REFUSED = [
    (dict(new_decoder_architecture=True), "new_decoder_architecture"),
    (dict(alibi=True), "alibi"),
    (dict(parallel_attn=False), "parallel_attn"),
    (dict(multi_query=False), "multi_query"),
    (dict(multi_query=False, num_kv_heads=1), "multi_query"),
    (dict(bias=True), "bias"),
    (dict(activation="relu"), "activation"),
    (dict(num_attention_heads=4), "head_dim"),
    (dict(rope_parameters={"rope_type": "linear", "rope_theta": 10000.0, "factor": 2.0}), "rotary"),
    (dict(hidden_size=32 * 7, num_attention_heads=7), "head_dim"),
    (dict(ffn_hidden_size=1800), "ffn_hidden_size"),
]


@pytest.mark.parametrize("kw,msg", REFUSED)
def test_unsupported_configs_are_rejected(kw, msg):
    LD.check_ln_decoder_config(_cfg())
    with pytest.raises(ValueError, match=msg):
        LD.check_ln_decoder_config(_cfg(**kw))


def test_hidden_not_a_multiple_of_64_is_rejected():
    """head_dim 64 implies hidden % 64 == 0; the check stands on its own for a config object that says otherwise."""
    cfg = types.SimpleNamespace(**{**_cfg().to_dict(), "model_type": "falcon", "hidden_size": 4544 + 32,
                                   "num_attention_heads": 71})
    with pytest.raises(ValueError, match="head_dim|multiple of 64"):
        LD.check_ln_decoder_config(cfg)


@pytest.mark.parametrize("kw,msg", REFUSED)
def test_rejects_before_reading_weights(tmp_path, kw, msg):
    """extract_embedding's Falcon branch refuses from the config alone: no weight file exists here."""
    from mertools_b200.extract import text
    d = tmp_path / "tools" / "transformers" / "m"
    d.mkdir(parents=True)
    _cfg(**kw).save_pretrained(str(d))
    with pytest.raises(ValueError, match=msg):
        text._ln_decoder_extractor(str(d), transformers.AutoConfig.from_pretrained(str(d)), "cpu")


@pytest.mark.parametrize("model_type", LD.REFINEDWEB_TYPES)
def test_refinedweb_checkpoints_are_refused(tmp_path, model_type):
    """The legacy remote-code Falcon format: refused by name, before AutoConfig (which does not know it) and before any
    weight is read."""
    from mertools_b200.extract import text
    d = tmp_path / "m"
    d.mkdir()
    (d / "config.json").write_text(json.dumps({"model_type": model_type, "hidden_size": 4544, "n_head": 71}))
    with pytest.raises(ValueError, match="RefinedWeb.*legacy"):
        text._refuse_remote_code_falcon(str(d))
    with pytest.raises(ValueError, match="legacy"):
        LD.check_ln_decoder_config(types.SimpleNamespace(model_type=model_type))
    text._refuse_remote_code_falcon(str(tmp_path))   # no config.json: AutoConfig reports that itself


def test_refuses_sentences_longer_than_max_positions():
    cfg = _cfg(max_position_embeddings=64, num_hidden_layers=3)
    net = _net(_sd(layers=3), cfg)
    with pytest.raises(ValueError, match="max_position_embeddings"):
        net.forward(np.arange(4, 69), [65])


def test_activation_budget_per_token():
    """~130 KB of activations per token at the Falcon-7B shape, counted on the padded rows."""
    assert 90e3 < LD.activation_bytes_per_token(4544, 18176, "falcon") < 160e3
