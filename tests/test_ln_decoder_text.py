"""CPU checks of the BLOOM / OPT branch of the text extractor (mertools_b200/extract/ln_decoder_text.py): the
orchestration with a torch fp32 backend against HF BloomModel / OPTModel (every hidden state) and against the golden of
the unmodified reference extract_embedding (tests/golden/make_golden_bloom_opt.py), the de-interleaved BLOOM QKV, the
ALiBi slopes, the tokenizer probes, the streaming weight loader on sharded prefixed checkpoints, and the configs the
path refuses."""
import gzip
import json
import os

import numpy as np
import pytest
import torch

from mertools_b200 import synthetic as S
from mertools_b200.extract import common
from mertools_b200.extract import ln_decoder_text as LD

transformers = pytest.importorskip("transformers")
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
C = S.LN_DECODER_SMALL_CFG
FAMILIES = ["bloom", "opt"]


def _cfg(family, **kw):
    if family == "bloom":
        base = dict(vocab_size=C["vocab"], hidden_size=C["hidden"], n_head=C["heads"], n_layer=C["layers"],
                    bos_token_id=0, eos_token_id=2, pad_token_id=1)
        base.update(kw)
        return transformers.BloomConfig(**base)
    base = dict(vocab_size=C["vocab"], hidden_size=C["hidden"], num_attention_heads=C["heads"], ffn_dim=C["ffn"],
                num_hidden_layers=C["layers"], max_position_embeddings=C["max_pos"], word_embed_proj_dim=C["hidden"],
                bos_token_id=2, eos_token_id=2, pad_token_id=1)
    base.update(kw)
    return transformers.OPTConfig(**base)


def _sd(family, seed=None, **kw):
    if family == "bloom":
        return S.bloom_state_dict(**({} if seed is None else dict(seed=seed)), **kw)
    return S.opt_state_dict(**({} if seed is None else dict(seed=seed)), **kw)


def _hf(family, sd, cfg):
    m = (transformers.BloomModel if family == "bloom" else transformers.OPTModel)(cfg).eval()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    return m


def _net(family, sd, cfg, dtype=torch.float32):
    fam, layers, heads, _, _, eps, max_pos = LD.net_dims(cfg)
    assert fam == family
    return LD.LnDecoderNet({LD._strip(k, family): torch.from_numpy(v) for k, v in sd.items()}, LD.TorchOps(dtype=dtype),
                           family, layers, heads, eps, max_pos)


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / np.abs(b).max())


@pytest.mark.parametrize("family", FAMILIES)
def test_torch_orchestration_matches_hf_every_hidden_state(family):
    """Three sentences packed (one crosses 64 tokens): positions / ALiBi restart, no attention across them.  The
    hidden_states tuple of OPTModel (output recorders in transformers 5) is h[0] = E[ids] + P[pos + 2], the layer
    outputs, and last_hidden_state = final_layer_norm(h[L])."""
    sd, cfg = _sd(family), _cfg(family)
    m = _hf(family, sd, cfg)
    rng = np.random.default_rng(0)
    sents = [rng.integers(4, C["vocab"], n) for n in (37, 70, 1)]
    with torch.no_grad():
        acc, hs = _net(family, sd, cfg).forward(np.concatenate(sents), [len(s) for s in sents], return_hidden=True)
        o = 0
        for s in sents:
            out = m(torch.from_numpy(s)[None], output_hidden_states=True)
            ref = out.hidden_states
            assert len(ref) == len(hs) == C["layers"] + 1
            for i, (r, h) in enumerate(zip(ref, hs)):
                assert _rel(h[o:o + len(s)], r[0]) < 2e-5, (i, _rel(h[o:o + len(s)], r[0]))
            assert torch.equal(ref[-1], out.last_hidden_state)
            assert _rel(acc[o:o + len(s)], torch.stack(ref)[[-4, -3, -2, -1]].sum(0)[0]) < 2e-5
            o += len(s)


def test_deinterleaved_bloom_qkv_reproduces_bloom_attention():
    """q | k | v blocks from the de-interleaved query_key_value give BloomAttention's per-head q, k, v."""
    from transformers.models.bloom.modeling_bloom import BloomAttention
    cfg = _cfg("bloom")
    att = BloomAttention(cfg, layer_idx=0).eval()
    sd = S.bloom_state_dict(layers=1)
    att.query_key_value.weight.data = torch.from_numpy(sd["h.0.self_attention.query_key_value.weight"])
    att.query_key_value.bias.data = torch.from_numpy(sd["h.0.self_attention.query_key_value.bias"])
    x = torch.randn(1, 9, C["hidden"])
    H, D = C["heads"], C["hidden"]
    with torch.no_grad():
        fused = att.query_key_value(x)
        q, k, v = att._reshape(fused)                              # [batch * heads, seq, 128] (k transposed in HF)
        w = LD.deinterleave_qkv(att.query_key_value.weight, H)
        b = LD.deinterleave_qkv(att.query_key_value.bias, H)
        ours = x[0] @ w.T + b
    blocks = [ours[:, i * D:(i + 1) * D].view(9, H, 128).transpose(0, 1) for i in range(3)]
    assert torch.equal(blocks[0], q.reshape(H, 9, 128))
    assert torch.equal(blocks[1], k.reshape(H, 9, 128)) or torch.equal(blocks[1], k.reshape(H, 128, 9).transpose(1, 2))
    assert torch.equal(blocks[2], v.reshape(H, 9, 128))


def test_alibi_slopes_match_build_alibi_tensor():
    from transformers.models.bloom.modeling_bloom import build_alibi_tensor
    for heads in range(1, 65):
        ref = build_alibi_tensor(torch.ones(1, 2, dtype=torch.long), heads, torch.float32)[:, 0, 1]
        assert torch.equal(LD.alibi_slopes(heads), ref), heads


def _golden(family):
    return np.load(os.path.join(G, f"{family}_text_golden.npz"))


def unpack_tokenizer(family, dest):
    """The committed tokenizer fixture of ``family`` as a loadable directory (its ``*.gz`` files decompressed)."""
    src = os.path.join(G, f"{family}_tokenizer")
    os.makedirs(dest, exist_ok=True)
    for f in os.listdir(src):
        with (gzip.open if f.endswith(".gz") else open)(os.path.join(src, f), "rb") as a, \
                open(os.path.join(dest, f[:-3] if f.endswith(".gz") else f), "wb") as b:
            b.write(a.read())


def _tokenizer(family, dest):
    from transformers import AutoTokenizer
    unpack_tokenizer(family, dest)
    return AutoTokenizer.from_pretrained(dest, use_fast=False)


@pytest.mark.parametrize("family,probe", [("bloom", (0, None)), ("opt", (1, None))])
def test_tokenizer_fixture_probe_and_ids(tmp_path, family, probe):
    from mertools_b200.extract.text import find_start_end_pos
    g, tok = _golden(family), _tokenizer(family, str(tmp_path / "tok"))
    assert find_start_end_pos(tok) == probe == (int(g["start"]), None if int(g["end"]) == 0 else int(g["end"]))
    cfg = _cfg(family)
    assert (tok.bos_token_id, tok.eos_token_id, tok.pad_token_id) == (cfg.bos_token_id, cfg.eos_token_id,
                                                                       cfg.pad_token_id)
    for i, (s, nan) in enumerate(zip(g["sentences"], g["isnan"])):
        if not nan:
            assert tok(str(s))["input_ids"] == g[f"ids{i}"].tolist(), i
    lens = [len(g[f"ids{i}"]) for i in range(len(g["sentences"])) if not g["isnan"][i]]
    assert max(lens) > 64 and min(lens) <= 2


@pytest.mark.parametrize("which", ["hf", "torch_backend"])
@pytest.mark.parametrize("family", FAMILIES)
def test_readout_matches_reference_golden(family, which):
    """The golden's features from HF BloomModel / OPTModel (the oracle) and from LnDecoderNet on the torch backend."""
    g = _golden(family)
    sd, cfg = _sd(family, seed=int(g["seed"])), _cfg(family)
    start = int(g["start"])
    idx = [i for i in range(len(g["sentences"])) if not g["isnan"][i]]
    ids = [g[f"ids{i}"] for i in idx]
    with torch.no_grad():
        if which == "hf":
            m = _hf(family, sd, cfg)
            rows = [torch.stack(m(torch.from_numpy(x)[None], output_hidden_states=True).hidden_states)[[-4, -3, -2, -1]]
                    .sum(0)[0].numpy() for x in ids]
        else:
            acc = _net(family, sd, cfg).forward(np.concatenate(ids), [len(x) for x in ids]).numpy()
            cu = np.concatenate([[0], np.cumsum([len(x) for x in ids])])
            rows = [acc[cu[j]:cu[j + 1]] for j in range(len(ids))]
    for j, i in enumerate(idx):
        for level in ("UTTERANCE", "FRAME"):
            ref = g[f"{level[:3].lower()}{i}"]
            got = common.save_feature(None, rows[j][start:], level, C["hidden"])
            assert got.shape == ref.shape and _rel(got, ref) < 2e-5, (which, i, level, _rel(got, ref))
    nan = [i for i in range(len(g["sentences"])) if g["isnan"][i]]
    assert nan and all(g[f"utt{i}"].dtype == np.float64 and not g[f"utt{i}"].any() for i in nan)


def _write_checkpoint(d, sd, fmt, dtype, prefix, shards=3):
    """A sharded checkpoint as save_pretrained writes one (shard files + index.json), keys under ``prefix`` and an
    lm_head when there is a prefix (a *ForCausalLM checkpoint)."""
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
@pytest.mark.parametrize("family,prefix", [("bloom", ""), ("bloom", "transformer."), ("opt", ""), ("opt", "model.")])
def test_streaming_loader_on_sharded_prefixed_checkpoints(tmp_path, family, prefix, fmt, dtype):
    """BloomModel / BloomForCausalLM (transformer.) and OPTModel (decoder.) / OPTForCausalLM (model.decoder.) keys."""
    sd = _sd(family, layers=3)
    d = str(tmp_path / "ckpt")
    _write_checkpoint(d, sd, fmt, dtype, prefix)
    got = LD.load_ln_decoder_weights(d, "cpu", family)
    want = {LD._strip(k, family): v for k, v in sd.items()}
    assert sorted(got) == sorted(want) and not any(k.startswith(("transformer.", "model.", "decoder.")) for k in got)
    for k, v in want.items():
        assert got[k].dtype == torch.float16
        assert torch.equal(got[k], torch.from_numpy(v).to(dtype).to(torch.float16)), k
    # the loaded names drive LnDecoderNet
    LD.LnDecoderNet(dict(got), LD.TorchOps(), family, 3, C["heads"], 1e-5, None if family == "bloom" else C["max_pos"])


def test_streaming_loader_refuses_non_finite(tmp_path):
    sd = _sd("opt", layers=3)
    sd["decoder.layers.1.fc1.weight"][3, 5] = 1e6    # overflows fp16
    d = str(tmp_path / "ckpt")
    _write_checkpoint(d, sd, "safetensors", torch.float32, "")
    with pytest.raises(ValueError, match="not finite"):
        LD.load_ln_decoder_weights(d, "cpu", "opt")


REFUSED = [
    ("bloom", dict(apply_residual_connection_post_layernorm=True), "apply_residual"),
    ("bloom", dict(slow_but_exact=True, pretraining_tp=2), "slow_but_exact"),
    ("bloom", dict(n_head=8), "head_dim"),
    ("opt", dict(do_layer_norm_before=False), "do_layer_norm_before"),
    ("opt", dict(word_embed_proj_dim=256), "word_embed_proj_dim"),
    ("opt", dict(enable_bias=False), "enable_bias"),
    ("opt", dict(layer_norm_elementwise_affine=False), "non-affine"),
    ("opt", dict(_remove_final_layer_norm=True), "_remove_final_layer_norm"),
    ("opt", dict(activation_function="gelu"), "activation_function"),
    ("opt", dict(num_attention_heads=8), "head_dim"),
]


@pytest.mark.parametrize("family,kw,msg", REFUSED)
def test_unsupported_configs_are_rejected(family, kw, msg):
    LD.check_ln_decoder_config(_cfg(family))
    with pytest.raises(ValueError, match=msg):
        LD.check_ln_decoder_config(_cfg(family, **kw))


@pytest.mark.parametrize("family,kw,msg", REFUSED)
def test_rejects_before_reading_weights(tmp_path, family, kw, msg):
    """extract_embedding's BLOOM / OPT branch refuses from the config alone: no weight file exists here."""
    from mertools_b200.extract import text
    d = tmp_path / "tools" / "transformers" / "m"
    d.mkdir(parents=True)
    _cfg(family, **kw).save_pretrained(str(d))
    with pytest.raises(ValueError, match=msg):
        text._ln_decoder_extractor(str(d), transformers.AutoConfig.from_pretrained(str(d)), "cpu")


def test_opt_refuses_sentences_longer_than_max_positions():
    cfg = _cfg("opt", max_position_embeddings=64)
    net = _net("opt", _sd("opt", layers=3, max_pos=64), cfg.__class__(**{**cfg.to_dict(), "num_hidden_layers": 3}))
    with pytest.raises(ValueError, match="max_position_embeddings"):
        net.forward(np.arange(4, 69), [65])


def test_activation_budget_per_token():
    """~100-150 KB of activations per token at the BLOOM-7B1 / OPT-13B shapes."""
    assert 80e3 < LD.activation_bytes_per_token(4096, 16384) < 160e3
    assert 100e3 < LD.activation_bytes_per_token(5120, 20480) < 200e3
