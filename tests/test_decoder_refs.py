"""CPU checks of the decoder-layer restatements of tests/_decoder_refs.py, which tests/test_decoder_stack_gpu.py holds
the LLaMA, BLOOM, OPT, GPT-2 and Falcon stacks to: the restatement is the torch nets' layer in float64, its bound
covers an fp32 emulation of the CUDA path's arithmetic, and it rejects each restated wiring fault by 4x or more."""
import numpy as np
import pytest
import torch

import _decoder_refs as DR
import _kernel_refs as R
from mertools_b200.extract import llama_text as LT
from mertools_b200.extract import ln_decoder_text as LD

_CACHE = {}


def loaded(family, sd):
    """An HF-named state dict as the loader hands it to the nets: prefixes stripped, GPT-2's Conv1D weights [out, in]."""
    out = {}
    for k, v in sd.items():
        t = torch.from_numpy(np.asarray(v))
        out[LD._strip(k, family)] = t.T.contiguous() if family == "gpt2" and k.endswith(LD.GPT2_CONV1D) else t
    return out


def _case(name):
    """(case, float64 torch-net hidden states) of a small case, cached."""
    if name not in _CACHE:
        c = DR.small_case(name)
        f, sd = c["family"], c["sd"]
        ops = (LT if f == "llama" else LD).TorchOps(dtype=torch.float64)
        if f == "llama":
            net = LT.LlamaNet(loaded(f, sd), ops, c["layers"], c["heads"], c["eps"], 10000.0, c["max_pos"])
            _, hs = net.forward(c["ids"], c["lens"], return_hidden=True)
        else:
            net = LD.LnDecoderNet(loaded(f, sd), ops, f, c["layers"], c["heads"], c["eps"], c["max_pos"])
            _, hs = net.forward(c["ids"], c["lens"], return_hidden=True, token_types=c["token_types"])
        c["tables"], c["slopes"] = DR.layer_tables(f, c["max_pos"] or 2048, heads=c["heads"])
        _CACHE[name] = (c, hs)
    return _CACHE[name]


def _layer(c, x, l, **kw):
    w = DR.decoder_weights(c["family"], c["sd"], l, c["heads"])
    return DR.decoder_layer(c["family"], w, x, c["lens"], c["heads"], c["eps"], c["tables"], c["slopes"], **kw)


@pytest.mark.parametrize("name", DR.SMALL_CASES)
def test_decoder_layer_is_the_torch_net_layer(name):
    """Without operand rounding, decoder_embedding, decoder_layer and final_norm are the family's TorchOps net in float64
    (LlamaNet / LnDecoderNet, which test_llama_text.py, test_ln_decoder_text.py, test_gpt2_text.py and test_falcon_text.py
    tie to HF) on that net's own hidden states, within 1e-12; every bound is positive."""
    c, hs = _case(name)
    f = c["family"]
    h0, e0 = DR.decoder_embedding(f, c["sd"], c["ids"], c["lens"], c["eps"], c["token_types"])
    worst = float((h0 - hs[0]).abs().max())
    n = c["layers"]
    for l in range(n):
        x, b = _layer(c, hs[l], l)
        if l == n - 1:
            x, b = DR.final_norm(f, c["sd"], x, b, c["eps"])
        worst = max(worst, float((x - hs[l + 1]).abs().max()))
        assert bool((b > 0).all()), l
    print(f"{name}: restatement vs TorchOps float64, max |diff| {worst:.1e} over hidden_states[0 .. {n}]")
    assert worst < 1e-12


@pytest.mark.parametrize("name", DR.SMALL_CASES)
def test_decoder_bound_covers_an_fp32_emulation(name):
    """An fp32 evaluation of each layer that rounds every operand the CUDA path stores (norm outputs, q | k | v, q | k
    after RoPE, P for P V, ctx, the FFN activation) to fp16 lands inside the float64 restatement's bound, at a ratio in
    (1e-3, 1]; the last layer through the final norm."""
    c, hs = _case(name)
    worst = []
    for l in range(c["layers"]):
        x = hs[l].float()
        ref, bound = _layer(c, x, l)
        emu, _ = _layer(c, x, l, emulate=True)
        if l == c["layers"] - 1:
            ref, bound = DR.final_norm(c["family"], c["sd"], ref, bound, c["eps"])
            emu = DR.final_norm(c["family"], c["sd"], emu.double(), torch.zeros_like(ref), c["eps"])[0]
        worst.append(float(R.bound_ratio(emu, ref, bound).max()))
    print(f"{name}: fp32 emulation / bound by layer " + ", ".join(f"{r:.3f}" for r in worst))
    assert all(1e-3 < r <= 1.0 for r in worst), worst


def test_decoder_bound_rejects_the_faults():
    """Each fault of DECODER_FAULTS, restated on layer 0 (or hidden_states[0]) of the cases the GPU test runs, leaves the
    bound by 4x or more on some element.  ALiBi as slope * j instead of slope * (j - i), or counted from the pack start,
    is a per-row constant the softmax cancels: not a fault, and so not listed."""
    worst = {}
    for fault, names in DR.DECODER_FAULTS.items():
        for name in DR.SMALL_CASES:
            c, hs = _case(name)
            if name not in names and c["family"] not in names:
                continue
            if fault in DR.EMBED_FAULTS:
                args = (c["family"], c["sd"], c["ids"], c["lens"], c["eps"], c["token_types"])
                ref, bound = DR.decoder_embedding(*args)
                got, _ = DR.decoder_embedding(*args, fault=fault)
            else:
                x = hs[0].float()
                ref, bound = _layer(c, x, 0)
                got, _ = _layer(c, x, 0, fault=fault)
            r = float(R.bound_ratio(got, ref, bound).max())
            if r >= worst.get(fault, ("", -1.0))[1]:
                worst[fault] = (name, r)
    print("fault / bound: " + ", ".join(f"{k} {v[1]:.3g} ({v[0]})" for k, v in worst.items()))
    assert set(worst) == set(DR.DECODER_FAULTS)
    assert all(v[1] >= 4 for v in worst.values()), worst


def test_rope_tables_at_head_dim_128_match_llama_rotary_embedding():
    """The fp32 cos / sin operands decoder_layer takes are HF's LlamaRotaryEmbedding values (its cat(freqs, freqs)
    halves), bit for bit, up to DECODER_MAX_POS."""
    from transformers import LlamaConfig
    from transformers.models.llama.modeling_llama import LlamaRotaryEmbedding
    cfg = LlamaConfig(hidden_size=512, num_attention_heads=4, max_position_embeddings=DR.DECODER_MAX_POS)
    cos, sin = LlamaRotaryEmbedding(cfg)(torch.zeros(1, 1, 128), torch.arange(DR.DECODER_MAX_POS)[None])
    (c, s), _ = DR.layer_tables("llama", DR.DECODER_MAX_POS)
    assert torch.equal(torch.cat([c, c], -1), cos[0]) and torch.equal(torch.cat([s, s], -1), sin[0])


def test_small_cases_cover_the_packing_edges():
    """Every case packs the edge lengths with most sentence starts off a multiple of 8; LLaMA, OPT and GPT-2 include a
    sentence of exactly max_position_embeddings tokens; ids 0 and vocab - 1 both occur."""
    for name in DR.SMALL_CASES:
        c = DR.small_case(name)
        starts = np.cumsum([0] + c["lens"][:-1])
        assert sum(s % 8 != 0 for s in starts) > len(starts) // 2, name
        assert c["ids"].min() == 0 and c["ids"].max() == c["vocab"] - 1
        if c["family"] in ("llama", "opt", "gpt2"):
            assert c["max_pos"] in c["lens"], name
