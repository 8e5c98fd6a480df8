"""Layer-by-layer float64 parity of the host-orchestrated decoder text stacks: LlamaTextEncoder (LLaMA) and
LnDecoderTextEncoder (BLOOM, OPT, GPT-2, Falcon), built on synthetic checkpoints.

Each case runs net.forward(ids, lens, return_hidden=True) over one packed batch and checks hidden_states[0] against
decoder_embedding and every hidden_states[l + 1] against decoder_layer(hidden_states[l]) (the last through final_norm),
elementwise |err| <= bound (tests/_decoder_refs.py).  Each layer is fed the GPU's own hidden state, so errors do not
compound down the stack; the float64 work runs on the GPU and is freed per layer.  The return_hidden=False readout must
equal the in-order fp32 sum h[L-3] + h[L-2] + h[L-1] + hidden_states[L] bit for bit: both go through the same residual
and final-norm epilogues, so any difference is a wiring bug, not rounding.  That run is profiled, and the one attention
kernel instance it launches is the family's (attention_kernel).  Falcon's pad columns (rows padded to a multiple of 128)
are exactly 0 in every hidden state and in the readout.  hidden_states[0] of OPT and GPT-2 is one or two fp32 adds of
fp16-exact rows, whose bound u |sum| per add is sharp (round to nearest stays within u / (1 + u) of the exact sum), so
ratios near 1 there are expected.

Small cases (synthetic.*_state_dict written as safetensors and read back through the product loaders, so the GPT-2
Conv1D transpose and the prefix handling are in the path): the packed lengths of DECODER_LENS, sentence starts mostly
off a multiple of 8, with a sentence of exactly max_position_embeddings tokens (320) for LLaMA, OPT and GPT-2; GPT-2 at
head_dim 64 with and without token types and at head_dim 96.  Full-width cases: 3 layers at the widths of LLaMA-13B,
BLOOM-7B1, OPT-13B, Wenzhong GPT-2 (head_dim 96) and Falcon-7B (4544 = 71 x 64 padded to 4608), and BLOOM at 12 heads
(the interleaved tail of alibi_slopes), on a few dozen tokens."""
import os
import time

import numpy as np
import pytest
import torch

import _decoder_refs as DR
import _kernel_refs as R
from mertools_b200.extract import llama_text as LT
from mertools_b200.extract import ln_decoder_text as LD

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _wall_time():
    t0 = time.time()
    yield
    print(f"\ntest_decoder_stack_gpu.py: {time.time() - t0:.1f} s wall time")


def _config(family, vocab, D, heads, F, layers, max_pos, eps):
    import transformers as T
    if family == "llama":
        return T.LlamaConfig(vocab_size=vocab, hidden_size=D, num_attention_heads=heads, intermediate_size=F,
                             num_hidden_layers=layers, max_position_embeddings=max_pos, rms_norm_eps=eps)
    if family == "bloom":
        return T.BloomConfig(vocab_size=vocab, hidden_size=D, n_head=heads, n_layer=layers, layer_norm_epsilon=eps)
    if family == "opt":
        return T.OPTConfig(vocab_size=vocab, hidden_size=D, num_attention_heads=heads, ffn_dim=F,
                           num_hidden_layers=layers, max_position_embeddings=max_pos, word_embed_proj_dim=D)
    if family == "gpt2":
        return T.GPT2Config(vocab_size=vocab, n_positions=max_pos, n_embd=D, n_layer=layers, n_head=heads, n_inner=F,
                            layer_norm_epsilon=eps)
    return T.FalconConfig(vocab_size=vocab, hidden_size=D, num_attention_heads=heads, ffn_hidden_size=F,
                          num_hidden_layers=layers, max_position_embeddings=max_pos, layer_norm_epsilon=eps)


def _encoder(family, sd_loaded, cfg, cuda):
    if family == "llama":
        return LT.LlamaTextEncoder(sd_loaded, cfg, device=cuda)
    return LD.LnDecoderTextEncoder(sd_loaded, cfg, device=cuda)


def _check_stack(enc, family, sd, heads, eps, max_pos, ids, lens, tt, tag, cuda):
    """Run the checks of the module docstring; returns the report line."""
    net = enc.net
    D = net.hidden
    hd = 64 if family == "falcon" else D // heads
    kw = {} if family == "llama" else dict(token_types=tt)
    acc_h, hs = net.forward(ids, lens, return_hidden=True, **kw)
    acc, names = R.attention_kernels(lambda: net.forward(ids, lens, **kw).clone())
    want = DR.attention_kernel(family, hd)
    assert names and all(want in n for n in names), (tag, want, names)
    n = len(hs) - 1
    seq = ((hs[n - 3] + hs[n - 2]) + hs[n - 1]) + hs[n]
    assert torch.equal(R.bits(acc), R.bits(seq)) and torch.equal(R.bits(acc_h), R.bits(seq)), tag
    if hs[0].shape[1] != D:                       # Falcon: padded rows
        assert family == "falcon" and hs[0].shape[1] == (D + 127) // 128 * 128
        assert all(bool((h[:, D:] == 0).all()) for h in hs) and bool((acc[:, D:] == 0).all()), tag
    h0, e0 = DR.decoder_embedding(family, sd, ids, lens, eps, tt, device=cuda)
    r0 = float(R.bound_ratio(hs[0][:, :D], h0, e0).max())
    assert r0 <= 1.0, (tag, r0)
    del h0, e0
    tables, slopes = DR.layer_tables(family, max_pos or 2048, heads=heads, device=cuda)
    worst = []
    for l in range(n):
        w = DR.decoder_weights(family, sd, l, heads, cuda)
        ref, bound = DR.decoder_layer(family, w, hs[l][:, :D], lens, heads, eps, tables, slopes)
        if l == n - 1:
            ref, bound = DR.final_norm(family, sd, ref, bound, eps, device=cuda)
        worst.append(float(R.bound_ratio(hs[l + 1][:, :D], ref, bound).max()))
        del w, ref, bound
        torch.cuda.empty_cache()
    line = (f"{tag} ({want}): hidden_states[0] {r0:.3f}; |err| / bound by layer "
            + ", ".join(f"{r:.3f}" for r in worst))
    print(line)
    assert all(r <= 1.0 for r in worst), (tag, worst)
    return line


@pytest.mark.parametrize("name", DR.SMALL_CASES)
def test_small_checkpoint_stack_layers_and_readout(cuda, tmp_path, name):
    from safetensors.torch import save_file
    c = DR.small_case(name)
    f, sd = c["family"], c["sd"]
    save_file({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in sd.items()},
              os.path.join(str(tmp_path), "model.safetensors"))
    if f == "llama":
        loaded = LT.load_llama_weights(str(tmp_path), cuda)
        D, F = loaded["embed_tokens.weight"].shape[1], loaded["layers.0.mlp.up_proj.weight"].shape[0]
    else:
        loaded = LD.load_ln_decoder_weights(str(tmp_path), cuda, f)
        up = {"bloom": "h.0.mlp.dense_h_to_4h.weight", "opt": "layers.0.fc1.weight", "gpt2": "h.0.mlp.c_fc.weight",
              "falcon": "h.0.mlp.dense_h_to_4h.weight"}[f]
        F = loaded[up].shape[0]
        D = loaded[up].shape[1]
    cfg = _config(f, c["vocab"], D, c["heads"], F, c["layers"], c["max_pos"] or 2048, c["eps"])
    enc = _encoder(f, loaded, cfg, cuda)
    _check_stack(enc, f, sd, c["heads"], c["eps"], c["max_pos"], c["ids"], c["lens"], c["token_types"], name, cuda)


# (family, hidden, heads, FFN): the widths of LLaMA-13B, BLOOM-7B1 (and BLOOM at 12 heads), OPT-13B, Wenzhong GPT-2 and
# Falcon-7B
FULL_WIDTH = {"llama": ("llama", 5120, 40, 13824), "bloom": ("bloom", 4096, 32, 16384), "bloom12": ("bloom", 1536, 12, 6144),
              "opt": ("opt", 5120, 40, 20480), "gpt2_96": ("gpt2", 3072, 32, 12288), "falcon": ("falcon", 4544, 71, 18176)}


def _full_width_sd(family, D, heads, F, cuda, vocab=1000, max_pos=2048, layers=3):
    """An HF-named fp16 state dict on the device: std-0.02 matrices, 0.02 biases, LayerNorm gains 1 + 0.1 N and biases
    0.1 N, std-1 embeddings (0.1 for learned positions); BLOOM's fused rows interleaved, GPT-2's Conv1D weights [in, out],
    Falcon's heads x q | k | v rows."""
    g = torch.Generator(device=cuda).manual_seed(17)

    def w(*shape, std=0.02):
        return (torch.randn(*shape, generator=g, device=cuda) * std).half()

    def ln(p, bias=True):
        return {p + ".weight": 1 + w(D, std=0.1), **({p + ".bias": w(D, std=0.1)} if bias else {})}

    def lin(p, out, inp, bias=True):
        return {p + ".weight": w(out, inp), **({p + ".bias": w(out)} if bias else {})}
    sd = {}
    if family == "llama":
        sd.update({"embed_tokens.weight": w(vocab, D, std=1.0), **ln("norm", False)})
        for i in range(layers):
            p = f"layers.{i}."
            for n in ("q_proj", "k_proj", "v_proj", "o_proj"):
                sd.update(lin(p + "self_attn." + n, D, D, False))
            sd.update({**lin(p + "mlp.gate_proj", F, D, False), **lin(p + "mlp.up_proj", F, D, False),
                       **lin(p + "mlp.down_proj", D, F, False), **ln(p + "input_layernorm", False),
                       **ln(p + "post_attention_layernorm", False)})
    elif family == "bloom":
        sd.update({"word_embeddings.weight": w(vocab, D, std=1.0), **ln("word_embeddings_layernorm"), **ln("ln_f")})
        for i in range(layers):
            p = f"h.{i}."
            sd.update({**ln(p + "input_layernorm"), **ln(p + "post_attention_layernorm"),
                       **lin(p + "self_attention.query_key_value", 3 * D, D), **lin(p + "self_attention.dense", D, D),
                       **lin(p + "mlp.dense_h_to_4h", F, D), **lin(p + "mlp.dense_4h_to_h", D, F)})
    elif family == "opt":
        sd.update({"embed_tokens.weight": w(vocab, D, std=1.0), "embed_positions.weight": w(max_pos + 2, D, std=0.1),
                   **ln("final_layer_norm")})
        for i in range(layers):
            p = f"layers.{i}."
            sd.update({**ln(p + "self_attn_layer_norm"), **ln(p + "final_layer_norm"), **lin(p + "fc1", F, D),
                       **lin(p + "fc2", D, F)})
            for n in ("q", "k", "v", "out"):
                sd.update(lin(p + f"self_attn.{n}_proj", D, D))
    elif family == "gpt2":
        sd.update({"wte.weight": w(vocab, D, std=1.0), "wpe.weight": w(max_pos, D, std=0.1), **ln("ln_f")})
        for i in range(layers):
            p = f"h.{i}."
            sd.update({**ln(p + "ln_1"), **ln(p + "ln_2")})
            for n, (i_, o_) in (("attn.c_attn", (D, 3 * D)), ("attn.c_proj", (D, D)), ("mlp.c_fc", (D, F)),
                                ("mlp.c_proj", (F, D))):
                sd.update({p + n + ".weight": w(i_, o_), p + n + ".bias": w(o_)})
    else:
        sd.update({"word_embeddings.weight": w(vocab, D, std=1.0), **ln("ln_f")})
        for i in range(layers):
            p = f"h.{i}."
            sd.update({**ln(p + "input_layernorm"), **lin(p + "self_attention.query_key_value", D + 128, D, False),
                       **lin(p + "self_attention.dense", D, D, False), **lin(p + "mlp.dense_h_to_4h", F, D, False),
                       **lin(p + "mlp.dense_4h_to_h", D, F, False)})
    return sd


@pytest.mark.parametrize("name", list(FULL_WIDTH))
def test_full_width_stack_layers_and_readout(cuda, name):
    family, D, heads, F = FULL_WIDTH[name]
    sd = _full_width_sd(family, D, heads, F, cuda)
    loaded = {k: (v.T.contiguous() if family == "gpt2" and k.endswith(LD.GPT2_CONV1D) else v) for k, v in sd.items()}
    cfg = _config(family, 1000, D, heads, F, 3, 2048, 1e-5)
    enc = _encoder(family, loaded, cfg, cuda)
    del loaded
    lens = [9, 1, 30, 17, 2]
    rng = np.random.default_rng(5)
    ids = rng.integers(0, 1000, sum(lens))
    ids[0], ids[-1] = 0, 999
    tt = rng.integers(0, 3, sum(lens)) if family == "gpt2" else None
    _check_stack(enc, family, sd, heads, 1e-5, None if family == "bloom" else 2048, ids, lens, tt,
                 f"{name} {D} x {heads}", cuda)
