"""BLOOM / OPT / GPT-2 / Falcon branch of the text extractor: the pre-LayerNorm decoder LLMs among those the reference
loads (MERBench/feature_extraction/text/extract_text_huggingface.py): ``bloom-7b1`` and ``opt-13b`` through plain
``AutoModel`` (:170-172) and ``falcon-7b`` (AutoModel, :188-190), run in fp16 (:193-196), and
``gpt2-chinese-cluecorpussmall`` (AutoModel, :188-190) and ``wenzhong2-gpt2-chinese`` (GPT2Model, :167-169), run in fp32;
one sentence per forward (:208-231).  Readout as for every text model:
``torch.stack(hidden_states)[[-4, -3, -2, -1]].sum(0)``, where the last term is the output of the final LayerNorm
(``ln_f`` / ``final_layer_norm``) and the other three are raw residual states.

Both families are one orchestration (``LnDecoderNet``) over an ``ops`` backend, as in llama_text.py:
- BLOOM: h[0] = word_embeddings_layernorm(E[ids]); causal attention with ALiBi (``mer_causal_alibi_attention_f16``),
  slopes from ``alibi_slopes``; tanh-GELU MLP (``MER_EPI_GELU_TANH``).  The fused ``query_key_value`` rows, interleaved
  per head as [head][q, k, v][128], are de-interleaved into q | k | v blocks at load time.
- OPT: h[0] = E[ids] + P[pos + 2] (learned positions, offset 2); plain causal attention (``mer_causal_attention_hd_f16``
  at head_dim 128, the kernel of ``mer_causal_attention_f16``); ReLU MLP (``MER_EPI_RELU | MER_EPI_OUT_F16``).
- GPT-2: h[0] = wte[ids] + wpe[pos] (+ wte[token_type_ids] when the tokenizer returns token types, as GPT2Model adds
  them); plain causal attention at head_dim 64, 96 or 128 (``mer_causal_attention_hd_f16``); tanh-GELU MLP (gelu_new).
  The Conv1D weights, stored [in, out], are transposed at load time; c_attn's columns are already q | k | v.
- Falcon (FalconModel with parallel_attn, multi_query, no biases, no ALiBi): h[0] = E[ids]; one LayerNorm y feeds both
  branches, x += dense(attn(y)) + dense_4h_to_h(gelu(dense_h_to_4h(y))).  query_key_value's rows are 71 q heads | one
  k head | one v head of 64; rotate-half rotary embedding on q and k (``mer_rope_hd_f16``), positions restarting at every
  sentence; every query head attends to the one k / v head (``mer_causal_mqa_attention_f16``); erf-GELU MLP
  (``MER_EPI_GELU``).  Hidden 4544 = 71 x 64 is not a multiple of the GEMM's 128-column tiles, so the CUDA backend keeps
  the residual stream, the readout and the LayerNorm output in rows padded to a multiple of 128 columns (zero pad columns,
  ``mer_layernorm_ld_f16``) and zero-pads the output rows of query_key_value, dense and dense_4h_to_h when it packs them.
``CudaOps``: fp16 weights and GEMM operands, fp32 biases, residual stream and readout, ``mer_layernorm_f16`` (for GPT-2
too, whose reference run is fp32: its features are saved as float32).
``TorchOps``: plain torch in HF's order of operations on unpadded weights (CPU tests, tests/test_ln_decoder_text.py,
tests/test_falcon_text.py).
"""
from __future__ import annotations

import math
import re

import numpy as np
import torch

from .common import stream_fp16_weights
from .llama_text import HEAD_DIM, rope_tables, rope_theta
from .packed_text import DeviceOps, PackedTextEncoder

OPT_POS_OFFSET = 2  # OPTLearnedPositionalEmbedding: position p reads row p + 2
GPT2_HEAD_DIMS = (64, 96, 128)  # the instances of mer_causal_attention_hd_f16
GPT2_CONV1D = ("attn.c_attn.weight", "attn.c_proj.weight", "mlp.c_fc.weight", "mlp.c_proj.weight")  # [in, out]
FALCON_HEAD_DIM = 64  # the instance of mer_causal_mqa_attention_f16
REFINEDWEB_TYPES = ("RefinedWebModel", "RefinedWeb")


# ---- configs --------------------------------------------------------------------------------------------------------
def _head_check(family, heads, hidden):
    if heads * HEAD_DIM != hidden:
        raise ValueError(f"{family} path: head_dim {hidden // heads} with {heads} heads and hidden {hidden} "
                         f"(head_dim 128 only)")


def refuse_refinedweb(model_type):
    """The first Falcon checkpoints name their model_type RefinedWebModel / RefinedWeb and ship their own model code.
    The reference's plain AutoModel call (no trust_remote_code) cannot load them, so neither does this path."""
    if model_type in REFINEDWEB_TYPES:
        raise ValueError(f"Falcon path: model_type {model_type!r} is the legacy remote-code Falcon checkpoint format; "
                         f"only model_type 'falcon' checkpoints (FalconModel of transformers) are supported")


def _rope_type(cfg):
    rope = getattr(cfg, "rope_parameters", None) or getattr(cfg, "rope_scaling", None) or {}
    return rope.get("rope_type", rope.get("type", "default")), rope


def check_ln_decoder_config(cfg):
    """Reject, before any weight is read, every BLOOM / OPT / GPT-2 / Falcon config this path does not compute exactly."""
    refuse_refinedweb(cfg.model_type)
    if cfg.model_type == "bloom":
        if getattr(cfg, "apply_residual_connection_post_layernorm", False):
            raise ValueError("BLOOM path: apply_residual_connection_post_layernorm is not supported")
        if getattr(cfg, "slow_but_exact", False) and getattr(cfg, "pretraining_tp", 1) > 1:
            raise ValueError("BLOOM path: slow_but_exact with pretraining_tp > 1 is not supported")
        _head_check("BLOOM", cfg.num_attention_heads, cfg.hidden_size)
    elif cfg.model_type == "opt":
        if not getattr(cfg, "do_layer_norm_before", True):
            raise ValueError("OPT path: do_layer_norm_before=False (post-LN OPT-350m) is not supported")
        if getattr(cfg, "word_embed_proj_dim", cfg.hidden_size) != cfg.hidden_size:
            raise ValueError(f"OPT path: word_embed_proj_dim {cfg.word_embed_proj_dim} != hidden_size "
                             f"{cfg.hidden_size} (project_in / project_out) is not supported")
        if not getattr(cfg, "enable_bias", True):
            raise ValueError("OPT path: enable_bias=False is not supported")
        if not getattr(cfg, "layer_norm_elementwise_affine", True):
            raise ValueError("OPT path: a non-affine LayerNorm (layer_norm_elementwise_affine=False) is not supported")
        if getattr(cfg, "_remove_final_layer_norm", False):
            raise ValueError("OPT path: _remove_final_layer_norm is not supported")
        if getattr(cfg, "activation_function", "relu") != "relu":
            raise ValueError(f"OPT path: activation_function {cfg.activation_function!r} is not supported (relu only)")
        _head_check("OPT", cfg.num_attention_heads, cfg.hidden_size)
    elif cfg.model_type == "gpt2":
        act = getattr(cfg, "activation_function", "gelu_new")
        if act not in ("gelu_new", "gelu_pytorch_tanh"):
            raise ValueError(f"GPT-2 path: activation_function {act!r} is not supported (tanh GELU only)")
        if not getattr(cfg, "scale_attn_weights", True):
            raise ValueError("GPT-2 path: scale_attn_weights=False is not supported")
        if getattr(cfg, "scale_attn_by_inverse_layer_idx", False):
            raise ValueError("GPT-2 path: scale_attn_by_inverse_layer_idx=True is not supported")
        if getattr(cfg, "add_cross_attention", False):
            raise ValueError("GPT-2 path: add_cross_attention=True is not supported")
        hidden, heads = cfg.hidden_size, cfg.num_attention_heads
        if hidden % heads or hidden // heads not in GPT2_HEAD_DIMS:
            raise ValueError(f"GPT-2 path: head_dim {hidden / heads:g} with {heads} heads and hidden {hidden} "
                             f"(head_dim 64, 96 or 128 only)")
        if hidden % 256:
            raise ValueError(f"GPT-2 path: hidden size {hidden} is not a multiple of 256 (mer_layernorm_f16)")
        if (cfg.n_inner or 4 * hidden) % 128:
            raise ValueError(f"GPT-2 path: n_inner {cfg.n_inner} is not a multiple of 128")
    elif cfg.model_type == "falcon":
        if getattr(cfg, "new_decoder_architecture", False):
            raise ValueError("Falcon path: new_decoder_architecture (Falcon-40B / 180B layout) is not supported")
        if getattr(cfg, "alibi", False):
            raise ValueError("Falcon path: alibi=True is not supported (rotary embedding only)")
        if not getattr(cfg, "parallel_attn", True):
            raise ValueError("Falcon path: parallel_attn=False is not supported")
        if not getattr(cfg, "multi_query", True):
            raise ValueError(f"Falcon path: multi_query=False ({getattr(cfg, 'num_kv_heads', None)} K / V heads) is not "
                             f"supported (one K / V head only)")
        if getattr(cfg, "bias", False):
            raise ValueError("Falcon path: bias=True is not supported")
        if getattr(cfg, "activation", "gelu") != "gelu":
            raise ValueError(f"Falcon path: activation {cfg.activation!r} is not supported (erf gelu only)")
        hidden, heads = cfg.hidden_size, cfg.num_attention_heads
        if hidden % heads or hidden // heads != FALCON_HEAD_DIM:
            raise ValueError(f"Falcon path: head_dim {hidden / heads:g} with {heads} heads and hidden {hidden} "
                             f"(head_dim 64 only)")
        rtype, rope = _rope_type(cfg)
        if rtype != "default" or set(rope) - {"rope_type", "rope_theta"}:
            raise ValueError(f"Falcon path: only the default rotary embedding is supported, got {rope}")
        if hidden % 64:
            raise ValueError(f"Falcon path: hidden size {hidden} is not a multiple of 64 (mer_layernorm_ld_f16)")
        if _falcon_ffn(cfg) % 128:
            raise ValueError(f"Falcon path: ffn_hidden_size {_falcon_ffn(cfg)} is not a multiple of 128")
    else:
        raise ValueError(f"not a BLOOM / OPT / GPT-2 / Falcon config: model_type {cfg.model_type!r}")


def _falcon_ffn(cfg):
    return getattr(cfg, "ffn_hidden_size", None) or 4 * cfg.hidden_size


def alibi_slopes(heads):
    """fp32 [heads]: the per-head ALiBi slopes of HF build_alibi_tensor, bit for bit.  For a head count that is not a
    power of two, the largest power of two below it gets the geometric sequence and the remaining heads take every
    other term of the sequence for twice that count."""
    p2 = 2 ** math.floor(math.log2(heads))
    base = torch.tensor(2 ** (-(2 ** -(math.log2(p2) - 3))), dtype=torch.float32)
    slopes = torch.pow(base, torch.arange(1, 1 + p2, dtype=torch.int32))
    if p2 != heads:
        extra = torch.tensor(2 ** (-(2 ** -(math.log2(2 * p2) - 3))), dtype=torch.float32)
        n = min(p2, heads - p2)
        slopes = torch.cat([slopes, torch.pow(extra, torch.arange(1, 1 + 2 * n, 2, dtype=torch.int32))])
    return slopes


# ---- streaming checkpoint loader ------------------------------------------------------------------------------------
def _strip(k, family):
    """Parameter name of BloomModel / GPT2Model / FalconModel (``h.0...``) / of OPTModel.decoder (``layers.0...``), or
    None to drop: lm_head, and the causal-mask buffers ``h.*.attn.bias`` / ``h.*.attn.masked_bias`` of older GPT-2 checkpoints."""
    if k.startswith("lm_head."):
        return None
    for p in (("model.", "decoder.") if family == "opt" else ("transformer.",)):
        if k.startswith(p):
            k = k[len(p):]
    if family == "gpt2" and re.fullmatch(r"h\.\d+\.attn\.(bias|masked_bias)", k):
        return None
    return k


def load_ln_decoder_weights(model_dir, device, family):
    """{name: fp16 tensor on ``device``} of a BLOOM (``family="bloom"``), OPT (``"opt"``), GPT-2 (``"gpt2"``) or
    Falcon (``"falcon"``) checkpoint, read one tensor at a time from safetensors or ``.bin`` shards (fp32 / fp16 / bf16).
    Names lose the ``transformer.`` (BloomForCausalLM, GPT2LMHeadModel, FalconForCausalLM) or ``model.`` / ``decoder.`` (OPTForCausalLM / OPTModel)
    prefixes; ``lm_head`` and GPT-2's mask buffers are dropped.  GPT-2's Conv1D weights (GPT2_CONV1D, stored [in, out])
    are transposed to the [out, in] of the other families.  A value that is not finite in fp16 is refused."""
    out = {}
    for k, t in stream_fp16_weights(model_dir, device, lambda k: _strip(k, family)):
        out[k] = t.t().contiguous() if family == "gpt2" and k.endswith(GPT2_CONV1D) else t
    return out


def deinterleave_qkv(t, heads, head_dim=HEAD_DIM):
    """Fused projection rows interleaved per head as [head][q, k, v][head_dim] (BLOOM's query_key_value, head_dim 128;
    DeBERTa's in_proj, 64), weight [3 D, D] or bias [3 D] -> q | k | v blocks."""
    shape = t.shape
    return t.reshape(heads, 3, head_dim, *shape[1:]).transpose(0, 1).reshape(shape).contiguous()


# ---- layer orchestration --------------------------------------------------------------------------------------------
class LnDecoderNet:
    """Backend-agnostic BloomModel / OPTModel.decoder / GPT2Model / FalconModel forward over packed sentences.  ``sd``:
    {name: tensor} as load_ln_decoder_weights names and lays them out; entries are popped as the backend takes them over.
    ``family``: "bloom", "opt", "gpt2" or "falcon".  ``ops``: weight, vector, embedding, embed, batch, layernorm,
    attention, linear_res, mlp, zeros_like, add_, and for Falcon falcon_embedding, falcon_qkv, falcon_out, mqa_attention,
    parallel_res.  ``theta``: Falcon's rotary base."""

    def __init__(self, sd, ops, family, n_layers, heads, eps, max_pos=None, theta=10000.0):
        assert family in ("bloom", "opt", "gpt2", "falcon") and n_layers >= 3, (family, n_layers)
        self.ops, self.family, self.n_layers, self.heads, self.eps, self.max_pos = ops, family, n_layers, heads, eps, max_pos
        self.layers = []
        if family == "falcon":
            assert max_pos is not None, "the rotary tables need max_position_embeddings"
            E = sd.pop("word_embeddings.weight")
            self.hidden = E.shape[1]
            self.embed = ops.falcon_embedding(E)
            self.emb_ln = self.pos = self.slopes = None
            self.cos, self.sin = (ops.vector(t) for t in rope_tables(max_pos, theta, self.hidden // heads))
            for i in range(n_layers):
                p = f"h.{i}."
                a, m = p + "self_attention.", p + "mlp."
                self.layers.append(dict(
                    ln1=(ops.vector(sd.pop(p + "input_layernorm.weight")), ops.vector(sd.pop(p + "input_layernorm.bias"))),
                    qkv=ops.falcon_qkv(sd.pop(a + "query_key_value.weight"), heads),
                    o=ops.falcon_out(sd.pop(a + "dense.weight")),
                    up=ops.weight(sd.pop(m + "dense_h_to_4h.weight")),
                    down=ops.falcon_out(sd.pop(m + "dense_4h_to_h.weight"))))
            self.ln_f = (ops.vector(sd.pop("ln_f.weight")), ops.vector(sd.pop("ln_f.bias")))
            self.act = "gelu"
        elif family == "bloom":
            self.embed = ops.embedding(sd.pop("word_embeddings.weight"))
            self.emb_ln = (ops.vector(sd.pop("word_embeddings_layernorm.weight")),
                           ops.vector(sd.pop("word_embeddings_layernorm.bias")))
            self.pos = None
            self.slopes = ops.vector(alibi_slopes(heads))
            for i in range(n_layers):
                p = f"h.{i}."
                a, m = p + "self_attention.", p + "mlp."
                self.layers.append(dict(
                    ln1=(ops.vector(sd.pop(p + "input_layernorm.weight")), ops.vector(sd.pop(p + "input_layernorm.bias"))),
                    qkv=ops.weight(deinterleave_qkv(sd.pop(a + "query_key_value.weight"), heads)),
                    b_qkv=ops.vector(deinterleave_qkv(sd.pop(a + "query_key_value.bias"), heads)),
                    o=ops.weight(sd.pop(a + "dense.weight")), b_o=ops.vector(sd.pop(a + "dense.bias")),
                    ln2=(ops.vector(sd.pop(p + "post_attention_layernorm.weight")),
                         ops.vector(sd.pop(p + "post_attention_layernorm.bias"))),
                    up=ops.weight(sd.pop(m + "dense_h_to_4h.weight")), b_up=ops.vector(sd.pop(m + "dense_h_to_4h.bias")),
                    down=ops.weight(sd.pop(m + "dense_4h_to_h.weight")),
                    b_down=ops.vector(sd.pop(m + "dense_4h_to_h.bias"))))
            self.ln_f = (ops.vector(sd.pop("ln_f.weight")), ops.vector(sd.pop("ln_f.bias")))
            self.act = "gelu_tanh"
        elif family == "gpt2":
            self.embed = ops.embedding(sd.pop("wte.weight"))
            self.emb_ln = None
            self.pos = ops.embedding(sd.pop("wpe.weight"))
            self.slopes = None
            for i in range(n_layers):
                p = f"h.{i}."
                a, m = p + "attn.", p + "mlp."
                self.layers.append(dict(
                    ln1=(ops.vector(sd.pop(p + "ln_1.weight")), ops.vector(sd.pop(p + "ln_1.bias"))),
                    qkv=ops.weight(sd.pop(a + "c_attn.weight")), b_qkv=ops.vector(sd.pop(a + "c_attn.bias")),
                    o=ops.weight(sd.pop(a + "c_proj.weight")), b_o=ops.vector(sd.pop(a + "c_proj.bias")),
                    ln2=(ops.vector(sd.pop(p + "ln_2.weight")), ops.vector(sd.pop(p + "ln_2.bias"))),
                    up=ops.weight(sd.pop(m + "c_fc.weight")), b_up=ops.vector(sd.pop(m + "c_fc.bias")),
                    down=ops.weight(sd.pop(m + "c_proj.weight")), b_down=ops.vector(sd.pop(m + "c_proj.bias"))))
            self.ln_f = (ops.vector(sd.pop("ln_f.weight")), ops.vector(sd.pop("ln_f.bias")))
            self.act = "gelu_tanh"
        else:
            self.embed = ops.embedding(sd.pop("embed_tokens.weight"))
            self.emb_ln = None
            self.pos = ops.embedding(sd.pop("embed_positions.weight"))
            self.slopes = None
            for i in range(n_layers):
                p = f"layers.{i}."
                a = p + "self_attn."
                self.layers.append(dict(
                    ln1=(ops.vector(sd.pop(p + "self_attn_layer_norm.weight")),
                         ops.vector(sd.pop(p + "self_attn_layer_norm.bias"))),
                    qkv=ops.weight(torch.cat([sd.pop(a + f"{n}_proj.weight") for n in "qkv"], 0)),
                    b_qkv=ops.vector(torch.cat([sd.pop(a + f"{n}_proj.bias") for n in "qkv"], 0)),
                    o=ops.weight(sd.pop(a + "out_proj.weight")), b_o=ops.vector(sd.pop(a + "out_proj.bias")),
                    ln2=(ops.vector(sd.pop(p + "final_layer_norm.weight")), ops.vector(sd.pop(p + "final_layer_norm.bias"))),
                    up=ops.weight(sd.pop(p + "fc1.weight")), b_up=ops.vector(sd.pop(p + "fc1.bias")),
                    down=ops.weight(sd.pop(p + "fc2.weight")), b_down=ops.vector(sd.pop(p + "fc2.bias"))))
            self.ln_f = (ops.vector(sd.pop("final_layer_norm.weight")), ops.vector(sd.pop("final_layer_norm.bias")))
            self.act = "relu"
        if family != "falcon":
            self.hidden = self.embed.shape[1]
        assert not any(k.startswith(("h.", "layers.")) for k in sd), f"unused layer weights: {sorted(sd)[:4]}"

    def forward(self, ids, lens, return_hidden=False, token_types=None):
        """ids: int64 [tokens] of packed sentences with lengths ``lens``; token_types: None or int64 [tokens] (GPT-2 adds
        wte[token_types], as GPT2Model does when it is passed token_type_ids).  Returns the readout
        h[L-3] + h[L-2] + h[L-1] + ln_f(h[L]) [tokens, hidden] (fp32 on the CUDA backend) and, with return_hidden, the HF
        hidden_states tuple as a list."""
        ops, n = self.ops, self.n_layers
        if self.max_pos is not None and max(lens) > self.max_pos:
            raise ValueError(f"a sentence of {max(lens)} tokens exceeds max_position_embeddings {self.max_pos}")
        b = ops.batch(lens)
        assert token_types is None or self.family == "gpt2", "token types are a GPT-2 input"
        if self.family == "bloom":
            x = ops.layernorm(ops.embed(self.embed, ids), *self.emb_ln, self.eps, out="f32")
        elif self.family == "falcon":
            x = ops.embed(self.embed, ids)
        else:
            pos = np.concatenate([np.arange(m) for m in lens]) + (OPT_POS_OFFSET if self.family == "opt" else 0)
            x = ops.embed(self.embed, ids) + ops.embed(self.pos, pos)
            if token_types is not None:
                x = x + ops.embed(self.embed, token_types)
        hs = [x.clone()] if return_hidden else None
        acc = ops.zeros_like(x)
        for i, L in enumerate(self.layers):
            if i == n - 3:            # h[0] (the embedding) when n == 3
                ops.add_(acc, x)
            y = ops.layernorm(x, *L["ln1"], self.eps)
            if self.family == "falcon":   # parallel attention: one LayerNorm output feeds both branches
                ctx = ops.mqa_attention(y, L["qkv"], b, self.heads, self.cos, self.sin)
                x = ops.parallel_res(ctx, L["o"], ops.mlp(y, L["up"], None, self.act), L["down"], x)
            else:
                ctx = ops.attention(y, L["qkv"], L["b_qkv"], b, self.heads, self.slopes)
                x = ops.linear_res(ctx, L["o"], L["b_o"], x)
                y = ops.layernorm(x, *L["ln2"], self.eps)
                x = ops.linear_res(ops.mlp(y, L["up"], L["b_up"], self.act), L["down"], L["b_down"], x)
            if n - 3 <= i < n - 1:
                ops.add_(acc, x)
            if return_hidden and i < n - 1:
                hs.append(x.clone())
        ops.layernorm(x, *self.ln_f, self.eps, acc=acc)
        if return_hidden:
            hs.append(ops.layernorm(x, *self.ln_f, self.eps, acc=ops.zeros_like(x)))
        return (acc, hs) if return_hidden else acc


class TorchOps:
    """Plain torch backend (CPU tests, fp32 by default): the same orchestration on torch operators, HF's order of
    operations (BloomAttention: baddbmm of alibi and q k^T / sqrt(128); OPTAttention: q scaled before the product;
    GPT2Attention scales the product instead, a rounding difference only)."""

    def __init__(self, device="cpu", dtype=torch.float32):
        self.device, self.dtype = torch.device(device), dtype

    def weight(self, t):
        return t.to(self.device, self.dtype)

    vector = embedding = falcon_embedding = falcon_out = weight

    def falcon_qkv(self, w, heads):
        return self.weight(w)

    def embed(self, table, ids):
        return table[torch.as_tensor(ids, device=self.device)]

    def zeros_like(self, x):
        return torch.zeros_like(x)

    def add_(self, acc, x):
        acc += x

    def batch(self, lens):
        return list(lens)

    def layernorm(self, x, g, b, eps, out="f16", acc=None):
        y = torch.nn.functional.layer_norm(x, (x.shape[-1],), g, b, eps)
        if acc is not None:
            acc += y
            return acc
        return y

    def attention(self, y, w_qkv, b_qkv, lens, heads, slopes):
        D = w_qkv.shape[0] // 3
        hd = D // heads
        qkv = y @ w_qkv.T + b_qkv
        ctx = torch.empty(y.shape[0], D, dtype=y.dtype, device=y.device)
        o = 0
        for n in lens:
            q, k, v = (qkv[o:o + n, i * D:(i + 1) * D].view(n, heads, hd).transpose(0, 1) for i in range(3))
            if slopes is not None:   # BLOOM: alibi.baddbmm(q, k^T, beta=1, alpha=1/sqrt(128)), alibi = slope * j
                alibi = slopes[:, None, None] * torch.arange(n, device=y.device, dtype=slopes.dtype)[None, None, :]
                sc = alibi.to(y.dtype) + (q @ k.transpose(1, 2)) * hd ** -0.5
            else:                    # OPT / GPT-2: (q * 1/sqrt(head_dim)) k^T
                sc = (q * hd ** -0.5) @ k.transpose(1, 2)
            sc = sc.masked_fill(torch.ones(n, n, dtype=torch.bool, device=y.device).triu(1), float("-inf"))
            p = torch.softmax(sc.to(torch.promote_types(sc.dtype, torch.float32)), dim=-1).to(y.dtype)
            ctx[o:o + n] = (p @ v).transpose(0, 1).reshape(n, D)
            o += n
        return ctx

    def mqa_attention(self, y, w_qkv, lens, heads, cos, sin):
        """FalconAttention (multi_query): q | k | v = y W^T with rows heads x hd | hd | hd, rotate-half rotary on q and
        k at positions 0 .. n-1 of each sentence, causal softmax(q k^T / sqrt(hd)) v with the one k / v head shared."""
        hd = w_qkv.shape[0] // (heads + 2)
        qkv = y @ w_qkv.T
        ctx = torch.empty(y.shape[0], heads * hd, dtype=y.dtype, device=y.device)
        rot = lambda t: torch.cat([-t[..., hd // 2:], t[..., :hd // 2]], -1)  # noqa: E731
        o = 0
        for n in lens:
            blk = qkv[o:o + n].view(n, heads + 2, hd).transpose(0, 1)            # [heads + 2, n, hd]
            c, s = (torch.cat([t[:n], t[:n]], -1).to(y.dtype) for t in (cos, sin))
            q, k, v = blk[:heads], blk[heads:heads + 1], blk[heads + 1:]
            q, k = q * c + rot(q) * s, k * c + rot(k) * s
            sc = (q @ k.transpose(1, 2)) * hd ** -0.5
            sc = sc.masked_fill(torch.ones(n, n, dtype=torch.bool, device=y.device).triu(1), float("-inf"))
            p = torch.softmax(sc.to(torch.promote_types(sc.dtype, torch.float32)), dim=-1).to(y.dtype)
            ctx[o:o + n] = (p @ v).transpose(0, 1).reshape(n, heads * hd)
            o += n
        return ctx

    def parallel_res(self, ctx, w_o, h, w_down, x):
        """FalconDecoderLayer with parallel_attn: (mlp + attn) + residual, in HF's order."""
        return x + (h @ w_down.T + ctx @ w_o.T)

    def linear_res(self, a, w, b, x):
        return x + (a @ w.T + b)

    def mlp(self, y, w, b, act):
        h = y @ w.T if b is None else y @ w.T + b
        if act == "relu":
            return torch.relu(h)
        if act == "gelu":
            return torch.nn.functional.gelu(h)
        return h * 0.5 * (1.0 + torch.tanh(0.79788456 * h * (1 + 0.044715 * h * h)))


class CudaOps(DeviceOps):
    """Product backend: fp16 weights and GEMM operands (MER_GEMM_F16) with fp32 biases, fp32 residual stream; every op
    is one or two libmer_b200.so launches.  ``timing``: see DeviceOps."""

    embedding = DeviceOps.weight

    def __init__(self, device="cuda"):
        import ctypes as C
        super().__init__("f16", device)
        L = self.L
        vp, i32, i64, f32 = C.c_void_p, C.c_int, C.c_longlong, C.c_float
        self._ln = L.declare("mer_layernorm_f16", [vp, vp, vp, vp, vp, vp, i64, i32, f32, vp])
        self._att = L.declare("mer_causal_attention_hd_f16", [vp, vp, i64, vp, vp, i32, i64, i32, i32, i32, vp])
        self._att_alibi = L.declare("mer_causal_alibi_attention_f16", [vp, vp, i64, vp, vp, i32, i64, i32, i32, vp, vp])
        self._ln_ld = L.declare("mer_layernorm_ld_f16", [vp, i64, vp, vp, vp, vp, vp, i64, i32, f32, vp])
        self._rope = L.declare("mer_rope_hd_f16", [vp, i64, i64, i32, i32, vp, i32, vp, vp, vp, i32, vp])
        self._att_mqa = L.declare("mer_causal_mqa_attention_f16", [vp, i64, vp, i64, vp, vp, i32, i64, i32, i32, vp])

    # ---- Falcon: hidden-wide rows padded to a multiple of 128 columns (mer_gemm's N), pad columns zero ----
    def falcon_embedding(self, t):
        """[vocab, hidden] -> fp16 [vocab, pad128(hidden)]: the gathered residual rows are born padded."""
        return self.weight(torch.nn.functional.pad(t, (0, _pad128(t.shape[1]) - t.shape[1])))

    def falcon_out(self, w):
        """dense / dense_4h_to_h [hidden, K] -> fp16 [pad128(hidden), K]: zero rows add nothing to the pad columns."""
        return self.weight(torch.nn.functional.pad(w, (0, 0, 0, _pad128(w.shape[0]) - w.shape[0])))

    def falcon_qkv(self, w, heads):
        """query_key_value [(heads + 2) hd, hidden] -> (fp16 [N, hidden], vt_col0): rows q (heads x hd) | k (hd) | zero
        rows | v (hd) with N = pad128((heads + 2) hd) and v in the last hd rows, so that the GEMM's V^T side output
        (columns vt_col0 = N - hd on) is exactly V^T."""
        hd = w.shape[0] // (heads + 2)
        qk = (heads + 1) * hd
        n = _pad128(qk + hd)
        out = torch.zeros(n, w.shape[1], dtype=w.dtype, device=w.device)
        out[:qk], out[n - hd:] = w[:qk], w[qk:]
        return self.weight(out), n - hd

    def mqa_attention(self, y, w_qkv, b, heads, cos, sin):
        """y: fp16 [T, pad128(hidden)] (first hidden columns valid) -> ctx fp16 [T, hidden]."""
        L, T = self.L, y.shape[0]
        w, vt_col0 = w_qkv
        n, hd = w.shape[0], w.shape[0] - vt_col0
        qkv = torch.empty(T, n, dtype=torch.float16, device=self.device)          # q | k rows (other columns unused)
        vt = torch.empty(hd, (T + 7) // 8 * 8, dtype=torch.float16, device=self.device)
        self._run("gemm", lambda: L.gemm(y, w, qkv, mode=L.MER_GEMM_F16, f16_out=True, vt=vt, vt_col0=vt_col0,
                                         a_row_stride=y.shape[1]))
        self._run("rope", lambda: L.check(self._rope(L.ptr(qkv), n, T, heads + 1, hd, L.ptr(b["cu"]), b["n"], None,
                                                     L.ptr(cos), L.ptr(sin), cos.shape[0], L.stream_ptr())))
        ctx = torch.empty(T, heads * hd, dtype=torch.float16, device=self.device)
        self._run("attention", lambda: L.check(self._att_mqa(L.ptr(qkv), n, L.ptr(vt), vt.shape[1], L.ptr(ctx),
                                                             L.ptr(b["cu"]), b["n"], T, b["max_len"], heads,
                                                             L.stream_ptr())))
        return ctx

    def parallel_res(self, ctx, w_o, h, w_down, x):
        """x += dense(ctx), then x += dense_4h_to_h(h), both in the GEMM's residual epilogue (HF adds mlp + attn first:
        a rounding difference only)."""
        self._run("gemm", lambda: self.L.gemm(ctx, w_o, x, res=x, mode=self.L.MER_GEMM_F16))
        self._run("gemm", lambda: self.L.gemm(h, w_down, x, res=x, mode=self.L.MER_GEMM_F16))
        return x

    def layernorm(self, x, g, b, eps, out="f16", acc=None):
        """out "f16": a new fp16 operand; "f32": a new fp32 row block; with acc: acc += y, returns acc.  Rows wider
        than gamma (Falcon's padded rows) are normalised over their first len(gamma) columns, outputs of the same
        pitch."""
        L = self.L
        y16 = y32 = None
        if acc is None:
            if out == "f16":
                y16 = torch.empty(x.shape, dtype=torch.float16, device=self.device)
            else:
                y32 = torch.empty(x.shape, dtype=torch.float32, device=self.device)
        if x.shape[1] != g.shape[0]:
            self._run("layernorm", lambda: L.check(self._ln_ld(L.ptr(x), x.shape[1], L.ptr(g), L.ptr(b), L.ptr(y16),
                                                               L.ptr(y32), L.ptr(acc), x.shape[0], g.shape[0], eps,
                                                               L.stream_ptr())))
        else:
            self._run("layernorm", lambda: L.check(self._ln(L.ptr(x), L.ptr(g), L.ptr(b), L.ptr(y16), L.ptr(y32),
                                                            L.ptr(acc), x.shape[0], x.shape[1], eps, L.stream_ptr())))
        return acc if acc is not None else (y16 if y16 is not None else y32)

    def attention(self, y, w_qkv, b_qkv, b, heads, slopes):
        L, T, D = self.L, y.shape[0], w_qkv.shape[0] // 3
        qkv = torch.empty(T, 3 * D, dtype=torch.float16, device=self.device)     # q | k rows (V columns unused)
        vt = torch.empty(D, (T + 7) // 8 * 8, dtype=torch.float16, device=self.device)
        self._run("gemm", lambda: L.gemm(y, w_qkv, qkv, bias=b_qkv, mode=L.MER_GEMM_F16, f16_out=True, vt=vt,
                                         vt_col0=2 * D))
        ctx = torch.empty(T, D, dtype=torch.float16, device=self.device)
        args = (L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(ctx), L.ptr(b["cu"]), b["n"], T, b["max_len"], heads)
        if slopes is not None:
            self._run("attention", lambda: L.check(self._att_alibi(*args, L.ptr(slopes), L.stream_ptr())))
        else:  # OPT scales q by 1/sqrt(128) before q k^T; the kernel scales the product: a rounding difference only
            self._run("attention", lambda: L.check(self._att(*args, D // heads, L.stream_ptr())))
        return ctx

    def mlp(self, y, w, bias, act):
        """act "gelu" (Falcon, erf form, no bias): y may be padded rows, the GEMM reads their first w.shape[1]
        columns."""
        L, T = self.L, y.shape[0]
        h = torch.empty(T, w.shape[0], dtype=torch.float16, device=self.device)
        self._run("gemm", lambda: L.gemm(y, w, h, bias=bias, mode=L.MER_GEMM_F16, f16_out=True, a_row_stride=y.shape[1],
                                         relu=(act == "relu"), gelu_tanh=(act == "gelu_tanh"), gelu=(act == "gelu")))
        return h


def _pad128(n):
    return (n + 127) // 128 * 128


def activation_bytes_per_token(hidden, ffn, family=None):
    """Device bytes one token of a packed pass holds at the peak of a layer: fp32 residual, readout and embedding
    gather, fp16 operands, q | k | v rows and V^T, ctx, and the fp16 FFN activation.  Falcon: padded fp32 rows and
    LayerNorm output, the padded QKV rows and one 64-row V^T."""
    if family == "falcon":
        w = _pad128(hidden)
        return w * (4 + 4 + 4 + 2) + (w + 128) * 2 + 64 * 2 + hidden * 2 + ffn * 2
    return hidden * (4 + 4 + 4 + 2 + 3 * 2 + 2 + 2) + ffn * 2


def net_dims(cfg):
    """(family, layers, heads, hidden, ffn, eps, max_pos) of a BLOOM / OPT / GPT-2 / Falcon config."""
    if cfg.model_type == "falcon":
        return ("falcon", cfg.num_hidden_layers, cfg.num_attention_heads, cfg.hidden_size, _falcon_ffn(cfg),
                float(cfg.layer_norm_epsilon), int(cfg.max_position_embeddings))
    if cfg.model_type == "bloom":
        return ("bloom", cfg.num_hidden_layers, cfg.num_attention_heads, cfg.hidden_size, 4 * cfg.hidden_size,
                float(cfg.layer_norm_epsilon), None)
    if cfg.model_type == "gpt2":
        return ("gpt2", cfg.n_layer, cfg.n_head, cfg.n_embd, cfg.n_inner or 4 * cfg.n_embd,
                float(cfg.layer_norm_epsilon), int(cfg.n_positions))
    return ("opt", cfg.num_hidden_layers, cfg.num_attention_heads, cfg.hidden_size, cfg.ffn_dim, 1e-5,
            int(cfg.max_position_embeddings))


class LnDecoderTextEncoder(PackedTextEncoder):
    """PackedTextEncoder over ``LnDecoderNet`` with the CUDA backend; token types are GPT-2's.  ``cfg``: the
    checkpoint's BloomConfig / OPTConfig / GPT2Config / FalconConfig; ``sd``: {name: tensor} (load_ln_decoder_weights)."""

    takes_token_types = True

    def __init__(self, sd, cfg, device="cuda"):
        check_ln_decoder_config(cfg)
        family, layers, heads, hidden, ffn, eps, self.max_pos = net_dims(cfg)
        self.ops = CudaOps(device)
        self.device = self.ops.device
        theta = rope_theta(cfg) if family == "falcon" else None
        self.net = LnDecoderNet(sd, self.ops, family, layers, heads, eps, self.max_pos, theta=theta)
        self.hidden, self.vocab_size = self.net.hidden, self.net.embed.shape[0]
        self.bytes_per_token = activation_bytes_per_token(hidden, ffn, family)
