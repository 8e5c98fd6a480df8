"""XLNet branch of the text extractor: ``chinese-xlnet-base``, ``xlnet-base-cased`` and ``xlnet-large-cased``
(MERBench/feature_extraction/text/extract_text_huggingface.py, the AutoModel + AutoTokenizer(use_fast=False) branch),
run by the reference in fp32, one sentence per forward.  Readout as for every text model: the sum of the last four
hidden states, where hidden state 0 is the raw word embedding (no positions, no LayerNorm).

XLNet (HF XLNetModel, attn_type "bi", content stream only) is a post-LN encoder with Transformer-XL relative attention:

    score[i, j] = ((q_i + r_w_bias) . k_j + (q_i + r_r_bias) . R[row(i - j)] + (q_i + r_s_bias) . seg_embed[s_ij]) / 8

- R: per layer, the sinusoidal rows pos_emb(d) = [sin(d inv_freq), cos(d inv_freq)] (float32, inv_freq =
  1 / 10000^(arange(0, d_model, 2) / d_model)) projected by the layer's ``r``; ``rel_table`` builds the rows and the
  distance -> row map, which is how clamp_len > 0 clamps the distance.  pos_emb does not depend on the layer, so the
  CUDA path projects it for every layer in one GEMM.
- s_ij = (token_type_i != token_type_j), one-hot over seg_embed; the term exists only when the model is called with
  token_type_ids, i.e. when the tokenizer's output carries them (``XlnetTextExtractor`` forwards them).
- q, k, v, o, r are [d_model, heads, 64] without bias; h = LN(h + o(attn)); h = LN(h + W2 act(W1 h + b1) + b2), act
  gelu (erf) or relu.

``XlnetNet`` is the orchestration over an ``ops`` backend, as in deberta_text.py: ``TorchOps`` is plain torch in HF's
order of operations (CPU tests, the restatement the GPU tests compare against), ``CudaOps`` runs every op as
libmer_b200.so launches: ``mer_gemm``, ``mer_layernorm``, ``mer_xlnet_attention``.  Operand format: BertEncoder's rule
and its MER_TEXT_PRECISION variable, "f16" at hidden 768 (fp16 operands and attention), "bf16x3" above (split-bf16 GEMM
operands, tf32 q | k | V^T and R in the attention); fp32 residual stream and readout in both.
"""
from __future__ import annotations

import math
import os

import numpy as np
import torch

from .deberta_text import LN_DIMS, activation_bytes_per_token
from .packed_text import DeviceOps, PackedTextEncoder
from .text import TokenIds, TokenTypeTextExtractor  # noqa: F401  (TokenIds: re-exported)

HEAD_DIM = 64
MAX_LEN = 512   # tokens per sentence the launch sizing assumes (XLNet has no max_position_embeddings)


# ---- configs --------------------------------------------------------------------------------------------------------
def check_xlnet_config(cfg):
    """Reject, before any weight is read, every XLNet config this path does not compute exactly."""
    if cfg.model_type != "xlnet":
        raise ValueError(f"not an XLNet config: model_type {cfg.model_type!r}")
    if cfg.attn_type != "bi":
        raise ValueError(f"XLNet path: attn_type {cfg.attn_type!r} is not supported (bi only)")
    if cfg.bi_data:
        raise ValueError("XLNet path: bi_data is not supported")
    if cfg.d_head != HEAD_DIM or cfg.n_head * cfg.d_head != cfg.d_model:
        raise ValueError(f"XLNet path: d_head {cfg.d_head} with {cfg.n_head} heads and d_model {cfg.d_model} "
                         "(64 only, n_head * d_head = d_model)")
    if cfg.d_model not in LN_DIMS:
        raise ValueError(f"XLNet path: d_model {cfg.d_model} (mer_layernorm rows: {LN_DIMS})")
    if cfg.ff_activation not in ("gelu", "relu"):
        raise ValueError(f"XLNet path: ff_activation {cfg.ff_activation!r} is not supported (gelu or relu)")


class XlnetDims:
    """The shape facts of an XLNetConfig the orchestration needs."""

    def __init__(self, cfg):
        self.layers, self.heads, self.hidden = cfg.n_layer, cfg.n_head, cfg.d_model
        self.ffn, self.eps = cfg.d_inner, float(cfg.layer_norm_eps)
        self.clamp_len, self.act = int(cfg.clamp_len), cfg.ff_activation


def rel_table(d_model, max_len, clamp_len=-1):
    """(pos_emb float32 [rows, d_model], int32 [2 max_len - 1]): the sinusoidal rows of the distances m .. -m in
    HF's float32 arithmetic (m = max_len - 1, or clamp_len when 0 < clamp_len < max_len - 1), and the row of distance
    d = i - j at index d + max_len - 1 (clamped to +-m)."""
    m = max_len - 1 if clamp_len <= 0 else min(clamp_len, max_len - 1)
    freq = torch.arange(0, d_model, 2.0, dtype=torch.int64).float()
    inv_freq = 1 / torch.pow(10000, (freq / d_model))
    pos = torch.arange(m, -m - 1, -1.0, dtype=torch.int64).float()      # row r holds distance m - r
    sin = torch.einsum("i,d->id", pos, inv_freq)
    table = torch.cat([torch.sin(sin), torch.cos(sin)], dim=-1)
    d = np.arange(-(max_len - 1), max_len)
    return table, (m - np.clip(d, -m, m)).astype(np.int32)


# ---- weights --------------------------------------------------------------------------------------------------------
def _strip(sd):
    """{name: tensor} of XLNetModel: a ``transformer.`` prefix dropped, the LM head and mask_emb dropped."""
    out = {}
    for k, v in sd.items():
        if k.startswith("transformer."):
            k = k[len("transformer."):]
        if k.startswith("lm_loss.") or k == "mask_emb":
            continue
        out[k] = torch.as_tensor(v)
    return out


def proj_weights(sd, prefix, d_model, heads):
    """The [d_model, heads, 64] parameters of layer ``prefix`` as GEMM weights [out, in]: q | k | v stacked
    [3 heads*64, d_model], o [d_model, heads*64] and r [heads*64, d_model]."""
    def w(n):
        return sd.pop(prefix + n).reshape(d_model, heads * HEAD_DIM)
    qkv = torch.cat([w("q").T, w("k").T, w("v").T])
    return qkv, w("o"), w("r").T


class XlnetNet:
    """Backend-agnostic XLNetModel forward over packed sentences.  ``sd``: {name: tensor} with XLNetModel names (a
    ``transformer.`` prefix is dropped, ``lm_loss.*`` / ``mask_emb`` ignored); ``dims``: XlnetDims.  ``ops``: weight,
    vector, embedding, operand, embed, batch, layernorm, rel_proj, attention, linear_res, ffn_up, zeros_like."""

    def __init__(self, sd, ops, dims):
        sd = _strip(sd)
        self.ops, self.d = ops, dims
        d, H = dims, dims.hidden
        self.word = ops.embedding(sd.pop("word_embedding.weight"))
        self.layers, w_r = [], []
        for i in range(d.layers):
            p = f"layer.{i}."
            a = p + "rel_attn."
            qkv, o, r = proj_weights(sd, a, H, d.heads)
            w_r.append(r)
            self.layers.append(dict(
                qkv=ops.weight(qkv), o=ops.weight(o),
                bias=tuple(ops.vector(sd.pop(a + n).float().contiguous())
                           for n in ("r_w_bias", "r_r_bias", "r_s_bias", "seg_embed")),
                ln1=(ops.vector(sd.pop(a + "layer_norm.weight")), ops.vector(sd.pop(a + "layer_norm.bias"))),
                up=ops.weight(sd.pop(p + "ff.layer_1.weight")), b_up=ops.vector(sd.pop(p + "ff.layer_1.bias")),
                down=ops.weight(sd.pop(p + "ff.layer_2.weight")), b_down=ops.vector(sd.pop(p + "ff.layer_2.bias")),
                ln2=(ops.vector(sd.pop(p + "ff.layer_norm.weight")), ops.vector(sd.pop(p + "ff.layer_norm.bias")))))
        self.w_r = ops.weight(torch.cat(w_r))          # [layers heads*64, d_model]: every layer's r in one GEMM
        assert not sd, f"unused weights: {sorted(sd)[:4]}"
        self.hidden = H
        self.scale = 1.0 / math.sqrt(HEAD_DIM)

    def forward(self, ids, lens, token_types=None, return_hidden=False):
        """ids: int64 [tokens] of packed sentences with lengths ``lens``; token_types: None (no segment term) or int
        [tokens].  Returns the readout (sum of hidden states n - 3 .. n, fp32 on the CUDA backend) and, with
        return_hidden, the HF hidden_states tuple as a list."""
        ops, d = self.ops, self.d
        n = d.layers
        table, rows = rel_table(d.hidden, max(lens), d.clamp_len)
        b = ops.batch(lens, rows, token_types)
        x = ops.embed(self.word, ids)                  # hs[0]: the raw word embedding
        acc = x.clone() if n <= 3 else ops.zeros_like(x)
        hs = [x.clone()] if return_hidden else None
        y = ops.operand(x)
        rel = ops.rel_proj(ops.operand(table), self.w_r, n)
        for i, L in enumerate(self.layers):
            ctx = ops.attention(y, L["qkv"], rel[i], L["bias"], b, d.heads, self.scale)
            x, y = ops.layernorm(ops.linear_res(ctx, L["o"], None, x), *L["ln1"], d.eps)
            into = acc if i + 1 >= n - 3 else None          # hidden state i + 1 is in the readout
            h = ops.linear_res(ops.ffn_up(y, L["up"], L["b_up"], d.act), L["down"], L["b_down"], x)
            x, y = ops.layernorm(h, *L["ln2"], d.eps, acc=into)
            if return_hidden:
                hs.append(x.clone())
        return (acc, hs) if return_hidden else acc


class TorchOps:
    """Plain torch backend (CPU tests, fp32 by default): the same orchestration in HF's order of operations."""

    def __init__(self, device="cpu", dtype=torch.float32):
        self.device, self.dtype = torch.device(device), dtype

    def weight(self, t):
        return torch.as_tensor(t).to(self.device, self.dtype)

    vector = embedding = operand = weight

    def embed(self, table, ids):
        return table[torch.as_tensor(ids, device=self.device)]

    def zeros_like(self, x):
        return torch.zeros_like(x)

    def batch(self, lens, rows, token_types):
        tt = None if token_types is None else torch.as_tensor(np.asarray(token_types), device=self.device).long()
        return dict(lens=list(lens), rows=torch.from_numpy(rows).long().to(self.device), max_len=max(lens), types=tt)

    def layernorm(self, x, g, b, eps, acc=None):
        y = torch.nn.functional.layer_norm(x, (x.shape[-1],), g, b, eps)
        if acc is not None:
            acc += y
        return y, y

    def rel_proj(self, table, w_r, layers):
        D = w_r.shape[0] // layers
        r = table @ w_r.T
        return [r[:, i * D:(i + 1) * D] for i in range(layers)]

    def attention(self, y, w_qkv, r, bias, b, heads, scale):
        D = heads * HEAD_DIM
        r_w, r_r, r_s, seg = bias
        qkv = y @ w_qkv.T
        kr = r.reshape(-1, heads, HEAD_DIM).transpose(0, 1)                       # [h, rows, 64]
        ctx = torch.empty(y.shape[0], D, dtype=y.dtype, device=y.device)
        o = 0
        for n in b["lens"]:
            q, k, v = (qkv[o:o + n, i * D:(i + 1) * D].view(n, heads, HEAD_DIM).transpose(0, 1) for i in range(3))
            i = torch.arange(n, device=y.device)
            row = b["rows"][(i[:, None] - i[None, :]) + b["max_len"] - 1].expand(heads, n, n)
            ac = (q + r_w[:, None]) @ k.transpose(1, 2)
            bd = torch.gather((q + r_r[:, None]) @ kr.transpose(1, 2), -1, row)
            sc = ac + bd
            if b["types"] is not None:
                t = b["types"][o:o + n]
                ef = torch.einsum("hid,shd->his", q + r_s[:, None], seg)               # [h, i, 2]
                diff = (t[:, None] != t[None, :]).long().expand(heads, n, n)
                sc = sc + torch.gather(ef, -1, diff)
            ctx[o:o + n] = (torch.softmax(sc * scale, dim=-1) @ v).transpose(0, 1).reshape(n, D)
            o += n
        return ctx

    def linear_res(self, a, w, b, x):
        y = a @ w.T
        return x + (y if b is None else y + b)

    def ffn_up(self, y, w, b, act):
        h = y @ w.T + b
        return torch.relu(h) if act == "relu" else torch.nn.functional.gelu(h)


class CudaOps(DeviceOps):
    """Product backend.  precision "f16": fp16 weights, GEMM operands, q | k | V^T and R (MER_GEMM_F16,
    MER_ATT_QKV_F16); "bf16x3": split-bf16 weights and operands (MER_GEMM_BF16X3), tf32-rounded q | k | V^T and R,
    ctx written as split rows.  fp32 biases, residual stream and readout; ``mer_layernorm`` writes the fp32 row, the
    next operand and the readout term in one pass.  ``timing``: see DeviceOps."""

    def batch(self, lens, rows, token_types):
        """DeviceOps.batch, with the distance -> table row map and the int32 token types (None: no segment term)."""
        tt = None if token_types is None else torch.as_tensor(np.asarray(token_types, np.int32), device=self.device)
        return dict(super().batch(lens), rows=torch.from_numpy(rows).to(self.device), types=tt)

    def rel_proj(self, table, w_r, layers):
        """Every layer's R = pos_emb @ r in one GEMM: [rows, layers heads*64] in the attention's operand format; layer
        i's table is the column block i (row pitch layers heads*64)."""
        out = torch.empty(table.shape[0], w_r.shape[0], dtype=self.op_dtype, device=self.device)
        self._run("gemm", lambda: self.L.gemm(table, w_r, out, mode=self.mode, f16_out=self.f16,
                                              round_out=not self.f16))
        D = w_r.shape[0] // layers
        return [out[:, i * D:(i + 1) * D] for i in range(layers)]

    def attention(self, y, w_qkv, r, bias, b, heads, scale):
        L, T, D = self.L, y.shape[0], heads * HEAD_DIM
        qkv = torch.empty(T, 3 * D, dtype=self.op_dtype, device=self.device)     # q | k rows (V columns unused)
        vt = torch.empty(D, (T + 7) // 8 * 8, dtype=self.op_dtype, device=self.device)
        self._run("gemm", lambda: L.gemm(y, w_qkv, qkv, mode=self.mode, f16_out=self.f16, round_out=not self.f16,
                                         vt=vt, vt_col0=2 * D))
        ctx = torch.empty(T, D, dtype=self.op_dtype, device=self.device)
        flags = (L.MER_ATT_QKV_F16 | L.MER_EPI_OUT_F16) if self.f16 else L.MER_EPI_SPLIT_BF16
        r_w, r_r, r_s, seg = bias
        self._run("attention", lambda: L.check(L.lib().mer_xlnet_attention(
            L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(r), r.stride(0), L.ptr(b["rows"]), L.ptr(r_w), L.ptr(r_r),
            L.ptr(r_s), L.ptr(seg), L.ptr(b["types"]), scale, L.ptr(ctx), L.ptr(b["cu"]), b["n"], T, b["max_len"],
            heads, flags, L.stream_ptr())))
        return ctx


class XlnetTextEncoder(PackedTextEncoder):
    """PackedTextEncoder over ``XlnetNet`` with the CUDA backend; token types give the segment term.  ``sd``: {name:
    tensor}; ``cfg``: the checkpoint's XLNetConfig.  ``precision``: None = MER_TEXT_PRECISION, else BertEncoder's rule
    ("f16" at hidden 768, "bf16x3" above)."""

    span = (0, -2)
    takes_token_types = True

    def __init__(self, sd, cfg, device="cuda", precision=None):
        check_xlnet_config(cfg)
        self.dims = d = XlnetDims(cfg)
        self.precision = precision or os.environ.get("MER_TEXT_PRECISION", "f16" if d.hidden == 768 else "bf16x3")
        self.ops = CudaOps(self.precision, device)
        self.device = self.ops.device
        self.net = XlnetNet(sd, self.ops, d)
        self.hidden, self.vocab_size = d.hidden, self.net.word.shape[0]
        self.bytes_per_token = activation_bytes_per_token(d.hidden, d.ffn)


XlnetTextExtractor = TokenTypeTextExtractor   # the token-type hook, under its XLNet name
