"""DeBERTa / DeBERTa-v2 branch of the text extractor: ``deberta-chinese-large`` (MERBench/feature_extraction/text/
extract_text_huggingface.py:164-166, AutoModel + BertTokenizer) and ``deberta-base``, ``deberta-large``,
``deberta-v2-xlarge``, ``deberta-v2-xxlarge`` (the AutoModel + AutoTokenizer branch), all run by the reference in fp32,
one sentence per forward (:193-231).  Readout as for every text model: the sum of the last four hidden states.

DeBERTa is a post-LN BERT-shaped encoder whose attention adds two relative-position terms (HF DisentangledSelfAttention,
pos_att_type c2p | p2c):

    score[i, j] = (q_i . k_j + q_i . PK[row(i - j)] + k_j . PQ[row(i - j)]) / sqrt(3 * 64)

- PK | PQ: per layer, the relative-position table projected once per layer (independent of the batch).  v1: pos_proj
  (no bias) | pos_q_proj of the raw table; v2: key_proj | query_proj with share_att_key (else pos_key_proj |
  pos_query_proj), applied to the LayerNorm'd table when norm_rel_ebd = "layer_norm".
- row(d) (``rel_rows``): v1 clamp(max_rel + d, 0, 2 max_rel - 1); v2 clamp(span + log_bucket(d), 0, 2 span - 1) with
  span = position_buckets (or max_rel + d without buckets).  Both c2p and p2c read that one row.
- h[0] = LayerNorm(E[ids] (+ P[pos] if position_biased_input) (+ T[0] if type_vocab_size > 0)); v2 checkpoints with a
  conv layer replace h[1] by LayerNorm(layer0_out + gelu(conv1d_k3(h[0]))), zero-padded at every sentence's edges.

``DebertaNet`` is the orchestration over an ``ops`` backend, as in ln_decoder_text.py: ``TorchOps`` is plain torch in
HF's order of operations (CPU tests, the restatement the GPU tests compare against), ``CudaOps`` runs every op as
libmer_b200.so launches: ``mer_gemm``, ``mer_layernorm``, ``mer_disentangled_attention``.  Operand format: BertEncoder's
rule and its MER_TEXT_PRECISION variable, "f16" at hidden 768 (fp16 operands and attention), "bf16x3" above (split-bf16
GEMM operands, tf32 q | k | V^T and tables in the attention); fp32 residual stream and readout in both.
"""
from __future__ import annotations

import math
import os

import numpy as np
import torch

from .ln_decoder_text import deinterleave_qkv
from .packed_text import DeviceOps, PackedTextEncoder

HEAD_DIM = 64
LN_DIMS = (512, 768, 1024, 1280, 1536)  # mer_layernorm's row widths


# ---- configs --------------------------------------------------------------------------------------------------------
def check_deberta_config(cfg):
    """Reject, before any weight is read, every DeBERTa / DeBERTa-v2 config this path does not compute exactly."""
    if cfg.model_type not in ("deberta", "deberta-v2"):
        raise ValueError(f"not a DeBERTa config: model_type {cfg.model_type!r}")
    if not getattr(cfg, "relative_attention", False):
        raise ValueError("DeBERTa path: relative_attention=False is not supported")
    pat = getattr(cfg, "pos_att_type", None) or []
    if isinstance(pat, str):
        pat = [x.strip() for x in pat.lower().split("|")]
    if sorted(pat) != ["c2p", "p2c"]:
        raise ValueError(f"DeBERTa path: pos_att_type {pat} is not supported (c2p and p2c only)")
    if getattr(cfg, "talking_head", False):
        raise ValueError("DeBERTa path: talking_head is not supported")
    head = getattr(cfg, "attention_head_size", None) or cfg.hidden_size // cfg.num_attention_heads
    if head != HEAD_DIM or cfg.num_attention_heads * HEAD_DIM != cfg.hidden_size:
        raise ValueError(f"DeBERTa path: head size {head} with {cfg.num_attention_heads} heads and hidden "
                         f"{cfg.hidden_size} (64 only)")
    if getattr(cfg, "embedding_size", cfg.hidden_size) not in (None, cfg.hidden_size):
        raise ValueError(f"DeBERTa path: embedding_size {cfg.embedding_size} != hidden_size {cfg.hidden_size} "
                         "(embed_proj) is not supported")
    if cfg.hidden_act != "gelu":
        raise ValueError(f"DeBERTa path: hidden_act {cfg.hidden_act!r} is not supported (gelu only)")
    if cfg.model_type == "deberta-v2":
        if getattr(cfg, "conv_kernel_size", 0) not in (0, 3):
            raise ValueError(f"DeBERTa path: conv_kernel_size {cfg.conv_kernel_size} is not supported (0 or 3)")
        if getattr(cfg, "conv_kernel_size", 0) > 0:
            if getattr(cfg, "conv_act", "tanh") != "gelu":
                raise ValueError(f"DeBERTa path: conv_act {getattr(cfg, 'conv_act', 'tanh')!r} is not supported "
                                 "(gelu only)")
            if getattr(cfg, "conv_groups", 1) != 1:
                raise ValueError(f"DeBERTa path: conv_groups {cfg.conv_groups} is not supported (1 only)")
        norm = [x.strip() for x in getattr(cfg, "norm_rel_ebd", "none").lower().split("|")]
        if set(norm) - {"none", "layer_norm"}:
            raise ValueError(f"DeBERTa path: norm_rel_ebd {cfg.norm_rel_ebd!r} is not supported")


class DebertaDims:
    """The shape and variant facts of a DebertaConfig / DebertaV2Config the orchestration needs."""

    def __init__(self, cfg):
        self.v2 = cfg.model_type == "deberta-v2"
        self.layers, self.heads, self.hidden = cfg.num_hidden_layers, cfg.num_attention_heads, cfg.hidden_size
        self.ffn, self.eps = cfg.intermediate_size, float(cfg.layer_norm_eps)
        mr = getattr(cfg, "max_relative_positions", -1)
        self.max_rel = mr if mr >= 1 else cfg.max_position_embeddings
        self.buckets = getattr(cfg, "position_buckets", -1) if self.v2 else -1
        self.span = self.buckets if self.buckets > 0 else self.max_rel
        self.share = self.v2 and getattr(cfg, "share_att_key", False)
        self.norm_rel = self.v2 and "layer_norm" in getattr(cfg, "norm_rel_ebd", "none").lower()
        self.conv = self.v2 and getattr(cfg, "conv_kernel_size", 0) > 0
        self.pos_biased = getattr(cfg, "position_biased_input", True)
        self.max_pos = cfg.max_position_embeddings
        self.type_vocab = cfg.type_vocab_size


def log_bucket(rel, buckets, max_position):
    """HF make_log_bucket_position on an int64 tensor of distances (torch float32 arithmetic, as transformers 5.x)."""
    sign = torch.sign(rel)
    mid = buckets // 2
    abs_pos = torch.where((rel < mid) & (rel > -mid), torch.tensor(mid - 1).type_as(rel), torch.abs(rel))
    log_pos = torch.ceil(torch.log(abs_pos / mid) / torch.log(torch.tensor((max_position - 1) / mid))
                         * (mid - 1)) + mid
    return torch.where(abs_pos <= mid, rel.type_as(log_pos), log_pos * sign).to(torch.long)


def rel_rows(dims, max_len):
    """int32 [2 max_len - 1]: the table row of distance d = i - j at index d + max_len - 1 (c2p and p2c alike)."""
    d = torch.arange(-(max_len - 1), max_len, dtype=torch.long)
    if dims.v2 and dims.buckets > 0:
        d = log_bucket(d, dims.buckets, dims.max_rel)
    return torch.clamp(d + dims.span, 0, 2 * dims.span - 1).to(torch.int32).numpy()


# ---- layer orchestration --------------------------------------------------------------------------------------------
def _strip(sd):
    """{name: tensor} of DebertaModel / DebertaV2Model: task-model prefixes dropped, heads (lm_predictions ...) too."""
    out = {}
    for k, v in sd.items():
        for p in ("deberta.",):
            if k.startswith(p):
                k = k[len(p):]
        if k.startswith(("embeddings.", "encoder.")) and not k.endswith("position_ids"):
            out[k] = torch.as_tensor(v)
    return out


class DebertaNet:
    """Backend-agnostic DebertaModel / DebertaV2Model forward over packed sentences.  ``sd``: {name: tensor} with
    DebertaModel names (a ``deberta.`` prefix is dropped); ``dims``: DebertaDims.  ``ops``: weight, operand, vector,
    embed, batch, layernorm, pos_proj, attention, linear_res, ffn_up, conv, zeros_like."""

    def __init__(self, sd, ops, dims):
        sd = _strip(sd)
        self.ops, self.d = ops, dims
        d, H, D = dims, dims.hidden, dims.heads * HEAD_DIM
        e = "embeddings."
        self.word = ops.embedding(sd.pop(e + "word_embeddings.weight"))
        self.pos = ops.embedding(sd.pop(e + "position_embeddings.weight")) if d.pos_biased else None
        self.type0 = ops.vector(sd.pop(e + "token_type_embeddings.weight")[0]) if d.type_vocab > 0 else None
        self.emb_ln = (ops.vector(sd.pop(e + "LayerNorm.weight")), ops.vector(sd.pop(e + "LayerNorm.bias")))
        rel = sd.pop("encoder.rel_embeddings.weight").float()[:2 * d.span]
        if d.norm_rel:
            rel = torch.nn.functional.layer_norm(rel, (H,), sd.pop("encoder.LayerNorm.weight").float(),
                                                 sd.pop("encoder.LayerNorm.bias").float(), d.eps)
        self.rel = ops.operand(rel)
        self.layers = []
        for i in range(d.layers):
            p = f"encoder.layer.{i}."
            a = p + "attention.self."
            if not d.v2:
                w_qkv = deinterleave_qkv(sd.pop(a + "in_proj.weight"), d.heads, HEAD_DIM)
                qb = sd.pop(a + "q_bias")
                b_qkv = torch.cat([qb, torch.zeros_like(qb), sd.pop(a + "v_bias")])
                w_pos = torch.cat([sd.pop(a + "pos_proj.weight"), sd.pop(a + "pos_q_proj.weight")])
                pb = sd.pop(a + "pos_q_proj.bias")
                b_pos = torch.cat([torch.zeros_like(pb), pb])
            else:
                names = ("query_proj", "key_proj", "value_proj")
                w_qkv = torch.cat([sd[a + n + ".weight"] for n in names])
                b_qkv = torch.cat([sd[a + n + ".bias"] for n in names])
                pk, pq = ("key_proj", "query_proj") if d.share else ("pos_key_proj", "pos_query_proj")
                w_pos = torch.cat([sd[a + pk + ".weight"], sd[a + pq + ".weight"]])
                b_pos = torch.cat([sd[a + pk + ".bias"], sd[a + pq + ".bias"]])
                for n in set(names) | {pk, pq}:
                    sd.pop(a + n + ".weight"), sd.pop(a + n + ".bias")
            self.layers.append(dict(
                qkv=ops.weight(w_qkv), b_qkv=ops.vector(b_qkv), pos=ops.weight(w_pos), b_pos=ops.vector(b_pos),
                o=ops.weight(sd.pop(p + "attention.output.dense.weight")),
                b_o=ops.vector(sd.pop(p + "attention.output.dense.bias")),
                ln1=(ops.vector(sd.pop(p + "attention.output.LayerNorm.weight")),
                     ops.vector(sd.pop(p + "attention.output.LayerNorm.bias"))),
                up=ops.weight(sd.pop(p + "intermediate.dense.weight")),
                b_up=ops.vector(sd.pop(p + "intermediate.dense.bias")),
                down=ops.weight(sd.pop(p + "output.dense.weight")), b_down=ops.vector(sd.pop(p + "output.dense.bias")),
                ln2=(ops.vector(sd.pop(p + "output.LayerNorm.weight")), ops.vector(sd.pop(p + "output.LayerNorm.bias")))))
        if d.conv:
            w = sd.pop("encoder.conv.conv.weight")        # [H, H, 3] -> [H, 3 H]: W[n, tap * H + c] = w[n, c, tap]
            self.conv = (ops.weight(w.permute(0, 2, 1).reshape(H, 3 * H)), ops.vector(sd.pop("encoder.conv.conv.bias")),
                         (ops.vector(sd.pop("encoder.conv.LayerNorm.weight")),
                          ops.vector(sd.pop("encoder.conv.LayerNorm.bias"))))
        assert not sd, f"unused weights: {sorted(sd)[:4]}"
        self.hidden = H
        # v1 scales q before both of its products (and PQ), v2 scales each product: the same value up to rounding
        self.scale = 1.0 / math.sqrt(3 * HEAD_DIM)

    def forward(self, ids, lens, return_hidden=False):
        """ids: int64 [tokens] of packed sentences with lengths ``lens``.  Returns the readout (sum of hidden states
        n - 3 .. n, fp32 on the CUDA backend) and, with return_hidden, the HF hidden_states tuple as a list."""
        ops, d = self.ops, self.d
        n = d.layers
        if d.pos_biased and max(lens) > d.max_pos:
            raise ValueError(f"a sentence of {max(lens)} tokens exceeds max_position_embeddings {d.max_pos}")
        b = ops.batch(lens, rel_rows(d, max(lens)))
        x = ops.embed(self.word, ids)
        if self.pos is not None:
            x = x + ops.embed(self.pos, np.concatenate([np.arange(m) for m in lens]))
        if self.type0 is not None:
            x = x + self.type0
        acc = ops.zeros_like(x)
        x, y = ops.layernorm(x, *self.emb_ln, d.eps, acc=acc if n <= 3 else None)
        hs = [x.clone()] if return_hidden else None
        y0 = y
        for i, L in enumerate(self.layers):
            pos = ops.pos_proj(self.rel, L["pos"], L["b_pos"])
            ctx = ops.attention(y, L["qkv"], L["b_qkv"], pos, b, d.heads, d.span, self.scale)
            x, y = ops.layernorm(ops.linear_res(ctx, L["o"], L["b_o"], x), *L["ln1"], d.eps)
            into = acc if i + 1 >= n - 3 else None          # hidden state i + 1 is in the readout
            conv = d.conv and i == 0
            h = ops.linear_res(ops.ffn_up(y, L["up"], L["b_up"]), L["down"], L["b_down"], x)
            x, y = ops.layernorm(h, *L["ln2"], d.eps, acc=None if conv else into)
            if conv:   # hs[1] = LayerNorm(layer0_out + gelu(conv(hs[0])))
                w, bias, ln = self.conv
                x, y = ops.layernorm(x + ops.conv(y0, w, bias, b), *ln, d.eps, acc=into)
            if return_hidden:
                hs.append(x.clone())
        return (acc, hs) if return_hidden else acc


class TorchOps:
    """Plain torch backend (CPU tests, fp32 by default): the same orchestration in HF's order of operations.
    ``v2`` selects where the 1/sqrt(3 * 64) scale goes: v1 divides q (before q k^T and c2p) and PQ, v2 divides k and
    each relative product."""

    def __init__(self, v2, device="cpu", dtype=torch.float32):
        self.v2, self.device, self.dtype = v2, torch.device(device), dtype

    def weight(self, t):
        return torch.as_tensor(t).to(self.device, self.dtype)

    vector = embedding = operand = weight

    def embed(self, table, ids):
        return table[torch.as_tensor(ids, device=self.device)]

    def zeros_like(self, x):
        return torch.zeros_like(x)

    def batch(self, lens, rows):
        return dict(lens=list(lens), rows=torch.from_numpy(rows).long().to(self.device), max_len=max(lens))

    def layernorm(self, x, g, b, eps, acc=None):
        y = torch.nn.functional.layer_norm(x, (x.shape[-1],), g, b, eps)
        if acc is not None:
            acc += y
        return y, y

    def pos_proj(self, rel, w, b):
        return rel @ w.T + b

    def attention(self, y, w_qkv, b_qkv, pos, b, heads, span, scale):
        D = heads * HEAD_DIM
        qkv = y @ w_qkv.T + b_qkv
        pk, pq = (pos[:, i * D:(i + 1) * D].view(-1, heads, HEAD_DIM).transpose(0, 1) for i in range(2))
        s = torch.sqrt(torch.tensor(HEAD_DIM * 3.0)).to(y.device, y.dtype)   # as HF scaled_size_sqrt
        ctx = torch.empty(y.shape[0], D, dtype=y.dtype, device=y.device)
        o = 0
        for n in b["lens"]:
            q, k, v = (qkv[o:o + n, i * D:(i + 1) * D].view(n, heads, HEAD_DIM).transpose(0, 1) for i in range(3))
            i = torch.arange(n, device=y.device)
            row = b["rows"][(i[:, None] - i[None, :]) + b["max_len"] - 1].expand(heads, n, n)   # [h, i, j]
            if self.v2:
                sc = q @ (k / s).transpose(1, 2)
                sc = sc + torch.gather(q @ pk.transpose(1, 2), -1, row) / s
                sc = sc + torch.gather(k @ pq.transpose(1, 2), -1, row.transpose(1, 2)).transpose(1, 2) / s
            else:
                q = q / s
                sc = q @ k.transpose(1, 2)
                sc = sc + torch.gather(q @ pk.transpose(1, 2), -1, row)
                sc = sc + torch.gather(k @ (pq / s).transpose(1, 2), -1, row.transpose(1, 2)).transpose(1, 2)
            ctx[o:o + n] = (torch.softmax(sc, dim=-1) @ v).transpose(0, 1).reshape(n, D)
            o += n
        return ctx

    def linear_res(self, a, w, b, x):
        return x + (a @ w.T + b)

    def ffn_up(self, y, w, b):
        return torch.nn.functional.gelu(y @ w.T + b)

    def conv(self, y0, w, bias, b):
        H = y0.shape[1]
        out, o = [], 0
        for n in b["lens"]:
            xs = y0[o:o + n].T[None]                                  # [1, H, n]
            out.append(torch.nn.functional.conv1d(xs, w.view(H, 3, H).permute(0, 2, 1), bias, padding=1)[0].T)
            o += n
        return torch.nn.functional.gelu(torch.cat(out))


class CudaOps(DeviceOps):
    """Product backend.  precision "f16": fp16 weights, GEMM operands, q | k | V^T and PK | PQ (MER_GEMM_F16,
    MER_ATT_QKV_F16); "bf16x3": split-bf16 weights and operands (MER_GEMM_BF16X3), tf32-rounded q | k | V^T and PK | PQ,
    ctx written as split rows.  fp32 biases, residual stream and readout; ``mer_layernorm`` writes the fp32 row, the
    next operand and the readout term in one pass.  ``timing``: see DeviceOps."""

    def __init__(self, precision, device="cuda"):
        import ctypes as C
        super().__init__(precision, device)
        vp, i32, i64, f32 = C.c_void_p, C.c_int, C.c_longlong, C.c_float
        self._att = self.L.declare("mer_disentangled_attention", [vp, vp, i64, vp, vp, i64, i32, vp, f32, vp, vp, i32,
                                                                  i64, i32, i32, i32, vp])

    def batch(self, lens, rows):
        """DeviceOps.batch, with the distance -> table row map and the conv operand rows of each token.  The rows are
        built before the first host-to-device copy, which waits for the previous pass: host work after it idles the
        GPU."""
        cu = np.zeros(len(lens) + 1, np.int64)
        cu[1:] = np.cumsum(lens)
        pad = np.concatenate([cu[s] + 2 * s + 1 + np.arange(m) for s, m in enumerate(lens)])  # conv operand rows
        return dict(super().batch(lens), rows=torch.from_numpy(rows).to(self.device),
                    pad=torch.from_numpy(pad).to(self.device))

    def pos_proj(self, rel, w, b):
        out = torch.empty(rel.shape[0], w.shape[0], dtype=self.op_dtype, device=self.device)
        self._run("gemm", lambda: self.L.gemm(rel, w, out, bias=b, mode=self.mode, f16_out=self.f16,
                                              round_out=not self.f16))
        return out

    def attention(self, y, w_qkv, b_qkv, pos, b, heads, span, scale):
        L, T, D = self.L, y.shape[0], heads * HEAD_DIM
        qkv = torch.empty(T, 3 * D, dtype=self.op_dtype, device=self.device)     # q | k rows (V columns unused)
        vt = torch.empty(D, (T + 7) // 8 * 8, dtype=self.op_dtype, device=self.device)
        self._run("gemm", lambda: L.gemm(y, w_qkv, qkv, bias=b_qkv, mode=self.mode, f16_out=self.f16,
                                         round_out=not self.f16, vt=vt, vt_col0=2 * D))
        ctx = torch.empty(T, D, dtype=self.op_dtype, device=self.device)
        flags = (L.MER_ATT_QKV_F16 | L.MER_EPI_OUT_F16) if self.f16 else L.MER_EPI_SPLIT_BF16
        self._run("attention", lambda: L.check(self._att(
            L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(pos), L.ptr(pos[:, D:]), pos.shape[1], span, L.ptr(b["rows"]),
            scale, L.ptr(ctx), L.ptr(b["cu"]), b["n"], T, b["max_len"], heads, flags, L.stream_ptr())))
        return ctx

    def conv(self, y0, w, bias, b):
        """gelu(conv1d_k3(h[0]) + bias) per token: one 3-tap GEMM over the operand rows laid out with a zero row before
        and after every sentence, so that no tap reads a neighbouring sentence."""
        T, H = y0.shape
        rows = T + 2 * b["n"]
        padded = torch.zeros(rows, H, dtype=y0.dtype, device=self.device)
        padded[b["pad"]] = y0
        out = torch.empty(rows - 2, H, dtype=torch.float32, device=self.device)
        self._run("gemm", lambda: self.L.gemm(padded, w, out, bias=bias, mode=self.mode, gelu=True, taps=3, K_inner=H,
                                              rows_per_batch=rows - 2, a_rows_dim=rows, a_row_stride=H))
        return out[b["pad"] - 1]


def activation_bytes_per_token(hidden, ffn):
    """Device bytes one token of a packed pass holds at the peak of a layer (4-byte operands: the bf16x3 bound):
    embedding gather, residual, LayerNorm row, operand, readout, q | k | v rows, V^T, ctx, conv rows, FFN activation."""
    return hidden * 4 * 11 + ffn * 4


class DebertaTextEncoder(PackedTextEncoder):
    """PackedTextEncoder over ``DebertaNet`` with the CUDA backend.  ``sd``: {name: tensor}; ``cfg``: the checkpoint's
    DebertaConfig / DebertaV2Config.  ``precision``: None = MER_TEXT_PRECISION, else BertEncoder's rule ("f16" at
    hidden 768, "bf16x3" above)."""

    span = (1, -1)

    def __init__(self, sd, cfg, device="cuda", precision=None):
        check_deberta_config(cfg)
        self.dims = d = DebertaDims(cfg)
        if d.hidden not in LN_DIMS:
            raise ValueError(f"DeBERTa path: hidden {d.hidden} (mer_layernorm rows: {LN_DIMS})")
        self.precision = precision or os.environ.get("MER_TEXT_PRECISION", "f16" if d.hidden == 768 else "bf16x3")
        self.ops = CudaOps(self.precision, device)
        self.device = self.ops.device
        self.net = DebertaNet(sd, self.ops, d)
        self.hidden, self.vocab_size = d.hidden, self.net.word.shape[0]
        self.bytes_per_token = activation_bytes_per_token(d.hidden, d.ffn)
