"""ALBERT branch of the text extractor: ``albert_chinese_tiny`` and ``albert_chinese_small`` (AutoModel + BertTokenizer,
MERBench/feature_extraction/text/extract_text_huggingface.py:164-166) and ``albert-base-v2``, ``albert-large-v2`` and
``albert-xxlarge-v2`` (the AutoModel + AutoTokenizer(use_fast=False) branch), run by the reference in fp32, one
sentence per forward.  Readout as for every text model: the sum of the last four hidden states, where hidden state 0 is
the output of ``embedding_hidden_mapping_in``.

ALBERT (HF AlbertModel, absolute positions) is a post-LN BERT layer applied ``num_hidden_layers`` times with ONE set of
weights:

    e = LN_128(word[ids] + token_type[0] + position[0 .. n-1]);  h_0 = e W_map^T + b_map    (hidden wide)
    a = LN(h + dense(softmax(q k^T / sqrt(hidden / heads)) v));  h' = LN(a + W_2 act(W_1 a + b_1) + b_2)

act is ``gelu`` (erf) or ``gelu_new`` (tanh form).  The single-sentence forward has token_type 0 everywhere.

``AlbertNet`` is the orchestration over an ``ops`` backend, as in xlnet_text.py: ``TorchOps`` is plain torch in HF's
order of operations (CPU tests, the restatement the GPU tests compare against), ``CudaOps`` runs every op as
libmer_b200.so launches: ``mer_gemm``, ``mer_layernorm`` / ``mer_layernorm_f16``, ``mer_attention_hd``,
``mer_split_bf16``.  The shared layer is packed once; every layer reads the same buffers.

Widths the kernels do not have directly are zero-padded at packing time (``AlbertDims``):
- a head of 26 columns (albert_chinese_tiny: 312 = 12 x 26) becomes 32: zero rows of W_q / W_k / W_v and zero bias for
  the pad, zero input columns of W_o.  q.k and P v are unchanged, and the score scale stays 1 / sqrt(26);
- the residual stream is padded to the next multiple of 128 columns (312 -> 384) and the FFN likewise (1248 -> 1280),
  with zero weight rows / columns and zero bias; LayerNorm runs with MER_LN_PAD (statistics over the valid columns, zero
  pad columns), so the pad stays exactly zero through the stack and is sliced off the features.
Operand format: BertEncoder's rule and its MER_TEXT_PRECISION variable, "f16" up to hidden 768 (fp16 operands and
attention), "bf16x3" above (split-bf16 GEMM operands, tf32 q | k | V^T); fp32 residual stream and readout in both.
"""
from __future__ import annotations

import math
import os

import numpy as np
import torch

from .deberta_text import activation_bytes_per_token
from .text import TextExtractor

KERNEL_HEAD_DIM = {26: 32, 32: 32, 64: 64}   # ALBERT head_dim -> the attention kernel's head_dim (26: zero-padded)
LN_WIDTHS = (128, 384, 512, 768, 1024, 1280, 1536)   # mer_layernorm's rows (MER_LN_PAD: valid width below one of them)
LN_F16_MAX = 8192                                    # mer_layernorm_f16: dim % 256 == 0, <= 8192
MAX_LEN = 512                                        # mer_attention_hd's longest row
ACTS = ("gelu", "gelu_new")
CHINESE_BERT_TOKENIZER = ("albert_chinese_tiny", "albert_chinese_small")   # reference :164-166


def _round128(n):
    return (n + 127) // 128 * 128


# ---- configs --------------------------------------------------------------------------------------------------------
def check_albert_config(cfg):
    """Reject, before any weight is read, every ALBERT config this path does not compute exactly."""
    if cfg.model_type != "albert":
        raise ValueError(f"not an ALBERT config: model_type {cfg.model_type!r}")
    if cfg.num_hidden_groups != 1 or cfg.inner_group_num != 1:
        raise ValueError(f"ALBERT path: num_hidden_groups {cfg.num_hidden_groups} / inner_group_num "
                         f"{cfg.inner_group_num} (1 / 1 only, as every released checkpoint)")
    H, heads = cfg.hidden_size, cfg.num_attention_heads
    if heads <= 0 or H % heads != 0:
        raise ValueError(f"ALBERT path: hidden {H} is not a multiple of {heads} heads")
    if H // heads not in KERNEL_HEAD_DIM:
        raise ValueError(f"ALBERT path: head_dim {H // heads} (26 -> padded 32, 32 or 64)")
    if cfg.hidden_act not in ACTS:
        raise ValueError(f"ALBERT path: hidden_act {cfg.hidden_act!r} is not supported ({' or '.join(ACTS)})")
    if getattr(cfg, "position_embedding_type", "absolute") != "absolute":
        raise ValueError(f"ALBERT path: position_embedding_type {cfg.position_embedding_type!r} (absolute only)")
    if cfg.embedding_size not in LN_WIDTHS:
        raise ValueError(f"ALBERT path: embedding_size {cfg.embedding_size} (mer_layernorm rows: {LN_WIDTHS})")
    if cfg.max_position_embeddings > MAX_LEN:
        raise ValueError(f"ALBERT path: max_position_embeddings {cfg.max_position_embeddings} (rows up to {MAX_LEN})")
    d = AlbertDims(cfg)
    if d.att % 128:
        raise ValueError(f"ALBERT path: {heads} heads x {d.khd} columns = {d.att} (mer_gemm: a multiple of 128)")
    if d.hidden_pad not in LN_WIDTHS and not (d.hidden_pad == H and H % 256 == 0 and H <= LN_F16_MAX):
        raise ValueError(f"ALBERT path: hidden {H} (LayerNorm rows: {LN_WIDTHS}, padded valid widths below them, or a "
                         f"multiple of 256 up to {LN_F16_MAX})")


class AlbertDims:
    """The shape facts of an AlbertConfig the orchestration needs, with the device padding: ``khd`` the kernel's head
    dim, ``att`` = heads * khd, ``hidden_pad`` / ``ffn_pad`` the residual / FFN widths rounded up to 128."""

    def __init__(self, cfg, pad=True):
        self.layers, self.heads, self.hidden = cfg.num_hidden_layers, cfg.num_attention_heads, cfg.hidden_size
        self.ffn, self.eps, self.act = cfg.intermediate_size, float(cfg.layer_norm_eps), cfg.hidden_act
        self.emb = cfg.embedding_size
        self.head_dim = self.hidden // self.heads
        self.scale = 1.0 / math.sqrt(self.head_dim)
        self.khd = KERNEL_HEAD_DIM.get(self.head_dim, self.head_dim) if pad else self.head_dim
        self.att = self.heads * self.khd
        self.hidden_pad = _round128(self.hidden) if pad else self.hidden
        self.ffn_pad = _round128(self.ffn) if pad else self.ffn


# ---- weights --------------------------------------------------------------------------------------------------------
LAYER = "encoder.albert_layer_groups.0.albert_layers.0."


def strip_albert(sd):
    """{name: tensor} of AlbertModel: an ``albert.`` prefix dropped; the MLM head (``predictions.*``), the sentence-order
    head (``sop_classifier.*``), the pooler and the ``position_ids`` / ``token_type_ids`` buffers dropped."""
    out = {}
    for k, v in sd.items():
        if k.startswith("albert."):
            k = k[len("albert."):]
        if k.startswith(("predictions.", "sop_classifier.", "pooler.")) or k.endswith(("position_ids",
                                                                                          "token_type_ids")):
            continue
        out[k] = torch.as_tensor(v)
    return out


def _pad_rows(w, rows):
    """[r, ...] -> [rows, ...] with zero rows appended."""
    if w.shape[0] == rows:
        return w
    return torch.cat([w, w.new_zeros((rows - w.shape[0],) + tuple(w.shape[1:]))])


def _pad_cols(w, cols):
    if w.shape[1] == cols:
        return w
    return torch.cat([w, w.new_zeros(w.shape[0], cols - w.shape[1])], dim=1)


def _head_rows(w, heads, hd, khd):
    """[heads*hd, ...] -> [heads*khd, ...]: each head's rows followed by khd - hd zero rows."""
    if hd == khd:
        return w
    w = w.reshape(heads, hd, *w.shape[1:])
    return torch.cat([w, w.new_zeros(heads, khd - hd, *w.shape[2:])], dim=1).reshape(heads * khd, *w.shape[2:])


def pack_layer(sd, d):
    """The shared layer as padded fp32 GEMM weights [out, in] and vectors: qkv [3 att, hidden_pad] (q | k | v, head
    rows padded), b_qkv [3 att], o [hidden_pad, att] (head input columns padded), up [ffn_pad, hidden_pad], down
    [hidden_pad, ffn_pad], LayerNorm vectors at hidden_pad."""
    H, hp, fp = d.hidden, d.hidden_pad, d.ffn_pad

    def lin(n):
        return sd.pop(LAYER + n + ".weight").float(), sd.pop(LAYER + n + ".bias").float()

    def vec(v, n):
        return _pad_rows(v, n)

    qkv, b_qkv = [], []
    for n in ("query", "key", "value"):
        w, b = lin("attention." + n)
        qkv.append(_pad_cols(_head_rows(w, d.heads, d.head_dim, d.khd), hp))
        b_qkv.append(_head_rows(b, d.heads, d.head_dim, d.khd))
    w_o, b_o = lin("attention.dense")
    w_o = _head_rows(w_o.T, d.heads, d.head_dim, d.khd).T          # input columns per head
    up, b_up = lin("ffn")
    down, b_down = lin("ffn_output")
    ln = lambda n: (vec(sd.pop(LAYER + n + ".weight").float(), hp), vec(sd.pop(LAYER + n + ".bias").float(), hp))  # noqa: E731
    assert H <= hp
    return dict(qkv=torch.cat(qkv), b_qkv=torch.cat(b_qkv), o=_pad_rows(w_o, hp), b_o=vec(b_o, hp),
                ln1=ln("attention.LayerNorm"), up=_pad_rows(_pad_cols(up, hp), fp), b_up=vec(b_up, fp),
                down=_pad_rows(_pad_cols(down, fp), hp), b_down=vec(b_down, hp), ln2=ln("full_layer_layer_norm"))


class AlbertNet:
    """Backend-agnostic AlbertModel forward over packed sentences.  ``sd``: {name: tensor} with AlbertModel names (see
    strip_albert); ``dims``: AlbertDims (pad=False: the unpadded restatement, TorchOps only).  ``ops``: weight, vector,
    embedding, embed, batch, zeros_like, layernorm, linear, attention, linear_res, ffn_up."""

    def __init__(self, sd, ops, dims):
        sd = strip_albert(sd)
        self.ops, self.d = ops, dims
        d = dims
        e = "embeddings."
        self.word = ops.embedding(sd.pop(e + "word_embeddings.weight").float())
        # token type 0 folded into the position rows (a single-sentence forward has type 0 everywhere)
        types = sd.pop(e + "token_type_embeddings.weight").float()
        self.pos_type = ops.embedding(sd.pop(e + "position_embeddings.weight").float() + types[0])
        self.ln_emb = (ops.vector(sd.pop(e + "LayerNorm.weight")), ops.vector(sd.pop(e + "LayerNorm.bias")))
        w_map = sd.pop("encoder.embedding_hidden_mapping_in.weight").float()
        b_map = sd.pop("encoder.embedding_hidden_mapping_in.bias").float()
        self.map = ops.weight(_pad_rows(w_map, d.hidden_pad))
        self.b_map = ops.vector(_pad_rows(b_map, d.hidden_pad))
        p = pack_layer(sd, d)
        self.layer = dict(
            qkv=ops.weight(p["qkv"]), b_qkv=ops.vector(p["b_qkv"]), o=ops.weight(p["o"]), b_o=ops.vector(p["b_o"]),
            ln1=tuple(ops.vector(t) for t in p["ln1"]), up=ops.weight(p["up"]), b_up=ops.vector(p["b_up"]),
            down=ops.weight(p["down"]), b_down=ops.vector(p["b_down"]), ln2=tuple(ops.vector(t) for t in p["ln2"]))
        assert not sd, f"unused weights: {sorted(sd)[:4]}"

    def forward(self, ids, lens, return_hidden=False):
        """ids: int64 [tokens] of packed sentences with lengths ``lens``.  Returns the readout (sum of hidden states
        n - 3 .. n, [tokens, hidden_pad], fp32 on the CUDA backend; pad columns zero) and, with return_hidden, the HF
        hidden_states tuple as a list (padded width)."""
        ops, d, L = self.ops, self.d, self.layer
        n = d.layers
        b = ops.batch(lens)
        pos = np.concatenate([np.arange(k) for k in lens])
        e = ops.embed(self.word, ids, self.pos_type, pos)
        _, e_op = ops.layernorm(e, *self.ln_emb, d.eps, d.emb, want_y=False)
        x, y = ops.linear(e_op, self.map, self.b_map)       # hs[0]: the mapped embedding, and its operand
        acc = x.clone() if n <= 3 else ops.zeros_like(x)
        hs = [x.clone()] if return_hidden else None
        for i in range(n):
            ctx = ops.attention(y, L["qkv"], L["b_qkv"], b, d)
            x, y = ops.layernorm(ops.linear_res(ctx, L["o"], L["b_o"], x), *L["ln1"], d.eps, d.hidden)
            into = acc if i + 1 >= n - 3 else None          # hidden state i + 1 is in the readout
            h = ops.linear_res(ops.ffn_up(y, L["up"], L["b_up"], d.act), L["down"], L["b_down"], x)
            x, y = ops.layernorm(h, *L["ln2"], d.eps, d.hidden, acc=into)
            if return_hidden:
                hs.append(x.clone())
        return (acc, hs) if return_hidden else acc


class TorchOps:
    """Plain torch backend (CPU tests, fp32 by default): the same orchestration in HF's order of operations, on the
    padded or unpadded packing."""

    def __init__(self, device="cpu", dtype=torch.float32):
        self.device, self.dtype = torch.device(device), dtype

    def weight(self, t):
        return torch.as_tensor(t).to(self.device, self.dtype)

    vector = embedding = weight

    def embed(self, word, ids, pos_type, pos):
        return word[torch.as_tensor(ids, device=self.device)] + pos_type[torch.as_tensor(pos, device=self.device)]

    def zeros_like(self, x):
        return torch.zeros_like(x)

    def batch(self, lens):
        return dict(lens=list(lens))

    def layernorm(self, x, g, b, eps, valid, acc=None, want_y=True):
        y = torch.zeros_like(x)
        y[:, :valid] = torch.nn.functional.layer_norm(x[:, :valid], (valid,), g[:valid], b[:valid], eps)
        if acc is not None:
            acc += y
        return y, y

    def linear(self, a, w, b):
        y = a @ w.T + b
        return y, y

    def attention(self, y, w_qkv, b_qkv, b, d):
        D, hd = d.att, d.khd
        qkv = y @ w_qkv.T + b_qkv
        ctx = torch.empty(y.shape[0], D, dtype=y.dtype, device=y.device)
        o = 0
        for n in b["lens"]:
            q, k, v = (qkv[o:o + n, i * D:(i + 1) * D].view(n, d.heads, hd).transpose(0, 1) for i in range(3))
            p = torch.softmax((q @ k.transpose(1, 2)) * d.scale, dim=-1)
            ctx[o:o + n] = (p @ v).transpose(0, 1).reshape(n, D)
            o += n
        return ctx

    def linear_res(self, a, w, b, x):
        return x + (a @ w.T + b)

    def ffn_up(self, y, w, b, act):
        return torch.nn.functional.gelu(y @ w.T + b, approximate="tanh" if act == "gelu_new" else "none")


class CudaOps:
    """Product backend.  precision "f16": fp16 weights, GEMM operands and q | k | V^T (MER_GEMM_F16, MER_ATT_QKV_F16);
    "bf16x3": split-bf16 weights and operands (MER_GEMM_BF16X3), tf32-rounded q | k | V^T, ctx written as split rows.
    fp32 biases, residual stream and readout.  LayerNorm: ``mer_layernorm`` at its widths (MER_LN_PAD for a padded
    row), ``mer_layernorm_f16`` at multiples of 256 beyond them (xxlarge's 4096; on bf16x3 followed by mer_split_bf16).
    ``timing``: None, or a list that collects (kernel class, start, end) CUDA events per launch."""

    def __init__(self, precision, device="cuda"):
        import ctypes as C

        from .. import _lib as L
        L.check(L.lib().mer_check_device())
        assert precision in ("f16", "bf16x3"), precision
        self.L, self.f16, self.device, self.timing = L, precision == "f16", torch.device(device), None
        self.mode = L.MER_GEMM_F16 if self.f16 else L.MER_GEMM_BF16X3
        self.op_dtype = torch.float16 if self.f16 else torch.float32
        vp, i32, i64, f32 = C.c_void_p, C.c_int, C.c_longlong, C.c_float
        self._att = L.declare("mer_attention_hd", [vp, vp, i64, vp, vp, i32, i64, i32, i32, i32, f32, i32, vp])
        self._ln16 = L.declare("mer_layernorm_f16", [vp, vp, vp, vp, vp, vp, i64, i32, f32, vp])

    def _run(self, klass, fn):
        if self.timing is None:
            return fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        r = fn()
        b.record()
        self.timing.append((klass, a, b))
        return r

    def weight(self, t):
        """fp32 rows -> GEMM operand: fp16, or split bf16 rows."""
        t = torch.as_tensor(t).to(self.device, torch.float32).contiguous()
        return t.half() if self.f16 else self.L.split_bf16(t)

    def vector(self, t):
        return torch.as_tensor(t).to(self.device, torch.float32).contiguous()

    embedding = vector

    def embed(self, word, ids, pos_type, pos):
        return word[torch.as_tensor(ids, device=self.device)] + pos_type[torch.as_tensor(pos, device=self.device)]

    def zeros_like(self, x):
        return torch.zeros_like(x)

    def batch(self, lens):
        cu = np.zeros(len(lens) + 1, np.int64)
        cu[1:] = np.cumsum(lens)
        return dict(cu=torch.from_numpy(cu.astype(np.int32)).to(self.device), n=len(lens), max_len=int(max(lens)))

    def layernorm(self, x, g, b, eps, valid, acc=None, want_y=True):
        """(y fp32 or None, y as the next GEMM operand); acc += y when given.  valid: the unpadded width."""
        L, T, W = self.L, x.shape[0], x.shape[1]
        op = torch.empty(x.shape, dtype=self.op_dtype, device=self.device)
        y = torch.empty_like(x) if want_y else None
        if W in LN_WIDTHS:
            flags = ((L.MER_LN_SPLIT_F16 if self.f16 else 0) | (L.MER_LN_ACC_ADD if acc is not None else 0)
                     | (L.MER_LN_PAD if valid != W else 0))
            self._run("layernorm", lambda: L.check(L.lib().mer_layernorm(
                L.ptr(x), L.ptr(g), L.ptr(b), L.ptr(y), L.ptr(op), L.ptr(acc), T, valid, eps, flags, L.stream_ptr())))
            return y, op
        assert valid == W, "padded rows need a mer_layernorm width"
        if y is None:
            y = torch.empty_like(x)
        self._run("layernorm", lambda: L.check(self._ln16(L.ptr(x), L.ptr(g), L.ptr(b), L.ptr(op) if self.f16 else None,
                                                          L.ptr(y), L.ptr(acc), T, W, eps, L.stream_ptr())))
        if not self.f16:
            self._run("split", lambda: L.check(L.lib().mer_split_bf16(L.ptr(y), L.ptr(op), T, W, L.stream_ptr())))
        return y, op

    def linear(self, a, w, bias):
        """(fp32 a @ w.T + bias, the same as the next GEMM operand): the embedding mapping, hidden state 0.  On f16 a
        second pass of the (K = embedding_size) GEMM writes the fp16 copy; on bf16x3 the fp32 rows are split."""
        L = self.L
        out = torch.empty(a.shape[0], w.shape[0], dtype=torch.float32, device=self.device)
        self._run("gemm", lambda: L.gemm(a, w, out, bias=bias, mode=self.mode))
        op = torch.empty(out.shape, dtype=self.op_dtype, device=self.device)
        if self.f16:
            self._run("gemm", lambda: L.gemm(a, w, op, bias=bias, mode=self.mode, f16_out=True))
        else:
            self._run("split", lambda: L.check(L.lib().mer_split_bf16(L.ptr(out), L.ptr(op), out.shape[0],
                                                                       out.shape[1], L.stream_ptr())))
        return out, op

    def attention(self, y, w_qkv, b_qkv, b, d):
        L, T, D = self.L, y.shape[0], d.att
        qkv = torch.empty(T, 3 * D, dtype=self.op_dtype, device=self.device)     # q | k rows (V columns unused)
        vt = torch.empty(D, (T + 7) // 8 * 8, dtype=self.op_dtype, device=self.device)
        self._run("gemm", lambda: L.gemm(y, w_qkv, qkv, bias=b_qkv, mode=self.mode, f16_out=self.f16,
                                         round_out=not self.f16, vt=vt, vt_col0=2 * D))
        ctx = torch.empty(T, D, dtype=self.op_dtype, device=self.device)
        flags = (L.MER_ATT_QKV_F16 | L.MER_EPI_OUT_F16) if self.f16 else L.MER_EPI_SPLIT_BF16
        self._run("attention", lambda: L.check(self._att(
            L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(ctx), L.ptr(b["cu"]), b["n"], T, b["max_len"], d.heads, d.khd,
            d.scale, flags, L.stream_ptr())))
        return ctx

    def linear_res(self, a, w, bias, x):
        self._run("gemm", lambda: self.L.gemm(a, w, x, bias=bias, res=x, mode=self.mode))
        return x

    def ffn_up(self, y, w, bias, act):
        h = torch.empty(y.shape[0], w.shape[0], dtype=self.op_dtype, device=self.device)
        if act == "gelu":
            self._run("gemm", lambda: self.L.gemm(y, w, h, bias=bias, mode=self.mode, gelu=True, f16_out=self.f16,
                                                  split_out=not self.f16))
        elif self.f16:
            self._run("gemm", lambda: self.L.gemm(y, w, h, bias=bias, mode=self.mode, gelu_tanh=True, f16_out=True))
        else:   # mer_gemm's tanh-GELU epilogue writes fp32 or fp16 only: fp32, then split for the FC2 operand
            f = torch.empty(y.shape[0], w.shape[0], dtype=torch.float32, device=self.device)
            self._run("gemm", lambda: self.L.gemm(y, w, f, bias=bias, mode=self.mode, gelu_tanh=True))
            self._run("split", lambda: self.L.check(self.L.lib().mer_split_bf16(
                self.L.ptr(f), self.L.ptr(h), f.shape[0], f.shape[1], self.L.stream_ptr())))
        return h


def default_precision(hidden):
    """BertEncoder's rule, MER_TEXT_PRECISION overriding it: "f16" up to hidden 768, "bf16x3" above."""
    return os.environ.get("MER_TEXT_PRECISION", "f16" if hidden <= 768 else "bf16x3")


class AlbertTextEncoder:
    """``forward(id_lists, start, end, want_tokens)`` (the contract TextExtractor drives) over ``AlbertNet`` with the
    CUDA backend.  ``sd``: {name: tensor}; ``cfg``: the checkpoint's AlbertConfig.  ``precision``: None =
    default_precision(hidden)."""

    def __init__(self, sd, cfg, device="cuda", precision=None):
        import ctypes as C

        from .. import _lib as L
        check_albert_config(cfg)
        self.dims = d = AlbertDims(cfg)
        self.precision = precision or default_precision(d.hidden)
        self.ops = CudaOps(self.precision, device)
        self.device = self.ops.device
        self.net = AlbertNet(sd, self.ops, d)
        self.hidden, self.vocab_size = d.hidden, self.net.word.shape[0]
        self.max_pos = self.net.pos_type.shape[0]
        self.bytes_per_token = activation_bytes_per_token(d.hidden_pad, d.ffn_pad)
        self._L = L
        self._seg = L.declare("mer_segment_reduce", [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                                     C.c_void_p, C.c_void_p])

    def forward(self, id_lists, start=0, end=-2, want_tokens=False):
        """id_lists: non-empty token id sequences of at most max_position_embeddings tokens.  Returns (utt [n, hidden] =
        mean over each sentence's kept range [start : len + end], tokens [sum len, hidden] | None), fp32."""
        L, d = self._L, self.dims
        lens = [len(x) for x in id_lists]
        assert all(n > 0 for n in lens), "empty sentences are handled by the caller (zeros)"
        assert max(lens) <= self.max_pos, f"a sentence of {max(lens)} tokens (max_position_embeddings {self.max_pos})"
        ids = np.concatenate([np.asarray(x, dtype=np.int64) for x in id_lists])
        assert ids.min() >= 0 and ids.max() < self.vocab_size, "token id outside the vocabulary"
        acc = self.net.forward(ids, lens)
        cu = np.zeros(len(lens) + 1, np.int64)
        cu[1:] = np.cumsum(lens)
        seg = np.stack([cu[:-1] + (start or 0), cu[1:] + (end or 0)]).astype(np.int32)
        seg = torch.from_numpy(np.maximum(seg, seg[:1])).to(self.device)   # empty kept range -> zeros (caller skips it)
        utt = torch.empty(len(lens), d.hidden_pad, dtype=torch.float32, device=self.device)
        L.check(self._seg(L.ptr(acc), L.ptr(seg[0]), L.ptr(seg[1]), len(lens), d.hidden_pad, 1, L.ptr(utt),
                          L.stream_ptr()))
        if d.hidden_pad != d.hidden:   # the pad columns are zero: slice them off
            utt = utt[:, :d.hidden].contiguous()
            acc = acc[:, :d.hidden].contiguous() if want_tokens else acc
        return utt, (acc if want_tokens else None)


def albert_tokenizer(model_name, model_dir):
    """The tokenizer the reference loads for an ALBERT model: BertTokenizer for albert_chinese_tiny / _small
    (:164-166), AutoTokenizer for every other name, both with use_fast=False."""
    from transformers import AutoTokenizer, BertTokenizer
    cls = BertTokenizer if model_name in CHINESE_BERT_TOKENIZER else AutoTokenizer
    return cls.from_pretrained(model_dir, use_fast=False)


AlbertTextExtractor = TextExtractor
