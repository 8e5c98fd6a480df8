"""LLaMA branch of the text extractor: the decoder LLMs of MERBench/feature_extraction/text/extract_text_huggingface.py
(``llama-7b-hf``, ``llama-13b-hf``, ``llama-2-7b``, ``Llama-2-13b-hf``, ``vicuna-7b-v0``, ``stable-vicuna-13b``,
``chinese-alpaca-2-13b``; :170-175), which the reference loads as HF ``LlamaModel`` and runs in fp16, one sentence per
forward (:193-231).  Readout as for every text model: ``torch.stack(hidden_states)[[-4, -3, -2, -1]].sum(0)``, where
for ``LlamaModel`` the last term is the output of the final ``norm`` and the other three are raw residual states.

The decoder layers are orchestrated here over kernel-level entry points through an ``ops`` backend (``CudaOps``: fp16
weights and operands on ``mer_gemm`` (MER_GEMM_F16), ``mer_rmsnorm``, ``mer_rope_f16``, ``mer_causal_attention_f16``,
``mer_swiglu_f16``; fp32 residual stream and readout), so that the orchestration runs against the reference golden
with a torch backend on CPU (``TorchOps``, tests/test_llama_text.py).  Sentences are packed back to back: one device
pass covers many of them.  Weights are read shard by shard, tensor by tensor, and converted to fp16 on the device
(``load_llama_weights``), so a 13 B checkpoint never exists as fp32 in host memory.
"""
from __future__ import annotations

import json
import os

import numpy as np
import torch

HEAD_DIM = 128


def check_llama_config(cfg):
    """Reject, before any weight is read, every config this path does not compute exactly: grouped-query attention,
    scaled / non-default rotary embeddings, biases, another activation, another head size."""
    heads = cfg.num_attention_heads
    kv = getattr(cfg, "num_key_value_heads", None) or heads
    if kv != heads:
        raise ValueError(f"LLaMA path: grouped-query attention (num_key_value_heads {kv} != {heads} heads) is not supported")
    rope = getattr(cfg, "rope_parameters", None) or getattr(cfg, "rope_scaling", None) or {}
    if rope.get("rope_type", rope.get("type", "default")) != "default" or set(rope) - {"rope_type", "rope_theta"}:
        raise ValueError(f"LLaMA path: only the default rotary embedding is supported, got {rope}")
    if getattr(cfg, "attention_bias", False) or getattr(cfg, "mlp_bias", False):
        raise ValueError("LLaMA path: attention_bias / mlp_bias checkpoints are not supported")
    if getattr(cfg, "hidden_act", "silu") != "silu":
        raise ValueError(f"LLaMA path: hidden_act {cfg.hidden_act!r} is not supported (silu only)")
    head_dim = getattr(cfg, "head_dim", None) or cfg.hidden_size // heads
    if head_dim != HEAD_DIM or heads * HEAD_DIM != cfg.hidden_size:
        raise ValueError(f"LLaMA path: head_dim {head_dim} with {heads} heads and hidden {cfg.hidden_size} "
                         f"(head_dim 128 only)")


def rope_theta(cfg):
    rope = getattr(cfg, "rope_parameters", None) or {}
    return float(rope.get("rope_theta", getattr(cfg, "rope_theta", 10000.0)))


def rope_tables(max_pos, theta, head_dim=HEAD_DIM):
    """cos / sin [max_pos, head_dim / 2] fp32 built as HF LlamaRotaryEmbedding (and FalconRotaryEmbedding) builds them:
    fp32 inv_freq, fp32 angle pos * inv_freq, torch.cos / torch.sin (the table's columns j and j + head_dim / 2 of HF's
    cat(freqs, freqs) are equal)."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.int64).to(torch.float32) / head_dim))
    freqs = torch.arange(max_pos, dtype=torch.int64).to(torch.float32)[:, None] * inv_freq[None, :]
    return freqs.cos().contiguous(), freqs.sin().contiguous()


# ---- streaming checkpoint loader ------------------------------------------------------------------------------------
def _checkpoint_files(model_dir, prefer_bin=False):
    kinds = [("pytorch_model.bin", "pytorch_model.bin.index.json"), ("model.safetensors", "model.safetensors.index.json")]
    if not prefer_bin:
        kinds.reverse()
    for single, index in kinds:
        if os.path.exists(os.path.join(model_dir, single)):
            return [os.path.join(model_dir, single)]
        if os.path.exists(os.path.join(model_dir, index)):
            shards = sorted(set(json.load(open(os.path.join(model_dir, index)))["weight_map"].values()))
            return [os.path.join(model_dir, s) for s in shards]
    raise FileNotFoundError(f"no model.safetensors / pytorch_model.bin (or their .index.json) under {model_dir}")


def _iter_tensors(path):
    if path.endswith(".safetensors"):
        from safetensors import safe_open
        with safe_open(path, framework="pt", device="cpu") as f:
            for k in f.keys():
                yield k, f.get_tensor(k)
    else:
        sd = torch.load(path, map_location="cpu", mmap=True, weights_only=True)
        for k in list(sd):
            yield k, sd.pop(k)


def load_llama_weights(model_dir, device, prefer_bin=False):
    """{LlamaModel parameter name: fp16 tensor on ``device``}, read one tensor at a time (safetensors through
    ``safe_open``, ``.bin`` through an mmap'ed ``torch.load``) from fp32 / fp16 / bf16 checkpoints.  Accepts the
    ``model.`` prefix of ``LlamaForCausalLM`` checkpoints and drops ``lm_head.weight`` and the rotary ``inv_freq``
    buffers some older checkpoints carry.  ``prefer_bin``: read ``pytorch_model.bin*`` when both formats exist (the
    reference loads Llama-2-13b-hf with ``use_safetensors=False``)."""
    out = {}
    for path in _checkpoint_files(model_dir, prefer_bin):
        for k, v in _iter_tensors(path):
            if k.startswith("model."):
                k = k[len("model."):]
            if k == "lm_head.weight" or k.endswith("rotary_emb.inv_freq"):
                continue
            t = v.to(device).to(torch.float16)
            if not bool(torch.isfinite(t).all()):
                raise ValueError(f"{path}: {k} is not finite in fp16")
            out[k] = t
    return out


# ---- layer orchestration --------------------------------------------------------------------------------------------
class LlamaNet:
    """Backend-agnostic LlamaModel forward over packed sentences.  ``sd``: {LlamaModel parameter name: tensor}; entries
    are consumed (popped) as the backend takes them over, so that a 13 B checkpoint is not held twice.  ``ops``:
    weight, vector, embed, batch, rmsnorm, attention, linear_res, mlp, add_ (see CudaOps)."""

    def __init__(self, sd, ops, n_layers, heads, eps, theta, max_pos):
        self.ops, self.heads, self.eps, self.n_layers, self.max_pos = ops, heads, eps, n_layers, max_pos
        assert n_layers >= 3, "the last-four readout needs at least 3 layers"
        self.embed = ops.embedding(sd.pop("embed_tokens.weight"))
        self.hidden = self.embed.shape[1]
        self.cos, self.sin = (ops.vector(t) for t in rope_tables(max_pos, theta))
        self.layers = []
        for i in range(n_layers):
            p = f"layers.{i}."
            a, m = p + "self_attn.", p + "mlp."
            self.layers.append(dict(
                ln1=ops.vector(sd.pop(p + "input_layernorm.weight")),
                qkv=ops.weight(torch.cat([sd.pop(a + "q_proj.weight"), sd.pop(a + "k_proj.weight"),
                                          sd.pop(a + "v_proj.weight")], 0)),
                o=ops.weight(sd.pop(a + "o_proj.weight")),
                ln2=ops.vector(sd.pop(p + "post_attention_layernorm.weight")),
                gate_up=ops.weight(torch.cat([sd.pop(m + "gate_proj.weight"), sd.pop(m + "up_proj.weight")], 0)),
                down=ops.weight(sd.pop(m + "down_proj.weight"))))
        self.norm = ops.vector(sd.pop("norm.weight"))
        assert not any(k.startswith("layers.") for k in sd), f"unused layer weights: {sorted(sd)[:4]}"

    def forward(self, ids, lens, return_hidden=False):
        """ids: int64 [tokens] of packed sentences with lengths ``lens`` (each <= max_position_embeddings).  Returns the
        readout h[L-3] + h[L-2] + h[L-1] + norm(h[L]) [tokens, hidden] (fp32 on the CUDA backend) and, with
        return_hidden, the HF hidden_states tuple as a list."""
        ops, n = self.ops, self.n_layers
        assert max(lens) <= self.max_pos, f"sentence of {max(lens)} tokens > max_position_embeddings {self.max_pos}"
        b = ops.batch(lens)
        x = ops.embed(self.embed, ids)
        hs = [x.clone()] if return_hidden else None
        acc = ops.zeros_like(x)
        for i, L in enumerate(self.layers):
            if i == n - 3:            # h[0] (the embedding) when n == 3
                ops.add_(acc, x)
            y = ops.rmsnorm(x, L["ln1"], self.eps)
            ctx = ops.attention(y, L["qkv"], b, self.heads, self.cos, self.sin)
            x = ops.linear_res(ctx, L["o"], x)
            y = ops.rmsnorm(x, L["ln2"], self.eps)
            x = ops.linear_res(ops.mlp(y, L["gate_up"]), L["down"], x)
            if i >= n - 3 and i < n - 1:
                ops.add_(acc, x)
            if return_hidden and i < n - 1:
                hs.append(x.clone())
        ops.rmsnorm(x, self.norm, self.eps, acc=acc)
        if return_hidden:
            hs.append(ops.rmsnorm(x, self.norm, self.eps, acc=ops.zeros_like(x)))
        return (acc, hs) if return_hidden else acc


class TorchOps:
    """Plain torch backend (CPU tests, fp32 by default): the same orchestration on torch operators, HF's order of
    operations."""

    def __init__(self, device="cpu", dtype=torch.float32):
        self.device, self.dtype = torch.device(device), dtype

    def weight(self, t):
        return t.to(self.device, self.dtype)

    vector = embedding = weight

    def embed(self, table, ids):
        return table[torch.as_tensor(ids, device=self.device)]

    def zeros_like(self, x):
        return torch.zeros_like(x)

    def add_(self, acc, x):
        acc += x

    def batch(self, lens):
        return list(lens)

    def _up(self, x):  # HF computes the norm statistics and the softmax in (at least) fp32
        return x.to(torch.promote_types(x.dtype, torch.float32))

    def rmsnorm(self, x, w, eps, acc=None):
        v = self._up(x).pow(2).mean(-1, keepdim=True)
        y = w * (self._up(x) * torch.rsqrt(v + eps)).to(x.dtype)
        if acc is not None:
            acc += y
            return acc
        return y

    def attention(self, y, w_qkv, lens, heads, cos, sin):
        D = heads * HEAD_DIM
        qkv = y @ w_qkv.T
        ctx = torch.empty(y.shape[0], D, dtype=y.dtype, device=y.device)
        o = 0
        for n in lens:
            c = torch.cat([cos[:n], cos[:n]], -1).to(y.dtype)[None]
            s = torch.cat([sin[:n], sin[:n]], -1).to(y.dtype)[None]
            q, k, v = (qkv[o:o + n, i * D:(i + 1) * D].view(n, heads, HEAD_DIM).transpose(0, 1) for i in range(3))
            rot = lambda t: torch.cat([-t[..., HEAD_DIM // 2:], t[..., :HEAD_DIM // 2]], -1)  # noqa: E731
            q, k = q * c + rot(q) * s, k * c + rot(k) * s
            sc = (q @ k.transpose(1, 2)) * HEAD_DIM ** -0.5
            sc = sc.masked_fill(torch.ones(n, n, dtype=torch.bool, device=y.device).triu(1), float("-inf"))
            p = torch.softmax(self._up(sc), dim=-1).to(y.dtype)
            ctx[o:o + n] = (p @ v).transpose(0, 1).reshape(n, D)
            o += n
        return ctx

    def linear_res(self, a, w, x):
        return x + a @ w.T

    def mlp(self, y, w_gu):
        gu = y @ w_gu.T
        h = gu.shape[1] // 2
        return torch.nn.functional.silu(gu[:, :h]) * gu[:, h:]


class CudaOps:
    """Product backend: fp16 weights and GEMM operands (MER_GEMM_F16), fp32 residual stream; every op is one or two
    libmer_b200.so launches.  With ``timing`` set to a list, each launch is bracketed by CUDA events and recorded as
    (kernel class, start, end) for the benchmark's time shares."""

    def __init__(self, device="cuda"):
        import ctypes as C

        from .. import _lib as L
        L.check(L.lib().mer_check_device())
        self.L, self.device, self.timing = L, torch.device(device), None
        vp, i32, i64, f32 = C.c_void_p, C.c_int, C.c_longlong, C.c_float
        self._rms = L.declare("mer_rmsnorm", [vp, vp, vp, vp, i64, i32, f32, vp])
        self._rope = L.declare("mer_rope_f16", [vp, i64, i64, i32, vp, i32, vp, vp, vp, i32, vp])
        self._att = L.declare("mer_causal_attention_f16", [vp, vp, i64, vp, vp, i32, i64, i32, i32, vp])
        self._swiglu = L.declare("mer_swiglu_f16", [vp, vp, i64, i32, vp])

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
        return t.to(self.device, torch.float16).contiguous()

    embedding = weight

    def vector(self, t):
        return t.to(self.device, torch.float32).contiguous()

    def embed(self, table, ids):
        return table[torch.as_tensor(ids, device=self.device)].float()

    def zeros_like(self, x):
        return torch.zeros_like(x)

    def add_(self, acc, x):
        acc += x

    def batch(self, lens):
        cu = np.zeros(len(lens) + 1, np.int32)
        cu[1:] = np.cumsum(lens)
        return dict(cu=torch.from_numpy(cu).to(self.device), n=len(lens), max_len=int(max(lens)))

    def rmsnorm(self, x, w, eps, acc=None):
        L = self.L
        y = None if acc is not None else torch.empty(x.shape, dtype=torch.float16, device=self.device)
        self._run("rmsnorm", lambda: L.check(self._rms(L.ptr(x), L.ptr(w), L.ptr(y), L.ptr(acc), x.shape[0], x.shape[1],
                                                       eps, L.stream_ptr())))
        return acc if acc is not None else y

    def attention(self, y, w_qkv, b, heads, cos, sin):
        L, T, D = self.L, y.shape[0], heads * HEAD_DIM
        qkv = torch.empty(T, 3 * D, dtype=torch.float16, device=self.device)     # q | k rows (V columns unused)
        vt = torch.empty(D, (T + 7) // 8 * 8, dtype=torch.float16, device=self.device)
        self._run("gemm", lambda: L.gemm(y, w_qkv, qkv, mode=L.MER_GEMM_F16, f16_out=True, vt=vt, vt_col0=2 * D))
        self._run("rope", lambda: L.check(self._rope(L.ptr(qkv), 3 * D, T, heads, L.ptr(b["cu"]), b["n"], None,
                                                     L.ptr(cos), L.ptr(sin), cos.shape[0], L.stream_ptr())))
        ctx = torch.empty(T, D, dtype=torch.float16, device=self.device)
        self._run("attention", lambda: L.check(self._att(L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(ctx), L.ptr(b["cu"]),
                                                         b["n"], T, b["max_len"], heads, L.stream_ptr())))
        return ctx

    def linear_res(self, a, w, x):
        self._run("gemm", lambda: self.L.gemm(a, w, x, res=x, mode=self.L.MER_GEMM_F16))
        return x

    def mlp(self, y, w_gu):
        L, T, two_i = self.L, y.shape[0], w_gu.shape[0]
        gu = torch.empty(T, two_i, dtype=torch.float32, device=self.device)
        self._run("gemm", lambda: L.gemm(y, w_gu, gu, mode=L.MER_GEMM_F16))
        h = torch.empty(T, two_i // 2, dtype=torch.float16, device=self.device)
        self._run("swiglu", lambda: L.check(self._swiglu(L.ptr(gu), L.ptr(h), T, two_i // 2, L.stream_ptr())))
        return h


def activation_bytes_per_token(hidden, intermediate):
    """Device bytes one token of a packed pass holds at the peak of a layer: fp32 residual + readout, fp16 operands,
    q | k rows and V^T, ctx, the fp32 gate | up output and its fp16 SwiGLU."""
    return hidden * (4 + 4 + 2 + 3 * 2 + 2 + 2) + intermediate * (2 * 4 + 2)


class LlamaTextEncoder:
    """``forward(id_lists, start, end, want_tokens)`` (the contract TextExtractor drives) over ``LlamaNet`` with the CUDA
    backend.  ``cfg``: the checkpoint's LlamaConfig; ``sd``: {name: tensor} (load_llama_weights)."""

    def __init__(self, sd, cfg, device="cuda"):
        import ctypes as C

        from .. import _lib as L
        check_llama_config(cfg)
        self.ops = CudaOps(device)
        self.device = self.ops.device
        self.max_pos = int(cfg.max_position_embeddings)
        self.net = LlamaNet(sd, self.ops, cfg.num_hidden_layers, cfg.num_attention_heads, float(cfg.rms_norm_eps),
                            rope_theta(cfg), self.max_pos)
        self.hidden, self.vocab_size = self.net.hidden, self.net.embed.shape[0]
        self.bytes_per_token = activation_bytes_per_token(self.hidden, cfg.intermediate_size)
        self._L = L
        self._seg = L.declare("mer_segment_reduce", [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                                     C.c_void_p, C.c_void_p])

    def forward(self, id_lists, start=1, end=None, want_tokens=False):
        """id_lists: non-empty token id sequences.  Returns (utt [n, hidden] = mean over each sentence's kept range
        [start : len + end], tokens [sum len, hidden] | None), fp32."""
        L = self._L
        lens = [len(x) for x in id_lists]
        assert all(n > 0 for n in lens), "empty sentences are handled by the caller (zeros)"
        if max(lens) > self.max_pos:
            raise ValueError(f"a sentence of {max(lens)} tokens exceeds max_position_embeddings {self.max_pos}")
        ids = np.concatenate([np.asarray(x, dtype=np.int64) for x in id_lists])
        assert ids.min() >= 0 and ids.max() < self.vocab_size, "token id outside the vocabulary"
        acc = self.net.forward(ids, lens)
        cu = np.zeros(len(lens) + 1, np.int64)
        cu[1:] = np.cumsum(lens)
        seg = np.stack([cu[:-1] + (start or 0), cu[1:] + (end or 0)]).astype(np.int32)
        seg = torch.from_numpy(np.maximum(seg, seg[:1])).to(self.device)   # empty kept range -> zeros (caller skips it)
        utt = torch.empty(len(lens), self.hidden, dtype=torch.float32, device=self.device)
        L.check(self._seg(L.ptr(acc), L.ptr(seg[0]), L.ptr(seg[1]), len(lens), self.hidden, 1, L.ptr(utt),
                          L.stream_ptr()))
        return utt, (acc if want_tokens else None)
