"""Host plumbing of the packed text branches (llama_text, ln_decoder_text, deberta_text, xlnet_text, albert_text):
``DeviceOps``, the base of their CUDA backends, and ``PackedTextEncoder``, the base of their encoders, whose
``forward`` is the contract TextExtractor drives.  Sentences are packed back to back, one device pass covers many of
them, and each sentence's features are the mean of the readout over its kept range."""
from __future__ import annotations

import numpy as np
import torch

from .. import _lib as L

_EPILOGUE = {"relu": "relu", "gelu_new": "gelu_tanh"}   # HF activation name -> mer_gemm epilogue flag (erf gelu aside)
_SPAN = object()   # forward's start / end default: the encoder's ``span``


def packed_token_types(id_lists, token_types=None):
    """int64 [sum len] of the token types of packed id lists, or None: ``token_types`` (one sequence per id list) when
    given, else the ``token_types`` TokenTypeTextExtractor attached to every id list (all or none of them)."""
    if token_types is None:
        found = [getattr(x, "token_types", None) for x in id_lists]
        assert all(t is None for t in found) or all(t is not None for t in found), "token types for some only"
        token_types = None if found[0] is None else found
    if token_types is None:
        return None
    assert [len(t) for t in token_types] == [len(x) for x in id_lists], "one token type per token"
    return np.concatenate([np.asarray(t, dtype=np.int64) for t in token_types])


def kept_ranges(lens, start, end):
    """int32 [2, n]: the packed rows [begin, end) of each sentence's kept range [start : len + end] (None: 0).  A
    sentence with nothing left gets begin == end, so its mean is zeros (TextExtractor saves zeros for it anyway)."""
    cu = np.zeros(len(lens) + 1, np.int64)
    cu[1:] = np.cumsum(lens)
    seg = np.stack([cu[:-1] + (start or 0), cu[1:] + (end or 0)]).astype(np.int32)
    return np.maximum(seg, seg[:1])


class DeviceOps:
    """Base of the CUDA backends: ``L`` (the libmer_b200.so bindings), ``device``, ``timing`` and the ops whose launches
    are the same in every family that has them.  precision "f16": fp16 weights and GEMM operands (MER_GEMM_F16);
    "bf16x3": split-bf16 weights and operands (MER_GEMM_BF16X3).  fp32 biases, residual stream and readout in both.
    ``timing``: None, or a list that collects (kernel class, start, end) CUDA events per launch, which the benchmark
    scripts turn into time shares."""

    f16 = True   # class default: the packing methods need only this and ``device``, not the library

    def __init__(self, precision, device="cuda"):
        L.check(L.lib().mer_check_device())
        assert precision in ("f16", "bf16x3"), precision
        self.L, self.f16, self.device, self.timing = L, precision == "f16", torch.device(device), None
        self.mode = L.MER_GEMM_F16 if self.f16 else L.MER_GEMM_BF16X3
        self.op_dtype = torch.float16 if self.f16 else torch.float32

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
        """-> GEMM operand: fp16, or split bf16 rows of the fp32 values."""
        t = torch.as_tensor(t)
        if self.f16:
            return t.to(self.device, torch.float16).contiguous()
        return self.L.split_bf16(t.to(self.device, torch.float32).contiguous())

    operand = weight

    def vector(self, t):
        return torch.as_tensor(t).to(self.device, torch.float32).contiguous()

    embedding = vector

    def embed(self, table, ids):
        return table[torch.as_tensor(ids, device=self.device)].float()

    def zeros_like(self, x):
        return torch.zeros_like(x)

    def add_(self, acc, x):
        acc += x

    def batch(self, lens):
        """The packed sentences as the kernels take them: int32 offsets ``cu`` [n + 1] on the device, ``n`` and
        ``max_len``."""
        cu = np.zeros(len(lens) + 1, np.int32)
        cu[1:] = np.cumsum(lens)
        return dict(cu=torch.from_numpy(cu).to(self.device), n=len(lens), max_len=int(max(lens)))

    def linear_res(self, a, w, bias, x):
        """x += a @ w.T (+ bias) in the GEMM's residual epilogue."""
        self._run("gemm", lambda: self.L.gemm(a, w, x, bias=bias, res=x, mode=self.mode))
        return x

    def layernorm(self, x, g, b, eps, acc=None):
        """``mer_layernorm``: (y fp32, y as the next GEMM operand) in one pass; acc += y when given."""
        L = self.L
        y = torch.empty_like(x)
        op = torch.empty(x.shape, dtype=self.op_dtype, device=self.device)
        flags = (L.MER_LN_SPLIT_F16 if self.f16 else 0) | (L.MER_LN_ACC_ADD if acc is not None else 0)
        self._run("layernorm", lambda: L.layernorm(x, g, b, y, eps=eps, y_split=op, acc=acc, flags=flags))
        return y, op

    def ffn_up(self, y, w, bias, act="gelu"):
        """act(y @ w.T + bias) as the next GEMM operand; act "gelu" (erf), "relu" or "gelu_new" (tanh form).  The
        ReLU and tanh-GELU epilogues write fp32 or fp16 only, so on bf16x3 they write fp32 rows that mer_split_bf16
        splits."""
        L = self.L
        h = torch.empty(y.shape[0], w.shape[0], dtype=self.op_dtype, device=self.device)
        if act == "gelu":
            self._run("gemm", lambda: L.gemm(y, w, h, bias=bias, mode=self.mode, gelu=True, f16_out=self.f16,
                                             split_out=not self.f16))
            return h
        epi = {_EPILOGUE[act]: True}
        if self.f16:
            self._run("gemm", lambda: L.gemm(y, w, h, bias=bias, mode=self.mode, f16_out=True, **epi))
        else:
            f = torch.empty(y.shape[0], w.shape[0], dtype=torch.float32, device=self.device)
            self._run("gemm", lambda: L.gemm(y, w, f, bias=bias, mode=self.mode, **epi))
            self._run("split", lambda: L.check(L.lib().mer_split_bf16(L.ptr(f), L.ptr(h), f.shape[0], f.shape[1],
                                                                       L.stream_ptr())))
        return h


class PackedTextEncoder:
    """``forward(id_lists, start, end, want_tokens, token_types)`` over a packed ``net``.  A family's __init__ checks
    the config before it touches the device or a weight, then sets ``net`` (``forward(ids, lens)`` -> the fp32 readout
    [tokens, width], width >= hidden with zero columns past hidden), ``device``, ``hidden``, ``vocab_size`` and
    ``bytes_per_token`` (what TextExtractor's launch size is budgeted by).  Class attributes: ``span``, the default
    kept range (start, end); ``max_pos``, the longest sentence accepted (None: no limit); ``takes_token_types``,
    whether ``net.forward`` takes token types."""

    span = (0, None)
    max_pos = None
    takes_token_types = False

    def forward(self, id_lists, start=_SPAN, end=_SPAN, want_tokens=False, token_types=None):
        """id_lists: non-empty token id sequences; token_types: None, or one int sequence per sentence (nets that take
        them).  When None, the ``token_types`` attribute TokenTypeTextExtractor attaches to each id list is used if
        present.  Returns (utt [n, hidden] = mean over each sentence's kept range [start : len + end], tokens
        [sum len, hidden] | None), fp32."""
        start = self.span[0] if start is _SPAN else start
        end = self.span[1] if end is _SPAN else end
        lens = [len(x) for x in id_lists]
        assert all(n > 0 for n in lens), "empty sentences are handled by the caller (zeros)"
        if self.max_pos is not None and max(lens) > self.max_pos:
            raise ValueError(f"a sentence of {max(lens)} tokens exceeds max_position_embeddings {self.max_pos}")
        ids = np.concatenate([np.asarray(x, dtype=np.int64) for x in id_lists])
        assert ids.min() >= 0 and ids.max() < self.vocab_size, "token id outside the vocabulary"
        if self.takes_token_types:
            tt = packed_token_types(id_lists, token_types)
            assert tt is None or (tt.min() >= 0 and tt.max() < self.vocab_size), "token type outside the vocabulary"
            acc = self.net.forward(ids, lens, token_types=tt)
        else:
            acc = self.net.forward(ids, lens)
        seg = torch.from_numpy(kept_ranges(lens, start, end)).to(self.device)
        width = acc.shape[1]
        utt = L.segment_reduce(acc, seg[0], seg[1], torch.empty(len(lens), width, dtype=torch.float32,
                                                                 device=self.device), dim=width, mean=True)
        if width != self.hidden:   # the pad columns are zero: slice them off
            utt = utt[:, :self.hidden].contiguous()
            acc = acc[:, :self.hidden].contiguous() if want_tokens else acc
        return utt, (acc if want_tokens else None)
