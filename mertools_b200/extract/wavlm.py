"""WavLM branch of the audio extractor (``wavlm-base`` / ``wavlm-large`` of
MERBench/feature_extraction/audio/extract_audio_huggingface.py:36-37, same readout as the other wav2vec2-style models
:93-100: sum of the last four hidden states).

WavLM = the wav2vec2 / HuBERT graph (feature encoder, projection, positional conv: ``mer_hubert_frontend``) with a
different attention: a bucketed relative position bias, computed once from layer 0's embedding and gated per layer,
head and query by a small projection of the layer input (HF modeling_wavlm.py WavLMAttention).  The layers are
orchestrated over kernel-level entry points through an ``ops`` backend (TF32 GEMMs, ``mer_layernorm``,
``mer_wavlm_gate``, ``mer_biased_attention``), so that the orchestration runs against the oracle with a torch backend on
CPU (tests/test_host_logic.py).  GPU parity test: tests/test_variants_gpu.py.
"""
from __future__ import annotations

import math

import numpy as np
import torch


def relative_buckets(T, num_buckets=320, max_distance=800):
    """WavLMAttention._relative_positions_bucket on ``j - i`` (float32 log arithmetic as in the original: the bucket
    boundaries depend on it).  int64 [T, T]."""
    rel = torch.arange(T)[None, :] - torch.arange(T)[:, None]
    nb = num_buckets // 2
    buckets = (rel > 0).to(torch.long) * nb
    rel = rel.abs()
    max_exact = nb // 2
    large = torch.log(rel.float() / max_exact) / math.log(max_distance / max_exact) * (nb - max_exact)
    large = torch.min((max_exact + large).to(torch.long), torch.full_like(rel, nb - 1))
    return (buckets + torch.where(rel < max_exact, rel, large)).numpy()


class WavLmNet:
    """Backend-agnostic orchestration of the WavLM transformer layers.  ``ops``: tensor, weight, operand, layernorm,
    linear, gate, biased_attention, add."""

    def __init__(self, state_dict, ops, eps=1e-5, max_distance=800):
        sd = {k: np.asarray(v, np.float32) for k, v in state_dict.items() if k.startswith("encoder.")}
        self.ops, self.eps, self.max_distance = ops, eps, max_distance
        self.d = d = sd["encoder.layers.0.attention.q_proj.weight"].shape[0]
        self.heads = d // 64
        # wavlm-large: LayerNorm feature extractor + do_stable_layer_norm (pre-LN layers), like the hubert-large family
        self.stable = "feature_extractor.conv_layers.1.layer_norm.weight" in state_dict
        self.rel_embed = sd["encoder.layers.0.attention.rel_attn_embed.weight"]          # [buckets, heads]
        self.enc_ln = (ops.tensor(sd["encoder.layer_norm.weight"]), ops.tensor(sd["encoder.layer_norm.bias"]))
        self.layers, self._bias = [], {}
        i = 0
        while f"encoder.layers.{i}.feed_forward.output_dense.weight" in sd:
            p = f"encoder.layers.{i}."
            a = p + "attention."
            self.layers.append(dict(
                qkv_w=ops.weight(np.concatenate([sd[a + "q_proj.weight"], sd[a + "k_proj.weight"], sd[a + "v_proj.weight"]], 0)),
                qkv_b=ops.tensor(np.concatenate([sd[a + "q_proj.bias"], sd[a + "k_proj.bias"], sd[a + "v_proj.bias"]])),
                o_w=ops.weight(sd[a + "out_proj.weight"]), o_b=ops.tensor(sd[a + "out_proj.bias"]),
                gate_w=ops.tensor(sd[a + "gru_rel_pos_linear.weight"]), gate_b=ops.tensor(sd[a + "gru_rel_pos_linear.bias"]),
                gate_c=ops.tensor(sd[a + "gru_rel_pos_const"].reshape(-1)),
                ln1=(ops.tensor(sd[p + "layer_norm.weight"]), ops.tensor(sd[p + "layer_norm.bias"])),
                w1=ops.weight(sd[p + "feed_forward.intermediate_dense.weight"]),
                b1=ops.tensor(sd[p + "feed_forward.intermediate_dense.bias"]),
                w2=ops.weight(sd[p + "feed_forward.output_dense.weight"]),
                b2=ops.tensor(sd[p + "feed_forward.output_dense.bias"]),
                ln2=(ops.tensor(sd[p + "final_layer_norm.weight"]), ops.tensor(sd[p + "final_layer_norm.bias"]))))
            i += 1

    def position_bias(self, T):
        """[heads, T, T] = rel_attn_embed[bucket(j - i)] (compute_bias), cached per T on the backend."""
        if T not in self._bias:
            b = self.rel_embed[relative_buckets(T, self.rel_embed.shape[0], self.max_distance)]      # [T, T, heads]
            self._bias[T] = self.ops.tensor(np.ascontiguousarray(b.transpose(2, 0, 1)))
        return self._bias[T]

    def hidden_states(self, h0, B, T):
        """h0: [B * T, D] = hidden_states[0] (mer_hubert_frontend).  Returns the HF tuple as a list of [B * T, D]."""
        ops, eps = self.ops, self.eps
        bias = self.position_bias(T)
        x, hs = h0, []
        for L in self.layers:
            hs.append(x)
            y = ops.layernorm(x, *L["ln1"], operand=False, eps=eps) if self.stable else x     # the attention input
            gate = ops.gate(y, self.heads, L["gate_w"], L["gate_b"], L["gate_c"])
            ctx = ops.biased_attention(ops.linear(ops.operand(y), L["qkv_w"], L["qkv_b"]), bias, gate, B, T, self.heads)
            if self.stable:
                x = ops.linear(ctx, L["o_w"], L["o_b"], res=x)
                y = ops.layernorm(x, *L["ln2"], operand=True, eps=eps)
                x = ops.linear(ops.linear(y, L["w1"], L["b1"], gelu=True, operand=True), L["w2"], L["b2"], res=x)
            else:
                x = ops.layernorm(ops.linear(ctx, L["o_w"], L["o_b"], res=x), *L["ln1"], operand=False, eps=eps)
                f = ops.linear(ops.linear(ops.operand(x), L["w1"], L["b1"], gelu=True, operand=True), L["w2"], L["b2"], res=x)
                x = ops.layernorm(f, *L["ln2"], operand=False, eps=eps)
        hs.append(ops.layernorm(x, *self.enc_ln, operand=False, eps=eps) if self.stable else x)
        return hs


def _cuda_ops(device):
    import ctypes as C

    from .whisper import CudaOps

    class Ops(CudaOps):
        def __init__(self, device):
            super().__init__(device)
            self._gate = self.L.declare("mer_wavlm_gate", [C.c_void_p, C.c_longlong, C.c_int, C.c_void_p, C.c_void_p,
                                                           C.c_void_p, C.c_void_p, C.c_void_p])
            self._batt = self.L.declare("mer_biased_attention", [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                                                 C.c_int, C.c_void_p, C.c_int, C.c_void_p])

        def operand(self, x):
            return self.L.round_tf32_(x.clone())

        def layernorm(self, x, g, b, operand, eps=1e-5):
            y = torch.empty_like(x)
            self.L.layernorm(x, g, b, y, eps=eps, flags=self.L.MER_LN_ROUND_TF32 if operand else 0)
            return y

        def gate(self, x, heads, w, b, c):
            out = torch.empty(x.shape[0], heads, dtype=torch.float32, device=self.device)
            self.L.check(self._gate(self.L.ptr(x), x.shape[0], heads, self.L.ptr(w), self.L.ptr(b), self.L.ptr(c),
                                    self.L.ptr(out), self.L.stream_ptr()))
            return out

        def biased_attention(self, qkv, bias, gate, B, T, heads):
            ctx = torch.empty(qkv.shape[0], qkv.shape[1] // 3, dtype=torch.float32, device=self.device)
            self.L.check(self._batt(self.L.ptr(qkv), self.L.ptr(bias), self.L.ptr(gate), B, T, heads, self.L.ptr(ctx), 1,
                                    self.L.stream_ptr()))
            return ctx
    return Ops(device)


class WavLmEncoder:
    """Same ``forward`` contract as ``HubertEncoder`` (what AudioExtractor drives): the front-end through
    ``mer_hubert_frontend`` on the HuBERT model struct, the WavLM layers through ``WavLmNet``."""

    def __init__(self, state_dict, device="cuda"):
        import ctypes as C

        from .. import _lib as L
        from ..encoders import HubertEncoder, MerHubertModel
        self.front = HubertEncoder(state_dict, device=device, conv_precision="bf16x3")  # (verified with split convolutions)
        self.device, self.hidden, self.n_layers = self.front.device, self.front.hidden, self.front.n_layers
        self.net = WavLmNet(state_dict, _cuda_ops(device))
        assert self.net.stable == bool(self.front.model.stable_layer_norm)
        self._L, self._C = L, C
        self._fe = L.declare("mer_hubert_frontend", [C.POINTER(MerHubertModel), C.c_void_p, C.c_int, C.c_int, C.c_int,
                                                     C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p])

    def num_frames(self, n_samples):
        return self.front.num_frames(n_samples)

    def forward(self, wave, normalize=True, want_frames=False, return_hidden=False):
        L, C = self._L, self._C
        assert wave.dtype == torch.float32 and wave.is_cuda and wave.dim() == 2
        wave = wave.contiguous()
        B, Ls = wave.shape
        T, D = self.num_frames(Ls), self.hidden
        assert T <= 1024, "rows of at most 10 s (the extractor's split_into_batch) give 499 frames"
        ws = self.front.ws.get(L.lib().mer_hubert_model_workspace_bytes(C.byref(self.front.model), B, Ls))
        h0 = torch.empty(B * T, D, dtype=torch.float32, device=self.device)
        L.check(self._fe(C.byref(self.front.model), L.ptr(wave), B, Ls, 1 if normalize else 0, L.ptr(ws), ws.numel(),
                         L.ptr(h0), L.stream_ptr()))
        hs = self.net.hidden_states(h0, B, T)
        frames = (hs[-1] + hs[-2] + hs[-3] + hs[-4]).view(B, T, D)
        utt = frames.mean(dim=1)
        if return_hidden:
            return utt, frames, torch.stack(hs).view(len(hs), B, T, D)
        return utt, (frames if want_frames else None)
