"""Whisper branch of the audio extractor: mirror of MERBench/feature_extraction/audio/extract_audio_huggingface.py:83-110
for ``whisper-base`` (d_model 512, 8 heads) and ``whisper-large-v2`` (1280, 20 heads).

``WhisperFeatureExtractor`` -> ``WhisperModel(input_features, decoder_input_ids=[[start, start]]).last_hidden_state[0]``
= the decoder's two output rows.  The network is orchestrated here over kernel-level entry points of libmer_b200.so —
``mer_whisper_logmel`` (front-end), ``mer_gemm`` (both convolutions as 3-tap GEMMs and every linear layer, TF32),
``mer_layernorm``, ``mer_attention`` (encoder, 1500 frames), ``mer_small_attention`` (decoder) — through a small
``ops`` backend, so that the orchestration (weight packing, layer order, residuals, position tables) can be run against
the reference golden with a torch backend on CPU (tests/test_host_logic.py); ``CudaOps`` is the product backend.
GPU parity test: tests/test_variants_gpu.py.
"""
from __future__ import annotations

import numpy as np
import torch

N_SAMPLES, N_FRAMES, N_MELS, MEL_LD = 480000, 3000, 80, 96


def whisper_mel_filters(n_freq=201, n_mel=N_MELS, fmin=0.0, fmax=8000.0, sr=16000):
    """[201, 80] Slaney-scale, Slaney-normalised triangular filter bank (the table WhisperFeatureExtractor builds)."""
    def hz_to_mel(f):
        f = np.asarray(f, dtype=np.float64)
        m = 3.0 * f / 200.0
        lg = f >= 1000.0
        m[lg] = 15.0 + np.log(f[lg] / 1000.0) * (27.0 / np.log(6.4))
        return m

    def mel_to_hz(m):
        m = np.asarray(m, dtype=np.float64)
        f = 200.0 * m / 3.0
        lg = m >= 15.0
        f[lg] = 1000.0 * np.exp((np.log(6.4) / 27.0) * (m[lg] - 15.0))
        return f
    fft_freqs = np.linspace(0, sr // 2, n_freq)
    f_pts = mel_to_hz(np.linspace(hz_to_mel(np.array([fmin]))[0], hz_to_mel(np.array([fmax]))[0], n_mel + 2))
    fdiff = np.diff(f_pts)
    slopes = f_pts[None, :] - fft_freqs[:, None]
    fb = np.maximum(0, np.minimum(-slopes[:, :-2] / fdiff[:-1], slopes[:, 2:] / fdiff[1:]))
    return (fb * (2.0 / (f_pts[2:n_mel + 2] - f_pts[:n_mel]))[None, :]).astype(np.float32)


class WhisperNet:
    """Backend-agnostic orchestration of WhisperModel for the reference's call.  ``ops`` provides: tensor, weight,
    logmel, conv1, conv2, layernorm, linear, self_attention, small_attention (see CudaOps)."""

    def __init__(self, state_dict, ops, heads=8):
        sd = {k: np.asarray(v, np.float32) for k, v in state_dict.items() if np.asarray(v).dtype.kind == "f"}
        self.ops, self.heads = ops, heads
        self.d = d = sd["encoder.conv2.weight"].shape[0]
        assert d == heads * 64 and sd["encoder.conv1.weight"].shape[1:] == (N_MELS, 3)
        w1 = np.zeros((d, 3, MEL_LD), np.float32)                       # [out][tap][mel padded to 96]
        w1[:, :, :N_MELS] = sd["encoder.conv1.weight"].transpose(0, 2, 1)
        self.conv1_w, self.conv1_b = ops.weight(w1.reshape(d, 3 * MEL_LD)), ops.tensor(sd["encoder.conv1.bias"])
        self.conv2_w = ops.weight(np.ascontiguousarray(sd["encoder.conv2.weight"].transpose(0, 2, 1)).reshape(d, 3 * d))
        self.conv2_b = ops.tensor(sd["encoder.conv2.bias"])
        self.enc_pos = sd["encoder.embed_positions.weight"]
        self.dec_pos, self.dec_tok = sd["decoder.embed_positions.weight"], sd["decoder.embed_tokens.weight"]
        zeros = np.zeros(d, np.float32)

        def ln(p):
            return ops.tensor(sd[p + ".weight"]), ops.tensor(sd[p + ".bias"])

        def attn(p, fused_kv_only=False):
            q, k, v = (sd[p + n + ".weight"] for n in ("q_proj", "k_proj", "v_proj"))
            out = dict(o_w=ops.weight(sd[p + "out_proj.weight"]), o_b=ops.tensor(sd[p + "out_proj.bias"]))
            if fused_kv_only:   # cross-attention: q from the decoder rows, k | v from the encoder output
                out.update(q_w=ops.weight(q), q_b=ops.tensor(sd[p + "q_proj.bias"]),
                           kv_w=ops.weight(np.concatenate([k, v], 0)),
                           kv_b=ops.tensor(np.concatenate([zeros, sd[p + "v_proj.bias"]])))
            else:               # k_proj has no bias
                out.update(qkv_w=ops.weight(np.concatenate([q, k, v], 0)),
                           qkv_b=ops.tensor(np.concatenate([sd[p + "q_proj.bias"], zeros, sd[p + "v_proj.bias"]])))
            return out

        def ffn(p):
            return dict(w1=ops.weight(sd[p + "fc1.weight"]), b1=ops.tensor(sd[p + "fc1.bias"]),
                        w2=ops.weight(sd[p + "fc2.weight"]), b2=ops.tensor(sd[p + "fc2.bias"]))
        self.enc_layers, self.dec_layers = [], []
        i = 0
        while f"encoder.layers.{i}.fc1.weight" in sd:
            p = f"encoder.layers.{i}."
            self.enc_layers.append(dict(ln1=ln(p + "self_attn_layer_norm"), att=attn(p + "self_attn."),
                                        ln2=ln(p + "final_layer_norm"), ffn=ffn(p)))
            i += 1
        self.enc_ln = ln("encoder.layer_norm")
        i = 0
        while f"decoder.layers.{i}.fc1.weight" in sd:
            p = f"decoder.layers.{i}."
            self.dec_layers.append(dict(ln1=ln(p + "self_attn_layer_norm"), att=attn(p + "self_attn."),
                                        lnc=ln(p + "encoder_attn_layer_norm"), cross=attn(p + "encoder_attn.", True),
                                        ln2=ln(p + "final_layer_norm"), ffn=ffn(p)))
            i += 1
        self.dec_ln = ln("decoder.layer_norm")

    def last_hidden_state(self, waves, start_token, n_tokens=2):
        """waves: list of 1-D float arrays (16 kHz).  Returns [B, n_tokens, d_model] (backend tensor)."""
        ops, d, H, B = self.ops, self.d, self.heads, len(waves)
        T = N_FRAMES // 2
        x = ops.conv2(ops.conv1(ops.logmel(waves), self.conv1_w, self.conv1_b), self.conv2_w, self.conv2_b,
                      ops.tensor(np.tile(self.enc_pos, (B, 1))))                       # [B * 1500, d] residual stream
        for L in self.enc_layers:
            y = ops.layernorm(x, *L["ln1"], operand=True)
            ctx = ops.self_attention(ops.linear(y, L["att"]["qkv_w"], L["att"]["qkv_b"], operand=True), B, T, H)
            x = ops.linear(ctx, L["att"]["o_w"], L["att"]["o_b"], res=x)
            y = ops.layernorm(x, *L["ln2"], operand=True)
            x = ops.linear(ops.linear(y, L["ffn"]["w1"], L["ffn"]["b1"], gelu=True, operand=True),
                           L["ffn"]["w2"], L["ffn"]["b2"], res=x)
        enc = ops.layernorm(x, *self.enc_ln, operand=True)
        y = ops.tensor(np.tile(self.dec_tok[start_token][None, :] + self.dec_pos[:n_tokens], (B, 1)))   # [B * n, d]
        for L in self.dec_layers:
            qkv = ops.linear(ops.layernorm(y, *L["ln1"], operand=True), L["att"]["qkv_w"], L["att"]["qkv_b"])
            ctx = ops.small_attention(qkv, 0, qkv, d, qkv, 2 * d, B, H, n_tokens, n_tokens, True)
            y = ops.linear(ctx, L["att"]["o_w"], L["att"]["o_b"], res=y)
            q = ops.linear(ops.layernorm(y, *L["lnc"], operand=True), L["cross"]["q_w"], L["cross"]["q_b"])
            kv = ops.linear(enc, L["cross"]["kv_w"], L["cross"]["kv_b"])                                  # [B * 1500, 2 d]
            ctx = ops.small_attention(q, 0, kv, 0, kv, d, B, H, n_tokens, T, False)
            y = ops.linear(ctx, L["cross"]["o_w"], L["cross"]["o_b"], res=y)
            h = ops.linear(ops.layernorm(y, *L["ln2"], operand=True), L["ffn"]["w1"], L["ffn"]["b1"], gelu=True, operand=True)
            y = ops.linear(h, L["ffn"]["w2"], L["ffn"]["b2"], res=y)
        return ops.layernorm(y, *self.dec_ln, operand=False).reshape(B, n_tokens, d)


class CudaOps:
    """Product backend: every op is one or two launches of libmer_b200.so kernels.  TF32 GEMMs: operands (``operand=True``
    outputs and the weights) are TF32-rounded fp32, everything else stays fp32."""

    def __init__(self, device="cuda"):
        import ctypes as C

        from .. import _lib as L
        L.check(L.lib().mer_check_device())
        self.L, self.C, self.device = L, C, torch.device(device)
        self._logmel = L.declare("mer_whisper_logmel", [C.c_void_p, C.c_int, C.c_longlong, C.c_void_p, C.c_void_p, C.c_int,
                                                        C.c_int, C.c_void_p, C.c_void_p])
        self._small = L.declare("mer_small_attention", [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                                                        C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                                        C.c_void_p])
        self.mel = self.tensor(whisper_mel_filters())

    def tensor(self, a):
        return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(self.device)

    def weight(self, a):
        return self.L.round_tf32_(self.tensor(a))

    def logmel(self, waves):
        L, B = self.L, len(waves)
        host = torch.zeros(B, N_SAMPLES, dtype=torch.float32)
        for i, w in enumerate(waves):
            n = min(len(w), N_SAMPLES)
            host[i, :n] = torch.from_numpy(np.asarray(w, np.float32)[:n])
        out = torch.empty(B, N_FRAMES, MEL_LD, dtype=torch.float32, device=self.device)
        scratch = torch.empty(B, dtype=torch.int32, device=self.device)
        L.check(self._logmel(L.ptr(host.to(self.device)), B, N_SAMPLES, L.ptr(self.mel), L.ptr(out), MEL_LD, 1,
                             L.ptr(scratch), L.stream_ptr()))
        return out

    def conv1(self, mel, w, b):
        """[B, 3000, 96] -> GELU(conv k3 p1) as a 3-tap GEMM, written into rows 1..3000 of a zeroed [B, 3002, d] buffer
        (the zero rows are conv2's padding)."""
        B, d = mel.shape[0], w.shape[0]
        out = torch.zeros(B, N_FRAMES + 2, d, dtype=torch.float32, device=self.device)
        self.L.gemm(mel.view(B * N_FRAMES, MEL_LD), w, out.view(-1, d), bias=b, gelu=True, round_out=True,
                    rows_per_batch=N_FRAMES, batches=B, a_rows_dim=N_FRAMES, K_inner=MEL_LD, taps=3, P=1,
                    a_row_stride=MEL_LD, a_batch_stride=N_FRAMES * MEL_LD, a_row0=-1,
                    out_bstride=N_FRAMES + 2, out_row0=1)
        return out

    def conv2(self, xpad, w, b, pos):
        """[B, 3002, d] (zero-padded) -> pos + GELU(conv k3 s2) = [B * 1500, d]: stride 2 through the two-phase row view."""
        B, rows, d = xpad.shape
        T = N_FRAMES // 2
        out = torch.empty(B * T, d, dtype=torch.float32, device=self.device)
        self.L.gemm(xpad.view(-1, d), w, out, bias=b, res=pos, gelu=True, rows_per_batch=T, batches=B,
                    a_rows_dim=rows // 2, K_inner=d, taps=3, P=2, a_phase_stride=d, a_row_stride=2 * d,
                    a_batch_stride=rows * d, out_bstride=T, res_bstride=T)
        return out

    def layernorm(self, x, g, b, operand):
        y = torch.empty_like(x)
        self.L.layernorm(x, g, b, y, eps=1e-5, flags=self.L.MER_LN_ROUND_TF32 if operand else 0)
        return y

    def linear(self, x, w, b, gelu=False, res=None, operand=False):
        out = torch.empty(x.shape[0], w.shape[0], dtype=torch.float32, device=self.device)
        self.L.gemm(x, w, out, bias=b, res=res, gelu=gelu, round_out=operand)
        return out

    def self_attention(self, qkv, B, T, heads):
        ctx = torch.empty(qkv.shape[0], qkv.shape[1] // 3, dtype=torch.float32, device=self.device)
        cu = torch.arange(0, (B + 1) * T, T, dtype=torch.int32, device=self.device)
        return self.L.attention(qkv, ctx, cu, T, heads, round_out=True)

    def small_attention(self, q, q0, k, k0, v, v0, B, heads, nq, nk, causal):
        L, d = self.L, heads * 64
        out = torch.empty(B * nq, d, dtype=torch.float32, device=self.device)
        f4 = lambda t, c0: self.C.c_void_p(t.data_ptr() + 4 * c0)   # noqa: E731  (column offset inside the rows)
        L.check(self._small(f4(q, q0), q.shape[1], f4(k, k0), k.shape[1], f4(v, v0), v.shape[1], B, heads, nq, nk,
                            1 if causal else 0, L.ptr(out), d, L.stream_ptr()))
        return L.round_tf32_(out)


class WhisperExtractor:
    """``extract()``'s Whisper branch for a list of waveforms: returns the arrays the reference saves (:103-110)."""

    def __init__(self, state_dict, start_token, device="cuda", heads=8, clips_per_launch=16):
        self.net = WhisperNet(state_dict, CudaOps(device), heads=heads)
        self.start_token, self.clips = int(start_token), clips_per_launch

    def extract_waves(self, waves, feature_level="UTTERANCE", save_files=None):
        res = []
        for s in range(0, len(waves), self.clips):
            feats = self.net.last_hidden_state(waves[s:s + self.clips], self.start_token).cpu().numpy()
            for f in feats:                                     # [2, D] per file
                f = np.array(f).squeeze()
                res.append(np.mean(f, axis=0) if feature_level == "UTTERANCE" and len(f.shape) != 1 else f)
        if save_files is not None:
            for path, r in zip(save_files, res):
                np.save(path, r)
        return res
