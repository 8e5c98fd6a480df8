"""dinov2-giant branch of the visual extractor (``DINO2_GIANT`` of
MERBench/feature_extraction/visual/extract_vision_huggingface.py:135-145): HF ``Dinov2Model`` with the SwiGLU MLP
(``use_swiglu_ffn``; hidden 1536, 24 heads, 40 layers), readout ``hidden_states[-1].sum(dim=1)`` per frame.

dinov2-large runs on the fused CLIP L/14 tower (``encoders.Dinov2Encoder``); the giant's width and MLP do not fit that
tower, so its layers are orchestrated over kernel-level entry points through an ``ops`` backend (TF32 linears,
``mer_layernorm`` at 1536 columns, the flash attention kernel over 257 tokens, ``mer_swiglu``), embeddings through
``PatchEmbedder`` (MER_VISION_EMBED_ONLY).  LayerScale is folded into each branch's last linear layer at load.
GPU parity test: tests/test_variants_gpu.py.
"""
from __future__ import annotations

import numpy as np
import torch


class Dinov2SwigluNet:
    """Backend-agnostic orchestration of Dinov2 layers with the SwiGLU MLP.  ``ops``: tensor, weight, layernorm,
    linear, self_attention, swiglu."""

    def __init__(self, state_dict, ops, eps=1e-6):
        sd = {k: np.asarray(v, np.float32) for k, v in state_dict.items() if k.startswith("encoder.")}
        self.ops, self.eps = ops, eps
        self.d = d = sd["encoder.layer.0.norm1.weight"].shape[0]
        self.heads = d // 64
        self.layers = []
        i = 0
        while f"encoder.layer.{i}.mlp.weights_out.weight" in sd:
            p = f"encoder.layer.{i}."
            a = p + "attention.attention."
            l1, l2 = sd[p + "layer_scale1.lambda1"], sd[p + "layer_scale2.lambda1"]
            self.layers.append(dict(
                ln1=(ops.tensor(sd[p + "norm1.weight"]), ops.tensor(sd[p + "norm1.bias"])),
                qkv_w=ops.weight(np.concatenate([sd[a + "query.weight"], sd[a + "key.weight"], sd[a + "value.weight"]], 0)),
                qkv_b=ops.tensor(np.concatenate([sd[a + "query.bias"], sd[a + "key.bias"], sd[a + "value.bias"]])),
                o_w=ops.weight(sd[p + "attention.output.dense.weight"] * l1[:, None]),
                o_b=ops.tensor(sd[p + "attention.output.dense.bias"] * l1),
                ln2=(ops.tensor(sd[p + "norm2.weight"]), ops.tensor(sd[p + "norm2.bias"])),
                w_in=ops.weight(sd[p + "mlp.weights_in.weight"]), b_in=ops.tensor(sd[p + "mlp.weights_in.bias"]),
                w_out=ops.weight(sd[p + "mlp.weights_out.weight"] * l2[:, None]),
                b_out=ops.tensor(sd[p + "mlp.weights_out.bias"] * l2)))
            i += 1
        assert self.layers, "not a SwiGLU Dinov2 checkpoint"

    def last_hidden(self, x, n_frames, tokens):
        """x: [n_frames * tokens, D] = hidden_states[0].  Returns hidden_states[-1] in the same layout."""
        ops = self.ops
        for L in self.layers:
            y = ops.layernorm(x, *L["ln1"], operand=True, eps=self.eps)
            ctx = ops.self_attention(ops.linear(y, L["qkv_w"], L["qkv_b"], operand=True), n_frames, tokens, self.heads)
            x = ops.linear(ctx, L["o_w"], L["o_b"], res=x)
            y = ops.layernorm(x, *L["ln2"], operand=True, eps=self.eps)
            x = ops.linear(ops.swiglu(ops.linear(y, L["w_in"], L["b_in"])), L["w_out"], L["b_out"], res=x)
        return x


def _cuda_ops(device):
    import ctypes as C

    from .wavlm import _cuda_ops as base

    ops = base(device)
    swiglu = ops.L.declare("mer_swiglu", [C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_void_p])

    def _swiglu(x):
        out = torch.empty(x.shape[0], x.shape[1] // 2, dtype=torch.float32, device=ops.device)
        ops.L.check(swiglu(ops.L.ptr(x), ops.L.ptr(out), x.shape[0], x.shape[1] // 2, 1, ops.L.stream_ptr()))
        return out
    ops.swiglu = _swiglu
    return ops


class Dinov2GiantEncoder:
    """``frame_features(uint8 CUDA [N, H, W, 3] BGR) -> [N, hidden]`` (the contract VisualExtractor drives); processor =
    BitImageProcessor of the checkpoint (shorter edge -> 256 bicubic, centre crop 224, rescale, ImageNet normalise)."""

    def __init__(self, state_dict, device="cuda", eps=1e-6, image=224, resize=256, mean=(0.485, 0.456, 0.406),
                 std=(0.229, 0.224, 0.225)):
        from .. import weights as W
        from ..encoders import clip_preprocess_geometry, dinov2_embedding_rows
        from .data2vec_vision import DeviceResizer, PatchEmbedder
        sd = W._np(state_dict)
        pw, cls, pos = dinov2_embedding_rows(sd, image)
        self.embed = PatchEmbedder(pw, cls + pos[0], pos[1:], device, image=image, mean=mean, std=std)
        self.device, self.hidden, self.tokens = self.embed.device, self.embed.hidden, self.embed.tokens
        self.image, self.resize_to, self._geometry = int(image), int(resize), clip_preprocess_geometry
        self.net = Dinov2SwigluNet(sd, _cuda_ops(device), eps=eps)
        self.resize = DeviceResizer(device)

    def frame_features(self, frames_bgr_u8):
        assert frames_bgr_u8.dtype == torch.uint8 and frames_bgr_u8.is_cuda and frames_bgr_u8.dim() == 4
        n, h, w, _ = frames_bgr_u8.shape
        nh, nw, _, _ = self._geometry(h, w, self.resize_to)
        frames = self.resize(frames_bgr_u8.contiguous(), nh, nw, 1)
        x = self.embed(frames, (nh - self.image) // 2, (nw - self.image) // 2)
        return self.net.last_hidden(x, n, self.tokens).view(n, self.tokens, self.hidden).sum(dim=1)
