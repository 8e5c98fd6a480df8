"""data2vec-vision branch of the visual extractor (``data2vec-vision-base-ft1k``: HF ``Data2VecVisionModel``, the BEiT
graph; MERBench/feature_extraction/visual/extract_vision_huggingface.py:124-133: every frame -> processor ->
``hidden_states[-1].sum(dim=1)``).

BEiT layers add a per-layer relative position bias to the attention scores, which the tensor-core attention kernels do not
take; the embeddings run through ``mer_clip_vision_forward`` (MER_VISION_EMBED_ONLY: patch gather + GEMM + class row)
and the layers are orchestrated over kernel-level entry points through an ``ops`` backend (TF32 linears,
``mer_layernorm``, ``mer_biased_attention``), so that the orchestration runs against the oracle with a torch backend on
CPU (tests/test_host_logic.py).  LayerScale is folded into each branch's last linear layer at load.
GPU parity test: tests/test_variants_gpu.py.
"""
from __future__ import annotations

import numpy as np
import torch


def relative_position_index(window=14):
    """Data2VecVisionRelativePositionBias.generate_relative_position_index: int64 [1 + w*w, 1 + w*w] into the
    (2w-1)^2 + 3 table (last three rows: cls->token, token->cls, cls->cls)."""
    n = (2 * window - 1) ** 2 + 3
    ys, xs = np.divmod(np.arange(window * window), window)
    rel = (ys[:, None] - ys[None, :] + window - 1) * (2 * window - 1) + (xs[:, None] - xs[None, :] + window - 1)
    idx = np.zeros((window * window + 1,) * 2, np.int64)
    idx[1:, 1:] = rel
    idx[0, :] = n - 3
    idx[:, 0] = n - 2
    idx[0, 0] = n - 1
    return idx


class BeitNet:
    """Backend-agnostic orchestration of the Data2VecVision / BEiT layers.  ``ops``: tensor, weight, operand,
    layernorm, linear, biased_attention."""

    def __init__(self, state_dict, ops, eps=1e-12, window=14):
        sd = {k: np.asarray(v, np.float32) for k, v in state_dict.items()}
        self.ops, self.eps = ops, eps
        self.d = d = sd["embeddings.cls_token"].shape[-1]
        self.heads, self.tokens = d // 64, window * window + 1
        idx = relative_position_index(window)
        zeros = np.zeros(d, np.float32)
        self.layers = []
        i = 0
        while f"encoder.layer.{i}.output.dense.weight" in sd:
            p = f"encoder.layer.{i}."
            a = p + "attention.attention."
            l1, l2 = sd[p + "lambda_1"], sd[p + "lambda_2"]
            # per-layer table (data2vec-vision, BEiT fine-tuned), else the encoder's shared one, else no bias
            table = sd.get(a + "relative_position_bias.relative_position_bias_table",
                           sd.get("encoder.relative_position_bias.relative_position_bias_table"))
            if table is None:
                table = np.zeros(((2 * window - 1) ** 2 + 3, self.heads), np.float32)
            assert table.shape == ((2 * window - 1) ** 2 + 3, self.heads), table.shape
            self.layers.append(dict(
                ln1=(ops.tensor(sd[p + "layernorm_before.weight"]), ops.tensor(sd[p + "layernorm_before.bias"])),
                qkv_w=ops.weight(np.concatenate([sd[a + "query.weight"], sd[a + "key.weight"], sd[a + "value.weight"]], 0)),
                qkv_b=ops.tensor(np.concatenate([sd[a + "query.bias"], zeros, sd[a + "value.bias"]])),   # key: no bias
                bias=ops.tensor(np.ascontiguousarray(table[idx].transpose(2, 0, 1))),                  # [heads, T, T]
                o_w=ops.weight(sd[p + "attention.output.dense.weight"] * l1[:, None]),
                o_b=ops.tensor(sd[p + "attention.output.dense.bias"] * l1),
                ln2=(ops.tensor(sd[p + "layernorm_after.weight"]), ops.tensor(sd[p + "layernorm_after.bias"])),
                w1=ops.weight(sd[p + "intermediate.dense.weight"]), b1=ops.tensor(sd[p + "intermediate.dense.bias"]),
                w2=ops.weight(sd[p + "output.dense.weight"] * l2[:, None]), b2=ops.tensor(sd[p + "output.dense.bias"] * l2)))
            i += 1

    def last_hidden(self, x, n_frames):
        """x: [n_frames * tokens, D] = hidden_states[0].  Returns hidden_states[-1] in the same layout."""
        ops = self.ops
        for L in self.layers:
            y = ops.layernorm(x, *L["ln1"], operand=True, eps=self.eps)
            ctx = ops.biased_attention(ops.linear(y, L["qkv_w"], L["qkv_b"]), L["bias"], None, n_frames, self.tokens, self.heads)
            x = ops.linear(ctx, L["o_w"], L["o_b"], res=x)
            y = ops.layernorm(x, *L["ln2"], operand=True, eps=self.eps)
            x = ops.linear(ops.linear(y, L["w1"], L["b1"], gelu=True, operand=True), L["w2"], L["b2"], res=x)
        return x


class PatchEmbedder:
    """``hidden_states[0]`` of a ViT-style model on the device: mer_clip_vision_forward with MER_VISION_EMBED_ONLY
    (BGR -> RGB, rescale, normalise, patch gather, TF32 patch GEMM, class row).  ``cls_row`` [D] = class token (+ its
    position), ``patch_rows`` [tokens - 1, D] = what is added to every frame's patch tokens (positions + conv bias).
    Shared by the host-orchestrated visual branches (data2vec-vision, dinov2-giant)."""

    def __init__(self, patch_weight, cls_row, patch_rows, device, image=224, mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5)):
        import ctypes as C

        from .. import _lib as L
        from .. import weights as W
        from ..encoders import MerClipVisionModel, _Workspace
        L.check(L.lib().mer_check_device())
        self.device = torch.device(device)
        pw = np.asarray(patch_weight, np.float32)
        D, _, p, _ = pw.shape
        assert D % 256 == 0 and image % p == 0, (pw.shape, image)
        self.hidden, self.image, self.tokens = int(D), int(image), (image // p) ** 2 + 1
        assert np.shape(cls_row) == (D,) and np.shape(patch_rows) == (self.tokens - 1, D)
        pk = self.pk = W.Packed(self.device)
        kpad = (3 * p * p + 31) // 32 * 32
        wflat = np.zeros((D, kpad), np.float32)
        wflat[:, :3 * p * p] = pw.reshape(D, 3 * p * p)
        m = MerClipVisionModel()
        m.n_layers, m.ln_eps = 0, 1e-6
        m.hidden, m.ffn, m.heads, m.patch, m.image, m.proj_dim, m.kpad = D, 4 * D, D // 64, p, image, D, kpad
        m.gemm_mode, m.variant = L.MER_GEMM_TF32, 2                                      # MER_VISION_EMBED_ONLY
        m.mean, m.std = (C.c_float * 3)(*mean), (C.c_float * 3)(*std)
        m.patch_w = pk.keep(wflat, tf32=True).data_ptr()
        m.cls_pos0 = pk.keep(np.asarray(cls_row, np.float32)).data_ptr()
        m.pos_rest = pk.keep(np.asarray(patch_rows, np.float32)).data_ptr()
        self.model = m
        self.ws = _Workspace(self.device)
        lib = L.lib()
        lib.mer_clip_vision_workspace_bytes.restype = C.c_longlong
        lib.mer_clip_vision_workspace_bytes.argtypes = [C.POINTER(MerClipVisionModel), C.c_int]
        self._fwd = L.declare("mer_clip_vision_forward", [C.POINTER(MerClipVisionModel), C.c_void_p, C.c_int, C.c_int,
                                                          C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_longlong,
                                                          C.c_void_p, C.c_void_p, C.c_void_p])
        self._L, self._C = L, C

    def __call__(self, frames_u8, crop_y0=0, crop_x0=0):
        """frames: uint8 CUDA [n, H, W, 3] BGR, already resized; the image x image window at (crop_y0, crop_x0) is
        embedded.  Returns fp32 [n * tokens, D]."""
        L, C = self._L, self._C
        n, h, w, _ = frames_u8.shape
        assert crop_y0 + self.image <= h and crop_x0 + self.image <= w
        ws = self.ws.get(L.lib().mer_clip_vision_workspace_bytes(C.byref(self.model), n))
        x = torch.empty(n * self.tokens, self.hidden, dtype=torch.float32, device=self.device)
        L.check(self._fwd(C.byref(self.model), L.ptr(frames_u8), n, h, w, crop_y0, crop_x0, L.ptr(ws), ws.numel(),
                          L.ptr(x), None, L.stream_ptr()))
        return x


class DeviceResizer:
    """Pillow-exact uint8 resize on the device (mer_resize_u8; filter 0 = bilinear, 1 = bicubic)."""

    def __init__(self, device):
        import ctypes as C

        from .. import _lib as L
        from ..encoders import _Workspace
        self.device, self.ws, self._L = torch.device(device), _Workspace(torch.device(device)), L
        L.lib().mer_resize_workspace_bytes.restype = C.c_longlong
        L.lib().mer_resize_workspace_bytes.argtypes = [C.c_int] * 5
        self._resize = L.declare("mer_resize_u8", [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                                   C.c_int, C.c_int, C.c_void_p, C.c_void_p])

    def __call__(self, frames_u8, out_h, out_w, filter=0):
        L = self._L
        n, h, w, _ = frames_u8.shape
        if (h, w) == (out_h, out_w):
            return frames_u8
        out = torch.empty(n, out_h, out_w, 3, dtype=torch.uint8, device=self.device)
        ws = self.ws.get(max(int(L.lib().mer_resize_workspace_bytes(n, h, w, out_h, out_w)), 1))
        L.check(self._resize(L.ptr(frames_u8), n, h, w, L.ptr(out), out_h, out_w, filter, L.ptr(ws), L.stream_ptr()))
        return out


class Data2VecVisionEncoder:
    """``frame_features(uint8 CUDA [N, H, W, 3] BGR) -> [N, hidden]`` (the contract VisualExtractor drives).  Processor:
    BeitImageProcessor as configured by the checkpoint's preprocessor_config.json — resize to size x size
    (``resample`` 2 = bilinear, 3 = bicubic; Pillow-exact on the device), optional centre crop, rescale, normalise;
    defaults = the 224 bilinear / mean 0.5 / std 0.5 processor of the reference's ViT-style checkpoints."""

    def __init__(self, state_dict, device="cuda", eps=1e-12, image=224, size=224, resample=2, center_crop=False,
                 mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5)):
        from .. import weights as W
        from .wavlm import _cuda_ops
        sd = W._np(state_dict)
        pw = np.asarray(sd["embeddings.patch_embeddings.projection.weight"], np.float32)
        D, p = pw.shape[0], pw.shape[-1]
        assert D in (768, 1024) and size >= image, (pw.shape, image, size)
        self.hidden, self.image, self.size = int(D), int(image), int(size)
        self.filter, self.center_crop = {2: 0, 3: 1}[int(resample)], bool(center_crop)
        self.tokens = (image // p) ** 2 + 1
        self.net = BeitNet(sd, _cuda_ops(device), eps=eps, window=image // p)
        # no absolute positions: the residual operand of the patch GEMM carries the conv bias alone
        bias = np.asarray(sd["embeddings.patch_embeddings.projection.bias"], np.float32)
        self.embed = PatchEmbedder(pw, np.asarray(sd["embeddings.cls_token"], np.float32).reshape(D),
                                   np.tile(bias, (self.tokens - 1, 1)), device, image=image, mean=mean, std=std)
        self.device = self.embed.device
        self.resize = DeviceResizer(device)

    @classmethod
    def from_pretrained(cls, model_dir, device="cuda"):
        import json
        import os

        from . import common
        kw = {}
        pc = os.path.join(model_dir, "preprocessor_config.json")
        if os.path.exists(pc):
            cfg = json.load(open(pc))
            size, crop = cfg.get("size", 224), cfg.get("crop_size", 224)
            size = size.get("height", 224) if isinstance(size, dict) else size
            crop = crop.get("height", 224) if isinstance(crop, dict) else crop
            do_crop = bool(cfg.get("do_center_crop", False))
            kw.update(size=int(size), image=int(crop if do_crop else size), center_crop=do_crop,
                      resample=int(cfg.get("resample", 2)), mean=cfg.get("image_mean", (0.5,) * 3),
                      std=cfg.get("image_std", (0.5,) * 3))
        return cls(common.load_hf_state_dict(model_dir), device=device, **kw)

    def frame_features(self, frames_bgr_u8):
        assert frames_bgr_u8.dtype == torch.uint8 and frames_bgr_u8.is_cuda and frames_bgr_u8.dim() == 4
        frames = self.resize(frames_bgr_u8.contiguous(), self.size, self.size, self.filter)
        off = (self.size - self.image) // 2
        n = frames.shape[0]
        x = self.embed(frames, off, off)
        return self.net.last_hidden(x, n).view(n, self.tokens, self.hidden).sum(dim=1)
