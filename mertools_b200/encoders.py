"""Device-side encoder objects: the "model" seam of the reference extractors.

Each class takes an HF-named ``state_dict`` (what ``AutoModel.from_pretrained(...).state_dict()``
holds in the reference, extract_*_huggingface.py) and exposes the fused forward + readout that the
reference spells as ``model(x, output_hidden_states=True).hidden_states`` followed by
``torch.stack(hs)[...]`` arithmetic.  All compute happens inside libmer_b200.so.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from . import _lib as L
from . import weights as W


class MerVitModel(C.Structure):
    _fields_ = [("n_layers", C.c_int), ("ln_eps", C.c_float), ("gemm_mode", C.c_int), ("patch_w", C.c_void_p),
                ("patch_b", C.c_void_p), ("cls_pos0", C.c_void_p), ("pos_rest", C.c_void_p),
                ("layers", C.POINTER(W.MerLayerWeights))]


class _Workspace:
    """Grow-only device scratch buffer (torch owns the memory)."""

    def __init__(self, device):
        self.device = device
        self.buf = None

    def get(self, nbytes):
        if self.buf is None or self.buf.numel() < nbytes:
            self.buf = None
            self.buf = torch.empty(int(nbytes), dtype=torch.uint8, device=self.device)
        return self.buf


class VitEncoder:
    """ViT-B/16 frame encoder (HF ``ViTModel``) + ``hidden_states[-1].sum(dim=1)`` readout.

    Reference: MERBench/feature_extraction/visual/extract_vision_huggingface.py:135-145.

    precision: "f16" (default) runs the 12 layers' linear layers on fp16 operands (LayerNorm / attention /
    GELU outputs and the weights stored as fp16, fp32 accumulation, fp32 residual stream); "tf32" keeps
    them as tf32-rounded fp32.  Both carry a 10-bit mantissa, i.e. the same products; fp16 halves the
    operand traffic and doubles the tensor-pipe rate.  MER_VIT_PRECISION overrides the default."""

    def __init__(self, state_dict, device="cuda", ln_eps=1e-12, precision=None):
        L.check(L.lib().mer_check_device())
        sd = W._np(state_dict)
        self.device = torch.device(device)
        self.pk = W.Packed(self.device)
        self.n_layers = W.count_layers(sd, VIT_PROBE)
        pw = sd["embeddings.patch_embeddings.projection.weight"]
        assert pw.shape == (768, 3, 16, 16), f"ViT-B/16 only, got patch weight {pw.shape}"
        pos = sd["embeddings.position_embeddings"][0]
        assert pos.shape == (197, 768), f"224x224 / patch 16 only, got pos {pos.shape}"
        self.patch_w = self.pk.keep(pw.reshape(768, 768), tf32=True)
        self.patch_b = self.pk.keep(sd["embeddings.patch_embeddings.projection.bias"])
        self.cls_pos0 = self.pk.keep(sd["embeddings.cls_token"].reshape(768) + pos[0])
        self.pos_rest = self.pk.keep(pos[1:])
        import os
        self.precision = precision or os.environ.get("MER_VIT_PRECISION", "f16")
        assert self.precision in ("f16", "tf32"), self.precision
        f16 = self.precision == "f16"
        self.layers = W.pack_layers(sd, W.VIT_NAMES, self.n_layers, self.pk, f16=f16)
        self.model = MerVitModel(self.n_layers, ln_eps, L.MER_GEMM_F16 if f16 else L.MER_GEMM_TF32,
                                 self.patch_w.data_ptr(),
                                 self.patch_b.data_ptr(), self.cls_pos0.data_ptr(),
                                 self.pos_rest.data_ptr(), self.layers)
        self.ws = _Workspace(self.device)
        self._fwd = L.declare("mer_vit_forward", [C.POINTER(MerVitModel), C.c_void_p, C.c_int,
                                                  C.c_void_p, C.c_longlong, C.c_void_p,
                                                  C.c_void_p, C.c_void_p])
        L.lib().mer_vit_workspace_bytes.restype = C.c_longlong
        L.lib().mer_vit_workspace_bytes.argtypes = [C.c_int]
        self._resize = L.declare("mer_resize_bilinear_u8", [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                                            C.c_int, C.c_int, C.c_void_p, C.c_void_p])
        L.lib().mer_resize_workspace_bytes.restype = C.c_longlong
        L.lib().mer_resize_workspace_bytes.argtypes = [C.c_int] * 5
        self.ws_resize = _Workspace(self.device)

    def resize_frames(self, frames_u8: torch.Tensor, size=224):
        """PIL-bilinear resize of uint8 CUDA frames [N,H,W,3] to [N,size,size,3] (the resize step of HF
        ViTImageProcessor, extract_vision_huggingface.py:137-138), bit-exact, on the device."""
        assert frames_u8.dtype == torch.uint8 and frames_u8.is_cuda and frames_u8.dim() == 4 \
            and frames_u8.shape[-1] == 3, f"frames must be uint8 CUDA [N,H,W,3], got {tuple(frames_u8.shape)}"
        n, h, w, _ = frames_u8.shape
        if (h, w) == (size, size):
            return frames_u8
        frames_u8 = frames_u8.contiguous()
        out = torch.empty(n, size, size, 3, dtype=torch.uint8, device=self.device)
        need = L.lib().mer_resize_workspace_bytes(n, h, w, size, size)
        ws = self.ws_resize.get(max(int(need), 1))
        L.check(self._resize(L.ptr(frames_u8), n, h, w, L.ptr(out), size, size, L.ptr(ws), L.stream_ptr()))
        return out

    def frame_features(self, frames_bgr_u8: torch.Tensor, return_hidden=False):
        """frames: uint8 CUDA tensor [N,H,W,3] (BGR); frames that are not 224x224 are resized first
        (PIL bilinear, as the HF processor does).  Returns [N,768] fp32 (CUDA)."""
        assert frames_bgr_u8.dtype == torch.uint8 and frames_bgr_u8.is_cuda
        frames = self.resize_frames(frames_bgr_u8, 224).contiguous()
        n = frames.shape[0]
        need = L.lib().mer_vit_workspace_bytes(n)
        ws = self.ws.get(need)
        out = torch.empty(n, 768, dtype=torch.float32, device=self.device)
        hidden = None
        if return_hidden:
            hidden = torch.empty(self.n_layers + 1, n * 197, 768, dtype=torch.float32,
                                 device=self.device)
        L.check(self._fwd(C.byref(self.model), L.ptr(frames), n, L.ptr(ws), ws.numel(),
                          L.ptr(out), L.ptr(hidden), L.stream_ptr()))
        if return_hidden:
            return out, hidden.view(self.n_layers + 1, n, 197, 768)
        return out


    def clip_features(self, frames_bgr_u8: torch.Tensor, frames_per_clip: int):
        """UTTERANCE-level features of equal-length clips: mean over each clip's frame features
        (np.mean(axis=0) at extract_vision_huggingface.py:187-188), on the device.  [C,768]."""
        n = frames_bgr_u8.shape[0]
        assert n % frames_per_clip == 0
        c = n // frames_per_clip
        ff = self.frame_features(frames_bgr_u8)
        key = (c, frames_per_clip)
        if getattr(self, "_clip_key", None) != key:
            self._clip_off = torch.arange(c + 1, dtype=torch.int32, device=self.device) * frames_per_clip
            self._clip_key = key
        out = torch.empty(c, 768, dtype=torch.float32, device=self.device)
        seg = L.declare("mer_segment_reduce", [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                               C.c_int, C.c_void_p, C.c_void_p])
        L.check(seg(L.ptr(ff), L.ptr(self._clip_off), L.ptr(self._clip_off[1:]), c, 768, 1, L.ptr(out),
                    L.stream_ptr()))
        return out


VIT_PROBE = "encoder.layer.{i}.layernorm_before.weight"


class MerNormWeights(C.Structure):
    _fields_ = [("g", C.c_void_p), ("b", C.c_void_p)]


class MerClipVisionModel(C.Structure):
    _fields_ = [("n_layers", C.c_int), ("ln_eps", C.c_float), ("hidden", C.c_int), ("ffn", C.c_int),
                ("heads", C.c_int), ("patch", C.c_int), ("image", C.c_int), ("proj_dim", C.c_int),
                ("kpad", C.c_int), ("gemm_mode", C.c_int), ("mean", C.c_float * 3), ("std", C.c_float * 3),
                ("patch_w", C.c_void_p), ("cls_pos0", C.c_void_p), ("pos_rest", C.c_void_p),
                ("pre_ln_g", C.c_void_p), ("pre_ln_b", C.c_void_p), ("post_ln_g", C.c_void_p),
                ("post_ln_b", C.c_void_p), ("proj_w", C.c_void_p), ("layers", C.POINTER(W.MerLayerWeights)), ("variant", C.c_int),
                ("rope_cos", C.c_void_p), ("rope_sin", C.c_void_p), ("rope_rows", C.c_int),
                ("ffn_norms", C.POINTER(MerNormWeights))]


MER_VISION_EVA02 = 3


CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


def clip_preprocess_geometry(h, w, size=224):
    """(new_h, new_w, crop_y0, crop_x0) of HF CLIPImageProcessor: the shorter edge becomes ``size`` (the longer
    one int(size * long / short)), then a centered size x size crop."""
    short, long = (w, h) if w <= h else (h, w)
    new_long = int(size * long / short)
    nh, nw = (new_long, size) if w <= h else (size, new_long)
    return nh, nw, (nh - size) // 2, (nw - size) // 2


def fold_conv_bn(w, gamma, beta, mean, var, eps=1e-5):
    """Eval-mode BatchNorm folded into the preceding bias-free convolution (float64 math):
    w' = w * gamma / sqrt(var + eps), b' = beta - mean * gamma / sqrt(var + eps)."""
    scale = np.asarray(gamma, np.float64) / np.sqrt(np.asarray(var, np.float64) + eps)
    return np.asarray(w, np.float64) * scale[:, None, None, None], \
        np.asarray(beta, np.float64) - np.asarray(mean, np.float64) * scale


class ClipVisionEncoder:
    """CLIP vision tower + projection (HF ``CLIPModel.get_image_features``) for clip-vit-base-patch32 and
    clip-vit-large-patch14, including the CLIPImageProcessor steps (bicubic resize of the shorter edge to
    224, center crop, rescale, normalise) on the device.

    Reference: MERBench/feature_extraction/visual/extract_vision_huggingface.py:114-122."""

    def __init__(self, state_dict, device="cuda", ln_eps=1e-5, image=224, precision=None, variant=0, mean=CLIP_MEAN,
                 std=CLIP_STD, resize=None):
        """variant / mean / std / resize: set by Dinov2Encoder (same tower, MER_VISION_DINOV2 readout).
        precision: None = "f16" up to 249 tokens per frame (B/32), else "tf32" (L/14: attention on fp16 q | k | V^T
        between tf32 linear layers); "f16" forces fp16 linear layers for longer sequences too (L/14: attention then
        runs the fp16 V^T kernel, past 505 tokens the fp32-operand kernel of attention.cu; env MER_CLIP_PRECISION=f16;
        not yet measured)."""
        L.check(L.lib().mer_check_device())
        sd = W._np(state_dict)
        self.device = torch.device(device)
        pk = self.pk = W.Packed(self.device)
        v = "vision_model."
        self.n_layers = W.count_layers(sd, v + "encoder.layers.{i}.layer_norm1.weight")
        pw = sd[v + "embeddings.patch_embedding.weight"]
        D, _, p, _ = pw.shape
        pos = sd[v + "embeddings.position_embedding.weight"]
        assert D in (768, 1024) and image % p == 0 and pos.shape == ((image // p) ** 2 + 1, D), (pw.shape, pos.shape)
        self.hidden, self.patch, self.image = int(D), int(p), image
        self.tokens = (image // p) ** 2 + 1
        self.variant, self.resize = int(variant), int(resize or image)
        self.proj_dim = int(sd["visual_projection.weight"].shape[0]) if variant == 0 else int(D)
        ffn = int(sd[v + "encoder.layers.0.mlp.fc2.weight"].shape[1])
        kpad = (3 * p * p + 31) // 32 * 32
        wflat = np.zeros((D, kpad), np.float32)
        wflat[:, :3 * p * p] = pw.reshape(D, 3 * p * p)
        # fp16 linear layers by default up to 249 tokens per frame: B/32 yes, L/14 (257) runs TF32
        import os
        precision = precision or os.environ.get("MER_CLIP_PRECISION")
        assert precision in (None, "f16", "tf32"), precision
        self.precision = precision or ("f16" if self.tokens <= 249 else "tf32")
        f16 = self.precision == "f16"
        self.layers = W.pack_layers(sd, W.CLIP_NAMES, self.n_layers, pk, f16=f16)
        m = MerClipVisionModel()
        m.n_layers, m.ln_eps = self.n_layers, ln_eps
        m.hidden, m.ffn, m.heads, m.patch, m.image, m.proj_dim, m.kpad = D, ffn, D // 64, p, image, self.proj_dim, kpad
        m.gemm_mode = L.MER_GEMM_F16 if f16 else L.MER_GEMM_TF32
        m.mean = (C.c_float * 3)(*mean)
        m.std = (C.c_float * 3)(*std)
        m.patch_w = pk.keep(wflat, tf32=True).data_ptr()
        m.cls_pos0 = pk.keep(sd[v + "embeddings.class_embedding"].reshape(D) + pos[0]).data_ptr()
        m.pos_rest = pk.keep(pos[1:]).data_ptr()
        m.variant = self.variant
        if self.variant == 0:
            m.pre_ln_g = pk.keep(sd[v + "pre_layrnorm.weight"]).data_ptr()
            m.pre_ln_b = pk.keep(sd[v + "pre_layrnorm.bias"]).data_ptr()
            m.post_ln_g = pk.keep(sd[v + "post_layernorm.weight"]).data_ptr()
            m.post_ln_b = pk.keep(sd[v + "post_layernorm.bias"]).data_ptr()
            m.proj_w = pk.keep(sd["visual_projection.weight"], tf32=True).data_ptr()
        elif self.variant == MER_VISION_EVA02:
            m.post_ln_g = pk.keep(sd[v + "post_layernorm.weight"]).data_ptr()
            m.post_ln_b = pk.keep(sd[v + "post_layernorm.bias"]).data_ptr()
            self.ffn_norms = (MerNormWeights * self.n_layers)()
            for i in range(self.n_layers):
                n_ = f"{v}encoder.layers.{i}.mlp.norm."
                self.ffn_norms[i].g = pk.keep(sd[n_ + "weight"]).data_ptr()
                self.ffn_norms[i].b = pk.keep(sd[n_ + "bias"]).data_ptr()
            m.ffn_norms = self.ffn_norms
            cos, sin = eva02_rope_tables(image // p)
            m.rope_cos, m.rope_sin = pk.keep(cos).data_ptr(), pk.keep(sin).data_ptr()
            m.rope_rows = cos.shape[0]
        m.layers = self.layers
        self.model = m
        self.ws, self.ws_resize = _Workspace(self.device), _Workspace(self.device)
        lib = L.lib()
        lib.mer_clip_vision_workspace_bytes.restype = C.c_longlong
        lib.mer_clip_vision_workspace_bytes.argtypes = [C.POINTER(MerClipVisionModel), C.c_int]
        lib.mer_resize_workspace_bytes.restype = C.c_longlong
        lib.mer_resize_workspace_bytes.argtypes = [C.c_int] * 5
        self._fwd = L.declare("mer_clip_vision_forward", [C.POINTER(MerClipVisionModel), C.c_void_p, C.c_int, C.c_int,
                                                          C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_longlong,
                                                          C.c_void_p, C.c_void_p, C.c_void_p])
        self._resize = L.declare("mer_resize_u8", [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                                   C.c_int, C.c_int, C.c_void_p, C.c_void_p])

    def preprocess_geometry(self, h, w):
        """(new_h, new_w, crop_y0, crop_x0) of CLIPImageProcessor: shorter edge -> image, center crop
        (Dinov2Encoder: shorter edge -> 256, then the 224 crop; Eva02Encoder overrides the crop rule)."""
        nh, nw, _, _ = clip_preprocess_geometry(h, w, self.resize)
        return nh, nw, (nh - self.image) // 2, (nw - self.image) // 2

    def frame_features(self, frames_bgr_u8: torch.Tensor, return_hidden=False):
        """frames: uint8 CUDA [N, H, W, 3] (BGR).  Returns image embeddings [N, proj_dim] fp32 (CUDA)."""
        assert frames_bgr_u8.dtype == torch.uint8 and frames_bgr_u8.is_cuda and frames_bgr_u8.dim() == 4
        frames = frames_bgr_u8.contiguous()
        n, h, w, _ = frames.shape
        nh, nw, y0, x0 = self.preprocess_geometry(h, w)
        if (nh, nw) != (h, w):
            out = torch.empty(n, nh, nw, 3, dtype=torch.uint8, device=self.device)
            need = L.lib().mer_resize_workspace_bytes(n, h, w, nh, nw)
            ws = self.ws_resize.get(max(int(need), 1))
            L.check(self._resize(L.ptr(frames), n, h, w, L.ptr(out), nh, nw, 1, L.ptr(ws), L.stream_ptr()))
            frames = out
        need = L.lib().mer_clip_vision_workspace_bytes(C.byref(self.model), n)
        ws = self.ws.get(need)
        emb = torch.empty(n, self.proj_dim, dtype=torch.float32, device=self.device)
        hidden = (torch.empty(self.n_layers + 1, n * self.tokens, self.hidden, dtype=torch.float32, device=self.device)
                  if return_hidden else None)
        L.check(self._fwd(C.byref(self.model), L.ptr(frames), n, nh, nw, y0, x0, L.ptr(ws), ws.numel(), L.ptr(emb),
                          L.ptr(hidden), L.stream_ptr()))
        if return_hidden:
            return emb, hidden.view(self.n_layers + 1, n, self.tokens, self.hidden)
        return emb


def dinov2_embedding_rows(sd, image=224):
    """(patch conv weight [D, 3, p, p], class token [D], position rows [1 + g*g, D]) of HF ``Dinov2Embeddings`` at an
    ``image`` x ``image`` input: the position table interpolated to the g x g patch grid (bicubic, align_corners=False:
    interpolate_pos_encoding of transformers 5.x) with the patch-conv bias folded into its patch rows."""
    pw = np.asarray(sd["embeddings.patch_embeddings.projection.weight"], np.float32)
    D, _, p, _ = pw.shape
    g = image // p
    pos = torch.from_numpy(np.asarray(sd["embeddings.position_embeddings"], np.float32))
    side = int(round((pos.shape[1] - 1) ** 0.5))
    assert side * side + 1 == pos.shape[1], pos.shape
    if side != g:
        grid = pos[:, 1:].reshape(1, side, side, D).permute(0, 3, 1, 2)
        grid = torch.nn.functional.interpolate(grid, size=(g, g), mode="bicubic", align_corners=False)
        pos = torch.cat([pos[:, :1], grid.permute(0, 2, 3, 1).reshape(1, g * g, D)], dim=1)
    pos = pos[0].numpy().copy()
    pos[1:] += np.asarray(sd["embeddings.patch_embeddings.projection.bias"], np.float32)
    return pw, np.asarray(sd["embeddings.cls_token"], np.float32).reshape(D), pos


def dinov2_to_clip_layout(state_dict, image=224):
    """HF ``Dinov2Model`` tensors re-expressed in the layout of the CLIP tower (what mer_clip_vision_forward walks), so
    that DINOv2 needs no kernel of its own:  the position table is interpolated to the image grid (bicubic,
    align_corners=False: Dinov2Embeddings.interpolate_pos_encoding of transformers 5.x), the patch-conv bias is folded
    into the patch rows of the position table (both are added to every patch token), LayerScale is folded into the
    branch's last linear layer (lambda * (W x + b) = (lambda W) x + lambda b).  Pure numpy / torch-CPU weight
    preparation, checked on CPU against HF in tests/test_host_logic.py."""
    sd = W._np(state_dict)
    pw, cls, pos = dinov2_embedding_rows(sd, image)
    v = "vision_model."
    out = {v + "embeddings.patch_embedding.weight": pw, v + "embeddings.class_embedding": cls,
           v + "embeddings.position_embedding.weight": pos}
    i = 0
    while f"encoder.layer.{i}.mlp.fc2.weight" in sd:
        assert f"encoder.layer.{i}.mlp.fc1.weight" in sd, "SwiGLU MLP (dinov2-giant) is not supported"
        s_, d_ = f"encoder.layer.{i}.", f"{v}encoder.layers.{i}."
        l1 = np.asarray(sd[s_ + "layer_scale1.lambda1"], np.float32)
        l2 = np.asarray(sd[s_ + "layer_scale2.lambda1"], np.float32)
        for a, b in (("norm1", "layer_norm1"), ("norm2", "layer_norm2"), ("attention.attention.query", "self_attn.q_proj"),
                     ("attention.attention.key", "self_attn.k_proj"), ("attention.attention.value", "self_attn.v_proj"),
                     ("mlp.fc1", "mlp.fc1")):
            out[d_ + b + ".weight"], out[d_ + b + ".bias"] = sd[s_ + a + ".weight"], sd[s_ + a + ".bias"]
        out[d_ + "self_attn.out_proj.weight"] = np.asarray(sd[s_ + "attention.output.dense.weight"], np.float32) * l1[:, None]
        out[d_ + "self_attn.out_proj.bias"] = np.asarray(sd[s_ + "attention.output.dense.bias"], np.float32) * l1
        out[d_ + "mlp.fc2.weight"] = np.asarray(sd[s_ + "mlp.fc2.weight"], np.float32) * l2[:, None]
        out[d_ + "mlp.fc2.bias"] = np.asarray(sd[s_ + "mlp.fc2.bias"], np.float32) * l2
        i += 1
    return out


class Dinov2Encoder(ClipVisionEncoder):
    """HF ``Dinov2Model`` (dinov2-large: 24 layers, hidden 1024, patch 14, 257 tokens at the 224 crop) with the reference's
    readout ``hidden_states[-1].sum(dim=1)`` per frame, on the CLIP L/14 tower kernels (MER_VISION_DINOV2): BitImageProcessor
    steps on the device (shorter edge -> 256 bicubic, centre crop 224, rescale, ImageNet normalise).  ``frame_features``
    returns [N, hidden].  dinov2-giant (SwiGLU MLP, hidden 1536) is not supported.

    Reference: MERBench/feature_extraction/visual/extract_vision_huggingface.py:135-145.  Not yet run on a GPU."""

    def __init__(self, state_dict, device="cuda", ln_eps=1e-6, image=224, resize=256, precision=None,
                 mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225)):
        super().__init__(dinov2_to_clip_layout(state_dict, image), device=device, ln_eps=ln_eps, image=image,
                         precision=precision, variant=1, mean=mean, std=std, resize=resize)


def eva02_rope_tables(grid, head_dim=64, temperature=10000.0):
    """(cos, sin) float32 [grid * grid, head_dim / 2] of timm ``RotaryEmbeddingCat(head_dim, in_pixels=False,
    feat_shape=(grid, grid), ref_feat_shape=(grid, grid))``, one entry per rotated pair (timm repeats each twice):
    bands[j] = 1 / temperature^(j / nb) (nb = head_dim / 4), patch (r, c) in row-major order, pairs [0, nb) at angle
    r * bands, pairs [nb, 2 nb) at c * bands.  Built with torch in float32 in timm's order of operations, so the tables
    are the ones the reference's model holds."""
    nb = head_dim // 4
    bands = 1.0 / (temperature ** (torch.arange(0, nb, 1, dtype=torch.int64).to(torch.float32) / nb))
    t = [torch.arange(grid, dtype=torch.int64).to(torch.float32) / grid * grid for _ in range(2)]
    pos = torch.stack(torch.meshgrid(*t, indexing="ij"), dim=-1).unsqueeze(-1) * bands   # [g, g, 2, nb]
    return pos.cos().reshape(grid * grid, 2 * nb).numpy(), pos.sin().reshape(grid * grid, 2 * nb).numpy()


EVA02_BLOCK_KEYS = ("norm1.weight", "norm1.bias", "attn.qkv.weight", "attn.q_bias", "attn.v_bias", "attn.proj.weight",
                    "attn.proj.bias", "norm2.weight", "norm2.bias", "mlp.fc1_g.weight", "mlp.fc1_g.bias",
                    "mlp.fc1_x.weight", "mlp.fc1_x.bias", "mlp.norm.weight", "mlp.norm.bias", "mlp.fc2.weight",
                    "mlp.fc2.bias")
EVA02_TOP_KEYS = ("cls_token", "pos_embed", "patch_embed.proj.weight", "patch_embed.proj.bias", "fc_norm.weight",
                  "fc_norm.bias")


def eva02_to_clip_layout(state_dict):
    """timm ``Eva`` tensors (eva02_base_patch14_224) re-expressed in the layout of the CLIP tower, for the
    MER_VISION_EVA02 variant of mer_clip_vision_forward: the fused qkv weight split into q / k / v with the bias
    q_bias | 0 | v_bias (Eva's k_bias is a zero buffer), the patch-conv bias folded into the patch rows of the position
    table, fc1 = rows fc1_g | fc1_x, mlp.norm and fc_norm carried as ``mlp.norm.*`` / ``post_layernorm.*``.  Widths come
    from the tensor shapes.  Keys the model does not use (other than ``head.*``) and missing keys are refused by name."""
    sd = W._np(state_dict)
    n = 0
    while f"blocks.{n}.norm1.weight" in sd:
        n += 1
    want = set(EVA02_TOP_KEYS) | {f"blocks.{i}.{k}" for i in range(n) for k in EVA02_BLOCK_KEYS}
    missing = sorted(want - set(sd))
    extra = sorted(k for k in set(sd) - want if not k.startswith("head."))
    if missing or extra or n == 0:
        raise ValueError(f"not an eva02 state_dict: missing {missing[:8]}{' ...' if len(missing) > 8 else ''}, "
                         f"unexpected {extra[:8]}{' ...' if len(extra) > 8 else ''}, {n} blocks")
    f32 = lambda k: np.asarray(sd[k], np.float32)  # noqa: E731
    pw = f32("patch_embed.proj.weight")
    D = pw.shape[0]
    pos = f32("pos_embed").reshape(-1, D).copy()
    pos[1:] += f32("patch_embed.proj.bias")
    v = "vision_model."
    out = {v + "embeddings.patch_embedding.weight": pw, v + "embeddings.class_embedding": f32("cls_token").reshape(D),
           v + "embeddings.position_embedding.weight": pos,
           v + "post_layernorm.weight": f32("fc_norm.weight"), v + "post_layernorm.bias": f32("fc_norm.bias")}
    for i in range(n):
        s_, d_ = f"blocks.{i}.", f"{v}encoder.layers.{i}."
        q, k, vv = np.split(f32(s_ + "attn.qkv.weight"), 3, axis=0)
        for name, w_, b_ in (("q_proj", q, f32(s_ + "attn.q_bias")), ("k_proj", k, np.zeros(D, np.float32)),
                             ("v_proj", vv, f32(s_ + "attn.v_bias"))):
            out[d_ + f"self_attn.{name}.weight"], out[d_ + f"self_attn.{name}.bias"] = w_, b_
        for a, b in (("norm1", "layer_norm1"), ("norm2", "layer_norm2"), ("attn.proj", "self_attn.out_proj"),
                     ("mlp.norm", "mlp.norm"), ("mlp.fc2", "mlp.fc2")):
            out[d_ + b + ".weight"], out[d_ + b + ".bias"] = f32(s_ + a + ".weight"), f32(s_ + a + ".bias")
        out[d_ + "mlp.fc1.weight"] = np.concatenate([f32(s_ + "mlp.fc1_g.weight"), f32(s_ + "mlp.fc1_x.weight")], 0)
        out[d_ + "mlp.fc1.bias"] = np.concatenate([f32(s_ + "mlp.fc1_g.bias"), f32(s_ + "mlp.fc1_x.bias")], 0)
    return out


EVA02_MEAN = CLIP_MEAN   # OPENAI_CLIP_MEAN / _STD: the registry values of eva02_base_patch14_224.mim_in22k
EVA02_STD = CLIP_STD


def eva02_preprocess_geometry(h, w, size=224, crop_pct=0.9):
    """(new_h, new_w, crop_y0, crop_x0) of timm's eval transform: torchvision Resize(floor(size / crop_pct)) of the
    shorter edge (the longer one int(scale * long / short)), then CenterCrop(size) at int(round((new - size) / 2.0))
    (Python's round-half-even, not the floor of HF's processors)."""
    scale = int(math.floor(size / crop_pct))
    nh, nw, _, _ = clip_preprocess_geometry(h, w, scale)
    return nh, nw, int(round((nh - size) / 2.0)), int(round((nw - size) / 2.0))


class Eva02Encoder(ClipVisionEncoder):
    """timm ``Eva`` (eva02_base_patch14_224.mim_in22k: 12 blocks, hidden 768, patch 14, 257 tokens) with the
    reference's ``model(batch)`` readout (num_classes=0: mean over the patch rows, then fc_norm) per frame, on the CLIP
    tower kernels (MER_VISION_EVA02): timm's eval transform on the device (shorter edge -> 248 bicubic, centre crop 224
    at torchvision's offset, rescale, OPENAI CLIP normalise).  ``frame_features`` returns [N, hidden].

    precision: "f16" (default) or "tf32" operands of the linear layers; attention takes fp16 q | k | V^T in both
    (profiles/eva02_precision_table.json).  eva02 large / giant (FFN width 2730) are refused by shape.

    Reference: MER2024/feature_extraction/visual/extract_vision_huggingface.py:127-131, 202-210."""

    def __init__(self, state_dict, device="cuda", ln_eps=1e-6, image=224, precision="f16"):
        assert precision in ("f16", "tf32"), precision
        super().__init__(eva02_to_clip_layout(state_dict), device=device, ln_eps=ln_eps, image=image,
                         precision=precision, variant=MER_VISION_EVA02, mean=EVA02_MEAN, std=EVA02_STD,
                         resize=int(math.floor(image / 0.9)))

    def preprocess_geometry(self, h, w):
        return eva02_preprocess_geometry(h, w, self.image)


class MerResnetConv(C.Structure):
    _fields_ = [("w", C.c_void_p), ("b", C.c_void_p), ("cin", C.c_int), ("cout", C.c_int), ("cout_pad", C.c_int),
                ("k", C.c_int), ("stride", C.c_int), ("pad", C.c_int), ("kpad", C.c_int)]


class MerResnet18Model(C.Structure):
    _fields_ = [("convs", MerResnetConv * 20), ("mean", C.c_float * 3), ("std", C.c_float * 3)]


class ResNet18Encoder:
    """torchvision resnet18 without its fc layer (the reference's ImageNet CNN extractor): BatchNorm folded
    into the convolutions at load, every convolution an fp16 im2col + wgmma GEMM with a ReLU epilogue.

    Reference: MERBench/feature_extraction/visual/extract_imagenet_embedding.py:47-55."""

    IMAGENET_MEAN = (0.485, 0.456, 0.406)
    IMAGENET_STD = (0.229, 0.224, 0.225)

    def __init__(self, state_dict, device="cuda", bn_eps=1e-5):
        L.check(L.lib().mer_check_device())
        sd = W._np(state_dict)
        self.device = torch.device(device)
        pk = self.pk = W.Packed(self.device)
        m = MerResnet18Model()
        specs = [("conv1", "bn1", 2, 3)]
        for li in range(1, 5):
            for b in range(2):
                p = f"layer{li}.{b}."
                stride = 2 if (li > 1 and b == 0) else 1
                specs += [(p + "conv1", p + "bn1", stride, 1), (p + "conv2", p + "bn2", 1, 1)]
                if p + "downsample.0.weight" in sd:
                    specs.append((p + "downsample.0", p + "downsample.1", stride, 0))
        assert len(specs) == 20, "not a torchvision resnet18 state_dict"
        for i, (cn, bn, stride, pad) in enumerate(specs):
            w = sd[cn + ".weight"]                                          # [cout, cin, k, k]
            wf, bf = fold_conv_bn(w, sd[bn + ".weight"], sd[bn + ".bias"], sd[bn + ".running_mean"],
                                  sd[bn + ".running_var"], bn_eps)
            cout, cin, k, _ = w.shape
            cout_pad = max(cout, 128)
            kk = k * k * cin
            kpad = 192 if i == 0 else kk
            wp = np.zeros((cout_pad, kpad), np.float32)
            wp[:cout, :kk] = wf.transpose(0, 2, 3, 1).reshape(cout, kk)       # (ky, kx, c) order
            bp = np.zeros(cout_pad, np.float32)
            bp[:cout] = bf
            c = m.convs[i]
            c.w, c.b = pk.keep(wp, f16=True).data_ptr(), pk.keep(bp).data_ptr()
            c.cin, c.cout, c.cout_pad, c.k, c.stride, c.pad, c.kpad = cin, cout, cout_pad, k, stride, pad, kpad
        m.mean = (C.c_float * 3)(*self.IMAGENET_MEAN)
        m.std = (C.c_float * 3)(*self.IMAGENET_STD)
        self.model = m
        self.feature_dim = 512
        self.ws, self.ws_resize = _Workspace(self.device), _Workspace(self.device)
        lib = L.lib()
        lib.mer_resnet18_workspace_bytes.restype = C.c_longlong
        lib.mer_resnet18_workspace_bytes.argtypes = [C.c_int]
        lib.mer_resize_workspace_bytes.restype = C.c_longlong
        lib.mer_resize_workspace_bytes.argtypes = [C.c_int] * 5
        self._fwd = L.declare("mer_resnet18_forward", [C.POINTER(MerResnet18Model), C.c_void_p, C.c_int, C.c_void_p,
                                                       C.c_longlong, C.c_void_p, C.c_void_p])
        self._resize = L.declare("mer_resize_u8", [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                                   C.c_int, C.c_int, C.c_void_p, C.c_void_p])

    def frame_features(self, frames_bgr_u8: torch.Tensor, max_frames=64):
        """frames: uint8 CUDA [N, H, W, 3] (BGR); transforms.Resize((224, 224)) on the device when needed.
        Returns [N, 512] fp32 (CUDA)."""
        assert frames_bgr_u8.dtype == torch.uint8 and frames_bgr_u8.is_cuda and frames_bgr_u8.dim() == 4
        frames = frames_bgr_u8.contiguous()
        n, h, w, _ = frames.shape
        if (h, w) != (224, 224):
            out = torch.empty(n, 224, 224, 3, dtype=torch.uint8, device=self.device)
            need = L.lib().mer_resize_workspace_bytes(n, h, w, 224, 224)
            ws = self.ws_resize.get(max(int(need), 1))
            L.check(self._resize(L.ptr(frames), n, h, w, L.ptr(out), 224, 224, 0, L.ptr(ws), L.stream_ptr()))
            frames = out
        feats = torch.empty(n, 512, dtype=torch.float32, device=self.device)
        for s in range(0, n, max_frames):  # the fp32 activations of conv1 cost 6.4 MB per frame
            m = min(max_frames, n - s)
            ws = self.ws.get(L.lib().mer_resnet18_workspace_bytes(m))
            L.check(self._fwd(C.byref(self.model), L.ptr(frames[s:s + m]), m, L.ptr(ws), ws.numel(),
                              L.ptr(feats[s:s + m]), L.stream_ptr()))
        return feats


class MerCnnOp(C.Structure):
    _fields_ = [("kind", C.c_int), ("conv", C.c_int), ("src", C.c_int), ("dst", C.c_int), ("res", C.c_int),
                ("relu", C.c_int), ("k", C.c_int), ("stride", C.c_int), ("pad", C.c_int), ("ceil_mode", C.c_int),
                ("p", C.c_int * 4)]


class MerCnnModel(C.Structure):
    _fields_ = [("convs", C.POINTER(MerResnetConv)), ("n_convs", C.c_int), ("ops", C.POINTER(MerCnnOp)),
                ("n_ops", C.c_int), ("gemm_mode", C.c_int), ("in_h", C.c_int), ("in_w", C.c_int),
                ("scale", C.c_float), ("mean", C.c_float * 3), ("std", C.c_float * 3), ("feat_dim", C.c_int)]


CNN_STEM, CNN_CONV, CNN_MAXPOOL, CNN_GAP, CNN_SE, CNN_CROP, CNN_SHAPE, CNN_SLICE, CNN_CBAM, CNN_AFFINE, CNN_UPADD, \
    CNN_MASKMUL = range(12)
FERPLUS_BLOCKS = (3, 4, 6, 3)


def ferplus_resnet50_tables(state_dict, pack, bn_eps=1e-5, pack_dense=None):
    """Conv and op tables of ``resnet50_ferplus_dag`` / ``senet50_ferplus_dag`` up to conv5_3_3x3_relu + the 7x7
    average pool, for mer_cnn_forward.  ``pack(w [cout_pad, kpad] fp32, b [cout_pad] fp32) -> (w_ptr, b_ptr)``
    places the folded weights (split bf16) and biases on the device; ``pack_dense`` (default: ``pack``) does the
    same for the plain fp32 squeeze-and-excitation matrices of the SENet (detected by its ``*_1x1_down`` keys).
    Returns (MerCnnModel, keep-alive list).
    Buffers: 0 = the residual stream (block input / output), 1 and 2 = block-internal, 3 = projection shortcut."""
    sd = W._np(state_dict)
    convs, ops = [], []
    se = "conv2_1_1x1_down.weight" in sd
    pack_dense = pack_dense or pack

    def add_dense(name):
        w = np.ascontiguousarray(sd[name + ".weight"][:, :, 0, 0], np.float32)   # [cout, cin]
        c = MerResnetConv()
        c.w, c.b = pack_dense(w, np.asarray(sd[name + ".bias"], np.float32))
        c.cin, c.cout, c.cout_pad, c.k, c.stride, c.pad, c.kpad = w.shape[1], w.shape[0], w.shape[0], 1, 1, 0, w.shape[1]
        convs.append(c)
        return len(convs) - 1

    def add_conv(name, stride, pad):
        w = sd[name + ".weight"]
        wf, bf = fold_conv_bn(w, sd[name + "_bn.weight"], sd[name + "_bn.bias"], sd[name + "_bn.running_mean"],
                              sd[name + "_bn.running_var"], bn_eps)
        cout, cin, k, _ = w.shape
        cout_pad, kk = max(cout, 128), k * k * cin
        kpad = 160 if cin == 3 else kk
        wp = np.zeros((cout_pad, kpad), np.float32)
        wp[:cout, :kk] = wf.transpose(0, 2, 3, 1).reshape(cout, kk)       # (ky, kx, c) order
        bp = np.zeros(cout_pad, np.float32)
        bp[:cout] = bf
        c = MerResnetConv()
        c.w, c.b = pack(wp, bp)
        c.cin, c.cout, c.cout_pad, c.k, c.stride, c.pad, c.kpad = cin, cout, cout_pad, k, stride, pad, kpad
        convs.append(c)
        return len(convs) - 1

    def op(kind, conv=-1, src=0, dst=0, res=-1, relu=0, k=0, stride=0, pad=0, ceil_mode=0):
        ops.append(MerCnnOp(kind, conv, src, dst, res, relu, k, stride, pad, ceil_mode))

    op(CNN_STEM, add_conv("conv1_7x7_s2", 2, 3), dst=1, relu=1)
    op(CNN_MAXPOOL, src=1, dst=0, k=3, stride=2, pad=0, ceil_mode=1)
    for si, nblk in enumerate(FERPLUS_BLOCKS):
        for b in range(1, nblk + 1):
            p = f"conv{si + 2}_{b}_"
            stride = 2 if (si > 0 and b == 1) else 1
            op(CNN_CONV, add_conv(p + "1x1_reduce", stride, 0), src=0, dst=1, relu=1)
            op(CNN_CONV, add_conv(p + "3x3", 1, 1), src=1, dst=2, relu=1)
            if si == 3 and b == nblk:
                op(CNN_GAP, src=2)
                break
            if b == 1:
                op(CNN_CONV, add_conv(p + "1x1_proj", stride, 0), src=0, dst=3, relu=0)
            shortcut = 3 if b == 1 else 0
            if se:   # y -> buffer 1 (no ReLU), then the gate, the shortcut add and the ReLU in one op
                op(CNN_CONV, add_conv(p + "1x1_increase", 1, 0), src=2, dst=1, relu=0)
                op(CNN_SE, add_dense(p + "1x1_down"), src=1, dst=0, res=shortcut, relu=1, k=add_dense(p + "1x1_up"))
            else:
                op(CNN_CONV, add_conv(p + "1x1_increase", 1, 0), src=2, dst=0, res=shortcut, relu=1)
    assert len(convs) == (52 + 30 if se else 52) and ops[-1].kind == CNN_GAP
    conv_arr = (MerResnetConv * len(convs))(*convs)
    op_arr = (MerCnnOp * len(ops))(*ops)
    m = MerCnnModel()
    m.convs, m.n_convs = conv_arr, len(convs)
    m.ops, m.n_ops = op_arr, len(ops)
    m.gemm_mode = L.MER_GEMM_BF16X3
    m.in_h = m.in_w = 224
    m.scale = 1.0
    m.mean = (C.c_float * 3)(131.0912, 103.8827, 91.4953)   # model.meta (resnet50_ferplus_dag.py:11-13); std 1
    m.std = (C.c_float * 3)(1.0, 1.0, 1.0)
    m.feat_dim = 512
    return m, [conv_arr, op_arr]


def manet_tables(state_dict, pack, pack_dense=None, bn_eps=1e-5):
    """Conv and op tables of the reference's MA-Net (manet/model/manet.py:156-270) for mer_cnn_forward:
    ``model(x, return_embedding=True)`` = cat(local branch [512], multi-scale branch [512]).
    ``pack`` places a GEMM weight matrix ([cout_pad, kpad] fp32 -> split bf16) and its bias, ``pack_dense`` the plain
    fp32 matrices of the CBAM gates.  Buffers: 0 = trunk output (28 x 28 x 128, read by all five branches),
    1..5 = branch scratch, 7 = multi-scale stream."""
    sd = W._np(state_dict)
    pack_dense = pack_dense or pack
    convs, ops = [], []

    def fold(conv, bn):
        return fold_conv_bn(sd[conv + ".weight"], sd[bn + ".weight"], sd[bn + ".bias"], sd[bn + ".running_mean"],
                            sd[bn + ".running_var"], bn_eps)

    def add_conv(conv, bn, stride, pad):
        wf, bf = fold(conv, bn)
        cout, cin, k, _ = wf.shape
        cout_pad, kk = max(cout, 128), k * k * cin
        kpad = 160 if cin == 3 else kk
        wp = np.zeros((cout_pad, kpad), np.float32)
        wp[:cout, :kk] = wf.transpose(0, 2, 3, 1).reshape(cout, kk)       # (ky, kx, c) order
        bp = np.zeros(cout_pad, np.float32)
        bp[:cout] = bf
        c = MerResnetConv()
        c.w, c.b = pack(wp, bp)
        c.cin, c.cout, c.cout_pad, c.k, c.stride, c.pad, c.kpad = cin, cout, cout_pad, k, stride, pad, kpad
        convs.append(c)
        return len(convs) - 1

    def add_dense(w, b, cin, cout, k=1):
        c = MerResnetConv()
        c.w, c.b = pack_dense(np.ascontiguousarray(w, np.float32), np.ascontiguousarray(b, np.float32))
        c.cin, c.cout, c.cout_pad, c.k, c.stride, c.pad, c.kpad = cin, cout, cout, k, 1, k // 2, w.size // max(cout, 1)
        convs.append(c)
        return len(convs) - 1

    def op(kind, conv=-1, src=0, dst=0, res=-1, relu=0, k=0, stride=0, pad=0, ceil_mode=0, p=(0, 0, 0, 0)):
        ops.append(MerCnnOp(kind, conv, src, dst, res, relu, k, stride, pad, ceil_mode, (C.c_int * 4)(*p)))

    def shortcut(pfx, src, dst, stride):
        if pfx + "downsample.0.weight" not in sd:
            return src
        op(CNN_CONV, add_conv(pfx + "downsample.0", pfx + "downsample.1", stride, 0), src=src, dst=dst)
        return dst

    def basic(pfx, stride):                   # stream in buffer 0, in place
        op(CNN_CONV, add_conv(pfx + "conv1", pfx + "bn1", stride, 1), src=0, dst=1, relu=1)
        idt = shortcut(pfx, 0, 2, stride)
        op(CNN_CONV, add_conv(pfx + "conv2", pfx + "bn2", 1, 1), src=1, dst=0, res=idt, relu=1)

    def attention(pfx, src, stride):          # AttentionBlock: src (1 or 5) -> buffer 5
        op(CNN_CONV, add_conv(pfx + "conv1", pfx + "bn1", stride, 1), src=src, dst=2, relu=1)
        op(CNN_CONV, add_conv(pfx + "conv2", pfx + "bn2", 1, 1), src=2, dst=3)
        idt = shortcut(pfx, src, 4, stride)
        g = pfx + "cbam."
        w1, w2 = sd[g + "ChannelGate.mlp.1.weight"], sd[g + "ChannelGate.mlp.3.weight"]
        l1 = add_dense(w1, sd[g + "ChannelGate.mlp.1.bias"], w1.shape[1], w1.shape[0])
        l2 = add_dense(w2, sd[g + "ChannelGate.mlp.3.bias"], w2.shape[1], w2.shape[0])
        ws, bs = fold(g + "SpatialGate.spatial.conv", g + "SpatialGate.spatial.bn")     # [1, 2, 7, 7], [1]
        sp = add_dense(ws.reshape(1, 98), bs.reshape(1), 2, 1, k=7)
        op(CNN_CBAM, l1, src=3, dst=5, res=idt, p=(l2, sp, 0, 0))

    def mulscale(pfx, src, stride):           # MulScaleBlock: src (0 or 7) -> buffer 7
        c1 = add_conv(pfx + "conv1", pfx + "bn1", stride, 1)
        planes = convs[c1].cout
        sw = planes // 4
        op(CNN_CONV, c1, src=src, dst=1, relu=1)                                  # t, split into 4 x sw channels
        idt = shortcut(pfx, src, 5, stride)
        op(CNN_SHAPE, src=1, dst=4, p=(planes, 0, 0, 0))                          # O = O_1 + O_2
        op(CNN_SHAPE, src=1, dst=3, p=(sw, 0, 0, 0))                              # relu(o_{i-1}) + sp_i
        for chain in (1, 2):
            for i in range(4):
                ci = add_conv(pfx + f"conv{chain}_2_{i + 1}", pfx + f"bn{chain}_2_{i + 1}", 1, 1)
                if i == 0:
                    op(CNN_CONV, ci, src=1, dst=2, p=(0, 0, 0, 0))                # conv(sp_0)
                else:
                    op(CNN_SLICE, src=2, dst=3, res=1, relu=1, p=(0, 0, sw, i * sw))
                    op(CNN_CONV, ci, src=3, dst=2)
                op(CNN_SLICE, src=2, dst=4, res=4 if chain == 2 else -1, p=(0, i * sw, sw, i * sw))
        if idt != 7:
            op(CNN_SHAPE, src=4, dst=7, p=(planes, 0, 0, 0))
        op(CNN_SLICE, src=4, dst=7, res=idt, relu=2, p=(0, 0, planes, 0))

    op(CNN_STEM, add_conv("conv1", "bn1", 2, 3), dst=1, relu=1)
    op(CNN_MAXPOOL, src=1, dst=0, k=3, stride=2, pad=1, ceil_mode=0)
    for b in range(2):
        basic(f"layer1.{b}.", 1)
    for b in range(2):
        basic(f"layer2.{b}.", 2 if b == 0 else 1)
    for pi, (y0, x0) in enumerate(((0, 0), (0, 14), (14, 0), (14, 14)), start=1):
        op(CNN_CROP, src=0, dst=1, p=(y0, x0, 14, 14))
        attention(f"layer3_1_p{pi}.0.", 1, 2)
        attention(f"layer3_1_p{pi}.1.", 5, 1)
        attention(f"layer4_1_p{pi}.0.", 5, 1)
        attention(f"layer4_1_p{pi}.1.", 5, 1)
        op(CNN_GAP, src=5, p=(0, 1 if pi > 1 else 0, 4, 0))       # mean of the 14 x 14 mosaic = mean of the 4 patch means
    mulscale("layer3_2.0.", 0, 2)
    mulscale("layer3_2.1.", 7, 1)
    mulscale("layer4_2.0.", 7, 2)
    mulscale("layer4_2.1.", 7, 1)
    op(CNN_GAP, src=7, p=(512, 0, 1, 0))
    conv_arr = (MerResnetConv * len(convs))(*convs)
    op_arr = (MerCnnOp * len(ops))(*ops)
    m = MerCnnModel()
    m.convs, m.n_convs = conv_arr, len(convs)
    m.ops, m.n_ops = op_arr, len(ops)
    m.gemm_mode = L.MER_GEMM_BF16X3
    m.in_h = m.in_w = 224
    m.scale = 1.0 / 255.0                                          # ToTensor only (extract_manet_embedding.py:60-61)
    m.mean = (C.c_float * 3)(0.0, 0.0, 0.0)
    m.std = (C.c_float * 3)(1.0, 1.0, 1.0)
    m.feat_dim = 1024
    return m, [conv_arr, op_arr]


def emonet_tables(state_dict, pack, pack_dense=None, bn_eps=1e-5):
    """Conv and op tables of the reference's EmoNet (emonet/models/emonet.py:173-222) for mer_cnn_forward: the 256-d
    embedding after the emotion tower's average pool.  Pre-activation ConvBlocks become AFFINE (BatchNorm + ReLU) ->
    CONV triples whose outputs land in channel slices next to the shortcut; the hourglass recursion keeps one
    skip buffer and one low-resolution buffer per level.
    Buffers: 0 = x (trunk, 64 x 64 x 256), 1 = the hourglass input ("previous"), 2 / 3 = the two modules' features,
    4 = heat-maps, 5 = concatenation, 6..10 = ConvBlock scratch, 11..14 = skip buffers, 15..18 = low buffers of
    hourglass levels 1..4, 19 / 20 = stem / tower ping-pong."""
    sd = W._np(state_dict)
    pack_dense = pack_dense or pack
    convs, ops = [], []
    A_, U1, U2, U3, R_ = 6, 7, 8, 9, 10

    def bn_affine(name):
        scale = np.asarray(sd[name + ".weight"], np.float64) / np.sqrt(np.asarray(sd[name + ".running_var"], np.float64) + bn_eps)
        return scale, np.asarray(sd[name + ".bias"], np.float64) - np.asarray(sd[name + ".running_mean"], np.float64) * scale

    def add_conv(name, stride=1, pad=0, post_bn=None, cin_pad=None, cout_real=None):
        w = np.asarray(sd[name + ".weight"], np.float64)
        b = np.asarray(sd[name + ".bias"], np.float64) if name + ".bias" in sd else np.zeros(w.shape[0])
        if post_bn is not None:                                # conv (+ bias) followed by a BatchNorm: fold
            sc, sh = bn_affine(post_bn)
            w, b = w * sc[:, None, None, None], b * sc + sh
        cout, cin, k, _ = w.shape
        cin_p = cin_pad or cin
        cout_r = cout_real or cout                             # channels declared real (zero rows beyond cout)
        cout_pad, kk = max(cout_r, 128), k * k * cin_p
        kpad = 160 if cin == 3 else kk
        wp = np.zeros((cout_pad, k, k, cin_p), np.float32)
        wp[:cout, :, :, :cin] = w.transpose(0, 2, 3, 1)
        wp = wp.reshape(cout_pad, k * k * cin_p)
        if kpad != kk:
            wp = np.concatenate([wp, np.zeros((cout_pad, kpad - kk), np.float32)], axis=1)
        bp = np.zeros(cout_pad, np.float32)
        bp[:cout] = b
        c = MerResnetConv()
        c.w, c.b = pack(np.ascontiguousarray(wp), bp)
        c.cin, c.cout, c.cout_pad, c.k, c.stride, c.pad, c.kpad = cin_p, cout_r, cout_pad, k, stride, pad, kpad
        convs.append(c)
        return len(convs) - 1

    def add_affine(bn_name):
        sc, sh = bn_affine(bn_name)
        c = MerResnetConv()
        c.w, c.b = pack_dense(sc.astype(np.float32), sh.astype(np.float32))
        c.cin = c.cout = c.cout_pad = c.kpad = len(sc)
        c.k, c.stride, c.pad = 1, 1, 0
        convs.append(c)
        return len(convs) - 1

    def op(kind, conv=-1, src=0, dst=0, res=-1, relu=0, k=0, stride=0, pad=0, ceil_mode=0, p=(0, 0, 0, 0)):
        ops.append(MerCnnOp(kind, conv, src, dst, res, relu, k, stride, pad, ceil_mode, (C.c_int * 4)(*p)))

    def block(pfx, src, dst):
        """ConvBlock (:20-64): dst = cat(o1, o2, o3) + shortcut; dst may be src when there is no downsample."""
        c1 = add_conv(pfx + "conv1", 1, 1)
        c2 = add_conv(pfx + "conv2", 1, 1)
        c3 = add_conv(pfx + "conv3", 1, 1)
        h, q = convs[c1].cout, convs[c2].cout                  # out / 2, out / 4
        op(CNN_AFFINE, add_affine(pfx + "bn1"), src=src, dst=A_, relu=1)
        op(CNN_CONV, c1, src=A_, dst=U1)
        op(CNN_AFFINE, add_affine(pfx + "bn2"), src=U1, dst=A_, relu=1)
        op(CNN_CONV, c2, src=A_, dst=U2)
        op(CNN_AFFINE, add_affine(pfx + "bn3"), src=U2, dst=A_, relu=1)
        op(CNN_CONV, c3, src=A_, dst=U3)
        if pfx + "downsample.2.weight" in sd:
            assert dst != src
            op(CNN_AFFINE, add_affine(pfx + "downsample.0"), src=src, dst=A_, relu=1)
            op(CNN_CONV, add_conv(pfx + "downsample.2"), src=A_, dst=R_)
            shortcut = R_
        else:
            shortcut = src
        if dst != src:
            op(CNN_SHAPE, src=U1, dst=dst, p=(h + 2 * q, 0, 0, 0))
        op(CNN_SLICE, src=U1, dst=dst, res=shortcut, p=(0, 0, h, 0))
        op(CNN_SLICE, src=U2, dst=dst, res=shortcut, p=(0, h, q, h))
        op(CNN_SLICE, src=U3, dst=dst, res=shortcut, p=(0, h + q, q, h + q))

    def hourglass(pfx, level, inp):
        """HourGlass._forward (:87-109); the result lands in the level's skip buffer."""
        up, low = 10 + level, 14 + level
        block(pfx + f"b1_{level}.", inp, up)
        op(CNN_MAXPOOL, src=inp, dst=low, k=2, stride=2)
        block(pfx + f"b2_{level}.", low, low)
        if level > 1:
            low2 = hourglass(pfx, level - 1, low)
        else:
            block(pfx + f"b2_plus_{level}.", low, low)
            low2 = low
        block(pfx + f"b3_{level}.", low2, low2)
        op(CNN_UPADD, src=low2, dst=up, res=up)
        return up

    op(CNN_STEM, add_conv("conv1", 2, 3, post_bn="bn1"), dst=19, relu=1)              # [128, 128, 64]
    block("conv2.", 19, 20)                                                           # -> 128 channels
    op(CNN_MAXPOOL, src=20, dst=19, k=2, stride=2)                                    # [64, 64, 128]
    block("conv3.", 19, 19)
    block("conv4.", 19, 0)                                                            # x
    op(CNN_SHAPE, src=0, dst=1, p=(256, 0, 0, 0))
    op(CNN_SLICE, src=0, dst=1, p=(0, 0, 256, 0))                                     # previous = x
    for i in range(2):
        hg = hourglass(f"m{i}.", 4, 1)
        block(f"top_m_{i}.", hg, hg)
        feat = 2 + i
        op(CNN_CONV, add_conv(f"conv_last{i}", post_bn=f"bn_end{i}"), src=hg, dst=feat if i == 1 else 20, relu=1)
        ll = feat if i == 1 else 20
        op(CNN_CONV, add_conv(f"l{i}", cout_real=128), src=ll, dst=4)                  # 68 heat-maps (+ 60 zero channels)
        if i < 1:
            op(CNN_CONV, add_conv(f"bl{i}"), src=ll, dst=feat)                          # the feature kept for module 0
            op(CNN_CONV, add_conv(f"al{i}", cin_pad=128), src=4, dst=A_)
            op(CNN_SLICE, src=feat, dst=1, res=1, p=(0, 0, 256, 0))                     # previous += ll
            op(CNN_SLICE, src=A_, dst=1, res=1, p=(0, 0, 256, 0))                       # previous += al(heat)
    op(CNN_SHAPE, src=0, dst=5, p=(768, 0, 0, 0))
    op(CNN_SLICE, src=0, dst=5, p=(0, 0, 256, 0))
    op(CNN_MASKMUL, src=2, dst=5, res=4, p=(0, 256, 256, 68))
    op(CNN_MASKMUL, src=3, dst=5, res=4, p=(0, 512, 256, 68))
    op(CNN_CONV, add_conv("conv1x1_input_emo_2"), src=5, dst=19)
    cur, other = 19, 20
    for i in range(4):
        block(f"emo_net_2.{2 * i}.", cur, cur)
        op(CNN_MAXPOOL, src=cur, dst=other, k=2, stride=2)
        cur, other = other, cur
    op(CNN_GAP, src=cur, p=(0, 0, 1, 0))
    conv_arr = (MerResnetConv * len(convs))(*convs)
    op_arr = (MerCnnOp * len(ops))(*ops)
    m = MerCnnModel()
    m.convs, m.n_convs = conv_arr, len(convs)
    m.ops, m.n_ops = op_arr, len(ops)
    m.gemm_mode = L.MER_GEMM_BF16X3
    m.in_h = m.in_w = 256
    m.scale = 1.0 / 255.0
    m.mean = (C.c_float * 3)(0.0, 0.0, 0.0)
    m.std = (C.c_float * 3)(1.0, 1.0, 1.0)
    m.feat_dim = 256
    return m, [conv_arr, op_arr]


class _CnnEncoder:
    """Shared driver of the table-driven CNN extractors: device-side PIL-bilinear resize (+ optional centre crop) to
    224 x 224, then mer_cnn_forward in chunks of frames."""

    def _setup(self, device, tables, feature_dim):
        L.check(L.lib().mer_check_device())
        self.device = torch.device(device)
        pk = self.pk = W.Packed(self.device)
        self.model, self._keep = tables(lambda wp, bp: (pk.keep(wp, split=True).data_ptr(), pk.keep(bp).data_ptr()),
                                        lambda w, b: (pk.keep(w).data_ptr(), pk.keep(b).data_ptr()))
        self.feature_dim = feature_dim
        self.ws, self.ws_resize = _Workspace(self.device), _Workspace(self.device)
        lib = L.lib()
        lib.mer_cnn_workspace_bytes.restype = C.c_longlong
        lib.mer_cnn_workspace_bytes.argtypes = [C.POINTER(MerCnnModel), C.c_int]
        lib.mer_resize_workspace_bytes.restype = C.c_longlong
        lib.mer_resize_workspace_bytes.argtypes = [C.c_int] * 5
        self._fwd = L.declare("mer_cnn_forward", [C.POINTER(MerCnnModel), C.c_void_p, C.c_int, C.c_void_p,
                                                  C.c_longlong, C.c_void_p, C.c_void_p])
        self._resize = L.declare("mer_resize_u8", [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                                   C.c_int, C.c_int, C.c_void_p, C.c_void_p])

    def preprocess_geometry(self, h, w):
        """(resized h, resized w, crop top, crop left) of the reference transform; default: Resize((224, 224))."""
        return 224, 224, 0, 0

    def frame_features(self, frames_bgr_u8: torch.Tensor, max_frames=64):
        """frames: uint8 CUDA [N, H, W, 3] (BGR) -> [N, feature_dim] fp32 (CUDA)."""
        assert frames_bgr_u8.dtype == torch.uint8 and frames_bgr_u8.is_cuda and frames_bgr_u8.dim() == 4
        frames = frames_bgr_u8.contiguous()
        n, h, w, _ = frames.shape
        nh, nw, top, left = self.preprocess_geometry(h, w)
        if (nh, nw) != (h, w):
            out = torch.empty(n, nh, nw, 3, dtype=torch.uint8, device=self.device)
            need = L.lib().mer_resize_workspace_bytes(n, h, w, nh, nw)
            ws = self.ws_resize.get(max(int(need), 1))
            L.check(self._resize(L.ptr(frames), n, h, w, L.ptr(out), nh, nw, 0, L.ptr(ws), L.stream_ptr()))
            frames = out
        if (nh, nw) != (224, 224):
            frames = frames[:, top:top + 224, left:left + 224].contiguous()
        feats = torch.empty(n, self.feature_dim, dtype=torch.float32, device=self.device)
        for s in range(0, n, max_frames):
            m = min(max_frames, n - s)
            nbytes = L.lib().mer_cnn_workspace_bytes(C.byref(self.model), m)
            L.check(0 if nbytes > 0 else 1)
            ws = self.ws.get(nbytes)
            L.check(self._fwd(C.byref(self.model), L.ptr(frames[s:s + m]), m, L.ptr(ws), ws.numel(),
                              L.ptr(feats[s:s + m]), L.stream_ptr()))
        return feats


class FerplusResnet50Encoder(_CnnEncoder):
    """``resnet50_ferplus_dag`` (or ``senet50_ferplus_dag``: same skeleton + a squeeze-and-excitation gate per block,
    picked up from the state_dict) up to ``conv5_3_3x3_relu`` + AvgPool2d(7) (what the reference's FER+ extractor keeps
    with its default ``--layer_name``): 52 BatchNorm-folded convolutions through the table-driven CNN executor
    (im2col + wgmma GEMMs on split-bf16 operands: fp16 operands measured 6e-4 in an fp32 emulation, too close
    to the 1e-3 bar), caffe-style strides, ceil-mode max-pool.

    Reference: MERBench/feature_extraction/visual/extract_ferplus_embedding.py:62-115,
    pytorch-benchmarks/model/resnet50_ferplus_dag.py:10-355."""

    def __init__(self, state_dict, device="cuda", bn_eps=1e-5):
        self._setup(device, lambda pack, dense: ferplus_resnet50_tables(state_dict, pack, bn_eps, pack_dense=dense), 512)

    def preprocess_geometry(self, h, w):
        """transforms.Resize(256) + CenterCrop(224) (extract_ferplus_embedding.py:68-70): resized (h, w) and the
        crop's (top, left)."""
        nh, nw = (256, int(256 * w / h)) if h <= w else (int(256 * h / w), 256)
        return nh, nw, int(round((nh - 224) / 2.0)), int(round((nw - 224) / 2.0))


class ManetEncoder(_CnnEncoder):
    """MA-Net (the RAF-DB checkpoint the reference extracts ``manet_<UTT|FRA>`` features with): ResNet-18 trunk, four
    14 x 14 patch branches of CBAM AttentionBlocks, a multi-scale branch of MulScaleBlocks; 1024-d embedding.
    120 BatchNorm-folded convolutions on split-bf16 wgmma GEMMs + 16 fused CBAM gates.

    Reference: MERBench/feature_extraction/visual/extract_manet_embedding.py:31-61,
    manet/model/manet.py:16-270, manet/model/attention.py:27-84."""

    def __init__(self, state_dict, device="cuda", bn_eps=1e-5):
        self._setup(device, lambda pack, dense: manet_tables(state_dict, pack, dense, bn_eps), 1024)


class EmonetEncoder(_CnnEncoder):
    """EmoNet (the 8-class AffectNet checkpoint the reference extracts ``emonet_<UTT|FRA>`` features with): stem,
    pre-activation ConvBlocks, two depth-4 hourglasses, heat-map mask, emotion tower; 256-d embedding.
    Faces are resized to 256 x 256 with the bit-exact cv2 INTER_LINEAR kernel (the reference's DataAugmentor).

    Reference: MERBench/feature_extraction/visual/extract_emonet_embedding.py:22-61,
    emonet/models/emonet.py:20-222, emonet/data_augmentation.py:68-87."""

    def __init__(self, state_dict, device="cuda", bn_eps=1e-5):
        self._setup(device, lambda pack, dense: emonet_tables(state_dict, pack, dense, bn_eps), 256)
        self._cv2 = L.declare("mer_resize_cv2_linear_u8", [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                                           C.c_int, C.c_void_p])

    def frame_features(self, frames_bgr_u8: torch.Tensor, max_frames=8):
        """frames: uint8 CUDA [N, H, W, 3] (BGR) -> [N, 256] fp32 (CUDA).  125 MB of workspace per frame."""
        assert frames_bgr_u8.dtype == torch.uint8 and frames_bgr_u8.is_cuda and frames_bgr_u8.dim() == 4
        frames = frames_bgr_u8.contiguous()
        n, h, w, _ = frames.shape
        if (h, w) != (256, 256):
            out = torch.empty(n, 256, 256, 3, dtype=torch.uint8, device=self.device)
            L.check(self._cv2(L.ptr(frames), n, h, w, L.ptr(out), 256, 256, L.stream_ptr()))
            frames = out
        feats = torch.empty(n, self.feature_dim, dtype=torch.float32, device=self.device)
        for s in range(0, n, max_frames):
            m = min(max_frames, n - s)
            nbytes = L.lib().mer_cnn_workspace_bytes(C.byref(self.model), m)
            L.check(0 if nbytes > 0 else 1)
            ws = self.ws.get(nbytes)
            L.check(self._fwd(C.byref(self.model), L.ptr(frames[s:s + m]), m, L.ptr(ws), ws.numel(),
                              L.ptr(feats[s:s + m]), L.stream_ptr()))
        return feats


class MerVggishModel(C.Structure):
    _fields_ = [("convs", MerResnetConv * 6), ("fc_w", C.c_void_p * 3), ("fc_b", C.c_void_p * 3)]


VGGISH_CONVS = ("conv1", "conv2", "conv3/conv3_1", "conv3/conv3_2", "conv4/conv4_1", "conv4/conv4_2")
VGGISH_FCS = ("fc1/fc1_1", "fc1/fc1_2", "fc2")
# torchvggish port (harritaylor/torchvggish, vggish-10086976.pth): same tensors under nn.Sequential names
_TORCHVGGISH = {"conv1": "features.0", "conv2": "features.3", "conv3/conv3_1": "features.6",
                "conv3/conv3_2": "features.8", "conv4/conv4_1": "features.11", "conv4/conv4_2": "features.13",
                "fc1/fc1_1": "embeddings.0", "fc1/fc1_2": "embeddings.2", "fc2": "embeddings.4"}


def vggish_tf_names(state_dict):
    """Accepts the TF checkpoint variables (``vggish/<scope>/weights|biases``, e.g. exported to .npz) or the
    state_dict of the torchvggish port (OIHW convs, [out, in] linears) and returns the TF-named / TF-laid-out
    dict the encoder packs from."""
    sd = W._np(state_dict)
    if "vggish/conv1/weights" in sd:
        return sd
    assert "features.0.weight" in sd, "neither TF VGGish variable names nor a torchvggish state_dict"
    out = {}
    for tf_name, pt in _TORCHVGGISH.items():
        w = sd[pt + ".weight"]
        out[f"vggish/{tf_name}/weights"] = w.transpose(2, 3, 1, 0) if w.ndim == 4 else w.T   # -> HWIO / [in, out]
        out[f"vggish/{tf_name}/biases"] = sd[pt + ".bias"]
    return out


def vggish_tables(state_dict, pack):
    """MerVggishModel from the TF-named (or torchvggish) weights.  ``pack(w [rows, K] fp32, b fp32) -> (w_ptr, b_ptr)``
    places one GEMM weight matrix (split bf16 on the device) and its bias."""
    sd = vggish_tf_names(state_dict)
    m = MerVggishModel()
    for i, name in enumerate(VGGISH_CONVS):
        w = sd[f"vggish/{name}/weights"]                                   # HWIO [3, 3, cin, cout]
        k, _, cin, cout = w.shape
        assert k == 3, name
        cout_pad, kk = max(cout, 128), 9 * cin
        kpad = 32 if i == 0 else kk
        wp = np.zeros((cout_pad, kpad), np.float32)
        wp[:cout, :kk] = w.transpose(3, 0, 1, 2).reshape(cout, kk)         # (ky, kx, c) order
        bp = np.zeros(cout_pad, np.float32)
        bp[:cout] = sd[f"vggish/{name}/biases"]
        c = m.convs[i]
        c.w, c.b = pack(wp, bp)
        c.cin, c.cout, c.cout_pad, c.k, c.stride, c.pad, c.kpad = cin, cout, cout_pad, 3, 1, 1, kpad
    for i, name in enumerate(VGGISH_FCS):
        w = sd[f"vggish/{name}/weights"]                                   # [in, out]
        m.fc_w[i], m.fc_b[i] = pack(np.ascontiguousarray(w.T, np.float32), np.asarray(sd[f"vggish/{name}/biases"], np.float32))
    return m


class VggishEncoder:
    """VGGish embedding network of the reference's audio extractor: six 3x3 convolutions as im2col + wgmma
    GEMMs with ReLU epilogues, 2x2 max-pools, three fully connected layers; all GEMMs on split-bf16 operands
    (MER_GEMM_BF16X3, ~fp32 accuracy: there is no normalisation between the nine layers).

    Reference: MERBench/feature_extraction/audio/vggish/vggish_slim.py:37-100 (graph),
    extract_vggish_embedding.py:30-49 (fetch of vggish/embedding for batches of log-mel examples)."""

    def __init__(self, state_dict, device="cuda"):
        L.check(L.lib().mer_check_device())
        self.device = torch.device(device)
        pk = self.pk = W.Packed(self.device)
        self.model = vggish_tables(state_dict, lambda w, b: (pk.keep(w, split=True).data_ptr(), pk.keep(b).data_ptr()))
        self.feature_dim = 128
        self.ws = _Workspace(self.device)
        lib = L.lib()
        lib.mer_vggish_workspace_bytes.restype = C.c_longlong
        lib.mer_vggish_workspace_bytes.argtypes = [C.c_int]
        self._fwd = L.declare("mer_vggish_forward", [C.POINTER(MerVggishModel), C.c_void_p, C.c_int, C.c_void_p,
                                                     C.c_longlong, C.c_void_p, C.c_void_p])

    def embeddings(self, examples: torch.Tensor, max_examples=256):
        """examples: fp32 CUDA [n, 96, 64] log-mel patches -> [n, 128] fp32 (CUDA).  Chunks of ``max_examples``
        bound the workspace (7.8 MB per example; the reference feeds 2048 at a time)."""
        assert examples.is_cuda and examples.dtype == torch.float32 and examples.shape[1:] == (96, 64)
        examples = examples.contiguous()
        n = examples.shape[0]
        out = torch.empty(n, 128, dtype=torch.float32, device=self.device)
        for s in range(0, n, max_examples):
            k = min(max_examples, n - s)
            ws = self.ws.get(L.lib().mer_vggish_workspace_bytes(k))
            L.check(self._fwd(C.byref(self.model), L.ptr(examples[s:s + k]), k, L.ptr(ws), ws.numel(),
                              L.ptr(out[s:s + k]), L.stream_ptr()))
        return out


class MerHubertModel(C.Structure):
    _fields_ = [("n_layers", C.c_int), ("ln_eps", C.c_float), ("conv0_w", C.c_void_p),
                ("gn_g", C.c_void_p), ("gn_b", C.c_void_p), ("conv_w", C.c_void_p * 6),
                ("fp_ln_g", C.c_void_p), ("fp_ln_b", C.c_void_p), ("fp_w", C.c_void_p),
                ("fp_b", C.c_void_p), ("pos_w", C.c_void_p), ("pos_w_bd", C.c_void_p), ("pos_b", C.c_void_p),
                ("enc_ln_g", C.c_void_p), ("enc_ln_b", C.c_void_p),
                ("layers", C.POINTER(W.MerLayerWeights)),
                ("hidden", C.c_int), ("ffn", C.c_int), ("heads", C.c_int), ("feat_norm_layer", C.c_int),
                ("stable_layer_norm", C.c_int), ("conv_b", C.c_void_p * 7), ("conv_ln_g", C.c_void_p * 7),
                ("conv_ln_b", C.c_void_p * 7), ("pos_window", C.c_int), ("layers_f16", C.POINTER(W.MerLayerWeights)),
                ("n_pos_layers", C.c_int), ("pos_taps", C.c_int), ("pos_layers_w", C.c_void_p * 8),
                ("pos_layers_b", C.c_void_p * 8), ("ln_ones", C.c_void_p), ("ln_zeros", C.c_void_p),
                ("conv_w_f16", C.c_void_p * 2), ("readout", C.c_int)]


MER_HUBERT_READOUT_LAST4, MER_HUBERT_READOUT_LAST = 0, 1   # MerHubertModel.readout (mer_b200.h)


def block_diagonal_pos_conv_weight(wpos, block_n=256, window=320, group=48):
    """[768 out][48 in][128 taps] grouped-conv weight -> dense [768][128 * window]: row o holds, for every
    tap k, its 48 input weights at columns k*window + (g*48 + i - win0(o)), zeros elsewhere, where
    win0 = floor(block_n * (o // block_n) / group) * group is the first input channel the GEMM reads for
    o's output column block (MerGemmDesc.a_col_group)."""
    n_out, cin, taps = wpos.shape
    out = np.zeros((n_out, taps, window), np.float32)
    for o0 in range(0, n_out, group):            # one group of outputs at a time
        g = o0 // group
        for o in range(o0, o0 + group):
            win0 = (block_n * (o // block_n) // group) * group
            off = g * group - win0
            assert 0 <= off and off + cin <= window, (o, off)
            out[o, :, off:off + cin] = wpos[o].T  # [taps][in]
    return out.reshape(n_out, taps * window)


def fold_pos_conv_weight(sd):
    """Effective weight of the weight-normed positional conv: g * v / ||v||_(dims 0,1)
    (HF modeling_hubert.py:45-92; torch weight_norm dim=2), float64 math, fp32 result."""
    pre = "encoder.pos_conv_embed.conv."
    if pre + "parametrizations.weight.original0" in sd:
        g, v = sd[pre + "parametrizations.weight.original0"], sd[pre + "parametrizations.weight.original1"]
    elif pre + "weight_g" in sd:
        g, v = sd[pre + "weight_g"], sd[pre + "weight_v"]
    else:
        return np.asarray(sd[pre + "weight"], dtype=np.float32)
    v = np.asarray(v, dtype=np.float64)
    norm = np.sqrt((v ** 2).sum(axis=(0, 1), keepdims=True))
    return (np.asarray(g, dtype=np.float64) * v / norm).astype(np.float32)


class HubertEncoder:
    """HF ``HubertModel`` / ``Wav2Vec2Model`` + the reference readout
    ``torch.stack(hidden_states)[[-4,-3,-2,-1]].sum(0)``.  Two families, recognised from the checkpoint:
    base (hidden 768, group-norm feature extractor, post-LN: hubert-base, wav2vec2-base) and large
    (hidden 1024, 16 heads, LayerNorm after every conv, conv biases, stable / pre-LN encoder: hubert-large,
    chinese-hubert-large, wav2vec2-large-lv60).  ``stable_layer_norm`` overrides the inference of
    ``config.do_stable_layer_norm`` from the feature extractor type (they coincide in every released checkpoint of
    the extractor's model list).  Two more combinations (GPU-tested in tests/test_variants_gpu.py): hidden 1024 on the
    group-norm extractor with post-LN layers (wav2vec2-large-960h) and ``Data2VecAudioModel``
    (data2vec-audio-base-960h: LayerNorm convs without biases, a chain of positional convs, post-LN).

    Reference: MERBench/feature_extraction/audio/extract_audio_huggingface.py:18-36,93-110."""

    def __init__(self, state_dict, device="cuda", ln_eps=1e-5, stable_layer_norm=None, stack_precision=None,
                 conv_precision=None, last_layer_only=False):
        """last_layer_only: the readout is ``hidden_states[-1]`` alone (MER2023's extract_transformers_embedding.py,
        ``layer_ids = [-1]``) instead of the sum of the last four."""
        L.check(L.lib().mer_check_device())
        sd = W._np(state_dict)
        self.device = torch.device(device)
        pk = self.pk = W.Packed(self.device)
        self.n_layers = W.count_layers(sd, "encoder.layers.{i}.layer_norm.weight")
        m = MerHubertModel()
        m.n_layers, m.ln_eps = self.n_layers, ln_eps
        m.readout = MER_HUBERT_READOUT_LAST if last_layer_only else MER_HUBERT_READOUT_LAST4
        w0 = sd["feature_extractor.conv_layers.0.conv.weight"]
        assert w0.shape == (512, 1, 10), f"wav2vec2-style feature extractor (512 x 10 conv0) only, got {w0.shape}"
        assert "feature_extractor.conv_layers.0.layer_norm.weight" in sd
        ln_convs = "feature_extractor.conv_layers.1.layer_norm.weight" in sd  # feat_extract_norm == "layer"
        self.hidden = int(sd["encoder.layer_norm.weight"].shape[0])
        ffn = int(sd["encoder.layers.0.feed_forward.intermediate_dense.weight"].shape[0])
        assert self.hidden in (768, 1024) and ffn % 128 == 0, (self.hidden, ffn)
        m.hidden, m.ffn, m.heads = self.hidden, ffn, self.hidden // 64
        data2vec = "encoder.pos_conv_embed.layers.0.conv.weight" in sd   # Data2VecAudioModel (data2vec-audio-base-960h)
        m.feat_norm_layer = 1 if ln_convs else 0
        m.stable_layer_norm = int((ln_convs and not data2vec) if stable_layer_norm is None else stable_layer_norm)
        m.conv0_w = pk.keep(w0.reshape(512, 10)).data_ptr()
        m.gn_g = pk.keep(sd["feature_extractor.conv_layers.0.layer_norm.weight"]).data_ptr()
        m.gn_b = pk.keep(sd["feature_extractor.conv_layers.0.layer_norm.bias"]).data_ptr()
        for i in range(7):
            pre = f"feature_extractor.conv_layers.{i}."
            has_b = pre + "conv.bias" in sd
            assert ln_convs or not has_b, "conv biases are implemented with the layer-norm feature extractor only"
            if ln_convs:
                if has_b:
                    m.conv_b[i] = pk.keep(sd[pre + "conv.bias"]).data_ptr()
                m.conv_ln_g[i] = pk.keep(sd[pre + "layer_norm.weight"]).data_ptr()
                m.conv_ln_b[i] = pk.keep(sd[pre + "layer_norm.bias"]).data_ptr()
        for i, k in enumerate((3, 3, 3, 3, 2, 2)):
            w = sd[f"feature_extractor.conv_layers.{i + 1}.conv.weight"]
            assert w.shape == (512, 512, k), w.shape
            m.conv_w[i] = pk.keep(np.ascontiguousarray(w.transpose(0, 2, 1)).reshape(512, k * 512),
                                  split=True).data_ptr()
        m.fp_ln_g = pk.keep(sd["feature_projection.layer_norm.weight"]).data_ptr()
        m.fp_ln_b = pk.keep(sd["feature_projection.layer_norm.bias"]).data_ptr()
        m.fp_w = pk.keep(sd["feature_projection.projection.weight"], split=True).data_ptr()
        m.fp_b = pk.keep(sd["feature_projection.projection.bias"]).data_ptr()
        gch = self.hidden // 16
        if data2vec:
            # a chain of k = 19 grouped convs, each as a windowed block-diagonal fp16 GEMM operand
            m.pos_window = 320 if gch == 48 else 256
            n_pos = W.count_layers(sd, "encoder.pos_conv_embed.layers.{i}.conv.weight")
            assert 0 < n_pos <= 8
            m.n_pos_layers = n_pos
            for l in range(n_pos):
                w = np.asarray(sd[f"encoder.pos_conv_embed.layers.{l}.conv.weight"], np.float32)
                assert w.shape[:2] == (self.hidden, gch) and w.shape[2] % 2 == 1, w.shape
                m.pos_taps = int(w.shape[2])
                m.pos_layers_w[l] = pk.keep(block_diagonal_pos_conv_weight(w, window=m.pos_window, group=gch),
                                            f16=True).data_ptr()
                m.pos_layers_b[l] = pk.keep(sd[f"encoder.pos_conv_embed.layers.{l}.conv.bias"]).data_ptr()
            m.ln_ones = pk.keep(np.ones(self.hidden, np.float32)).data_ptr()
            m.ln_zeros = pk.keep(np.zeros(self.hidden, np.float32)).data_ptr()
        wpos = None if data2vec else fold_pos_conv_weight(sd)
        assert data2vec or wpos.shape == (self.hidden, gch, 128), wpos.shape
        # the weights as a windowed block-diagonal fp16 matrix for the GEMM form of the conv
        # (MerHubertModel.pos_w_bd in mer_b200.h): 48-channel groups need a 320-wide window per 256-column
        # block, 64-channel groups exactly 256.  MER_POSCONV_LEGACY=1 keeps the mma.sync kernel (base only)
        import os
        m.pos_window = 320 if gch == 48 else 256
        if not data2vec:
            legacy = bool(os.environ.get("MER_POSCONV_LEGACY")) and gch == 48
            if gch == 48:
                wp = wpos.reshape(16, 48, 48, 128).transpose(0, 3, 1, 2)  # [g][tap][out][in]
                m.pos_w = pk.keep(np.ascontiguousarray(wp), tf32=True).data_ptr()
            m.pos_w_bd = None if legacy else \
                pk.keep(block_diagonal_pos_conv_weight(wpos, window=m.pos_window, group=gch), f16=True).data_ptr()
            m.pos_b = pk.keep(sd["encoder.pos_conv_embed.conv.bias"]).data_ptr()
        m.enc_ln_g = pk.keep(sd["encoder.layer_norm.weight"]).data_ptr()
        m.enc_ln_b = pk.keep(sd["encoder.layer_norm.bias"]).data_ptr()
        self.layers = W.pack_layers(sd, W.HUBERT_NAMES, self.n_layers, pk, split=True)
        m.layers = self.layers
        # Operand format of the transformer layers (the conv feature encoder always runs BF16X3):
        #  * post-LN base family (HuBERT-base, wav2vec2-base, data2vec-audio): "f16" by default since round 2 -- one
        #    MMA per product instead of three; emulated readout error at 12 layers 3.3e-4 against 4e-5
        #    (scripts/precision_table.py), measured in tests/test_bench_config_gpu.py; MER_AUDIO_PRECISION=bf16x3
        #    (or stack_precision="bf16x3") keeps the split operands.
        #  * large (pre-LN) family: BF16X3 by default, "f16" opt-in (MER_HUBERT_LARGE_PRECISION=f16; clips of <= 249
        #    frames then run the stack on fp16 operands like the ViT, longer ones keep BF16X3).
        import os as _os
        if m.stable_layer_norm:
            self.stack_precision = stack_precision or _os.environ.get("MER_HUBERT_LARGE_PRECISION", "bf16x3")
        else:
            self.stack_precision = stack_precision or _os.environ.get("MER_AUDIO_PRECISION", "f16")
        assert self.stack_precision in ("bf16x3", "f16"), self.stack_precision
        if self.stack_precision == "f16":
            self.layers_f16 = W.pack_layers(sd, W.HUBERT_NAMES, self.n_layers, pk, f16=True)
            m.layers_f16 = self.layers_f16
        # Operand format of conv1 / conv2 (77 % of the conv stack's flops), group-norm family with fp16 layers only:
        # "f16" (default there) runs them as ONE fp16 MMA per product, conv3..6 and the feature projection stay BF16X3.
        # Emulated readout error at 12 layers (4 checkpoints x clips): 3.5e-4 mean / 4.2e-4 max against 3.2e-4 / 3.7e-4
        # with every conv on split operands; conv1..6 in fp16 would be 4.4e-4 / 5.1e-4
        # (scripts/precision_conv_layers.py).  MER_AUDIO_CONV_PRECISION=bf16x3 / conv_precision="bf16x3" opts out.
        default_conv = "f16" if (self.stack_precision == "f16" and not ln_convs and not m.stable_layer_norm and
                                 self.hidden == 768 and self.n_layers <= 12) else "bf16x3"  # the emulated configuration
        self.conv_precision = conv_precision or _os.environ.get("MER_AUDIO_CONV_PRECISION", default_conv)
        assert self.conv_precision in ("bf16x3", "f16"), self.conv_precision
        if self.conv_precision == "f16":
            assert not ln_convs, "fp16 conv1 / conv2 operands are implemented for the group-norm feature encoder"
            for i in range(2):
                w = sd[f"feature_extractor.conv_layers.{i + 1}.conv.weight"]
                m.conv_w_f16[i] = pk.keep(np.ascontiguousarray(w.transpose(0, 2, 1)).reshape(512, 3 * 512),
                                          f16=True).data_ptr()
        self.model = m
        self.ws = _Workspace(self.device)
        lib = L.lib()
        lib.mer_hubert_model_workspace_bytes.restype = C.c_longlong
        lib.mer_hubert_model_workspace_bytes.argtypes = [C.POINTER(MerHubertModel), C.c_int, C.c_int]
        lib.mer_hubert_num_frames.argtypes = [C.c_int]
        self._fwd = L.declare("mer_hubert_forward", [C.POINTER(MerHubertModel), C.c_void_p, C.c_int,
                                                     C.c_int, C.c_int, C.c_void_p, C.c_longlong,
                                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p])

    def num_frames(self, n_samples):
        return L.lib().mer_hubert_num_frames(int(n_samples))

    def forward(self, wave: torch.Tensor, normalize=True, want_frames=False, return_hidden=False):
        """wave: fp32 CUDA [B, L] (equal-length rows).  Returns (utt [B,D], frames [B,T,D]|None
        [, hidden [(layers+1), B, T, D]]), D = 768 or 1024."""
        assert wave.dtype == torch.float32 and wave.is_cuda and wave.dim() == 2
        wave = wave.contiguous()
        B, Ls = wave.shape
        T = self.num_frames(Ls)
        D = self.hidden
        ws = self.ws.get(L.lib().mer_hubert_model_workspace_bytes(C.byref(self.model), B, Ls))
        utt = torch.empty(B, D, dtype=torch.float32, device=self.device)
        frames = torch.empty(B, T, D, dtype=torch.float32, device=self.device) if want_frames else None
        hidden = (torch.empty(self.n_layers + 1, B, T, D, dtype=torch.float32, device=self.device)
                  if return_hidden else None)
        L.check(self._fwd(C.byref(self.model), L.ptr(wave), B, Ls, 1 if normalize else 0, L.ptr(ws),
                          ws.numel(), L.ptr(frames), L.ptr(utt), L.ptr(hidden), L.stream_ptr()))
        if return_hidden:
            return utt, frames, hidden
        return utt, frames


def _hubert_forward_ragged(self, rows: torch.Tensor, lengths, normalize=True, want_frames=False):
    """rows: fp32 CUDA [B, Lmax]; row b holds ``lengths[b]`` samples (the rest is ignored when ``normalize``, and must
    be finite otherwise).  Every clip is computed as if it were forwarded alone (mer_hubert_forward_ragged).
    Returns (utt [B, D], frames): frames = list of [T_b, D] tensors (views of one packed tensor) or None."""
    assert rows.dtype == torch.float32 and rows.is_cuda and rows.dim() == 2
    rows = rows.contiguous()
    B, Lmax = rows.shape
    lengths = [int(n) for n in lengths]
    assert len(lengths) == B and all(0 < n <= Lmax for n in lengths)
    tb = [self.num_frames(n) for n in lengths]
    D = self.hidden
    ws = self.ws.get(L.lib().mer_hubert_model_workspace_bytes(C.byref(self.model), B, Lmax))
    utt = torch.empty(B, D, dtype=torch.float32, device=self.device)
    packed = torch.empty(sum(tb), D, dtype=torch.float32, device=self.device) if want_frames else None
    fwd = L.declare("mer_hubert_forward_ragged", [C.POINTER(MerHubertModel), C.c_void_p, C.POINTER(C.c_int), C.c_int,
                                                  C.c_int, C.c_int, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p,
                                                  C.c_void_p])
    L.check(fwd(C.byref(self.model), L.ptr(rows), (C.c_int * B)(*lengths), B, Lmax, 1 if normalize else 0, L.ptr(ws),
                ws.numel(), L.ptr(packed), L.ptr(utt), L.stream_ptr()))
    return utt, (list(torch.split(packed, tb)) if want_frames else None)


HubertEncoder.forward_ragged = _hubert_forward_ragged


class MerBertModel(C.Structure):
    _fields_ = [("n_layers", C.c_int), ("ln_eps", C.c_float), ("word_emb", C.c_void_p),
                ("pos_emb", C.c_void_p), ("type_emb0", C.c_void_p), ("emb_ln_g", C.c_void_p),
                ("emb_ln_b", C.c_void_p), ("layers", C.POINTER(W.MerLayerWeights)),
                ("hidden", C.c_int), ("ffn", C.c_int), ("heads", C.c_int),
                ("layers_f16", C.POINTER(W.MerLayerWeights))]


class MerBertEmbedProjection(C.Structure):
    _fields_ = [("emb_dim", C.c_int), ("word_emb", C.c_void_p), ("pos_emb", C.c_void_p), ("type_emb0", C.c_void_p),
                ("emb_ln_g", C.c_void_p), ("emb_ln_b", C.c_void_p), ("proj_w", C.c_void_p), ("proj_w_f16", C.c_void_p),
                ("proj_b", C.c_void_p)]


# keys of an ElectraForPreTraining / ElectraForMaskedLM checkpoint that ElectraModel does not have (the prefix
# ``electra.`` is already gone, common.normalise_hf_keys), and the registered buffers some checkpoints carry
_BERT_IGNORED_PREFIXES = ("discriminator_predictions.", "generator_predictions.", "generator_lm_head.")
_BERT_IGNORED_KEYS = ("embeddings.position_ids", "embeddings.token_type_ids")


def bert_model_state(state_dict):
    """The tensors of the base model (BertModel / RobertaModel / ElectraModel) in a prefix-free checkpoint, as numpy:
    ELECTRA's discriminator / generator heads and the position / token-type id buffers are dropped."""
    return {k: v for k, v in W._np(state_dict).items()
            if k not in _BERT_IGNORED_KEYS and not k.startswith(_BERT_IGNORED_PREFIXES)}


class BertEncoder:
    """BERT-architecture encoders (HF ``BertModel`` / ``RobertaModel`` / ``ElectraModel``; hidden 768 or 1024: BERT,
    RoBERTa, MacBERT, PERT, LERT, ELECTRA base and large; hidden 256: LERT-small, and ELECTRA-small with its factorised
    128-wide embedding + ``embeddings_project``) over a packed variable-length batch + the reference readout (sum of
    the last four hidden states, strip specials, mean).

    Reference: MERBench/feature_extraction/text/extract_text_huggingface.py:222-249."""

    def __init__(self, state_dict, device="cuda", ln_eps=1e-12, position_offset=0, precision=None):
        """precision: operand format of the layers' linear products.  "f16" (default for the 12-layer base models since
        round 2; env MER_TEXT_PRECISION): one fp16 MMA per product, readout error 2.9e-4 at 12 layers; "bf16x3" (default
        for the 24-layer -large models and the hidden-256 small ones): three bf16 MMAs on (hi, lo) pairs, 3.5e-5
        (scripts/precision_table.py; hidden 256: scripts/precision_table_electra.py)."""
        L.check(L.lib().mer_check_device())
        sd = bert_model_state(state_dict)
        self.device = torch.device(device)
        pk = self.pk = W.Packed(self.device)
        self.position_offset = position_offset  # 0 = BERT, 2 = RoBERTa (pad_token_id + 1)
        self.n_layers = W.count_layers(sd, "encoder.layer.{i}.output.LayerNorm.weight")
        m = MerBertModel()
        m.n_layers, m.ln_eps = self.n_layers, ln_eps
        self.word = pk.keep(sd["embeddings.word_embeddings.weight"])
        self.pos = pk.keep(sd["embeddings.position_embeddings.weight"])
        self.vocab_size, self.max_pos = self.word.shape[0], self.pos.shape[0]
        # ELECTRA with embedding_size != hidden_size: the E-wide embedding is projected to the hidden size
        projected = "embeddings_project.weight" in sd
        self.emb_dim = int(self.word.shape[1])
        # base (768 / 12 heads / 3072), -large (1024 / 16 / 4096) or small (256 / 4 / 1024) checkpoints
        self.hidden = int(sd["embeddings_project.weight"].shape[0]) if projected else self.emb_dim
        ffn = int(sd["encoder.layer.0.intermediate.dense.weight"].shape[0])
        assert self.hidden in (256, 768, 1024) and ffn % 128 == 0, \
            f"hidden {self.hidden} / ffn {ffn}: hidden 256, 768 or 1024 and ffn % 128 == 0 are on the H100 path"
        assert not projected or (self.emb_dim in (128, 256) and self.emb_dim != self.hidden and 2 * self.emb_dim <= ffn), \
            f"embedding size {self.emb_dim} -> hidden {self.hidden}: a projected embedding of 128 or 256 is on the H100 path"
        m.hidden, m.ffn, m.heads = self.hidden, ffn, self.hidden // 64
        emb = dict(word_emb=self.word.data_ptr(), pos_emb=self.pos.data_ptr(),
                   type_emb0=pk.keep(sd["embeddings.token_type_embeddings.weight"][0]).data_ptr(),
                   emb_ln_g=pk.keep(sd["embeddings.LayerNorm.weight"]).data_ptr(),
                   emb_ln_b=pk.keep(sd["embeddings.LayerNorm.bias"]).data_ptr())
        self.layers = W.pack_layers(sd, W.BERT_NAMES, self.n_layers, pk, split=True)
        m.layers = self.layers
        import os as _os
        # hidden 256: bf16x3, the emulated f16 readout error of the x5 stress checkpoint is 1.1e-2 at 12 layers
        self.precision = precision or _os.environ.get("MER_TEXT_PRECISION", "f16" if self.hidden == 768 else "bf16x3")
        assert self.precision in ("bf16x3", "f16"), self.precision
        if self.precision == "f16":
            self.layers_f16 = W.pack_layers(sd, W.BERT_NAMES, self.n_layers, pk, f16=True)
            m.layers_f16 = self.layers_f16
        self.proj = None
        if projected:  # the tables go to the projection struct; the model's stay NULL (not read)
            pr = self.proj = MerBertEmbedProjection()
            pr.emb_dim = self.emb_dim
            for k, v in emb.items():
                setattr(pr, k, v)
            w = sd["embeddings_project.weight"]
            if self.precision == "f16":
                pr.proj_w_f16 = pk.keep(w, f16=True).data_ptr()
            else:
                pr.proj_w = pk.keep(w, split=True).data_ptr()
            pr.proj_b = pk.keep(sd["embeddings_project.bias"]).data_ptr()
        else:
            for k, v in emb.items():
                setattr(m, k, v)
        self.model = m
        self.ws = _Workspace(self.device)
        lib = L.lib()
        lib.mer_bert_model_workspace_bytes.restype = C.c_longlong
        lib.mer_bert_model_workspace_bytes.argtypes = [C.POINTER(MerBertModel), C.c_int, C.c_int]
        vp, i32 = C.c_void_p, C.c_int
        if projected:
            fwd = L.declare("mer_bert_forward_projected", [C.POINTER(MerBertModel), C.POINTER(MerBertEmbedProjection),
                                                           vp, vp, vp, i32, i32, i32, vp, vp, vp, C.c_longlong, vp, vp,
                                                           vp, vp])
            self._fwd = lambda model, *args: fwd(model, C.byref(self.proj), *args)
        else:
            self._fwd = L.declare("mer_bert_forward", [C.POINTER(MerBertModel), vp, vp, vp, i32, i32, i32,
                                                       vp, vp, vp, C.c_longlong, vp, vp, vp, vp])

    def forward_packed(self, ids, seqlen, start=1, end=-1):
        """Device fast path for n sentences of identical length: ids int32 CUDA [n, seqlen].  Position
        ids / cu_seqlens / kept ranges are built once per (n, seqlen) on the device.
        Returns (utt [n,768], None)."""
        assert ids.is_cuda and ids.dtype == torch.int32 and ids.shape[1] == seqlen
        n = ids.shape[0]
        key = (n, seqlen, start, end)
        if getattr(self, "_packed_key", None) != key:
            ar = torch.arange(n + 1, dtype=torch.int32, device=self.device) * seqlen
            pos = (torch.arange(seqlen, dtype=torch.int32, device=self.device) + self.position_offset).repeat(n)
            self._packed = (ar, pos.contiguous(), (ar[:-1] + (start or 0)).contiguous(),
                            (ar[1:] + (end if end is not None else 0)).contiguous())
            self._packed_key = key
        cu, pos, seg_b, seg_e = self._packed
        n_tok = n * seqlen
        ws = self.ws.get(L.lib().mer_bert_model_workspace_bytes(C.byref(self.model), n_tok, n))
        utt = torch.empty(n, self.hidden, dtype=torch.float32, device=self.device)
        L.check(self._fwd(C.byref(self.model), L.ptr(ids.contiguous()), L.ptr(pos), L.ptr(cu), n, n_tok,
                          seqlen, L.ptr(seg_b), L.ptr(seg_e), L.ptr(ws), ws.numel(), None, L.ptr(utt),
                          None, L.stream_ptr()))
        return utt, None

    def forward(self, id_lists, start=1, end=-1, want_tokens=False, return_hidden=False):
        """id_lists: list of non-empty python/numpy int sequences (one tokenised sentence each).
        Returns (utt [n,768], tokens [sum T,768]|None [, hidden, cu_seqlens])."""
        lens = [len(x) for x in id_lists]
        assert all(n > 0 for n in lens), "empty sentences are handled by the caller (zeros)"
        assert max(lens) + self.position_offset <= self.max_pos, "sentence longer than position table"
        ids = np.concatenate([np.asarray(x, dtype=np.int64) for x in id_lists])
        assert ids.min() >= 0 and ids.max() < self.vocab_size, "token id outside the vocabulary"
        cu = np.zeros(len(lens) + 1, dtype=np.int32)
        cu[1:] = np.cumsum(lens)
        pos = np.concatenate([np.arange(n) for n in lens]).astype(np.int32) + self.position_offset
        e = end if end is not None else 0
        seg_b = (cu[:-1] + (start or 0)).astype(np.int32)
        seg_e = (cu[1:] + e).astype(np.int32)
        host = np.concatenate([ids.astype(np.int32), pos, cu, seg_b, seg_e])
        dev = torch.from_numpy(host).pin_memory().to(self.device, non_blocking=True)
        n_tok, n_seq = int(cu[-1]), len(lens)
        d_ids, d_pos = dev[:n_tok], dev[n_tok:2 * n_tok]
        d_cu = dev[2 * n_tok:2 * n_tok + n_seq + 1]
        d_b = dev[2 * n_tok + n_seq + 1:2 * n_tok + 2 * n_seq + 1]
        d_e = dev[2 * n_tok + 2 * n_seq + 1:]
        ws = self.ws.get(L.lib().mer_bert_model_workspace_bytes(C.byref(self.model), n_tok, n_seq))
        utt = torch.empty(n_seq, self.hidden, dtype=torch.float32, device=self.device)
        toks = torch.empty(n_tok, self.hidden, dtype=torch.float32, device=self.device) if want_tokens else None
        hidden = (torch.empty(self.n_layers + 1, n_tok, self.hidden, dtype=torch.float32, device=self.device)
                  if return_hidden else None)
        L.check(self._fwd(C.byref(self.model), L.ptr(d_ids), L.ptr(d_pos), L.ptr(d_cu), n_seq, n_tok,
                          max(lens), L.ptr(d_b), L.ptr(d_e), L.ptr(ws), ws.numel(), L.ptr(toks),
                          L.ptr(utt), L.ptr(hidden), L.stream_ptr()))
        if return_hidden:
            return utt, toks, hidden, cu
        return utt, toks
