"""VideoMAE branch of the visual extractor: mirror of MERBench/feature_extraction/visual/extract_vision_huggingface.py:
147-159 (``videomae-base`` / ``videomae-large``: 16 uniformly resampled frames -> VideoMAEImageProcessor ->
``VideoMAEModel(...).last_hidden_state`` [1568, D] -> mean over the 196 patches of each of the 8 tubelets -> [8, D]).

The encoder is orchestrated over kernel-level entry points of libmer_b200.so through the same ``ops`` backend as the
Whisper branch (``mer_videomae_patchify`` + the patch-embedding GEMM, TF32 linears, ``mer_layernorm``, ``mer_attention``
over 1568 tokens), so that the orchestration runs against the oracle with a torch backend on CPU
(tests/test_host_logic.py).  GPU parity test: tests/test_variants_gpu.py.
"""
from __future__ import annotations

import numpy as np
import torch

from .visual import resample_frames_uniform

TOKENS, TUBELETS, PATCHES = 1568, 8, 196


def sinusoid_table(n_position, d):
    """HF modeling_videomae.get_sinusoid_encoding_table (fixed position embeddings)."""
    pos = np.arange(n_position, dtype=np.float64)[:, None]
    tab = pos / np.power(10000.0, 2 * (np.arange(d) // 2) / d)[None, :]
    tab[:, 0::2] = np.sin(tab[:, 0::2])
    tab[:, 1::2] = np.cos(tab[:, 1::2])
    return tab.astype(np.float32)


class VideoMaeNet:
    """Backend-agnostic orchestration of VideoMAEModel (final LayerNorm when the checkpoint has one).
    ``ops``: tensor, weight, patchify, layernorm, linear, self_attention."""

    def __init__(self, state_dict, ops, eps=1e-12):
        sd = {k: np.asarray(v, np.float32) for k, v in state_dict.items()}
        self.ops, self.eps = ops, eps
        w = sd["embeddings.patch_embeddings.projection.weight"]                      # [D, 3, 2, 16, 16]
        self.d = d = w.shape[0]
        assert w.shape[1:] == (3, 2, 16, 16) and d % 64 == 0
        self.heads = d // 64
        self.patch_w, self.patch_b = ops.weight(w.reshape(d, -1)), ops.tensor(sd["embeddings.patch_embeddings.projection.bias"])
        self.pos = sinusoid_table(TOKENS, d)
        zeros = np.zeros(d, np.float32)
        # self-supervised checkpoints (use_mean_pooling=False: videomae-base / -large) close with VideoMAEModel.layernorm
        self.final_ln = ((ops.tensor(sd["layernorm.weight"]), ops.tensor(sd["layernorm.bias"]))
                         if "layernorm.weight" in sd else None)
        self.layers = []
        i = 0
        while f"encoder.layer.{i}.output.dense.weight" in sd:
            p = f"encoder.layer.{i}."
            a = p + "attention.attention."
            self.layers.append(dict(
                ln1=(ops.tensor(sd[p + "layernorm_before.weight"]), ops.tensor(sd[p + "layernorm_before.bias"])),
                qkv_w=ops.weight(np.concatenate([sd[a + "query.weight"], sd[a + "key.weight"], sd[a + "value.weight"]], 0)),
                qkv_b=ops.tensor(np.concatenate([sd[a + "q_bias"], zeros, sd[a + "v_bias"]])),
                o_w=ops.weight(sd[p + "attention.output.dense.weight"]), o_b=ops.tensor(sd[p + "attention.output.dense.bias"]),
                ln2=(ops.tensor(sd[p + "layernorm_after.weight"]), ops.tensor(sd[p + "layernorm_after.bias"])),
                w1=ops.weight(sd[p + "intermediate.dense.weight"]), b1=ops.tensor(sd[p + "intermediate.dense.bias"]),
                w2=ops.weight(sd[p + "output.dense.weight"]), b2=ops.tensor(sd[p + "output.dense.bias"])))
            i += 1

    def last_hidden_state(self, frames_bgr_u8, mean, std):
        """frames: uint8 [B * 16, 224, 224, 3] BGR (backend array).  Returns [B, 1568, D]."""
        ops = self.ops
        B = frames_bgr_u8.shape[0] // 16
        x = ops.linear(ops.patchify(frames_bgr_u8, mean, std), self.patch_w, self.patch_b,
                       res=ops.tensor(np.tile(self.pos, (B, 1))))                   # conv3d + bias + positions
        for L in self.layers:
            y = ops.layernorm(x, *L["ln1"], operand=True, eps=self.eps)
            ctx = ops.self_attention(ops.linear(y, L["qkv_w"], L["qkv_b"], operand=True), B, TOKENS, self.heads)
            x = ops.linear(ctx, L["o_w"], L["o_b"], res=x)
            y = ops.layernorm(x, *L["ln2"], operand=True, eps=self.eps)
            x = ops.linear(ops.linear(y, L["w1"], L["b1"], gelu=True, operand=True), L["w2"], L["b2"], res=x)
        if self.final_ln is not None:
            x = ops.layernorm(x, *self.final_ln, operand=False, eps=self.eps)
        return x.reshape(B, TOKENS, self.d)


def _cuda_ops(device):
    """The Whisper branch's CudaOps plus the VideoMAE patch gather."""
    import ctypes as C

    from .whisper import CudaOps

    class Ops(CudaOps):
        def __init__(self, device):
            super().__init__(device)
            self._patchify = self.L.declare("mer_videomae_patchify", [C.c_void_p, C.c_int, C.POINTER(C.c_float),
                                                                      C.POINTER(C.c_float), C.c_void_p, C.c_void_p])

        def patchify(self, frames, mean, std):
            n = frames.shape[0] // 16
            out = torch.empty(n * TOKENS, 1536, dtype=torch.float32, device=self.device)
            self.L.check(self._patchify(self.L.ptr(frames.contiguous()), n, (C.c_float * 3)(*mean), (C.c_float * 3)(*std),
                                        self.L.ptr(out), self.L.stream_ptr()))
            return out

        def layernorm(self, x, g, b, operand, eps=1e-5):
            y = torch.empty_like(x)
            self.L.layernorm(x, g, b, y, eps=eps, flags=self.L.MER_LN_ROUND_TF32 if operand else 0)
            return y
    return Ops(device)


class VideoMaeExtractor:
    """One video -> the array the reference saves: FRAME [8, D] (one row per tubelet), UTTERANCE [D]."""

    def __init__(self, state_dict, device="cuda", mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225), eps=1e-12):
        import ctypes as C

        from .. import _lib as L
        self.ops = _cuda_ops(device)
        self.net = VideoMaeNet(state_dict, self.ops, eps=eps)
        self.mean, self.std, self.device = tuple(mean), tuple(std), self.ops.device
        L.lib().mer_resize_workspace_bytes.restype = C.c_longlong
        L.lib().mer_resize_workspace_bytes.argtypes = [C.c_int] * 5
        self._resize = L.declare("mer_resize_u8", [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                                   C.c_int, C.c_void_p, C.c_void_p])
        self._L = L

    @classmethod
    def from_pretrained(cls, model_dir, device="cuda"):
        """Checkpoint directory of the reference (``transformers/videomae-base``): weights + the processor's mean / std
        and the config's layer_norm_eps."""
        import json
        import os

        from . import common
        kw = {}
        pc, mc = os.path.join(model_dir, "preprocessor_config.json"), os.path.join(model_dir, "config.json")
        if os.path.exists(pc):
            cfg = json.load(open(pc))
            kw.update(mean=cfg.get("image_mean", (0.485, 0.456, 0.406)), std=cfg.get("image_std", (0.229, 0.224, 0.225)))
        if os.path.exists(mc):
            kw.update(eps=float(json.load(open(mc)).get("layer_norm_eps", 1e-12)))
        return cls(common.load_hf_state_dict(model_dir), device=device, **kw)

    def extract_clips(self, clips, feature_level="UTTERANCE", nframe=None, save_files=None):
        """Same call shape as VisualExtractor.extract_clips (``nframe`` is fixed at 16 by the model)."""
        from . import common
        res = [self.extract_clip(c, feature_level) for c in clips]
        if save_files is not None:
            for path, r in zip(save_files, res):
                common.save_feature(path, r, feature_level, self.net.d)
        return res

    def preprocess(self, frames_bgr):
        """resample_frames_uniform(frames, 16) + the processor's geometry (shortest edge -> 224, PIL bilinear; centre
        crop 224) on the device; rescale / normalise happen in the patch gather."""
        L = self._L
        f = torch.from_numpy(np.ascontiguousarray(resample_frames_uniform(np.asarray(frames_bgr), 16))).to(self.device)
        n, h, w, _ = f.shape
        nh, nw = (224, int(224 * w / h)) if h <= w else (int(224 * h / w), 224)
        if (nh, nw) != (h, w):
            out = torch.empty(n, nh, nw, 3, dtype=torch.uint8, device=self.device)
            ws = torch.empty(max(int(L.lib().mer_resize_workspace_bytes(n, h, w, nh, nw)), 1), dtype=torch.uint8, device=self.device)
            L.check(self._resize(L.ptr(f), n, h, w, L.ptr(out), nh, nw, 0, L.ptr(ws), L.stream_ptr()))
            f = out
        top, left = (nh - 224) // 2, (nw - 224) // 2
        return f[:, top:top + 224, left:left + 224].contiguous()

    def extract_clip(self, frames_bgr, feature_level="UTTERANCE"):
        hs = self.net.last_hidden_state(self.preprocess(frames_bgr), self.mean, self.std)       # [1, 1568, D]
        emb = hs.reshape(TUBELETS, PATCHES, -1).mean(dim=1).cpu().numpy().squeeze()             # [8, D]
        return np.mean(emb, axis=0) if feature_level == "UTTERANCE" and emb.ndim == 2 else emb
