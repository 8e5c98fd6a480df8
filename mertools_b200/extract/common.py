"""Shared host-side pieces of the extractors: checkpoint loading and the .npy feature contract."""
from __future__ import annotations

import json
import os

import numpy as np


_PREFIXES = ("vit.", "hubert.", "bert.", "roberta.", "wav2vec2.", "data2vec_audio.", "electra.", "videomae.", "wavlm.",
             "data2vec_vision.", "dinov2.")


def _read_weights_file(path):
    if path.endswith(".safetensors"):
        from safetensors.numpy import load_file
        return load_file(path)
    import torch
    return {k: v.float().numpy() for k, v in torch.load(path, map_location="cpu").items()}


def normalise_hf_keys(sd):
    """The key fixes ``from_pretrained`` applies before matching a checkpoint to the model (the reference loads with
    ``AutoModel.from_pretrained``, e.g. extract_text_huggingface.py:163-190): the task-model prefix is dropped
    (``bert.``, ``hubert.`` ...), and the pre-2019 TensorFlow-style LayerNorm names ``*.gamma`` / ``*.beta`` still
    carried by bert-base-chinese / bert-base-uncased become ``*.weight`` / ``*.bias``."""
    out = {}
    for k, v in sd.items():
        for pre in _PREFIXES:
            if k.startswith(pre):
                k = k[len(pre):]
                break
        if k.endswith(".gamma") or k == "gamma":
            k = k[:-5] + "weight"
        elif k.endswith(".beta") or k == "beta":
            k = k[:-4] + "bias"
        out[k] = np.asarray(v, dtype=np.float32)
    return out


def load_hf_state_dict(model_dir):
    """HF checkpoint directory -> {name: numpy fp32} without instantiating the HF model (only the tensors are
    needed here).  Single-file checkpoints (``model.safetensors`` / ``pytorch_model.bin``) and sharded ones
    (``model.safetensors.index.json`` / ``pytorch_model.bin.index.json`` with their ``weight_map``)."""
    for single in ("model.safetensors", "pytorch_model.bin"):
        path = os.path.join(model_dir, single)
        if os.path.exists(path):
            return normalise_hf_keys(_read_weights_file(path))
    for index in ("model.safetensors.index.json", "pytorch_model.bin.index.json"):
        path = os.path.join(model_dir, index)
        if os.path.exists(path):
            shards = sorted(set(json.load(open(path))["weight_map"].values()))
            sd = {}
            for shard in shards:
                sd.update(_read_weights_file(os.path.join(model_dir, shard)))
            return normalise_hf_keys(sd)
    raise AssertionError(f"no model.safetensors / pytorch_model.bin (or their .index.json) under {model_dir}")


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
        import torch
        sd = torch.load(path, map_location="cpu", mmap=True, weights_only=True)
        for k in list(sd):
            yield k, sd.pop(k)


def stream_fp16_weights(model_dir, device, rename, prefer_bin=False):
    """Yield (name, fp16 tensor on ``device``) for every tensor of a checkpoint, read one at a time (safetensors through
    ``safe_open``, ``.bin`` through an mmap'ed ``torch.load``) from fp32 / fp16 / bf16 shards, so that a large
    checkpoint never exists as fp32 in host memory.  Safetensors are read when both formats exist, ``.bin`` with
    ``prefer_bin``.  ``rename(key)``: the name to yield, or None to skip the tensor.  A value that is not finite
    in fp16 is refused."""
    import torch
    for path in _checkpoint_files(model_dir, prefer_bin):
        for k, v in _iter_tensors(path):
            k = rename(k)
            if k is None:
                continue
            t = v.to(device).to(torch.float16)
            if not bool(torch.isfinite(t).all()):
                raise ValueError(f"{path}: {k} is not finite in fp16")
            yield k, t


def read_do_normalize(model_dir, default=True):
    """``do_normalize`` of the checkpoint's ``preprocessor_config.json``: the reference builds
    ``Wav2Vec2FeatureExtractor.from_pretrained(model_file)`` (extract_audio_huggingface.py:60-64), which applies the
    zero-mean / unit-variance step only when the checkpoint says so (hubert-base-ls960 and wavlm-base ship false)."""
    path = os.path.join(model_dir, "preprocessor_config.json")
    if not os.path.exists(path):
        return default
    return bool(json.load(open(path)).get("do_normalize", default))


def save_feature(save_file, embeddings, feature_level, feature_dim):
    """The on-disk contract shared by the three scripts (extract_vision_huggingface.py:175-189,
    extract_text_huggingface.py:235-249): UTTERANCE -> 1-D [D] (mean over rows when 2-D),
    FRAME -> 2-D [T, D]; empty -> zeros (float64, as np.zeros in the reference)."""
    emb = np.array(embeddings).squeeze()
    if feature_level == "FRAME":
        if emb.size == 0:
            emb = np.zeros((1, feature_dim))
        elif emb.ndim == 1:
            emb = emb[np.newaxis, :]
    else:
        if emb.size == 0:
            emb = np.zeros((feature_dim,))
        elif emb.ndim == 2:
            emb = np.mean(emb, axis=0)
    if save_file is not None:
        np.save(save_file, emb)
    return emb
