"""CPU restatement of MER2024's VideoMAE face-clip extractor (feature_extraction/visual/extract_sun_videomae.py over the
vendored videomae package) for the sun_videomae tests, tests/golden/make_golden_sun_videomae.py and
scripts/bench_sun_videomae.py, composed from the oracle's helpers (oracle/encoders.py ``_ln`` / ``_linear`` / ``_mha``):

    frames  -> PIL bilinear resize to S x S (video_transforms.Resize((S, S)))
            -> float32(p) / 255, (x - mean) / std in fp32 (ClipToTensor, Normalize)
    clip    -> Conv3d (2, 16, 16) patch embedding + the fixed sinusoid table
            -> pre-LN blocks (qkv without key bias, erf-GELU MLP, LayerNorm eps 1e-6) -> norm -> mean over the tokens
    video   -> 4 views per frame id (kinetics.py:VideoClsDatasetFrame), float64 np.mean per id (final_test)

plus the synthetic checkpoints (pretrain layout: ``model`` key, ``encoder.`` prefix, decoder keys) and videos the golden
and the tests share.  The view planning here is written independently of mertools_b200.extract.sun_videomae, straight
from the dataset's index rules."""
import numpy as np
import torch
import torch.nn.functional as F
from PIL import Image

from oracle import encoders as E

MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
SHAPES = {"vit_base_patch16_160": (160, 768, 12), "vit_base_patch16_224": (224, 768, 12),
          "vit_large_patch16_224": (224, 1024, 16)}   # img, dim, heads


def synth_video(n, h=112, w=112, seed=0):
    """uint8 [n, h, w, 3]: a smooth face-like gradient per frame plus noise, drifting over time."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    base = 128 + 60 * np.sin(yy[None, :, :, None] / 9.0 + np.arange(3)[None, None, None, :])
    base = base + 40 * np.cos(xx[None, :, :, None] / 13.0 + np.arange(n)[:, None, None, None] * 0.3)
    return np.clip(base + rng.normal(0, 20, (n, h, w, 3)), 0, 255).astype(np.uint8)


def synth_checkpoint(dim, layers, seed=0):
    """A pretraining checkpoint of a ``dim``-wide, ``layers``-deep encoder: {'model': {'encoder.*', 'decoder.*',
    'mask_token', 'encoder_to_decoder.weight', 'encoder.pos_embed'}} (float32 torch tensors)."""
    rng = np.random.default_rng(seed)
    f = 4 * dim
    t = lambda *s, std=0.02: torch.from_numpy((rng.standard_normal(s) * std).astype(np.float32))  # noqa: E731
    sd = {"encoder.patch_embed.proj.weight": t(dim, 3, 2, 16, 16, std=0.03), "encoder.patch_embed.proj.bias": t(dim)}
    for i in range(layers):
        p = f"encoder.blocks.{i}."
        sd.update({
            p + "norm1.weight": 1 + t(dim, std=0.1), p + "norm1.bias": t(dim),
            p + "attn.qkv.weight": t(3 * dim, dim, std=0.05), p + "attn.q_bias": t(dim, std=0.1),
            p + "attn.v_bias": t(dim, std=0.1),
            p + "attn.proj.weight": t(dim, dim), p + "attn.proj.bias": t(dim),
            p + "norm2.weight": 1 + t(dim, std=0.1), p + "norm2.bias": t(dim),
            p + "mlp.fc1.weight": t(f, dim), p + "mlp.fc1.bias": t(f),
            p + "mlp.fc2.weight": t(dim, f), p + "mlp.fc2.bias": t(dim),
        })
    sd.update({"encoder.norm.weight": 1 + t(dim, std=0.1), "encoder.norm.bias": t(dim),
               "encoder.pos_embed": t(1, 8, dim), "mask_token": t(1, 1, 384),
               "encoder_to_decoder.weight": t(384, dim), "decoder.blocks.0.mlp.fc1.weight": t(16, 384),
               "decoder.norm.weight": t(384)})
    return {"model": sd}


def model_params(ckpt):
    """The checkpoint's encoder parameters under the model's names (prefix stripped; other keys dropped)."""
    return {k[8:]: v for k, v in ckpt["model"].items() if k.startswith("encoder.") and k != "encoder.pos_embed"}


# ---- data path ----
def resize(frames, S):
    """Image.fromarray(f).convert('RGB'), resized to (S, S) with PIL bilinear, per frame."""
    return np.stack([np.asarray(Image.fromarray(f).convert("RGB").resize((S, S), Image.BILINEAR)) for f in frames])


def clip_tensor(resized, rows):
    """ClipToTensor + Normalize of the 16 frames ``rows`` of the resized video: fp32 [3, 16, S, S]."""
    x = torch.from_numpy(resized[list(rows)].astype(np.float64)).permute(3, 0, 1, 2).float()
    x = torch.div(x, 255)
    mean = torch.as_tensor(MEAN, dtype=torch.float32)[:, None, None, None]
    std = torch.as_tensor(STD, dtype=torch.float32)[:, None, None, None]
    return (x - mean) / std


def views(n, feature_level, sampling_rate=4):
    """[(frame id, 16 frame rows)] in the dataset's item order (kinetics.py:49-107, 111-125)."""
    def rows(idxs):
        while len(idxs) < 16:
            idxs.append(idxs[-1])
        buf = [np.arange(n)[min(i, n - 1)] for i in idxs]     # numpy indexing: negative indices wrap
        step = max(1.0 * (len(buf) - 16) / (2 - 1), 0)
        return buf, step

    items = []
    for ck in range(2):
        for _cp in range(2):
            if feature_level == "UTTERANCE":
                buf, step = rows(list(range(0, n, sampling_rate)))
                items.append((0, tuple(int(r) for r in buf[int(ck * step):int(ck * step) + 16])))
                continue
            for f in range(n):
                if f < 10:
                    s, e = 0, 16
                elif f > n - 10:
                    s, e = n - 17, n - 1
                else:
                    s, e = f - 8, f + 8
                buf, step = rows(list(range(s, e)))
                items.append((f, tuple(int(r) for r in buf[int(ck * step):int(ck * step) + 16])))
    return items


# ---- model ----
def sinusoid(n, d):
    return E.videomae_sinusoid_table(n, d)


def view_features(params, clips, heads, eps=1e-6, dtype=torch.float32):
    """VisionTransformer.forward_features (use_mean_pooling=False): clips [B, 3, 16, S, S] -> [B, D]."""
    x = clips.to(dtype)
    w = E._t(params, "patch_embed.proj.weight", dtype)
    x = F.conv3d(x, w, E._t(params, "patch_embed.proj.bias", dtype), stride=(2, 16, 16)).flatten(2).transpose(1, 2)
    x = x + sinusoid(x.shape[1], x.shape[2]).to(x.device, dtype)
    D = x.shape[-1]
    i = 0
    while f"blocks.{i}.attn.qkv.weight" in params:
        p = f"blocks.{i}."
        y = E._ln(x, params, p + "norm1", eps, dtype)
        bias = torch.cat([E._t(params, p + "attn.q_bias", dtype), torch.zeros(D, dtype=dtype, device=x.device),
                          E._t(params, p + "attn.v_bias", dtype)])
        qkv = F.linear(y, E._t(params, p + "attn.qkv.weight", dtype), bias)
        x = x + E._linear(E._mha(qkv[..., :D], qkv[..., D:2 * D], qkv[..., 2 * D:], heads), params, p + "attn.proj", dtype)
        h = F.gelu(E._linear(E._ln(x, params, p + "norm2", eps, dtype), params, p + "mlp.fc1", dtype))
        x = x + E._linear(h, params, p + "mlp.fc2", dtype)
        i += 1
    return E._ln(x, params, "norm", eps, dtype).mean(1)


def final_test(items, feats, feature_level):
    """engine_for_finetuning.py:final_test on per-item features (fp32 [D] each, item order)."""
    saved = {}
    for (fid, _), f in zip(items, feats):
        saved.setdefault("%010d" % fid, []).append(np.asarray(f, np.float32).tolist())
    emb = np.array([np.mean(saved[k], axis=0) for k in sorted(saved)]).squeeze()
    if feature_level == "FRAME":
        return emb[np.newaxis, :] if emb.ndim == 1 else emb
    return np.mean(emb, axis=0) if emb.ndim == 2 else emb


def video_features(params, frames, model, feature_level, sampling_rate=4, dtype=torch.float32, batch=8):
    """The saved array of one video (float64), every distinct view computed once in ``dtype``."""
    S, _, heads = SHAPES[model]
    rs = resize(frames, S)
    items = views(len(frames), feature_level, sampling_rate)
    uniq = list(dict.fromkeys(r for _, r in items))
    out = {}
    with torch.no_grad():
        for s in range(0, len(uniq), batch):
            chunk = uniq[s:s + batch]
            f = view_features(params, torch.stack([clip_tensor(rs, r) for r in chunk]), heads, dtype=dtype)
            out.update({r: f[j].float().numpy() if dtype == torch.float32 else f[j].numpy() for j, r in enumerate(chunk)})
    if dtype == torch.float32:
        return final_test(items, [out[r] for _, r in items], feature_level)
    # float64: the exact mean of the per-view values
    emb = {}
    for fid, r in items:
        emb.setdefault(fid, []).append(out[r])
    arr = np.array([np.mean(emb[k], axis=0) for k in sorted(emb)])
    return arr if feature_level == "FRAME" else arr.mean(0)
