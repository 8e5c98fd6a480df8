"""Float64 restatement of what the MER_VISION_EVA02 tower computes, from the CLIP-layout tensors of
``eva02_to_clip_layout`` and the loader's rotary tables, plus the synthetic faces of the EVA02 golden.  CPU only."""
import numpy as np
import torch

from mertools_b200 import encoders as E


def synth_faces(n, h=112, w=112, seed=0):
    """uint8 [n, h, w, 3] BGR frames: smooth gradients plus noise, so that the resize and crop are exercised."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([(yy * 255 // max(h - 1, 1)), (xx * 255 // max(w - 1, 1)), ((yy + xx) * 127 // max(h + w - 2, 1))],
                    -1)
    noise = rng.integers(-40, 41, size=(n, h, w, 3))
    return np.clip(base[None] + noise, 0, 255).astype(np.uint8)


def _ln(x, g, b, eps):
    m = x.mean(-1, keepdim=True)
    v = ((x - m) ** 2).mean(-1, keepdim=True)
    return (x - m) / torch.sqrt(v + eps) * g + b


def f16(t):
    return t.to(torch.float16).to(torch.float64)


def tf32(t):
    """round-to-nearest (ties away) to 10 mantissa bits, as cvt.rna.tf32.f32"""
    b = t.to(torch.float32).view(torch.int32)
    return ((b + 0x1000) & ~0x1fff).view(torch.float32).to(torch.float64)


def forward(layout, pixels, eps=1e-6, heads=12, return_hidden=False, op=None):
    """pixels: float [N, 3, S, S] normalised.  Returns the features [N, D] (float64) and, with return_hidden, the
    hidden states [(layers + 1), N, tokens, D] (state 0 = embeddings).

    op (emulation of the device's operand formats, None = exact): f16 or tf32 applied to both operands of every linear
    layer of the blocks; q | k (after the rotation), V and the attention probabilities then go through fp16, as the
    fp16 V^T attention kernel takes them in both formats."""
    d64 = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.float64)  # noqa: E731
    o = op or (lambda t: t)
    a16 = f16 if op else (lambda t: t)
    v = "vision_model."
    pw = d64(layout[v + "embeddings.patch_embedding.weight"])
    D, _, p, _ = pw.shape
    x = torch.nn.functional.conv2d(pixels.double(), pw, stride=p).flatten(2).transpose(1, 2)
    pos = d64(layout[v + "embeddings.position_embedding.weight"])
    cls = d64(layout[v + "embeddings.class_embedding"]) + pos[0]
    x = torch.cat([cls.expand(x.shape[0], 1, D), x + pos[1:]], 1)
    N, T, _ = x.shape
    cos, sin = (d64(t) for t in E.eva02_rope_tables(int(round((T - 1) ** 0.5))))

    def rope(t):   # t [N, H, T, 64]; class row untouched
        a, b = t[..., 1:, 0::2], t[..., 1:, 1::2]
        out = t.clone()
        out[..., 1:, 0::2] = a * cos - b * sin
        out[..., 1:, 1::2] = b * cos + a * sin
        return out

    hidden = [x]
    i = 0
    while f"{v}encoder.layers.{i}.layer_norm1.weight" in layout:
        g = lambda k: d64(layout[f"{v}encoder.layers.{i}.{k}"])  # noqa: E731
        h = o(_ln(x, g("layer_norm1.weight"), g("layer_norm1.bias"), eps))
        q, k, vv = (a16(h @ o(g(f"self_attn.{n}.weight")).T + g(f"self_attn.{n}.bias"))
                    for n in ("q_proj", "k_proj", "v_proj"))
        q, k, vv = (t.reshape(N, T, heads, 64).transpose(1, 2) for t in (q, k, vv))
        q, k = a16(rope(q)), a16(rope(k))
        a = a16(torch.softmax(q @ k.transpose(-1, -2) / 8.0, -1)) @ vv
        ctx = o(a.transpose(1, 2).reshape(N, T, D))
        x = x + ctx @ o(g("self_attn.out_proj.weight")).T + g("self_attn.out_proj.bias")
        h = o(_ln(x, g("layer_norm2.weight"), g("layer_norm2.bias"), eps))
        u = h @ o(g("mlp.fc1.weight")).T + g("mlp.fc1.bias")
        gate, val = u.chunk(2, -1)
        m = o(_ln(torch.nn.functional.silu(gate) * val, g("mlp.norm.weight"), g("mlp.norm.bias"), eps))
        x = x + m @ o(g("mlp.fc2.weight")).T + g("mlp.fc2.bias")
        hidden.append(x)
        i += 1
    feats = _ln(x[:, 1:].mean(1), d64(layout[v + "post_layernorm.weight"]), d64(layout[v + "post_layernorm.bias"]), eps)
    return (feats, torch.stack(hidden)) if return_hidden else feats


def pixels_from_frames(frames_bgr, transform):
    """The reference's per-frame host path: cv2 BGR -> RGB -> PIL -> timm eval transform, stacked."""
    from PIL import Image
    return torch.stack([transform(Image.fromarray(np.ascontiguousarray(f[..., ::-1]))) for f in frames_bgr])
