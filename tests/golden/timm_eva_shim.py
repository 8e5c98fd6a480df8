"""Stand-in for the ``timm`` / ``timm.data`` calls of the visual extractor's EVACLIP_VIT branch
(MER2024/feature_extraction/visual/extract_vision_huggingface.py:127-131, 202-210), which this image cannot install:
``create_model('eva02_base_patch14_224.mim_in22k', pretrained=True, num_classes=0, pretrained_cfg_overlay=...)``,
``data.resolve_model_data_config`` and ``data.create_transform``.  It restates timm 0.9.7's eva.py,
pos_embed_sincos.py, mlp.py and transforms_factory.py for that one tag and nothing more; the transforms are real
torchvision transforms.  Used by make_golden_eva02.py and tests/test_eva02.py.

``DEPTH`` (None = the tag's 12 blocks) shortens the model for the golden."""
import math
import sys
import types

import torch
import torch.nn.functional as F
from torch import nn

MODEL = "eva02_base_patch14_224.mim_in22k"
OPENAI_CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
DEPTH = None


def freq_bands(num_bands, temperature=10000.0, step=1):
    exp = torch.arange(0, num_bands, step, dtype=torch.int64).to(torch.float32) / num_bands
    return 1.0 / (temperature ** exp)


def build_rotary_pos_embed(feat_shape, dim, ref_feat_shape):
    """RotaryEmbeddingCat(dim, in_pixels=False, feat_shape, ref_feat_shape).get_embed(): cat([sin, cos], -1) with
    each pair's angle repeated for its two elements; 'ij' grid, so the row (y) bands come first."""
    bands = freq_bands(dim // 4)
    t = [torch.arange(s, dtype=torch.int64).to(torch.float32) for s in feat_shape]
    t = [x / f * r for x, f, r in zip(t, feat_shape, ref_feat_shape)]
    grid = torch.stack(torch.meshgrid(*t, indexing="ij"), dim=-1).unsqueeze(-1)
    pos = grid * bands
    n = feat_shape[0] * feat_shape[1]
    sin = pos.sin().reshape(n, -1).repeat_interleave(2, -1)
    cos = pos.cos().reshape(n, -1).repeat_interleave(2, -1)
    return torch.cat([sin, cos], -1)


def rot(x):
    return torch.stack([-x[..., 1::2], x[..., ::2]], -1).reshape(x.shape)


def apply_rot_embed_cat(x, emb):
    sin_emb, cos_emb = emb.tensor_split(2, -1)
    return x * cos_emb + rot(x) * sin_emb


class EvaAttention(nn.Module):
    def __init__(self, dim, num_heads):
        super().__init__()
        self.num_heads = num_heads
        self.qkv = nn.Linear(dim, 3 * dim, bias=False)
        self.q_bias = nn.Parameter(torch.zeros(dim))
        self.register_buffer("k_bias", torch.zeros(dim), persistent=False)
        self.v_bias = nn.Parameter(torch.zeros(dim))
        self.proj = nn.Linear(dim, dim)

    def forward(self, x, rope):
        B, N, C = x.shape
        qkv = F.linear(x, self.qkv.weight, torch.cat((self.q_bias, self.k_bias, self.v_bias)))
        q, k, v = qkv.reshape(B, N, 3, self.num_heads, -1).permute(2, 0, 3, 1, 4).unbind(0)
        q = torch.cat([q[:, :, :1, :], apply_rot_embed_cat(q[:, :, 1:, :], rope)], 2).type_as(v)
        k = torch.cat([k[:, :, :1, :], apply_rot_embed_cat(k[:, :, 1:, :], rope)], 2).type_as(v)
        x = F.scaled_dot_product_attention(q, k, v)
        return self.proj(x.transpose(1, 2).reshape(B, N, C))


class SwiGLU(nn.Module):
    def __init__(self, dim, hidden, eps):
        super().__init__()
        self.fc1_g = nn.Linear(dim, hidden)
        self.fc1_x = nn.Linear(dim, hidden)
        self.act = nn.SiLU()
        self.norm = nn.LayerNorm(hidden, eps=eps)
        self.fc2 = nn.Linear(hidden, dim)

    def forward(self, x):
        return self.fc2(self.norm(self.act(self.fc1_g(x)) * self.fc1_x(x)))


class EvaBlock(nn.Module):
    def __init__(self, dim, num_heads, hidden, eps):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=eps)
        self.attn = EvaAttention(dim, num_heads)
        self.norm2 = nn.LayerNorm(dim, eps=eps)
        self.mlp = SwiGLU(dim, hidden, eps)

    def forward(self, x, rope):
        x = x + self.attn(self.norm1(x), rope=rope)
        return x + self.mlp(self.norm2(x))


class Eva(nn.Module):
    """eva02_base_patch14_224: img 224, patch 14, embed 768, 12 heads, mlp_ratio 4 * 2 / 3 with swiglu_mlp and
    scale_mlp, use_rot_pos_emb with ref_feat_shape (16, 16), LayerNorm eps 1e-6, global_pool 'avg' (norm Identity,
    fc_norm LayerNorm), num_classes 0 (head Identity)."""

    def __init__(self, depth=12, img_size=224, patch_size=14, embed_dim=768, num_heads=12, mlp_ratio=4 * 2 / 3):
        super().__init__()
        g = img_size // patch_size
        self.patch_embed = nn.Module()
        self.patch_embed.proj = nn.Conv2d(3, embed_dim, patch_size, patch_size)
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
        self.pos_embed = nn.Parameter(torch.zeros(1, g * g + 1, embed_dim))
        self.register_buffer("rope", build_rotary_pos_embed((g, g), embed_dim // num_heads, (16, 16)), persistent=False)
        hidden = int(embed_dim * mlp_ratio)
        self.blocks = nn.ModuleList(EvaBlock(embed_dim, num_heads, hidden, 1e-6) for _ in range(depth))
        self.fc_norm = nn.LayerNorm(embed_dim, eps=1e-6)
        self.head = nn.Identity()
        self.pretrained_cfg = dict(input_size=(3, img_size, img_size), interpolation="bicubic", crop_pct=0.9,
                                   crop_mode="center", mean=OPENAI_CLIP_MEAN, std=OPENAI_CLIP_STD)

    def forward_features(self, x):
        x = self.patch_embed.proj(x).flatten(2).transpose(1, 2)
        x = torch.cat([self.cls_token.expand(x.shape[0], -1, -1), x], dim=1) + self.pos_embed
        for blk in self.blocks:
            x = blk(x, rope=self.rope)
        return x

    def forward(self, x):
        x = self.forward_features(x)
        return self.head(self.fc_norm(x[:, 1:].mean(dim=1)))


def create_model(model_name, pretrained=False, num_classes=None, pretrained_cfg_overlay=None, **kwargs):
    assert model_name == MODEL and num_classes == 0 and not kwargs, (model_name, num_classes, kwargs)
    model = Eva(depth=DEPTH or 12)
    if pretrained:
        from safetensors.torch import load_file
        sd = load_file(pretrained_cfg_overlay["file"])
        sd = {k: v for k, v in sd.items() if not k.startswith("head.")}   # num_classes=0 drops the classifier
        model.load_state_dict(sd, strict=True)
    return model


def resolve_model_data_config(model):
    return dict(model.pretrained_cfg)


def create_transform(input_size, interpolation="bicubic", mean=None, std=None, crop_pct=0.9, crop_mode="center",
                     is_training=False, **kwargs):
    """transforms_imagenet_eval: Resize(floor(size / crop_pct)) of the shorter edge, CenterCrop(size), ToTensor,
    Normalize."""
    from torchvision import transforms
    assert not is_training and crop_mode == "center" and interpolation == "bicubic"
    size = input_size[-1]
    return transforms.Compose([
        transforms.Resize(math.floor(size / crop_pct), interpolation=transforms.InterpolationMode.BICUBIC),
        transforms.CenterCrop(size), transforms.ToTensor(),
        transforms.Normalize(mean=torch.tensor(mean), std=torch.tensor(std))])


def install():
    """Register ``timm`` and ``timm.data`` in sys.modules (replacing any other stand-in)."""
    import importlib.machinery
    timm = types.ModuleType("timm")
    data = types.ModuleType("timm.data")
    # importers that probe for timm (transformers' availability checks) look at the spec
    timm.__spec__ = importlib.machinery.ModuleSpec("timm", None)
    data.__spec__ = importlib.machinery.ModuleSpec("timm.data", None)
    data.resolve_model_data_config, data.create_transform = resolve_model_data_config, create_transform
    timm.create_model, timm.data = create_model, data
    sys.modules.update({"timm": timm, "timm.data": data})
