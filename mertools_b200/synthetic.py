"""Deterministic synthetic checkpoints and inputs (there is no network: no pretrained weights).

Produces HF-named ``state_dict``s (numpy, float32) for ViT-B/16, HuBERT-base and BERT/RoBERTa-base
(SURVEY.md Appendix A), seeded with ``numpy.random.default_rng`` so that the golden-fixture
generator (which loads them into the HF classes the reference scripts instantiate), the oracle,
the CUDA path, bench.py and the GPU box all see bit-identical weights without shipping them.

Values are drawn tensor by tensor in a fixed order; ``scale`` multiplies every matrix weight of
the transformer layers (the "stress checkpoint" of SURVEY.md Appendix A: scale 4 gives peaky
softmax rows, large GELU arguments and LayerNorm inputs with large means).
"""
from __future__ import annotations

import numpy as np

VIT_CFG = dict(hidden=768, heads=12, ffn=3072, layers=12, image=224, patch=16, eps=1e-12)
HUBERT_CFG = dict(hidden=768, heads=12, ffn=3072, layers=12, conv_dim=512,
                  conv_kernel=(10, 3, 3, 3, 3, 2, 2), conv_stride=(5, 2, 2, 2, 2, 2, 2),
                  pos_kernel=128, pos_groups=16, eps=1e-5)
BERT_CFG = dict(hidden=768, heads=12, ffn=3072, layers=12, max_pos=512, type_vocab=2, eps=1e-12)


class _Gen:
    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.sd = {}

    def normal(self, name, shape, std):
        self.sd[name] = (self.rng.standard_normal(shape, dtype=np.float32) * np.float32(std))
        return self.sd[name]

    def ln(self, prefix, dim):
        self.sd[prefix + ".weight"] = (1.0 + 0.1 * self.rng.standard_normal(dim)).astype(np.float32)
        self.sd[prefix + ".bias"] = (0.1 * self.rng.standard_normal(dim)).astype(np.float32)

    def linear(self, prefix, out_dim, in_dim, std):
        self.normal(prefix + ".weight", (out_dim, in_dim), std)
        self.normal(prefix + ".bias", (out_dim,), 0.02)


def vit_state_dict(seed=0, layers=12, scale=1.0):
    """Keys of ``transformers.ViTModel(ViTConfig(num_hidden_layers=layers))`` (with pooler)."""
    c = VIT_CFG
    g = _Gen(seed)
    d = c["hidden"]
    g.normal("embeddings.cls_token", (1, 1, d), 0.02)
    g.normal("embeddings.position_embeddings", (1, (c["image"] // c["patch"]) ** 2 + 1, d), 0.02)
    g.normal("embeddings.patch_embeddings.projection.weight", (d, 3, c["patch"], c["patch"]), 0.02)
    g.normal("embeddings.patch_embeddings.projection.bias", (d,), 0.02)
    std = 0.02 * scale
    for i in range(layers):
        p = f"encoder.layer.{i}."
        for n in ("query", "key", "value"):
            g.linear(p + f"attention.attention.{n}", d, d, std)
        g.linear(p + "attention.output.dense", d, d, std)
        g.linear(p + "intermediate.dense", c["ffn"], d, std)
        g.linear(p + "output.dense", d, c["ffn"], std)
        g.ln(p + "layernorm_before", d)
        g.ln(p + "layernorm_after", d)
    g.ln("layernorm", d)
    g.linear("pooler.dense", d, d, 0.02)
    return g.sd


CLIP_CFGS = dict(b32=dict(hidden=768, heads=12, ffn=3072, layers=12, patch=32, proj=512),
                 l14=dict(hidden=1024, heads=16, ffn=4096, layers=24, patch=14, proj=768))


def clip_vision_state_dict(seed=4, variant="b32", layers=None, scale=1.0, image=224):
    """Vision-tower keys of ``transformers.CLIPModel`` (clip-vit-base-patch32 / clip-vit-large-patch14):
    ``vision_model.*`` and ``visual_projection.weight``."""
    c = CLIP_CFGS[variant]
    layers = c["layers"] if layers is None else layers
    g = _Gen(seed)
    d, p = c["hidden"], c["patch"]
    v = "vision_model."
    g.normal(v + "embeddings.class_embedding", (d,), 0.02)
    g.normal(v + "embeddings.patch_embedding.weight", (d, 3, p, p), 0.02)
    g.normal(v + "embeddings.position_embedding.weight", ((image // p) ** 2 + 1, d), 0.02)
    g.ln(v + "pre_layrnorm", d)
    std = 0.02 * scale
    for i in range(layers):
        q = f"{v}encoder.layers.{i}."
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            g.linear(q + f"self_attn.{n}", d, d, std)
        g.ln(q + "layer_norm1", d)
        g.linear(q + "mlp.fc1", c["ffn"], d, std)
        g.linear(q + "mlp.fc2", d, c["ffn"], std)
        g.ln(q + "layer_norm2", d)
    g.ln(v + "post_layernorm", d)
    g.normal("visual_projection.weight", (c["proj"], d), 0.03)
    return g.sd


def resnet18_state_dict(seed=6):
    """Keys of ``torchvision.models.resnet18()`` without fc (conv*/bn* with running statistics), He-style conv
    init and non-trivial BatchNorm statistics / affines so that the folding is exercised."""
    rng = np.random.default_rng(seed)
    sd = {}

    def conv(name, cout, cin, k):
        sd[name + ".weight"] = (rng.standard_normal((cout, cin, k, k)) * np.sqrt(2.0 / (cin * k * k))).astype(np.float32)

    def bn(name, c):
        sd[name + ".weight"] = rng.uniform(0.5, 1.5, c).astype(np.float32)
        sd[name + ".bias"] = (0.2 * rng.standard_normal(c)).astype(np.float32)
        sd[name + ".running_mean"] = (0.2 * rng.standard_normal(c)).astype(np.float32)
        sd[name + ".running_var"] = rng.uniform(0.5, 1.5, c).astype(np.float32)

    conv("conv1", 64, 3, 7)
    bn("bn1", 64)
    cin = 64
    for li, cout in enumerate((64, 128, 256, 512), start=1):
        for b in range(2):
            pre = f"layer{li}.{b}."
            conv(pre + "conv1", cout, cin if b == 0 else cout, 3)
            bn(pre + "bn1", cout)
            conv(pre + "conv2", cout, cout, 3)
            bn(pre + "bn2", cout)
            if b == 0 and li > 1:
                conv(pre + "downsample.0", cout, cin, 1)
                bn(pre + "downsample.1", cout)
        cin = cout
    return sd


def vggish_state_dict(seed=8):
    """Variables of the reference's VGGish graph under their TF checkpoint names (vggish_slim.py:63-99): conv
    kernels HWIO, fully connected [in, out].  He-style scales and non-zero biases (the checkpoint-less default,
    N(0, 0.01) with zero biases, would drive every activation to ~0 after nine ReLU layers)."""
    rng = np.random.default_rng(seed)
    sd = {}
    cin = 1
    for name, cout in (("conv1", 64), ("conv2", 128), ("conv3/conv3_1", 256), ("conv3/conv3_2", 256),
                       ("conv4/conv4_1", 512), ("conv4/conv4_2", 512)):
        sd[f"vggish/{name}/weights"] = (rng.standard_normal((3, 3, cin, cout)) * np.sqrt(2.0 / (9 * cin))).astype(np.float32)
        sd[f"vggish/{name}/biases"] = (0.1 * rng.standard_normal(cout)).astype(np.float32)
        cin = cout
    for name, k, n in (("fc1/fc1_1", 12288, 4096), ("fc1/fc1_2", 4096, 4096), ("fc2", 4096, 128)):
        sd[f"vggish/{name}/weights"] = (rng.standard_normal((k, n)) * np.sqrt(2.0 / k)).astype(np.float32)
        sd[f"vggish/{name}/biases"] = (0.1 * rng.standard_normal(n)).astype(np.float32)
    return sd


FERPLUS_BLOCKS = (3, 4, 6, 3)   # bottlenecks in conv2_x .. conv5_x


def ferplus_resnet50_state_dict(seed=9, se=False):
    """Parameters of the reference's ``resnet50_ferplus_dag`` (pytorch-benchmarks/model/resnet50_ferplus_dag.py:10-176):
    caffe-style ResNet-50 (stride on the 1x1 reduce / proj of conv3_1, conv4_1, conv5_1), one BatchNorm per conv,
    a 1x1 classifier conv with bias.  He-style conv scales, non-trivial BatchNorm statistics.
    ``se=True``: ``senet50_ferplus_dag`` (senet50_ferplus_dag.py:8-253) = the same skeleton plus a squeeze-and-
    excitation pair ``<block>_1x1_down`` (C -> C/16) / ``<block>_1x1_up`` (C/16 -> C), both with bias, per block."""
    rng = np.random.default_rng(seed)
    sd = {}

    def conv_bn(name, cout, cin, k, gain=1.0):
        sd[name + ".weight"] = (rng.standard_normal((cout, cin, k, k)) * np.sqrt(2.0 / (cin * k * k))).astype(np.float32)
        sd[name + "_bn.weight"] = (gain * rng.uniform(0.5, 1.5, cout)).astype(np.float32)
        sd[name + "_bn.bias"] = (0.2 * rng.standard_normal(cout)).astype(np.float32)
        sd[name + "_bn.running_mean"] = (0.2 * rng.standard_normal(cout)).astype(np.float32)
        sd[name + "_bn.running_var"] = rng.uniform(0.5, 1.5, cout).astype(np.float32)
        sd[name + "_bn.num_batches_tracked"] = np.zeros((), np.int64)

    conv_bn("conv1_7x7_s2", 64, 3, 7, gain=0.02)   # inputs are raw pixels minus the mean (|x| up to ~160)
    cin = 64
    for si, nblk in enumerate(FERPLUS_BLOCKS):
        mid, cout = 64 << si, 256 << si
        for b in range(1, nblk + 1):
            p = f"conv{si + 2}_{b}_"
            conv_bn(p + "1x1_reduce", mid, cin, 1)
            conv_bn(p + "3x3", mid, mid, 3)
            conv_bn(p + "1x1_increase", cout, mid, 1, gain=0.5)
            if se:
                sd[p + "1x1_down.weight"] = (rng.standard_normal((cout // 16, cout, 1, 1)) * np.sqrt(1.0 / cout)).astype(np.float32)
                sd[p + "1x1_down.bias"] = (0.2 * rng.standard_normal(cout // 16)).astype(np.float32)
                sd[p + "1x1_up.weight"] = (rng.standard_normal((cout, cout // 16, 1, 1)) * np.sqrt(16.0 / cout)).astype(np.float32)
                sd[p + "1x1_up.bias"] = (0.5 * rng.standard_normal(cout)).astype(np.float32)
            if b == 1:
                conv_bn(p + "1x1_proj", cout, cin, 1)
            cin = cout
    sd["classifier.weight"] = (0.02 * rng.standard_normal((8, 2048, 1, 1))).astype(np.float32)
    sd["classifier.bias"] = np.zeros(8, np.float32)
    return sd


def manet_state_dict(seed=10):
    """Parameters of the reference's MA-Net (``manet(num_classes=7)``, feature_extraction/visual/manet/model/manet.py:
    156-220): a ResNet-18 trunk up to layer2, a local branch of four 14 x 14 patches through AttentionBlocks (CBAM)
    ``layer3_1_p1..4`` / ``layer4_1_p1..4``, a multi-scale branch of MulScaleBlocks ``layer3_2`` / ``layer4_2``, two
    classifier heads.  He-style conv scales, non-trivial BatchNorm statistics."""
    rng = np.random.default_rng(seed)
    sd = {}

    def conv(name, cout, cin, k):
        sd[name + ".weight"] = (rng.standard_normal((cout, cin, k, k)) * np.sqrt(2.0 / (cin * k * k))).astype(np.float32)

    def bn(name, c, gain=1.0):
        sd[name + ".weight"] = (gain * rng.uniform(0.5, 1.5, c)).astype(np.float32)
        sd[name + ".bias"] = (0.2 * rng.standard_normal(c)).astype(np.float32)
        sd[name + ".running_mean"] = (0.2 * rng.standard_normal(c)).astype(np.float32)
        sd[name + ".running_var"] = rng.uniform(0.5, 1.5, c).astype(np.float32)
        sd[name + ".num_batches_tracked"] = np.zeros((), np.int64)

    def downsample(p, cin, cout):
        conv(p + "downsample.0", cout, cin, 1)
        bn(p + "downsample.1", cout)

    def basic(p, cin, cout, ds):
        conv(p + "conv1", cout, cin, 3); bn(p + "bn1", cout)
        conv(p + "conv2", cout, cout, 3); bn(p + "bn2", cout, 0.5)
        if ds:
            downsample(p, cin, cout)

    def attention(p, cin, cout, ds):
        basic(p, cin, cout, ds)
        r = cout // 16
        sd[p + "cbam.ChannelGate.mlp.1.weight"] = (rng.standard_normal((r, cout)) * np.sqrt(1.0 / cout)).astype(np.float32)
        sd[p + "cbam.ChannelGate.mlp.1.bias"] = (0.2 * rng.standard_normal(r)).astype(np.float32)
        sd[p + "cbam.ChannelGate.mlp.3.weight"] = (rng.standard_normal((cout, r)) * np.sqrt(1.0 / r)).astype(np.float32)
        sd[p + "cbam.ChannelGate.mlp.3.bias"] = (0.3 * rng.standard_normal(cout)).astype(np.float32)
        sd[p + "cbam.SpatialGate.spatial.conv.weight"] = (rng.standard_normal((1, 2, 7, 7)) * 0.2).astype(np.float32)
        bn(p + "cbam.SpatialGate.spatial.bn", 1)

    def mulscale(p, cin, cout, ds):
        conv(p + "conv1", cout, cin, 3); bn(p + "bn1", cout)
        sw = cout // 4
        for chain in (1, 2):
            for i in range(1, 5):
                conv(p + f"conv{chain}_2_{i}", sw, sw, 3)
                bn(p + f"bn{chain}_2_{i}", sw, 0.5)
        if ds:
            downsample(p, cin, cout)

    conv("conv1", 64, 3, 7); bn("bn1", 64)
    basic("layer1.0.", 64, 64, False); basic("layer1.1.", 64, 64, False)
    basic("layer2.0.", 64, 128, True); basic("layer2.1.", 128, 128, False)
    for pi in range(1, 5):
        attention(f"layer3_1_p{pi}.0.", 128, 256, True); attention(f"layer3_1_p{pi}.1.", 256, 256, False)
        attention(f"layer4_1_p{pi}.0.", 256, 512, True); attention(f"layer4_1_p{pi}.1.", 512, 512, False)
    mulscale("layer3_2.0.", 128, 256, True); mulscale("layer3_2.1.", 256, 256, False)
    mulscale("layer4_2.0.", 256, 512, True); mulscale("layer4_2.1.", 512, 512, False)
    for h in ("fc_1", "fc_2"):
        sd[h + ".weight"] = (0.02 * rng.standard_normal((7, 512))).astype(np.float32)
        sd[h + ".bias"] = np.zeros(7, np.float32)
    return sd


def emonet_state_dict(seed=11):
    """Parameters of the reference's ``EmoNet()`` (feature_extraction/visual/emonet/models/emonet.py:20-170;
    ``nn.InstanceNorm2d = nn.BatchNorm2d`` there, so every norm is a BatchNorm with running statistics): stem conv with
    bias, pre-activation ConvBlocks, two depth-4 hourglasses with their heads, the emotion tower."""
    rng = np.random.default_rng(seed)
    sd = {}

    def bn(name, c):
        sd[name + ".weight"] = rng.uniform(0.5, 1.5, c).astype(np.float32)
        sd[name + ".bias"] = (0.2 * rng.standard_normal(c)).astype(np.float32)
        sd[name + ".running_mean"] = (0.2 * rng.standard_normal(c)).astype(np.float32)
        sd[name + ".running_var"] = rng.uniform(0.5, 1.5, c).astype(np.float32)
        sd[name + ".num_batches_tracked"] = np.zeros((), np.int64)

    def conv(name, cout, cin, k, bias=False, gain=1.0):
        sd[name + ".weight"] = (gain * rng.standard_normal((cout, cin, k, k)) * np.sqrt(2.0 / (cin * k * k))).astype(np.float32)
        if bias:
            sd[name + ".bias"] = (0.1 * rng.standard_normal(cout)).astype(np.float32)

    def block(p, cin, cout):
        bn(p + "bn1", cin); conv(p + "conv1", cout // 2, cin, 3, gain=0.3)
        bn(p + "bn2", cout // 2); conv(p + "conv2", cout // 4, cout // 2, 3, gain=0.5)
        bn(p + "bn3", cout // 4); conv(p + "conv3", cout // 4, cout // 4, 3, gain=0.5)
        if cin != cout:
            bn(p + "downsample.0", cin); conv(p + "downsample.2", cout, cin, 1)

    def hourglass(p, level):
        block(p + f"b1_{level}.", 256, 256); block(p + f"b2_{level}.", 256, 256)
        if level > 1:
            hourglass(p, level - 1)
        else:
            block(p + f"b2_plus_{level}.", 256, 256)
        block(p + f"b3_{level}.", 256, 256)

    conv("conv1", 64, 3, 7, bias=True); bn("bn1", 64)
    block("conv2.", 64, 128); block("conv3.", 128, 128); block("conv4.", 128, 256)
    for i in range(2):
        hourglass(f"m{i}.", 4)
        block(f"top_m_{i}.", 256, 256)
        conv(f"conv_last{i}", 256, 256, 1, bias=True); bn(f"bn_end{i}", 256)
        conv(f"l{i}", 68, 256, 1, bias=True, gain=0.3)
        if i < 1:
            conv(f"bl{i}", 256, 256, 1, bias=True); conv(f"al{i}", 256, 68, 1, bias=True)
    conv("conv1x1_input_emo_2", 256, 768, 1, bias=True)
    for i in range(4):
        block(f"emo_net_2.{2 * i}.", 256, 256)
    sd["emo_fc_2.0.weight"] = (rng.standard_normal((128, 256)) * np.sqrt(2.0 / 256)).astype(np.float32)
    sd["emo_fc_2.0.bias"] = np.zeros(128, np.float32)
    bn("emo_fc_2.1", 128)
    sd["emo_fc_2.3.weight"] = (rng.standard_normal((10, 128)) * np.sqrt(1.0 / 128)).astype(np.float32)
    sd["emo_fc_2.3.bias"] = np.zeros(10, np.float32)
    return sd


WHISPER_BASE_CFG = dict(d_model=512, heads=8, ffn=2048, enc_layers=6, dec_layers=6, mels=80, src_pos=1500, tgt_pos=448,
                        vocab=51865, start_token=50258)


def whisper_state_dict(seed=13, enc_layers=6, dec_layers=6, vocab=64, cfg=WHISPER_BASE_CFG):
    """Keys of ``transformers.WhisperModel`` (whisper-base shape; a small vocabulary keeps the fixture light — the
    reference only ever embeds ``decoder_start_token_id``): encoder convs / sinusoid-initialised (here random)
    position table / pre-LN layers (k_proj without bias), decoder with self- and cross-attention."""
    g = _Gen(seed)
    d, f = cfg["d_model"], cfg["ffn"]
    g.normal("encoder.conv1.weight", (d, cfg["mels"], 3), np.sqrt(2.0 / (3 * cfg["mels"])))
    g.normal("encoder.conv1.bias", (d,), 0.05)
    g.normal("encoder.conv2.weight", (d, d, 3), np.sqrt(2.0 / (3 * d)))
    g.normal("encoder.conv2.bias", (d,), 0.05)
    g.normal("encoder.embed_positions.weight", (cfg["src_pos"], d), 0.1)
    g.normal("decoder.embed_tokens.weight", (vocab, d), 0.3)
    g.normal("decoder.embed_positions.weight", (cfg["tgt_pos"], d), 0.1)

    def attn(p):
        for n in ("q_proj", "v_proj", "out_proj"):
            g.linear(p + n, d, d, 0.03)
        g.normal(p + "k_proj.weight", (d, d), 0.03)
    for i in range(enc_layers):
        p = f"encoder.layers.{i}."
        attn(p + "self_attn.")
        g.ln(p + "self_attn_layer_norm", d)
        g.linear(p + "fc1", f, d, 0.03)
        g.linear(p + "fc2", d, f, 0.03)
        g.ln(p + "final_layer_norm", d)
    g.ln("encoder.layer_norm", d)
    for i in range(dec_layers):
        p = f"decoder.layers.{i}."
        attn(p + "self_attn.")
        g.ln(p + "self_attn_layer_norm", d)
        attn(p + "encoder_attn.")
        g.ln(p + "encoder_attn_layer_norm", d)
        g.linear(p + "fc1", f, d, 0.03)
        g.linear(p + "fc2", d, f, 0.03)
        g.ln(p + "final_layer_norm", d)
    g.ln("decoder.layer_norm", d)
    return g.sd


def dinov2_state_dict(seed=17, layers=24, hidden=1024, ffn=4096, patch=14, n_pos_side=37, swiglu=False):
    """Keys of ``transformers.Dinov2Model`` (dinov2-large shape: 24 layers, hidden 1024, 16 heads, patch 14, position
    table for 518 / 14 = 37 x 37 patches + the class token, LayerScale after the attention and MLP branches)."""
    g = _Gen(seed)
    g.normal("embeddings.cls_token", (1, 1, hidden), 0.02)
    g.normal("embeddings.mask_token", (1, hidden), 0.02)
    g.normal("embeddings.position_embeddings", (1, n_pos_side * n_pos_side + 1, hidden), 0.05)
    g.normal("embeddings.patch_embeddings.projection.weight", (hidden, 3, patch, patch), 0.02)
    g.normal("embeddings.patch_embeddings.projection.bias", (hidden,), 0.02)
    for i in range(layers):
        p = f"encoder.layer.{i}."
        g.ln(p + "norm1", hidden)
        for n in ("query", "key", "value"):
            g.linear(p + f"attention.attention.{n}", hidden, hidden, 0.02)
        g.linear(p + "attention.output.dense", hidden, hidden, 0.02)
        g.sd[p + "layer_scale1.lambda1"] = (0.5 + 0.5 * g.rng.random(hidden)).astype(np.float32)
        g.ln(p + "norm2", hidden)
        if swiglu:   # dinov2-giant: Dinov2SwiGLUFFN, hidden_features = (int(4 * hidden * 2 / 3) + 7) // 8 * 8
            hf = (int(4 * hidden * 2 / 3) + 7) // 8 * 8
            g.linear(p + "mlp.weights_in", 2 * hf, hidden, 0.02)
            g.linear(p + "mlp.weights_out", hidden, hf, 0.02)
        else:
            g.linear(p + "mlp.fc1", ffn, hidden, 0.02)
            g.linear(p + "mlp.fc2", hidden, ffn, 0.02)
        g.sd[p + "layer_scale2.lambda1"] = (0.5 + 0.5 * g.rng.random(hidden)).astype(np.float32)
    g.ln("layernorm", hidden)
    return g.sd


def data2vec_vision_state_dict(seed=19, layers=12, hidden=768, ffn=3072, heads=12, patch=16, window=14):
    """Keys of ``transformers.Data2VecVisionModel`` (data2vec-vision-base-ft1k: BEiT graph; no absolute positions, a
    relative position bias table per layer, key projection without bias, LayerScale ``lambda_1`` / ``lambda_2``)."""
    g = _Gen(seed)
    g.normal("embeddings.cls_token", (1, 1, hidden), 0.02)
    g.normal("embeddings.patch_embeddings.projection.weight", (hidden, 3, patch, patch), 0.02)
    g.normal("embeddings.patch_embeddings.projection.bias", (hidden,), 0.02)
    for i in range(layers):
        p = f"encoder.layer.{i}."
        g.sd[p + "lambda_1"] = (0.5 + 0.5 * g.rng.random(hidden)).astype(np.float32)
        g.sd[p + "lambda_2"] = (0.5 + 0.5 * g.rng.random(hidden)).astype(np.float32)
        g.linear(p + "attention.attention.query", hidden, hidden, 0.02)
        g.normal(p + "attention.attention.key.weight", (hidden, hidden), 0.02)
        g.linear(p + "attention.attention.value", hidden, hidden, 0.02)
        g.normal(p + "attention.attention.relative_position_bias.relative_position_bias_table",
                 ((2 * window - 1) ** 2 + 3, heads), 0.5)
        g.linear(p + "attention.output.dense", hidden, hidden, 0.02)
        g.linear(p + "intermediate.dense", ffn, hidden, 0.02)
        g.linear(p + "output.dense", hidden, ffn, 0.02)
        g.ln(p + "layernorm_before", hidden)
        g.ln(p + "layernorm_after", hidden)
    return g.sd


def videomae_state_dict(seed=15, layers=12, hidden=768, ffn=3072, final_norm=False):
    """Keys of ``transformers.VideoMAEModel`` (videomae-base shape): tubelet patch embedding Conv3d(3, 768, (2, 16, 16)),
    pre-LN layers whose attention carries separate ``q_bias`` / ``v_bias`` (no key bias); the position table is a fixed
    sinusoid, not a parameter."""
    g = _Gen(seed)
    g.normal("embeddings.patch_embeddings.projection.weight", (hidden, 3, 2, 16, 16), 0.02)
    g.normal("embeddings.patch_embeddings.projection.bias", (hidden,), 0.02)
    for i in range(layers):
        p = f"encoder.layer.{i}."
        for n in ("query", "key", "value"):
            g.normal(p + f"attention.attention.{n}.weight", (hidden, hidden), 0.02)
        g.normal(p + "attention.attention.q_bias", (hidden,), 0.02)
        g.normal(p + "attention.attention.v_bias", (hidden,), 0.02)
        g.linear(p + "attention.output.dense", hidden, hidden, 0.02)
        g.ln(p + "layernorm_before", hidden)
        g.ln(p + "layernorm_after", hidden)
        g.linear(p + "intermediate.dense", ffn, hidden, 0.02)
        g.linear(p + "output.dense", hidden, ffn, 0.02)
    if final_norm:   # use_mean_pooling=False (self-supervised checkpoints): VideoMAEModel.layernorm closes the encoder
        g.ln("layernorm", hidden)
    return g.sd


HUBERT_LARGE_CFG = dict(HUBERT_CFG, hidden=1024, heads=16, ffn=4096, layers=24)


def hubert_state_dict(seed=1, layers=12, scale=1.0, large=False, data2vec=False, group_norm=False, wavlm=False):
    """Keys of ``transformers.HubertModel(HubertConfig(num_hidden_layers=layers))``; ``large=True``: the
    hubert-large / chinese-hubert-large family (hidden 1024, 16 heads, FFN 4096, feat_extract_norm="layer",
    conv_bias=True, do_stable_layer_norm=True) -- same parameter names plus conv biases and one LayerNorm
    per conv layer.  ``data2vec=True``: ``Data2VecAudioModel(Data2VecAudioConfig())`` (data2vec-audio-base-960h):
    a LayerNorm after every bias-free conv, five positional conv layers (k = 19, 16 groups, bias; each followed by
    an affine-free LayerNorm and GELU), post-LN layers."""
    """``large=True, group_norm=True``: wav2vec2-large-960h (hidden 1024 with the base feature extractor: GroupNorm on
    conv0, no conv biases, post-LN layers)."""
    c = HUBERT_LARGE_CFG if large else HUBERT_CFG
    ln_convs = (large and not group_norm) or data2vec
    g = _Gen(seed)
    d, cd = c["hidden"], c["conv_dim"]
    g.sd["masked_spec_embed"] = g.rng.random(d, dtype=np.float32)
    cin = 1
    for i, k in enumerate(c["conv_kernel"]):
        g.normal(f"feature_extractor.conv_layers.{i}.conv.weight", (cd, cin, k),
                 np.sqrt(2.0 / (cin * k)))
        if large and not group_norm and not data2vec and not wavlm:   # data2vec-audio-large / wavlm-large: no conv biases
            g.normal(f"feature_extractor.conv_layers.{i}.conv.bias", (cd,), 0.05)
        if i == 0 or ln_convs:
            g.ln(f"feature_extractor.conv_layers.{i}.layer_norm", cd)
        cin = cd
    g.ln("feature_projection.layer_norm", cd)
    g.linear("feature_projection.projection", d, cd, 0.04)
    pk, pg = c["pos_kernel"], c["pos_groups"]
    if data2vec:
        for l in range(5):
            g.normal(f"encoder.pos_conv_embed.layers.{l}.conv.weight", (d, d // pg, 19), np.sqrt(2.0 / (19 * d // pg)))
            g.normal(f"encoder.pos_conv_embed.layers.{l}.conv.bias", (d,), 0.05)
    else:
        g.normal("encoder.pos_conv_embed.conv.bias", (d,), 0.02)
    v = None if data2vec else g.normal("encoder.pos_conv_embed.conv.parametrizations.weight.original1", (d, d // pg, pk),
                 2.0 * np.sqrt(1.0 / (pk * d)))
    if not data2vec:
        norm = np.sqrt((v.astype(np.float64) ** 2).sum(axis=(0, 1), keepdims=True))
        g.sd["encoder.pos_conv_embed.conv.parametrizations.weight.original0"] = (
            norm * (1.0 + 0.1 * g.rng.standard_normal(norm.shape))).astype(np.float32)
    g.ln("encoder.layer_norm", d)
    std = 0.02 * scale
    for i in range(layers):
        p = f"encoder.layers.{i}."
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            g.linear(p + f"attention.{n}", d, d, std)
        if wavlm:   # WavLMAttention: gate parameters on every layer, the bucket embedding (320 x heads) on layer 0 only
            g.linear(p + "attention.gru_rel_pos_linear", 8, 64, 0.3)
            g.sd[p + "attention.gru_rel_pos_const"] = (1.0 + 0.3 * g.rng.standard_normal((1, c["heads"], 1, 1))).astype(np.float32)
            if i == 0:
                g.normal(p + "attention.rel_attn_embed.weight", (320, c["heads"]), 0.5)
        g.ln(p + "layer_norm", d)
        g.linear(p + "feed_forward.intermediate_dense", c["ffn"], d, std)
        g.linear(p + "feed_forward.output_dense", d, c["ffn"], std)
        g.ln(p + "final_layer_norm", d)
    return g.sd


def bert_state_dict(vocab_size, seed=2, layers=12, scale=1.0, max_pos=None, type_vocab=None, large=False):
    """Keys of ``transformers.BertModel`` / ``RobertaModel`` (identical names, SURVEY App. A)."""
    c = dict(BERT_CFG, hidden=1024, heads=16, ffn=4096) if large else BERT_CFG   # large: bert-large / roberta-large
    g = _Gen(seed)
    d = c["hidden"]
    g.normal("embeddings.word_embeddings.weight", (vocab_size, d), 0.05)
    g.normal("embeddings.position_embeddings.weight", (max_pos or c["max_pos"], d), 0.05)
    g.normal("embeddings.token_type_embeddings.weight", (type_vocab or c["type_vocab"], d), 0.05)
    g.ln("embeddings.LayerNorm", d)
    std = 0.02 * scale
    for i in range(layers):
        p = f"encoder.layer.{i}."
        for n in ("query", "key", "value"):
            g.linear(p + f"attention.self.{n}", d, d, std)
        g.linear(p + "attention.output.dense", d, d, std)
        g.ln(p + "attention.output.LayerNorm", d)
        g.linear(p + "intermediate.dense", c["ffn"], d, std)
        g.linear(p + "output.dense", d, c["ffn"], std)
        g.ln(p + "output.LayerNorm", d)
    g.linear("pooler.dense", d, d, 0.02)
    return g.sd


LLAMA_SMALL_CFG = dict(vocab=4000, hidden=512, heads=4, ffn=1408, layers=6, max_pos=2048)


def llama_state_dict(seed=21, vocab=4000, hidden=512, ffn=1408, layers=6, scale=1.0):
    """Keys of ``transformers.LlamaModel`` (head_dim 128: hidden / 128 heads).  Every value is rounded to fp16 and
    stored as fp32, like the fp16 checkpoints the LLaMA family ships: the fp16 device copy is then exact and the parity
    bar measures the computation alone.  ``scale`` multiplies every layer matrix (stress checkpoints)."""
    g = _Gen(seed)
    g.normal("embed_tokens.weight", (vocab, hidden), 0.5)
    std = 0.03 * scale
    for i in range(layers):
        p = f"layers.{i}."
        for n in ("q_proj", "k_proj", "v_proj", "o_proj"):
            g.normal(p + f"self_attn.{n}.weight", (hidden, hidden), std)
        g.normal(p + "mlp.gate_proj.weight", (ffn, hidden), std)
        g.normal(p + "mlp.up_proj.weight", (ffn, hidden), std)
        g.normal(p + "mlp.down_proj.weight", (hidden, ffn), std)
        for n in ("input_layernorm", "post_attention_layernorm"):
            g.sd[p + n + ".weight"] = (1.0 + 0.1 * g.rng.standard_normal(hidden)).astype(np.float32)
    g.sd["norm.weight"] = (1.0 + 0.1 * g.rng.standard_normal(hidden)).astype(np.float32)
    return {k: v.astype(np.float16).astype(np.float32) for k, v in g.sd.items()}


LN_DECODER_SMALL_CFG = dict(vocab=4000, hidden=512, heads=4, ffn=2048, layers=6, max_pos=2048)


def bloom_state_dict(seed=23, vocab=4000, hidden=512, layers=6, scale=1.0):
    """Keys of ``transformers.BloomModel`` (head_dim 128: hidden / 128 heads, FFN 4 x hidden), fused
    ``query_key_value`` in HF's per-head interleaved row order.  Values rounded to fp16 and stored as fp32 (as
    llama_state_dict); ``scale`` multiplies every layer matrix (stress checkpoints)."""
    g = _Gen(seed)
    g.normal("word_embeddings.weight", (vocab, hidden), 0.5)
    g.ln("word_embeddings_layernorm", hidden)
    std = 0.03 * scale
    for i in range(layers):
        p = f"h.{i}."
        g.ln(p + "input_layernorm", hidden)
        g.linear(p + "self_attention.query_key_value", 3 * hidden, hidden, std)
        g.linear(p + "self_attention.dense", hidden, hidden, std)
        g.ln(p + "post_attention_layernorm", hidden)
        g.linear(p + "mlp.dense_h_to_4h", 4 * hidden, hidden, std)
        g.linear(p + "mlp.dense_4h_to_h", hidden, 4 * hidden, std)
    g.ln("ln_f", hidden)
    return {k: v.astype(np.float16).astype(np.float32) for k, v in g.sd.items()}


def opt_state_dict(seed=25, vocab=4000, hidden=512, ffn=2048, layers=6, max_pos=2048, scale=1.0):
    """Keys of ``transformers.OPTModel`` (``decoder.*``; position table of max_pos + 2 rows, pre-LN layers with biases,
    head_dim 128).  Values rounded to fp16 and stored as fp32; ``scale`` multiplies every layer matrix."""
    g = _Gen(seed)
    d = "decoder."
    g.normal(d + "embed_tokens.weight", (vocab, hidden), 0.5)
    g.normal(d + "embed_positions.weight", (max_pos + 2, hidden), 0.1)
    std = 0.03 * scale
    for i in range(layers):
        p = f"{d}layers.{i}."
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            g.linear(p + f"self_attn.{n}", hidden, hidden, std)
        g.ln(p + "self_attn_layer_norm", hidden)
        g.linear(p + "fc1", ffn, hidden, std)
        g.linear(p + "fc2", hidden, ffn, std)
        g.ln(p + "final_layer_norm", hidden)
    g.ln(d + "final_layer_norm", hidden)
    return {k: v.astype(np.float16).astype(np.float32) for k, v in g.sd.items()}


# The Falcon checkpoint of tests/golden/falcon_text_golden.npz: head_dim 64 like falcon-7b, with a hidden size (7 x 64 = 448)
# and a QKV width (9 x 64 = 576) that, like falcon-7b's 4544 and 4672, are not multiples of 128.
FALCON_SMALL_CFG = dict(vocab=4000, hidden=448, heads=7, ffn=1792, layers=6, max_pos=2048)


def falcon_state_dict(seed=43, vocab=4000, hidden=448, heads=7, ffn=1792, layers=6, scale=1.0):
    """Keys of ``transformers.FalconModel`` with parallel attention, multi-query and no biases: query_key_value rows
    heads x 64 q | 64 k | 64 v.  Values rounded to fp16 and stored as fp32 (as llama_state_dict); ``scale`` multiplies
    every layer matrix (stress checkpoints)."""
    g = _Gen(seed)
    hd = hidden // heads
    g.normal("word_embeddings.weight", (vocab, hidden), 0.5)
    std = 0.03 * scale
    for i in range(layers):
        p = f"h.{i}."
        g.ln(p + "input_layernorm", hidden)
        g.normal(p + "self_attention.query_key_value.weight", (hidden + 2 * hd, hidden), std)
        g.normal(p + "self_attention.dense.weight", (hidden, hidden), std)
        g.normal(p + "mlp.dense_h_to_4h.weight", (ffn, hidden), std)
        g.normal(p + "mlp.dense_4h_to_h.weight", (hidden, ffn), std)
    g.ln("ln_f", hidden)
    return {k: v.astype(np.float16).astype(np.float32) for k, v in g.sd.items()}


# The two GPT-2 checkpoints of tests/golden/gpt2_text_golden.npz, by the reference's model name: gpt2-chinese at head_dim
# 64 over the BERT fixture vocabulary (tests/golden/text_vocab.txt), Wenzhong at head_dim 96 over the byte-level BPE of
# tests/golden/opt_tokenizer.
GPT2_GOLDEN_CFGS = {
    "gpt2-chinese-cluecorpussmall": dict(seed=29, vocab=2629, hidden=256, heads=4, ffn=1024, layers=6, max_pos=1024),
    "wenzhong2-gpt2-chinese": dict(seed=31, vocab=4000, hidden=768, heads=8, ffn=3072, layers=6, max_pos=1024),
}


def gpt2_state_dict(seed=29, vocab=2629, hidden=256, ffn=1024, layers=6, max_pos=1024, scale=1.0):
    """Keys of ``transformers.GPT2Model`` with its Conv1D layout (c_attn / c_proj / c_fc weights [in, out]; c_attn's
    columns q | k | v).  Values rounded to fp16 and stored as fp32 (as llama_state_dict); ``scale`` multiplies every
    layer matrix (stress checkpoints)."""
    g = _Gen(seed)
    g.normal("wte.weight", (vocab, hidden), 0.5)
    g.normal("wpe.weight", (max_pos, hidden), 0.1)
    std = 0.03 * scale

    def conv1d(prefix, in_dim, out_dim):
        g.normal(prefix + ".weight", (in_dim, out_dim), std)
        g.normal(prefix + ".bias", (out_dim,), 0.02)
    for i in range(layers):
        p = f"h.{i}."
        g.ln(p + "ln_1", hidden)
        conv1d(p + "attn.c_attn", hidden, 3 * hidden)
        conv1d(p + "attn.c_proj", hidden, hidden)
        g.ln(p + "ln_2", hidden)
        conv1d(p + "mlp.c_fc", hidden, ffn)
        conv1d(p + "mlp.c_proj", ffn, hidden)
    g.ln("ln_f", hidden)
    return {k: v.astype(np.float16).astype(np.float32) for k, v in g.sd.items()}


# The two DeBERTa checkpoints of tests/golden/deberta_text_golden.npz: v1 as deberta-large (no absolute positions, c2p |
# p2c over max_relative_positions, raw relative table) at base width; v2 as deberta-v2-xlarge (log buckets, LayerNorm'd
# table, share_att_key, conv layer, no token types) at width 512.  HF config keywords.
DEBERTA_GOLDEN_CFGS = {
    "v1": dict(vocab_size=None, hidden_size=768, num_attention_heads=12, intermediate_size=1536, num_hidden_layers=4,
               max_position_embeddings=512, max_relative_positions=-1, relative_attention=True,
               pos_att_type=["c2p", "p2c"], position_biased_input=False, type_vocab_size=0, layer_norm_eps=1e-7),
    "v2": dict(vocab_size=None, hidden_size=512, num_attention_heads=8, intermediate_size=1024, num_hidden_layers=5,
               max_position_embeddings=512, max_relative_positions=-1, relative_attention=True, position_buckets=32,
               norm_rel_ebd="layer_norm", share_att_key=True, pos_att_type=["p2c", "c2p"], conv_kernel_size=3,
               conv_act="gelu", position_biased_input=False, type_vocab_size=0, layer_norm_eps=1e-7),
}


def deberta_state_dict(cfg, v2, seed=27, scale=1.0):
    """Keys of ``transformers.DebertaModel`` (v2 False) / ``DebertaV2Model`` (v2 True) for a dict of HF config keywords
    (as DEBERTA_GOLDEN_CFGS; vocab_size set).  v1: per-head interleaved ``in_proj`` with ``q_bias`` / ``v_bias`` and
    ``pos_proj`` / ``pos_q_proj``; v2: query / key / value projections (plus ``pos_key_proj`` / ``pos_query_proj``
    without share_att_key), ``encoder.LayerNorm`` with norm_rel_ebd, ``encoder.conv`` with conv_kernel_size.  ``scale``
    multiplies every layer matrix (stress checkpoints)."""
    g = _Gen(seed)
    d, ffn, std = cfg["hidden_size"], cfg["intermediate_size"], 0.03 * scale
    mr = cfg.get("max_relative_positions", -1)
    mr = mr if mr >= 1 else cfg["max_position_embeddings"]
    span = cfg["position_buckets"] if v2 and cfg.get("position_buckets", -1) > 0 else mr
    g.normal("embeddings.word_embeddings.weight", (cfg["vocab_size"], d), 0.5)
    if cfg.get("position_biased_input", True):
        g.normal("embeddings.position_embeddings.weight", (cfg["max_position_embeddings"], d), 0.1)
    if cfg.get("type_vocab_size", 0) > 0:
        g.normal("embeddings.token_type_embeddings.weight", (cfg["type_vocab_size"], d), 0.1)
    g.ln("embeddings.LayerNorm", d)
    for i in range(cfg["num_hidden_layers"]):
        p = f"encoder.layer.{i}."
        a = p + "attention.self."
        if v2:
            for n in ("query_proj", "key_proj", "value_proj"):
                g.linear(a + n, d, d, std)
            if not cfg.get("share_att_key", False):
                g.linear(a + "pos_key_proj", d, d, std)
                g.linear(a + "pos_query_proj", d, d, std)
        else:
            g.normal(a + "in_proj.weight", (3 * d, d), std)
            g.normal(a + "q_bias", (d,), 0.02)
            g.normal(a + "v_bias", (d,), 0.02)
            g.normal(a + "pos_proj.weight", (d, d), std)
            g.linear(a + "pos_q_proj", d, d, std)
        g.linear(p + "attention.output.dense", d, d, std)
        g.ln(p + "attention.output.LayerNorm", d)
        g.linear(p + "intermediate.dense", ffn, d, std)
        g.linear(p + "output.dense", d, ffn, std)
        g.ln(p + "output.LayerNorm", d)
    g.normal("encoder.rel_embeddings.weight", (2 * span, d), 0.5)
    if v2 and "layer_norm" in cfg.get("norm_rel_ebd", "none"):
        g.ln("encoder.LayerNorm", d)
    if v2 and cfg.get("conv_kernel_size", 0) > 0:
        g.normal("encoder.conv.conv.weight", (d, d, cfg["conv_kernel_size"]), std)
        g.normal("encoder.conv.conv.bias", (d,), 0.02)
        g.ln("encoder.conv.LayerNorm", d)
    return g.sd


# The two XLNet checkpoints of tests/golden/xlnet_text_golden.npz: "base" as chinese-xlnet-base (768 wide, 12 heads,
# relu) at 4 layers; "large" as xlnet-large-cased (1024 wide, 16 heads, gelu) at 3 layers, so that hidden state 0 (the
# raw word embedding) enters the last-four readout.  HF XLNetConfig keywords.
XLNET_GOLDEN_CFGS = {
    "base": dict(vocab_size=None, d_model=768, n_head=12, d_inner=1536, n_layer=4, ff_activation="relu",
                 layer_norm_eps=1e-12, dropout=0.0),
    "large": dict(vocab_size=None, d_model=1024, n_head=16, d_inner=2048, n_layer=3, ff_activation="gelu",
                  layer_norm_eps=1e-12, dropout=0.0),
}


def xlnet_state_dict(cfg, seed=33, scale=1.0):
    """Keys of ``transformers.XLNetModel`` for a dict of HF config keywords (as XLNET_GOLDEN_CFGS; vocab_size set):
    ``word_embedding``, ``mask_emb`` and per layer ``rel_attn.{q,k,v,o,r}`` [d_model, n_head, 64] (no bias), the
    r_w / r_r / r_s biases, ``seg_embed`` [2, n_head, 64], and the post-LN feed-forward.  ``scale`` multiplies every
    layer matrix (stress checkpoints)."""
    g = _Gen(seed)
    d, ffn, h = cfg["d_model"], cfg["d_inner"], cfg["n_head"]
    std = 0.03 * scale
    g.normal("mask_emb", (1, 1, d), 0.02)
    g.normal("word_embedding.weight", (cfg["vocab_size"], d), 0.5)
    for i in range(cfg["n_layer"]):
        a = f"layer.{i}.rel_attn."
        for n in ("q", "k", "v", "o", "r"):
            g.normal(a + n, (d, h, d // h), std)
        for n in ("r_r_bias", "r_s_bias", "r_w_bias"):
            g.normal(a + n, (h, d // h), 0.3)
        g.normal(a + "seg_embed", (2, h, d // h), 0.3)
        g.ln(a + "layer_norm", d)
        f = f"layer.{i}.ff."
        g.ln(f + "layer_norm", d)
        g.linear(f + "layer_1", ffn, d, std)
        g.linear(f + "layer_2", d, ffn, std)
    return g.sd


# ALBERT (AlbertConfig keywords).  Goldens: albert_chinese_tiny (312 = 12 heads of 26, padded to 32 on the device),
# albert_chinese_small (384 = 12 x 32) and albert-base-v2 at 3 layers (hidden state 0 enters the readout).  PUBLISHED:
# the five checkpoints' shapes, for the bench and the full-width tests (seeded weights; vocab and depth as given).
ALBERT_GOLDEN_CFGS = {
    "tiny": dict(vocab_size=None, embedding_size=128, hidden_size=312, num_attention_heads=12, intermediate_size=1248,
                 num_hidden_layers=4, hidden_act="gelu", layer_norm_eps=1e-12, hidden_dropout_prob=0.0,
                 attention_probs_dropout_prob=0.0, classifier_dropout_prob=0.0),
    "small": dict(vocab_size=None, embedding_size=128, hidden_size=384, num_attention_heads=12, intermediate_size=1536,
                  num_hidden_layers=4, hidden_act="gelu", layer_norm_eps=1e-12, hidden_dropout_prob=0.0,
                  attention_probs_dropout_prob=0.0, classifier_dropout_prob=0.0),
    "base": dict(vocab_size=None, embedding_size=128, hidden_size=768, num_attention_heads=12, intermediate_size=3072,
                 num_hidden_layers=3, hidden_act="gelu_new", layer_norm_eps=1e-12, hidden_dropout_prob=0.0,
                 attention_probs_dropout_prob=0.0, classifier_dropout_prob=0.0),
}
ALBERT_PUBLISHED_CFGS = {
    "albert_chinese_tiny": dict(ALBERT_GOLDEN_CFGS["tiny"], vocab_size=21128),
    "albert_chinese_small": dict(ALBERT_GOLDEN_CFGS["small"], vocab_size=21128, num_hidden_layers=6),
    "albert-base-v2": dict(ALBERT_GOLDEN_CFGS["base"], vocab_size=30000, num_hidden_layers=12),
    "albert-large-v2": dict(ALBERT_GOLDEN_CFGS["base"], vocab_size=30000, hidden_size=1024, num_attention_heads=16,
                            intermediate_size=4096, num_hidden_layers=24),
    "albert-xxlarge-v2": dict(ALBERT_GOLDEN_CFGS["base"], vocab_size=30000, hidden_size=4096, num_attention_heads=64,
                              intermediate_size=16384, num_hidden_layers=12),
}


def albert_state_dict(cfg, seed=41, scale=1.0):
    """Keys of ``transformers.AlbertModel`` (with pooler) for a dict of AlbertConfig keywords (as ALBERT_GOLDEN_CFGS;
    vocab_size set): the 128-wide embeddings and their LayerNorm, ``encoder.embedding_hidden_mapping_in`` and the ONE
    shared layer ``encoder.albert_layer_groups.0.albert_layers.0``.  ``scale`` multiplies every layer matrix (stress
    checkpoints)."""
    g = _Gen(seed)
    e, d, ffn = cfg["embedding_size"], cfg["hidden_size"], cfg["intermediate_size"]
    std = 0.03 * scale
    g.normal("embeddings.word_embeddings.weight", (cfg["vocab_size"], e), 0.5)
    g.normal("embeddings.position_embeddings.weight", (cfg.get("max_position_embeddings", 512), e), 0.1)
    g.normal("embeddings.token_type_embeddings.weight", (cfg.get("type_vocab_size", 2), e), 0.1)
    g.ln("embeddings.LayerNorm", e)
    g.linear("encoder.embedding_hidden_mapping_in", d, e, 0.08)
    p = "encoder.albert_layer_groups.0.albert_layers.0."
    g.ln(p + "full_layer_layer_norm", d)
    for n in ("query", "key", "value", "dense"):
        g.linear(p + "attention." + n, d, d, std)
    g.ln(p + "attention.LayerNorm", d)
    g.linear(p + "ffn", ffn, d, std)
    g.linear(p + "ffn_output", d, ffn, std)
    g.linear("pooler", d, d, 0.02)
    return g.sd


def fusion_state_dict(seed=3, audio_dim=768, text_dim=768, video_dim=768, hidden=128,
                      out1=6, out2=1, feat_type="utt"):
    """Keys of toolkit/models/attention.py:Attention, nn.Linear / nn.LSTM-style
    uniform(-1/sqrt(fan), 1/sqrt(fan)) init, in construction order (attention.py:21-34).  feat_type 'utt':
    MLPEncoder per modality; 'frm_align' / 'frm_unalign': LSTMEncoder (encoder.py:45-72)."""
    rng = np.random.default_rng(seed)
    sd = {}

    def lin(prefix, o, i):
        b = 1.0 / np.sqrt(i)
        sd[prefix + ".weight"] = rng.uniform(-b, b, (o, i)).astype(np.float32)
        sd[prefix + ".bias"] = rng.uniform(-b, b, (o,)).astype(np.float32)

    def mlp(prefix, i):
        lin(prefix + ".linear_1", hidden, i)
        lin(prefix + ".linear_2", hidden, hidden)
        lin(prefix + ".linear_3", hidden, hidden)

    def lstm(prefix, i):
        b = 1.0 / np.sqrt(hidden)
        sd[prefix + ".rnn.weight_ih_l0"] = rng.uniform(-b, b, (4 * hidden, i)).astype(np.float32)
        sd[prefix + ".rnn.weight_hh_l0"] = rng.uniform(-b, b, (4 * hidden, hidden)).astype(np.float32)
        sd[prefix + ".rnn.bias_ih_l0"] = rng.uniform(-b, b, (4 * hidden,)).astype(np.float32)
        sd[prefix + ".rnn.bias_hh_l0"] = rng.uniform(-b, b, (4 * hidden,)).astype(np.float32)
        lin(prefix + ".linear_1", hidden, hidden)

    enc = mlp if feat_type == "utt" else lstm
    enc("audio_encoder", audio_dim)
    enc("text_encoder", text_dim)
    enc("video_encoder", video_dim)
    mlp("attention_mlp", hidden * 3)
    lin("fc_att", 3, hidden)
    lin("fc_out_1", out1, hidden)
    lin("fc_out_2", out2, hidden)
    return sd


# ---- synthetic inputs (SURVEY.md §8d) ---------------------------------------------------------
def synth_frames(n_clips, n_frames=8, size=224, seed=0):
    """uint8 BGR face crops, [n_clips, n_frames, H, W, 3] ~ U{0..255}."""
    rng = np.random.default_rng(1000 + seed)
    return rng.integers(0, 256, (n_clips, n_frames, size, size, 3), dtype=np.uint8)


def synth_waves(n_clips, n_samples=80000, seed=0):
    """int16 waveforms round(3000 * N(0,1)) at 16 kHz, [n_clips, n_samples]."""
    rng = np.random.default_rng(2000 + seed)
    return np.round(3000.0 * rng.standard_normal((n_clips, n_samples))).astype(np.int16)


def fusion_topn_state_dict(feat_dims, seed=8, hidden=128, out1=6, out2=1):
    """Keys of MER2026 toolkit/models/attention_topn.py:Attention_TOPN in construction order."""
    rng = np.random.default_rng(seed)
    sd = {}

    def lin(prefix, o, i):
        b = 1.0 / np.sqrt(i)
        sd[prefix + ".weight"] = rng.uniform(-b, b, (o, i)).astype(np.float32)
        sd[prefix + ".bias"] = rng.uniform(-b, b, (o,)).astype(np.float32)

    def mlp(prefix, i):
        lin(prefix + ".linear_1", hidden, i)
        lin(prefix + ".linear_2", hidden, hidden)
        lin(prefix + ".linear_3", hidden, hidden)

    for i, d in enumerate(feat_dims):
        mlp(f"encoder{i}", d)
    mlp("attention_mlp", hidden * len(feat_dims))
    lin("fc_att", len(feat_dims), hidden)
    lin("fc_out_1", out1, hidden)
    lin("fc_out_2", out2, hidden)
    return sd


def synth_fusion_sequences(n, lens=(9, 5, 12), dim=768, seed=0):
    """Frame-level batch as pad_to_maxlen_pre_modality (read_data.py:118-125) hands it to the model:
    [n, T_m, dim] per modality, shorter clips zero-padded IN FRONT."""
    rng = np.random.default_rng(4000 + seed)
    out = []
    for T in lens:
        x = rng.standard_normal((n, T, dim), dtype=np.float32)
        for i in range(n):
            pad = int(rng.integers(0, max(1, T // 2)))
            x[i, :pad] = 0.0
        out.append(x)
    emo = rng.integers(0, 6, n).astype(np.int64)
    val = rng.uniform(-3, 3, n).astype(np.float32)
    return out[0], out[1], out[2], emo, val


def synth_fusion_features(n, dim=768, seed=0):
    rng = np.random.default_rng(3000 + seed)
    a, t, v = (rng.standard_normal((n, dim), dtype=np.float32) for _ in range(3))
    emo = rng.integers(0, 6, n).astype(np.int64)
    val = rng.uniform(-3, 3, n).astype(np.float32)
    return a, t, v, emo, val


EMOS_MER = ("neutral", "angry", "happy", "sad", "worried", "surprise")  # toolkit/globals.py:2


def write_mer2023_corpus(root, n_train=32, n_test=8, dim=768, seed=0, frame_level=False, dims=None,
                         numeric_val=False):
    """A MER2023-format corpus under ``root`` (SURVEY.md §8d, config C1): ``label-6way.npz`` with the
    ``{split}_corpus`` dict-of-dicts of toolkit/dataloader/mer2023.py:82-104 (every 7th valence left '' = missing)
    and N(0,1) float32 ``.npy`` features under ``features/{synA,synT,synV}-UTT/`` (and ``-FRA`` with 2..39 / 2..5
    rows per clip when ``frame_level``).  ``dims``: (audio, text, video) widths instead of ``dim`` for all three.
    ``numeric_val``: every valence a number, test3's the -10 placeholder of the released label file -- what
    MER2023/main-release.py reads (its loader turns the valences into a float tensor).  Returns (label_path,
    feature_root)."""
    import os
    rng = np.random.default_rng(seed)
    corp = {}
    for split, n in (("train", n_train), ("test1", n_test), ("test2", n_test), ("test3", n_test)):
        if numeric_val:
            corp[f"{split}_corpus"] = {
                f"{split}_{i:04d}": {"emo": EMOS_MER[int(rng.integers(0, 6))],
                                     "val": -10.0 if split == "test3" else float(rng.uniform(-3, 3))}
                for i in range(n)}
            continue
        corp[f"{split}_corpus"] = {
            f"{split}_{i:04d}": {"emo": EMOS_MER[int(rng.integers(0, 6))],
                                 "val": float(rng.uniform(-3, 3)) if i % 7 else ""}
            for i in range(n)}
    label_path = os.path.join(root, "label-6way.npz")
    np.savez(label_path, **corp)
    feats = os.path.join(root, "features")
    sets = [("synA-UTT", 0), ("synT-UTT", 0), ("synV-UTT", 0)]
    if frame_level:
        sets += [("synA-FRA", 40), ("synT-FRA", 6), ("synV-FRA", 6)]
    for si, (fname, hi) in enumerate(sets):
        width = dim if dims is None else dims[si % 3]
        os.makedirs(os.path.join(feats, fname), exist_ok=True)
        for split in corp.values():
            for name in split:
                shape = (int(rng.integers(2, hi)), width) if hi else (width,)
                np.save(os.path.join(feats, fname, name + ".npy"), rng.standard_normal(shape).astype(np.float32))
    return label_path, feats


# The label files of the MERBench corpora other than MER2023, in the formats their preprocessing scripts write
# (MERBench/toolkit/preprocess/cmumosi.py:70-86, cmumosei.py:130-142, sims.py:83-101, simsv2.py:67-77,
# iemocap.py:101-106, meld.py:57-80): (file name, splits, number of emotion classes or 0 for a sentiment corpus, valence
# range).  Every sentiment split holds some valences of exactly 0, which the acc-2 rule drops.
MERBENCH_LABELS = {
    "CMUMOSI": ("label.npz", ("train", "val", "test"), 0, 3.0),
    "CMUMOSEI": ("label.npz", ("train", "val", "test"), 0, 3.0),
    "SIMS": ("label.npz", ("train", "val", "test"), 0, 1.0),
    "SIMSv2": ("label.npz", ("train", "val", "test"), 0, 1.0),
    "IEMOCAPFour": ("label_4way.npz", ("whole",), 4, None),
    "IEMOCAPSix": ("label_6way.npz", ("whole",), 6, None),
    "MELD": ("label.npz", ("train", "val", "test"), 7, None),
}
MERBENCH_DIMS = (48, 64, 40)   # synA / synT / synV widths (the same in every corpus: cross-corpus runs share them)


def write_merbench_corpus(root, dataset, n=(40, 12, 12), seed=0, frame_level=False):
    """A ``dataset``-format corpus (a key of MERBENCH_LABELS) under ``root``: its label file with the
    ``{split}_corpus`` dicts the preprocessors write -- sentiment corpora ``{'emo': 0, 'val': v}`` with v on the
    corpus' label grid (CMU: steps of 1/3 in [-3, 3], SIMS: steps of 0.2 in [-1, 1]); IEMOCAP ``whole_corpus``
    ``{'emo': idx, 'val': -10}`` named ``Ses0{s}{F|M}_...`` with the five sessions interleaved, n[0] clips in all;
    MELD ``{'emo': idx, 'val': -10}`` -- and N(0,1) float32 ``.npy`` features under ``features/{synA,synT,synV}-UTT/``
    (and ``-FRA`` with 2..39 / 2..5 / 2..5 rows per clip when ``frame_level``).  ``n`` = clips per split, in the order
    of the corpus' splits.  Returns (label_path, feature_root)."""
    import os
    fname, splits, n_emo, vmax = MERBENCH_LABELS[dataset]
    rng = np.random.default_rng(seed)
    corp = {}
    for si, split in enumerate(splits):
        c = {}
        for i in range(n[si]):
            if split == "whole":
                sess = int(rng.integers(1, 6)) if i >= 5 else i + 1        # every session present
                name = f"Ses0{sess}{'FM'[i % 2]}_impro{i % 7:02d}_{'FM'[(i // 2) % 2]}{i:03d}"
            else:
                name = f"{split}_{dataset.lower()}_{i:04d}"
            if n_emo:
                c[name] = {"emo": int(rng.integers(0, n_emo)), "val": -10}
            else:
                steps = 9 if vmax == 3.0 else 5
                c[name] = {"emo": 0, "val": 0.0 if i % 5 == 0 else float(rng.integers(-steps, steps + 1)) * vmax / steps}
        corp[f"{split}_corpus"] = c
    os.makedirs(root, exist_ok=True)
    label_path = os.path.join(root, fname)
    np.savez(label_path, **corp)
    feats = os.path.join(root, "features")
    sets = [(f"syn{m}-UTT", 0, d) for m, d in zip("ATV", MERBENCH_DIMS)]
    if frame_level:
        sets += [(f"syn{m}-FRA", hi, d) for m, hi, d in zip("ATV", (40, 6, 6), MERBENCH_DIMS)]
    for fdir, hi, dim in sets:
        os.makedirs(os.path.join(feats, fdir), exist_ok=True)
        for split in corp.values():
            for name in split:
                shape = (int(rng.integers(2, hi)), dim) if hi else (dim,)
                np.save(os.path.join(feats, fdir, name + ".npy"), rng.standard_normal(shape).astype(np.float32))
    return label_path, feats


# Feature directories of a synthetic MER2026 corpus: every entry of MER2026's three rank lists
# (main_release.RANK_LISTS), named the way func_name_conversion resolves them -- the face extractors as `<dir>_UTT`,
# the rest as `<dir>-UTT` -- with a few different widths; videomae-large keeps 2..4 rows per clip (mean over time).
MER2026_FEATURE_DIRS = {
    "wavlm-base-UTT": 96, "chinese-wav2vec2-base-UTT": 96, "chinese-wav2vec2-large-UTT": 128,
    "chinese-hubert-large-UTT": 128, "chinese-hubert-base-UTT": 96,
    "chinese-roberta-wwm-ext-UTT": 96, "chinese-roberta-wwm-ext-large-UTT": 128, "chinese-macbert-base-UTT": 96,
    "chinese-macbert-large-UTT": 128,
    "videomae-large-UTT": 128, "resnet50face_UTT": 64, "emonet_UTT": 40, "senet50face_UTT": 64,
    "clip-vit-base-patch32-UTT": 64, "clip-vit-large-patch14-UTT": 100,
}


def write_mer2026_corpus(root, n_train=80, n_test=20, seed=0, dims=None):
    """A MER2024 / 25 / 26-format corpus under ``root``: ``track1_label_6way.npz`` with the ``train_corpus`` /
    ``test1_corpus`` dicts of toolkit/dataloader/mer2026.py:83-99 (emotion labels only) and N(0,1) float32 ``.npy``
    utterance features under ``features/<dir>/`` for every directory of ``dims`` (default MER2026_FEATURE_DIRS:
    name -> width).  Returns (label_path, feature_root)."""
    import os
    dims = MER2026_FEATURE_DIRS if dims is None else dims
    rng = np.random.default_rng(seed)
    corp = {f"{split}_corpus": {f"{split}_{i:04d}": {"emo": EMOS_MER[int(rng.integers(0, 6))]} for i in range(n)}
            for split, n in (("train", n_train), ("test1", n_test))}
    label_path = os.path.join(root, "track1_label_6way.npz")
    np.savez(label_path, **corp)
    feats = os.path.join(root, "features")
    for fname, dim in dims.items():
        os.makedirs(os.path.join(feats, fname), exist_ok=True)
        for split in corp.values():
            for name in split:
                shape = (int(rng.integers(2, 5)), dim) if fname.startswith("videomae") else (dim,)
                np.save(os.path.join(feats, fname, name + ".npy"), rng.standard_normal(shape).astype(np.float32))
    return label_path, feats


# ELECTRA (ElectraConfig keywords).  Goldens: ``small`` (the factorised 128-wide embedding + embeddings_project into
# hidden 256, 4 heads of 64, FFN 1024), ``base`` (embedding_size == hidden_size: BERT's graph) and ``lert_small`` (a
# hidden-256 BertModel, as chinese-lert-small).  PUBLISHED: the checkpoints' shapes (seeded weights; vocab as given).
ELECTRA_GOLDEN_CFGS = {
    "small": dict(vocab_size=None, embedding_size=128, hidden_size=256, num_attention_heads=4, intermediate_size=1024,
                  num_hidden_layers=5, hidden_act="gelu", layer_norm_eps=1e-12, hidden_dropout_prob=0.0,
                  attention_probs_dropout_prob=0.0),
    "base": dict(vocab_size=None, embedding_size=768, hidden_size=768, num_attention_heads=12, intermediate_size=3072,
                 num_hidden_layers=4, hidden_act="gelu", layer_norm_eps=1e-12, hidden_dropout_prob=0.0,
                 attention_probs_dropout_prob=0.0),
    "lert_small": dict(vocab_size=None, embedding_size=256, hidden_size=256, num_attention_heads=4,
                       intermediate_size=1024, num_hidden_layers=4, hidden_act="gelu", layer_norm_eps=1e-12,
                       hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0),
}
ELECTRA_PUBLISHED_CFGS = {
    "chinese-electra-180g-small": dict(ELECTRA_GOLDEN_CFGS["small"], vocab_size=21128, num_hidden_layers=12),
    "chinese-lert-small": dict(ELECTRA_GOLDEN_CFGS["lert_small"], vocab_size=21128, num_hidden_layers=12),
    "chinese-electra-180g-base": dict(ELECTRA_GOLDEN_CFGS["base"], vocab_size=21128, num_hidden_layers=12),
    "chinese-electra-180g-large": dict(ELECTRA_GOLDEN_CFGS["base"], vocab_size=21128, embedding_size=1024,
                                       hidden_size=1024, num_attention_heads=16, intermediate_size=4096,
                                       num_hidden_layers=24),
}


def electra_state_dict(cfg, seed=51, scale=1.0, pretraining=False):
    """Keys of ``transformers.ElectraModel`` for a dict of ElectraConfig keywords (as ELECTRA_GOLDEN_CFGS; vocab_size
    set): the E-wide embeddings and their LayerNorm, ``embeddings_project`` when embedding_size != hidden_size, and
    BERT's post-LN layers.  ``pretraining``: the keys of ``ElectraForPreTraining`` instead (``electra.`` prefix and the
    discriminator head).  ``scale`` multiplies every layer matrix (stress checkpoints)."""
    g = _Gen(seed)
    e, d, ffn = cfg["embedding_size"], cfg["hidden_size"], cfg["intermediate_size"]
    std = 0.03 * scale
    g.normal("embeddings.word_embeddings.weight", (cfg["vocab_size"], e), 0.5)
    g.normal("embeddings.position_embeddings.weight", (cfg.get("max_position_embeddings", 512), e), 0.1)
    g.normal("embeddings.token_type_embeddings.weight", (cfg.get("type_vocab_size", 2), e), 0.1)
    g.ln("embeddings.LayerNorm", e)
    if e != d:
        g.linear("embeddings_project", d, e, 0.08)
    for i in range(cfg["num_hidden_layers"]):
        p = f"encoder.layer.{i}."
        for n in ("query", "key", "value"):
            g.linear(p + f"attention.self.{n}", d, d, std)
        g.linear(p + "attention.output.dense", d, d, std)
        g.ln(p + "attention.output.LayerNorm", d)
        g.linear(p + "intermediate.dense", ffn, d, std)
        g.linear(p + "output.dense", d, ffn, std)
        g.ln(p + "output.LayerNorm", d)
    if not pretraining:
        return g.sd
    sd = {"electra." + k: v for k, v in g.sd.items()}
    g.sd = sd
    g.linear("discriminator_predictions.dense", d, d, 0.02)
    g.linear("discriminator_predictions.dense_prediction", 1, d, 0.02)
    return g.sd


def eva02_state_dict(seed=27, layers=12, scale=1.0, hidden=768, patch=14, image=224):
    """Keys of timm ``Eva`` as ``create_model('eva02_base_patch14_224', num_classes=0)`` holds them (hidden 768, 12
    heads, patch 14, 257 tokens, SwiGLU hidden int(768 * 4 * 2 / 3) = 2048 with its LayerNorm, fc_norm; the zero
    k_bias and the rotary table are non-persistent buffers, so not keys).  ``scale`` multiplies every block matrix
    (stress checkpoints)."""
    g = _Gen(seed)
    d, hf = hidden, int(hidden * 4 * 2 / 3)
    g.normal("cls_token", (1, 1, d), 0.02)
    g.normal("pos_embed", (1, (image // patch) ** 2 + 1, d), 0.02)
    g.normal("patch_embed.proj.weight", (d, 3, patch, patch), 0.02)
    g.normal("patch_embed.proj.bias", (d,), 0.02)
    std = 0.02 * scale
    for i in range(layers):
        p = f"blocks.{i}."
        g.ln(p + "norm1", d)
        g.normal(p + "attn.qkv.weight", (3 * d, d), std)
        g.normal(p + "attn.q_bias", (d,), 0.02)
        g.normal(p + "attn.v_bias", (d,), 0.02)
        g.linear(p + "attn.proj", d, d, std)
        g.ln(p + "norm2", d)
        g.linear(p + "mlp.fc1_g", hf, d, std)
        g.linear(p + "mlp.fc1_x", hf, d, std)
        g.ln(p + "mlp.norm", hf)
        g.linear(p + "mlp.fc2", d, hf, std)
    g.ln("fc_norm", d)
    return g.sd
