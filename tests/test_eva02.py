"""CPU tests of the EVA02 branch of the visual extractor (eva02_base_patch14_224.mim_in22k): the conventions the timm
stand-in pins, the loader's layout against the float64 restatement, refusals and the CLI."""
import math
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)

import _eva02_ref as R  # noqa: E402
import timm_eva_shim as T  # noqa: E402
from mertools_b200 import encoders as E  # noqa: E402
from mertools_b200 import synthetic as S  # noqa: E402
from mertools_b200.extract import visual as V  # noqa: E402


def _closed_form_angles(grid=16, nb=16):
    """float64 [grid^2, 2 nb]: pair i < nb at r / 10000^(i / nb), pair nb + i at c / 10000^(i / nb), p = r * grid + c."""
    r, c = np.divmod(np.arange(grid * grid), grid)
    bands = 1.0 / 10000.0 ** (np.arange(nb) / nb)
    return np.concatenate([r[:, None] * bands, c[:, None] * bands], 1)


def test_rope_table_matches_closed_form():
    cos, sin = E.eva02_rope_tables(16)
    assert cos.shape == sin.shape == (256, 32) and cos.dtype == np.float32
    ang = _closed_form_angles()
    # float32 bands and products: a few ulps of angles up to 15
    np.testing.assert_allclose(cos, np.cos(ang), rtol=0, atol=4e-6)
    np.testing.assert_allclose(sin, np.sin(ang), rtol=0, atol=4e-6)
    # row (y) bands first: patch (r=0, c=1) turns only the x pairs
    assert np.all(sin[1, :16] == 0) and np.all(sin[1, 16:] != 0)
    assert np.all(sin[16, 16:] == 0) and np.all(sin[16, :16] != 0)


def test_shim_rope_buffer_is_the_loader_table_repeated():
    emb = T.build_rotary_pos_embed((16, 16), 64, (16, 16))
    sin, cos = emb.tensor_split(2, -1)
    c, s = E.eva02_rope_tables(16)
    assert torch.equal(cos, torch.from_numpy(c).repeat_interleave(2, -1))
    assert torch.equal(sin, torch.from_numpy(s).repeat_interleave(2, -1))


def test_rotation_pairs_are_interleaved():
    x = torch.randn(3, 64, dtype=torch.float64)
    ang = torch.rand(3, 32, dtype=torch.float64) * 6
    emb = torch.cat([ang.sin().repeat_interleave(2, -1), ang.cos().repeat_interleave(2, -1)], -1)
    y = T.apply_rot_embed_cat(x, emb)
    c, s = ang.cos(), ang.sin()
    assert torch.allclose(y[:, 0::2], x[:, 0::2] * c - x[:, 1::2] * s)
    assert torch.allclose(y[:, 1::2], x[:, 1::2] * c + x[:, 0::2] * s)


def test_class_row_is_not_rotated():
    torch.manual_seed(0)
    att = T.EvaAttention(128, 2).double()
    rope = T.build_rotary_pos_embed((2, 2), 64, (16, 16)).double()
    x = torch.randn(1, 5, 128, dtype=torch.float64)
    q = torch.nn.functional.linear(x, att.qkv.weight, torch.cat((att.q_bias, att.k_bias, att.v_bias)))
    q = q.reshape(1, 5, 3, 2, 64).permute(2, 0, 3, 1, 4)[0]
    q_rot = torch.cat([q[:, :, :1], T.apply_rot_embed_cat(q[:, :, 1:], rope)], 2)
    assert torch.equal(q_rot[:, :, 0], q[:, :, 0]) and not torch.equal(q_rot[:, :, 1:], q[:, :, 1:])


def test_k_bias_is_a_zero_buffer():
    att = T.EvaAttention(768, 12)
    assert torch.count_nonzero(att.k_bias) == 0 and "k_bias" not in att.state_dict()
    assert {"q_bias", "v_bias", "qkv.weight"} <= set(att.state_dict())


def test_gate_is_silu_of_fc1_g_and_norm_follows_the_product():
    torch.manual_seed(1)
    m = T.SwiGLU(16, 32, 1e-6).double()
    torch.nn.init.normal_(m.norm.weight)
    x = torch.randn(4, 16, dtype=torch.float64)
    p = torch.nn.functional.silu(m.fc1_g(x)) * m.fc1_x(x)
    want = m.fc2(torch.nn.functional.layer_norm(p, (32,), m.norm.weight, m.norm.bias, 1e-6))
    assert torch.allclose(m(x), want)
    swapped = torch.nn.functional.silu(m.fc1_x(x)) * m.fc1_g(x)
    assert not torch.allclose(m(x), m.fc2(torch.nn.functional.layer_norm(swapped, (32,), m.norm.weight, m.norm.bias,
                                                                       1e-6)))


def test_pooling_happens_before_fc_norm():
    torch.manual_seed(2)
    T.DEPTH = 1
    try:
        m = T.create_model(T.MODEL, pretrained=False, num_classes=0).double().eval()
    finally:
        T.DEPTH = None
    torch.nn.init.normal_(m.fc_norm.weight)
    x = torch.randn(2, 3, 224, 224, dtype=torch.float64)
    with torch.no_grad():
        f = m.forward_features(x)
        out = m(x)
    assert torch.allclose(out, m.fc_norm(f[:, 1:].mean(1)))
    assert not torch.allclose(out, m.fc_norm(f[:, 1:]).mean(1))


@pytest.mark.parametrize("h,w,y0,x0", [(112, 112, 12, 12), (120, 100, 36, 12), (137, 112, 40, 12)])
def test_transform_geometry_matches_torchvision(h, w, y0, x0):
    from PIL import Image
    nh, nw, gy, gx = E.eva02_preprocess_geometry(h, w)
    assert (gy, gx) == (y0, x0) and min(nh, nw) == 248
    if (h, w) == (137, 112):   # excess 79: half-even rounds up, the floor rule would not
        assert (nh - 224) // 2 == 39
    frames = R.synth_faces(2, h, w, seed=3)
    tf = T.create_transform(**T.resolve_model_data_config(T.Eva(depth=0)))
    got = R.pixels_from_frames(frames, tf)
    for i, f in enumerate(frames):
        img = Image.fromarray(np.ascontiguousarray(f[..., ::-1])).resize((nw, nh), Image.BICUBIC)
        a = np.asarray(img, np.float32)[gy:gy + 224, gx:gx + 224] / 255.0
        want = (torch.from_numpy(a).permute(2, 0, 1) - torch.tensor(E.EVA02_MEAN)[:, None, None]) / \
            torch.tensor(E.EVA02_STD)[:, None, None]
        torch.testing.assert_close(got[i], want, rtol=0, atol=1e-6)


def test_data_config_is_the_registry_values():
    cfg = T.resolve_model_data_config(T.Eva(depth=0))
    assert cfg["crop_pct"] == 0.9 and cfg["interpolation"] == "bicubic" and cfg["input_size"] == (3, 224, 224)
    assert tuple(cfg["mean"]) == E.EVA02_MEAN and tuple(cfg["std"]) == E.EVA02_STD
    assert math.floor(224 / cfg["crop_pct"]) == 248


def test_layout_and_oracle_reproduce_the_stand_in():
    sd = S.eva02_state_dict(5, layers=2)
    T.DEPTH = 2
    try:
        m = T.Eva(depth=2)
        m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    finally:
        T.DEPTH = None
    m.eval()
    tf = T.create_transform(**T.resolve_model_data_config(m))
    px = R.pixels_from_frames(R.synth_faces(3, 112, 112, seed=4), tf)
    with torch.no_grad():
        want = m(px).double()
    got = R.forward(E.eva02_to_clip_layout(sd), px)
    err = float((got - want).abs().max() / want.abs().max())
    assert err < 1e-5, err


def test_layout_shapes():
    lay = E.eva02_to_clip_layout(S.eva02_state_dict(6, layers=1))
    v = "vision_model.encoder.layers.0."
    assert lay[v + "mlp.fc1.weight"].shape == (4096, 768) and lay[v + "mlp.fc2.weight"].shape == (768, 2048)
    assert lay[v + "mlp.norm.weight"].shape == (2048,) and np.all(lay[v + "self_attn.k_proj.bias"] == 0)
    assert lay["vision_model.embeddings.position_embedding.weight"].shape == (257, 768)


def test_loader_refuses_unknown_and_missing_keys():
    sd = S.eva02_state_dict(7, layers=1)
    E.eva02_to_clip_layout({**sd, "head.weight": np.zeros((10, 768), np.float32)})   # the classifier is allowed
    with pytest.raises(ValueError, match="blocks.0.attn.k_bias"):
        E.eva02_to_clip_layout({**sd, "blocks.0.attn.k_bias": np.zeros(768, np.float32)})
    no_fc = {k: v for k, v in sd.items() if not k.startswith("fc_norm.")}
    with pytest.raises(ValueError, match="fc_norm.bias.*fc_norm.weight"):
        E.eva02_to_clip_layout(no_fc)
    no_norm = {k: v for k, v in sd.items() if k != "blocks.0.mlp.norm.weight"}
    with pytest.raises(ValueError, match="blocks.0.mlp.norm.weight"):
        E.eva02_to_clip_layout(no_norm)


def test_cli_names_and_checkpoint_path():
    import types
    p = V.build_parser().parse_args(["--dataset", "D", "--model_name", V.EVACLIP_VIT, "--feature_level", "FRAME",
                                     "--gpu", "0"])
    assert p.model_name == "eva02_base_patch14_224.mim_in22k"
    assert f"{p.model_name.split('.')[0]}-{p.feature_level[:3]}" == "eva02_base_patch14_224-FRA"
    cfg = types.SimpleNamespace(PATH_TO_PRETRAINED_MODELS="/models")
    assert V.timm_checkpoint_path(cfg, p.model_name) == \
        "/models/timm/eva02_base_patch14_224.mim_in22k/model.safetensors"


def test_timm_state_dict_round_trip(tmp_path):
    from safetensors.numpy import save_file
    sd = S.eva02_state_dict(8, layers=1)
    f = tmp_path / "model.safetensors"
    save_file(sd, str(f))
    got = V.load_timm_state_dict(str(f))
    assert set(got) == set(sd) and all(np.array_equal(got[k].numpy(), sd[k]) for k in sd)
