"""CPU tests of the MER2024 VideoMAE face-clip extractor (mertools_b200/extract/sun_videomae.py): the CPU restatement
against the golden of the unmodified reference driver, the view planning against the dataset's own index decisions,
the float64 readout after de-duplication, the checkpoint rules and the CLI."""
import argparse
import os

import numpy as np
import pytest
import torch

import _sun_videomae_ref as R
from mertools_b200.extract import sun_videomae as SV

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "sun_videomae_golden.npz")
LENGTHS = (1, 5, 12, 16, 17, 19, 40, 64, 65, 150)
NONSQUARE = {40: (120, 100)}
SEEDS = {"base160": ("vit_base_patch16_160", 2, 11), "base224": ("vit_base_patch16_224", 2, 12),
         "large224": ("vit_large_patch16_224", 1, 13)}


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def video(n):
    h, w = NONSQUARE.get(n, (112, 112))
    return R.synth_video(n, h, w, seed=100 + n)


def params(case):
    model, blocks, seed = SEEDS[case]
    return R.model_params(R.synth_checkpoint(R.SHAPES[model][1], blocks, seed))


@pytest.mark.parametrize("case,level,n", [("base160", "UTTERANCE", n) for n in (1, 17, 40, 64, 65, 150)]
                         + [("base160", "FRAME", 12), ("base224", "FRAME", 19), ("base224", "UTTERANCE", 150),
                            ("large224", "UTTERANCE", 65)])
def test_reference_restatement_matches_golden(golden, case, level, n):
    got = R.video_features(params(case), video(n), SEEDS[case][0], level)
    ref = golden[f"feat/{case}/{level}/{n}"]
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() <= 1e-5 * np.abs(ref).max()


def test_clip_tensors_match_golden(golden):
    for name, (S, n, level, item) in {"sq160": (160, 65, "UTTERANCE", 3), "ns224": (224, 40, "FRAME", 37),
                                      "wrap160": (160, 12, "FRAME", 10)}.items():
        rows = SV.plan_views(n, level)[item][1]
        x = R.clip_tensor(R.resize(video(n), S), rows)[:, :2, :32, :].numpy()
        assert np.array_equal(x, golden[f"clip/{name}"]), name


@pytest.mark.parametrize("level", ["UTTERANCE", "FRAME"])
@pytest.mark.parametrize("n", LENGTHS)
def test_view_planning_matches_dataset(golden, level, n):
    items = SV.plan_views(n, level)
    assert [f for f, _ in items] == golden[f"fid/{level}/{n}"].tolist()
    assert np.array_equal(np.array([r for _, r in items]), golden[f"idx/{level}/{n}"])
    assert items == R.views(n, level)


def test_python_wrap_below_17_frames():
    # n = 12, frame 10: window [-5, 11), index -5 is frame 7
    rows = SV.plan_views(12, "FRAME")[10][1]
    assert rows == (7, 8, 9, 10, 11, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10)


def test_distinct_view_counts():
    # UTTERANCE: one view for <= 64 frames, two above; FRAME: the first 10 and the last 9 frames share a window
    assert len({r for _, r in SV.plan_views(64, "UTTERANCE")}) == 1
    assert len({r for _, r in SV.plan_views(65, "UTTERANCE")}) == 2
    assert len({r for _, r in SV.plan_views(150, "FRAME")}) == 150 - 10 - 9 + 2


@pytest.mark.parametrize("level,n", [("UTTERANCE", 1), ("UTTERANCE", 150), ("FRAME", 1), ("FRAME", 12), ("FRAME", 40)])
def test_readout_after_dedup_is_bit_identical(level, n):
    items = SV.plan_views(n, level)
    rng = np.random.default_rng(n)
    feats = {r: rng.standard_normal(64).astype(np.float32) for r in dict.fromkeys(r for _, r in items)}
    got = SV.readout(items, feats, level)
    ref = R.final_test(items, [feats[r] for _, r in items], level)
    assert got.dtype == np.float64 and got.shape == ref.shape
    assert np.array_equal(got, ref)
    assert got.shape == ((n, 64) if level == "FRAME" else (64,))


def test_empty_video_is_refused():
    with pytest.raises(ValueError, match="0 frames"):
        SV.plan_views(0, "UTTERANCE")


# ---- checkpoint rules ----
class _Arbitrary:
    """An object weights_only unpickling must refuse."""


def _ckpt(dim=768, layers=1):
    return R.synth_checkpoint(dim, layers, seed=5)


@pytest.mark.parametrize("key", ["model", "module", None])
@pytest.mark.parametrize("prefix", ["encoder.", "backbone.", ""])
def test_checkpoint_keys_and_prefixes(key, prefix):
    enc = {prefix + k[8:]: v for k, v in _ckpt()["model"].items() if k.startswith("encoder.")}
    enc["decoder.norm.weight"] = torch.ones(384)
    ck = {key: enc, "epoch": 3} if key else enc
    sd = SV.model_state_dict(ck, "vit_base_patch16_224", n_layers=1)
    ref = R.model_params(_ckpt())
    assert set(sd) == set(ref)
    for k in sd:
        assert np.array_equal(sd[k], ref[k].numpy()), k


def test_checkpoint_defaults_and_ignored_keys():
    enc = dict(_ckpt()["model"])
    for k in ["encoder.blocks.0.norm1.weight", "encoder.blocks.0.norm1.bias", "encoder.blocks.0.attn.q_bias",
              "encoder.blocks.0.attn.v_bias", "encoder.blocks.0.mlp.fc1.bias", "encoder.norm.weight"]:
        del enc[k]
    enc["encoder.blocks.0.gamma_1"] = torch.full((768,), 7.0)
    enc["encoder.head.weight"] = torch.zeros(6, 768)
    sd = SV.model_state_dict({"model": enc}, "vit_base_patch16_224", n_layers=1)
    assert (sd["blocks.0.norm1.weight"] == 1).all() and (sd["blocks.0.norm1.bias"] == 0).all()
    assert (sd["blocks.0.attn.q_bias"] == 0).all() and (sd["blocks.0.attn.v_bias"] == 0).all()
    assert (sd["blocks.0.mlp.fc1.bias"] == 0).all() and (sd["norm.weight"] == 1).all()
    assert not any("gamma" in k or "head" in k or "decoder" in k or "pos_embed" in k for k in sd)


@pytest.mark.parametrize("drop", ["encoder.patch_embed.proj.weight", "encoder.patch_embed.proj.bias",
                                  "encoder.blocks.0.attn.qkv.weight", "encoder.blocks.0.attn.proj.weight",
                                  "encoder.blocks.0.mlp.fc1.weight", "encoder.blocks.0.mlp.fc2.weight"])
def test_checkpoint_missing_random_init_weight_is_refused(drop):
    ck = _ckpt()
    del ck["model"][drop]
    with pytest.raises(ValueError, match="missing"):
        SV.model_state_dict(ck, "vit_base_patch16_224", n_layers=1)


def test_checkpoint_shape_mismatch_is_refused():
    with pytest.raises(ValueError, match="does not fit"):
        SV.model_state_dict(_ckpt(dim=1024), "vit_base_patch16_224", n_layers=1)   # a large checkpoint on the base model
    with pytest.raises(ValueError, match="missing"):
        SV.model_state_dict(_ckpt(layers=1), "vit_base_patch16_224")                # 12 blocks expected


def test_load_checkpoint_weights_only(tmp_path):
    ck = _ckpt()
    ck["args"] = argparse.Namespace(model="vit_base_patch16_224", lr=1e-3)
    p = tmp_path / "checkpoint-7.pth"
    torch.save(ck, p)
    sd = SV.load_checkpoint(str(p), "vit_base_patch16_224", n_layers=1)
    assert np.array_equal(sd["blocks.0.attn.qkv.weight"], ck["model"]["encoder.blocks.0.attn.qkv.weight"].numpy())
    torch.save({"model": ck["model"], "obj": _Arbitrary()}, p)
    with pytest.raises(Exception, match="weights_only|Unsupported global"):
        SV.load_checkpoint(str(p), "vit_base_patch16_224", n_layers=1)


# ---- CLI ----
def test_save_dir_name():
    assert SV.save_dir_name("videomae/pretrain_models/videomae-base-VoxCeleb2/checkpoint-99.pth",
                            "UTTERANCE") == "videomae-base-VoxCeleb2-99-UTT"
    assert SV.save_dir_name("m/videomae-large-K400-mer2023/checkpoint-49.pth", "FRAME") == "videomae-large-K400-mer2023-49-FRA"


def _args(*extra):
    return SV.parse_args(["--model", "vit_base_patch16_160", "--input_size", "160", "--short_side_size", "160",
                          "--finetune", "x/videomae-base/checkpoint-1.pth", *extra])


def test_cli_accepts_reference_command_line():
    a = _args("--batch_size", "64", "--dataset", "MER2023", "--feature_level", "FRAME", "--debug", "--drop_path", "0.1")
    SV.check_args(a)
    assert a.batch_size == 64 and a.feature_level == "FRAME" and a.debug


@pytest.mark.parametrize("extra,match", [
    (["--model", "vit_small_patch16_224"], "--model"),
    (["--attn_type", "factorised"], "--attn_type"),
    (["--use_mean_pooling"], "--use_mean_pooling"),
    (["--num_frames", "8"], "--num_frames"),
    (["--tubelet_size", "1"], "--tubelet_size"),
    (["--num_segments", "2"], "--num_segments"),
    (["--test_num_segment", "1"], "--test_num_segment"),
    (["--test_num_crop", "3"], "--test_num_crop"),
    (["--short_side_size", "224"], "--short_side_size"),
    (["--input_size", "224", "--short_side_size", "224"], "--input_size"),
    (["--feature_level", "SEGMENT"], "--feature_level"),
    (["--finetune", ""], "--finetune"),
    (["--device", "cpu"], "--device"),
])
def test_cli_refusals(extra, match):
    with pytest.raises(ValueError, match=match):
        SV.check_args(_args(*extra))
