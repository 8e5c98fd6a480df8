"""GPU parity of the visual hot path against the oracle (bit-identical weights and inputs).

Tolerance (north_star): 1e-3 relative fp32, measured as max|got - ref| / max|ref| over the tensor
and as the relative L2 norm.  The CUDA path computes the linear layers' products on fp16 operands
(default) or TF32 operands (both 10-bit mantissas, round-to-nearest), attention in TF32, all with fp32
accumulation; everything else in fp32.  Both precisions must pass.
"""
import os

import numpy as np
import pytest
import torch

from mertools_b200 import synthetic as S
from oracle import encoders as E
from oracle import pipeline as P

pytestmark = pytest.mark.gpu
TOL = 1e-3


def rel(got, ref):
    got, ref = got.double(), ref.double()
    return float((got - ref).abs().max() / ref.abs().max()), float((got - ref).norm() / ref.norm())


@pytest.mark.parametrize("precision", ["f16", "tf32"])
@pytest.mark.parametrize("layers,scale", [(2, 1.0), (12, 1.0), (4, 3.0)])
def test_vit_hidden_states_and_readout(cuda, layers, scale, precision):
    from mertools_b200.encoders import VitEncoder
    sd = S.vit_state_dict(seed=0, layers=layers, scale=scale)
    frames = S.synth_frames(1, 3, seed=11)[0]
    enc = VitEncoder(sd, device=cuda, precision=precision)
    feats, hidden = enc.frame_features(torch.from_numpy(frames).to(cuda), return_hidden=True)
    torch.cuda.synchronize()
    ref_hs = E.vit_hidden_states(sd, P.vit_preprocess(frames), layers=layers)
    worst = 0.0
    for l in range(layers + 1):
        m, l2 = rel(hidden[l].cpu(), ref_hs[l])
        worst = max(worst, m)
        assert m < 4 * TOL, f"hidden state {l}: max-rel {m:.2e} l2-rel {l2:.2e}"
    ref_feat = torch.stack(ref_hs)[-1].sum(dim=1)
    m, l2 = rel(feats.cpu(), ref_feat)
    assert m < TOL and l2 < TOL, f"readout: max-rel {m:.2e} l2-rel {l2:.2e} (worst hidden {worst:.2e})"


def test_vit_clip_feature_matches_oracle_pipeline(cuda):
    """8-frame clips -> UTTERANCE feature, through the public extractor API."""
    from mertools_b200.extract import visual
    sd = S.vit_state_dict(seed=0, layers=12)
    clips = S.synth_frames(2, 8, seed=12)
    ext = visual.VisualExtractor(sd, device=cuda)
    got = ext.extract_clips([c for c in clips], feature_level="UTTERANCE", nframe=None)
    for g, c in zip(got, clips):
        ref = P.visual_clip_features(sd, c, nframe=None, layers=12)
        assert g.dtype == np.float32 and g.shape == (768,)
        m = np.abs(g - ref).max() / np.abs(ref).max()
        assert m < TOL, f"clip feature max-rel {m:.2e}"


def test_vit_batch_invariance(cuda):
    """The reference runs 32-frame batches; features must not depend on how frames are batched."""
    from mertools_b200.encoders import VitEncoder
    sd = S.vit_state_dict(seed=0, layers=2)
    frames = torch.from_numpy(S.synth_frames(1, 5, seed=13)[0]).to(cuda)
    enc = VitEncoder(sd, device=cuda)
    a = enc.frame_features(frames).clone()
    b = torch.cat([enc.frame_features(frames[:2]).clone(), enc.frame_features(frames[2:]).clone()])
    # not bit-identical: the V^T attention aligns each sequence's key axis to a 16-byte boundary of
    # the packed token buffer, so the fp32 summation order depends on where a frame sits in the batch;
    # a 1e-7 difference that crosses a tf32 rounding boundary of a GEMM operand becomes 5e-4 on that
    # element, hence ~1e-5 on the output
    d = float((a - b).abs().max() / a.abs().max())
    assert d < 2e-4, f"batch dependence {d:.2e}"


@pytest.mark.parametrize("hw", [(112, 112), (300, 260), (57, 91), (448, 224), (224, 100), (1, 1)])
def test_resize_kernel_is_bit_exact(cuda, hw):
    """mer_resize_bilinear_u8 == the oracle's Pillow restatement (itself pinned to Pillow), byte for byte."""
    from mertools_b200.encoders import VitEncoder
    rng = np.random.default_rng(hw[0] * 7 + hw[1])
    frames = rng.integers(0, 256, (3, hw[0], hw[1], 3), dtype=np.uint8)
    enc = VitEncoder(S.vit_state_dict(seed=0, layers=1), device=cuda)
    got = enc.resize_frames(torch.from_numpy(frames).to(cuda), 224).cpu().numpy()
    ref = P.pil_resize_bilinear_u8(frames, 224, 224)
    assert got.shape == ref.shape and np.array_equal(got, ref)


def test_mixed_frame_sizes_in_one_call(cuda):
    """Clips of different crop sizes (and an empty clip) in one extractor call."""
    from mertools_b200.extract import visual
    sd = S.vit_state_dict(seed=0, layers=2)
    a = S.synth_frames(1, 3, size=112, seed=21)[0]
    b = S.synth_frames(1, 2, size=224, seed=22)[0]
    ext = visual.VisualExtractor(sd, device=cuda)
    got = ext.frame_features([a, np.zeros((0, 112, 112, 3), np.uint8), b])
    assert got[1].shape == (0, 768)
    for g, c in ((got[0], a), (got[2], b)):
        ref = P.visual_clip_features(sd, c, nframe=None, layers=2, feature_level="FRAME")
        assert np.abs(g - ref).max() / np.abs(ref).max() < TOL


@pytest.mark.parametrize("variant,layers,hw", [("b32", 3, (224, 224)), ("b32", 2, (112, 112)), ("l14", 2, (224, 224)),
                                                ("l14", 2, (150, 100))])
def test_clip_vision_tower_matches_oracle(cuda, variant, layers, hw):
    """CLIP branch (extract_vision_huggingface.py:114-122): bicubic shorter-edge resize + center crop +
    normalise on the device, patch 32 / 14 embedding, pre_layrnorm, quick-GELU layers (fp16 operands for the
    50-token B/32, TF32 + the long-sequence attention for the 257-token L/14), post_layernorm, projection."""
    from mertools_b200.encoders import ClipVisionEncoder
    c = S.CLIP_CFGS[variant]
    sd = S.clip_vision_state_dict(seed=4, variant=variant, layers=layers)
    rng = np.random.default_rng(31)
    frames = rng.integers(0, 256, (3, hw[0], hw[1], 3), dtype=np.uint8)
    enc = ClipVisionEncoder(sd, device=cuda)
    assert enc.precision == ("f16" if variant == "b32" else "tf32")
    emb, hidden = enc.frame_features(torch.from_numpy(frames).to(cuda), return_hidden=True)
    torch.cuda.synchronize()
    tsd = {k: torch.from_numpy(v) for k, v in sd.items()}
    ref_emb, ref_hs = E.clip_image_features(tsd, P.clip_preprocess(frames), layers=layers, heads=c["heads"])
    for l in range(layers + 1):
        m, l2 = rel(hidden[l].cpu(), ref_hs[l])
        assert m < 4 * TOL, f"hidden state {l}: max-rel {m:.2e} l2-rel {l2:.2e}"
    m, l2 = rel(emb.cpu(), ref_emb)
    assert emb.shape == (3, c["proj"]) and m < TOL and l2 < TOL, f"image embeds: max-rel {m:.2e} l2-rel {l2:.2e}"


def test_clip_through_the_visual_extractor(cuda):
    """The extractor recognises a CLIP checkpoint, keeps every frame (no resampling) and writes [proj] / [T, proj]."""
    from mertools_b200.extract import visual
    sd = S.clip_vision_state_dict(seed=4, variant="b32", layers=2)
    clips = [c for c in S.synth_frames(2, 5, size=112, seed=41)]
    ext = visual.VisualExtractor(sd, device=cuda)
    utt = ext.extract_clips(clips, "UTTERANCE", nframe=None)
    fra = ext.extract_clips(clips, "FRAME", nframe=None)
    tsd = {k: torch.from_numpy(v) for k, v in sd.items()}
    for u, f, c in zip(utt, fra, clips):
        ref = P.clip_visual_features(tsd, c, layers=2, heads=12, feature_level="FRAME")
        assert u.shape == (512,) and f.shape == (5, 512)
        assert np.abs(f - ref).max() / np.abs(ref).max() < TOL
        assert np.abs(u - ref.mean(0)).max() / np.abs(ref.mean(0)).max() < TOL


@pytest.mark.parametrize("hw", [(112, 112), (300, 260), (57, 91)])
def test_bicubic_resize_kernel_is_bit_exact(cuda, hw):
    import ctypes as C
    from mertools_b200 import _lib as L
    rng = np.random.default_rng(hw[0] + hw[1])
    frames = rng.integers(0, 256, (2, hw[0], hw[1], 3), dtype=np.uint8)
    dev = torch.from_numpy(frames).to(cuda)
    out = torch.empty(2, 224, 224, 3, dtype=torch.uint8, device=cuda)
    lib = L.lib()
    lib.mer_resize_workspace_bytes.restype = C.c_longlong
    lib.mer_resize_workspace_bytes.argtypes = [C.c_int] * 5
    ws = torch.empty(max(1, lib.mer_resize_workspace_bytes(2, hw[0], hw[1], 224, 224)), dtype=torch.uint8, device=cuda)
    fn = L.declare("mer_resize_u8", [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                     C.c_void_p, C.c_void_p])
    L.check(fn(L.ptr(dev), 2, hw[0], hw[1], L.ptr(out), 224, 224, 1, L.ptr(ws), L.stream_ptr()))
    assert np.array_equal(out.cpu().numpy(), P.pil_resize_bilinear_u8(frames, 224, 224, filter="bicubic"))


@pytest.mark.parametrize("hw,n", [((224, 224), 3), ((112, 112), 2)])
def test_resnet18_frame_features_match_oracle(cuda, hw, n):
    """ImageNet CNN extractor (extract_imagenet_embedding.py): Resize + ToTensor + Normalize, 20 BN-folded
    convolutions as fp16 im2col GEMMs with ReLU / residual epilogues, max-pool, global average pool."""
    from mertools_b200.encoders import ResNet18Encoder
    sd = S.resnet18_state_dict(seed=6)
    frames = np.random.default_rng(51).integers(0, 256, (n, hw[0], hw[1], 3), dtype=np.uint8)
    enc = ResNet18Encoder(sd, device=cuda)
    got = enc.frame_features(torch.from_numpy(frames).to(cuda)).cpu()
    tsd = {k: torch.from_numpy(v) for k, v in sd.items()}
    ref = E.resnet18_features(tsd, P.imagenet_preprocess(frames))
    m, l2 = rel(got, ref)
    assert got.shape == (n, 512) and m < TOL and l2 < TOL, f"resnet18 features: max-rel {m:.2e} l2-rel {l2:.2e}"


def test_imagenet_extractor_save_rules(cuda, tmp_path):
    """imagenet_UTT / imagenet_FRA outputs through the mirrored script, incl. a one-frame video."""
    import types
    from mertools_b200.extract import imagenet
    sd = S.resnet18_state_dict(seed=6)
    face = tmp_path / "face"
    clips = {"vidA": S.synth_frames(1, 3, seed=61)[0], "vidB": S.synth_frames(1, 1, size=112, seed=62)[0]}
    for vid, c in clips.items():
        os.makedirs(face / vid)
        np.save(face / vid / f"{vid}.npy", c)
    cfg = types.SimpleNamespace(PATH_TO_RAW_FACE={"D": str(face)}, PATH_TO_FEATURES={"D": str(tmp_path / "feat")})
    tsd = {k: torch.from_numpy(v) for k, v in sd.items()}
    for level in ("UTTERANCE", "FRAME"):
        imagenet.main(imagenet.build_parser().parse_args(["--dataset=D", f"--feature_level={level}", "--gpu=0"]),
                      config=cfg, state_dict=sd)
        for vid, c in clips.items():
            got = np.load(tmp_path / "feat" / f"imagenet_{level[:3]}" / f"{vid}.npy")
            ref = P.imagenet_clip_features(tsd, c, feature_level=level)
            assert got.shape == ref.shape and np.abs(got - ref).max() / np.abs(ref).max() < TOL
