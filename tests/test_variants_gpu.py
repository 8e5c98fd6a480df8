"""GPU parity of the kernel variants and of the wider extractor families (SURVEY.md §8f rows N2-N4).

Part of the always-on `-m gpu` suite.  Kernel level: the two V^T attention kernels on their own (fp16 operands: ViT; TF32
operands: HuBERT / BERT) on ragged batches in every ctx format against a float64 softmax(Q K^T / 8) V of the same
operand values (HF eager attention, modeling_vit.py:171-196) under attention_tc_bound; packed GELU / conv0 forms
against the scalar ones.  Extractor level: ragged
HuBERT batches, FER+ ResNet-50 / SENet-50, MA-Net, EmoNet, MS-Celeb, VGGish, Whisper, WavLM, data2vec-audio /
-vision, wav2vec2-large-960h, BERT-large, CLIP L/14 with fp16 linears, DINOv2 (-giant), VideoMAE, the device path of
load_video_from_npy -- each against its oracle and, where the reference code runs, a golden of the unmodified
reference."""
import os

import pytest
import torch

import _kernel_refs as R
from mertools_b200 import _lib as L

pytestmark = pytest.mark.gpu
HEADS, HD = 3, 64
LENS_F16 = [197, 197, 5, 1, 64, 128, 129, 249, 16, 17, 200, 33]
LENS_TC = LENS_F16 + [253, 250]


def _operands(lens, dtype, cuda, align, scale=1.5):
    g = torch.Generator().manual_seed(7)
    tokens = sum(lens)
    qkv = (torch.randn(tokens, 3 * HEADS * HD, generator=g) * scale).to(dtype).to(cuda)
    if dtype == torch.float32:
        L.round_tf32_(qkv)
    ld = (tokens + align - 1) // align * align
    vt = torch.zeros(HEADS * HD, ld, dtype=dtype, device=cuda)
    vt[:, :tokens] = qkv[:, 2 * HEADS * HD:].T
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    return qkv, vt, torch.tensor(cu, dtype=torch.int32, device=cuda), cu


def _run(qkv, vt, cu, lens, fmt):
    """ctx of mer_attention's V^T route in format fmt (fp16 rows, fp32, tf32-rounded fp32, or recombined split rows)."""
    dt = torch.float16 if fmt == "f16" else torch.float32
    ctx = torch.full((qkv.shape[0], HEADS * HD), float("nan"), dtype=dt, device=qkv.device)
    L.attention(qkv, ctx, cu, max(lens), HEADS, vt=vt, round_out=fmt == "tf32", split_out=fmt == "split",
                f16_out=fmt == "f16")
    torch.cuda.synchronize()
    return (L.unsplit_bf16(ctx) if fmt == "split" else ctx).double()


def _within_bound(out, qkv, lens, fmt):
    """Worst |out - float64| / attention_tc_bound (tests/_kernel_refs.py) for ctx in format fmt."""
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    return R.tc_bound_ratio(out, qkv, cu, HEADS, fmt)


@pytest.mark.parametrize("fmt,scale", [("f16", 1.5), ("f16", 4.0), ("fp32", 1.5), ("tf32", 1.5), ("split", 1.5)])
def test_attention_f16_kernel_vs_float64(cuda, fmt, scale):
    """The fp16 V^T route of mer_attention (the short kernel for this batch's 249-token maximum only under
    MER_ATT_SHORT=1, else the tiled kernel) on a ragged batch, in every ctx format and on peaked rows."""
    qkv, vt, cu, _ = _operands(LENS_F16, torch.float16, cuda, 8, scale)
    out = _run(qkv, vt, cu, LENS_F16, fmt)
    assert torch.isfinite(out).all()
    err = _within_bound(out, qkv, LENS_F16, fmt)
    assert err <= 1.0, err  # fp16 P, fp32 sums and the ctx format's rounding


@pytest.mark.parametrize("fmt", ["fp32", "f16"])
def test_attention_tf32_kernel_vs_float64(cuda, fmt):
    qkv, vt, cu, _ = _operands(LENS_TC, torch.float32, cuda, 4)
    out = _run(qkv, vt, cu, LENS_TC, fmt)
    assert torch.isfinite(out).all()
    err = _within_bound(out, qkv, LENS_TC, fmt)
    assert err <= 1.0, err  # TF32-rounded P, fp32 sums and the ctx format's rounding


def _with_env(env, val, fn):
    old = os.environ.get(env)
    os.environ[env] = val
    try:
        out = fn()
        torch.cuda.synchronize()
        return out
    finally:
        if old is None:
            os.environ.pop(env, None)
        else:
            os.environ[env] = old


def test_gemm_packed_gelu_epilogue(cuda):
    """MER_GELU_PACKED=1 (erf-GELU on value pairs, FFMA2 / FMUL2) against the scalar epilogue and float64, for
    the two operand formats FC1 writes: fp16 (ViT) and split bf16 (HuBERT / BERT)."""
    g = torch.Generator().manual_seed(3)
    M, K, N = 777, 768, 1024
    a = torch.randn(M, K, generator=g) * 0.5
    w = torch.randn(N, K, generator=g) * 0.05
    bias = (torch.randn(N, generator=g) * 0.1).to(cuda)

    def gelu64(x):
        return 0.5 * x * (1.0 + torch.erf(x / 2.0 ** 0.5))

    # fp16 operands and output
    a16, w16 = a.half().to(cuda), w.half().to(cuda)
    ref = gelu64(a16.double().cpu() @ w16.double().cpu().T + bias.double().cpu())
    outs = []
    for flag in ("0", "1"):
        out = torch.empty(M, N, dtype=torch.float16, device=cuda)
        _with_env("MER_GELU_PACKED", flag, lambda: L.gemm(a16, w16, out, bias=bias, gelu=True, mode=L.MER_GEMM_F16,
                                                          f16_out=True))
        outs.append(out.double().cpu())
        assert float((outs[-1] - ref).abs().max() / ref.abs().max()) < 1e-3
    assert float((outs[0] - outs[1]).abs().max() / ref.abs().max()) < 6e-4  # at most an fp16 ulp apart
    # split bf16 operands and output
    a_s, w_s = L.split_bf16(a.to(cuda)), L.split_bf16(w.to(cuda))
    ref = gelu64(a.double() @ w.double().T + bias.double().cpu())
    outs = []
    for flag in ("0", "1"):
        out = torch.empty(M, N, dtype=torch.float32, device=cuda)
        _with_env("MER_GELU_PACKED", flag, lambda: L.gemm(a_s, w_s, out, bias=bias, gelu=True,
                                                          mode=L.MER_GEMM_BF16X3, split_out=True))
        outs.append(L.unsplit_bf16(out).double().cpu())
        assert float((outs[-1] - ref).abs().max() / ref.abs().max()) < 3e-5
    assert float((outs[0] - outs[1]).abs().max() / ref.abs().max()) < 1e-5


def test_vggish_embeddings_match_oracle(cuda):
    """VGGish network (vggish_slim.py:37-100) on split-bf16 wgmma GEMMs against the fp32 restatement."""
    import numpy as np

    from mertools_b200 import synthetic as S
    from mertools_b200.encoders import VggishEncoder
    from oracle import encoders as E
    sd = S.vggish_state_dict(seed=8)
    x = np.random.default_rng(9).normal(-2.0, 2.0, (5, 96, 64)).astype(np.float32)
    got = VggishEncoder(sd, device=cuda).embeddings(torch.from_numpy(x).to(cuda), max_examples=3).cpu()
    ref = E.vggish_embeddings({k: torch.from_numpy(v) for k, v in sd.items()}, torch.from_numpy(x))
    assert got.shape == (5, 128)
    assert float((got - ref).abs().max() / ref.abs().max()) < 1e-3
    # the same patches through the reference's own graph definition (tests/golden/make_golden_vggish.py)
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vggish_golden.npz"))
    assert np.array_equal(g["patches"], x)
    gold = torch.from_numpy(g["patch_embeddings"])
    assert float((got - gold).abs().max() / gold.abs().max()) < 1e-3


def test_vggish_extractor_files(cuda, tmp_path):
    """extract_vggish_embedding.extract mirror: wav -> log-mel examples (0.5 s / 0.05 s hops) -> embeddings ->
    vggish_UTT / vggish_FRA save rules, against the oracle pipeline on the same waveform."""
    import sys
    import types

    import numpy as np
    from scipy.io import wavfile

    from mertools_b200 import synthetic as S
    from mertools_b200.extract import vggish
    from oracle import encoders as E
    from oracle import pipeline as P
    sd = S.vggish_state_dict(seed=8)
    rng = np.random.default_rng(4)
    wave = np.clip(np.round(3000 * rng.standard_normal(16000 * 3)), -32768, 32767).astype(np.int16)
    wav = tmp_path / "clipA.wav"
    wavfile.write(wav, 16000, wave)
    stub = types.ModuleType("soundfile")
    stub.read = lambda path, dtype=None: (wavfile.read(path)[1], wavfile.read(path)[0])
    sys.modules.setdefault("soundfile", stub)
    tsd = {k: torch.from_numpy(v) for k, v in sd.items()}
    for level, hop in (("UTTERANCE", 0.5), ("FRAME", 0.05)):
        out = tmp_path / level
        out.mkdir()
        vggish.extract([str(wav)], str(out), level, state_dict=sd, device="cuda:0")
        got = np.load(out / "clipA.npy")
        ex = P.waveform_to_examples(wave / 32768.0, hop)
        ref = E.vggish_embeddings(tsd, torch.from_numpy(ex.astype(np.float32))).numpy()
        ref = ref.mean(0) if level == "UTTERANCE" else ref
        assert got.shape == ref.shape and np.abs(got - ref).max() / np.abs(ref).max() < 1e-3
    # the clips of the golden: outputs of the UNMODIFIED reference extract() (graph definition + loop + save rules)
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vggish_golden.npz"))
    paths = []
    for name, n, seed in zip(g["clip_names"], g["clip_samples"], g["clip_seeds"]):
        paths.append(str(tmp_path / f"{name}.wav"))
        wavfile.write(paths[-1], 16000, S.synth_waves(1, int(n), seed=int(seed))[0].astype(np.int16))
    for level in ("UTTERANCE", "FRAME"):
        out = tmp_path / ("golden_" + level)
        out.mkdir()
        vggish.extract(paths, str(out), level, state_dict=sd, device="cuda:0")
        for name in g["clip_names"]:
            got, ref = np.load(out / f"{name}.npy"), g[f"{name}_{level}"]
            assert got.shape == ref.shape and np.abs(got - ref).max() / np.abs(ref).max() < 1e-3, (name, level)


def test_hubert_packed_conv0_and_switches_keep_parity(cuda):
    """HuBERT-base with the legacy conv0 form (MER_CONV0_PACKED=0: one channel per thread) and with MER_GELU_PACKED=1
    against the default kernels (tight), and the defaults against the oracle."""
    import numpy as np

    from mertools_b200 import synthetic as S
    from mertools_b200.encoders import HubertEncoder
    from oracle import encoders as E
    from oracle import pipeline as P
    sd = S.hubert_state_dict(seed=1, layers=4)
    wav = (S.synth_waves(2, 40000, seed=23).astype(np.float64) / 32768.0).astype(np.float32)
    # the split-operand stack: ~fp32 products, so that a 1e-7 difference in the front-end stays a 1e-7 difference (on
    # fp16 operands it can cross a rounding boundary and show up as 1e-4) and the TF32 attention kernel is in the path
    enc = HubertEncoder(sd, device=cuda, stack_precision="bf16x3")
    dev = torch.from_numpy(wav).to(cuda)

    def run():
        utt, frames = enc.forward(dev, normalize=True, want_frames=True)[:2]
        return frames.double().cpu()

    base = run()
    torch.cuda.synchronize()
    ref_hs = E.hubert_hidden_states(sd, torch.from_numpy(np.stack([P.wav2vec2_normalize(w) for w in wav])), layers=4)
    ref = torch.stack(ref_hs)[[-4, -3, -2, -1]].sum(dim=0).double()
    scale = float(ref.abs().max())
    assert float((base.reshape(ref.shape) - ref).abs().max()) / scale < 2e-3
    for env, val in (("MER_CONV0_PACKED", "0"), ("MER_GELU_PACKED", "1")):
        got = _with_env(env, val, run)
        assert float((got - base).abs().max()) / scale < 5e-5, env
    # conv1 / conv2 on fp16 operands (the default next to fp16 layers): the fp16-row forms of the conv0 kernels (two
    # channels per thread, and one with MER_CONV0_PACKED=0: an ulp apart before the fp16 rounding) agree, and the choice
    # of conv operand format is independent of the layers' (here: split layers + fp16 conv1 / conv2) and stays inside the
    # parity bar
    assert enc.conv_precision == "bf16x3" and HubertEncoder(sd, device=cuda).conv_precision == "f16"
    enc = HubertEncoder(sd, device=cuda, stack_precision="bf16x3", conv_precision="f16")
    f16c = run()
    assert float((f16c.reshape(ref.shape) - ref).abs().max()) / scale < 2e-3
    err = float((f16c - base).abs().max()) / scale
    print(f"fp16 conv1 / conv2 against split: {err:.2e}")
    assert 0 < err < 1e-3
    assert float((_with_env("MER_CONV0_PACKED", "0", run) - f16c).abs().max()) / scale < 2e-4


@pytest.mark.parametrize("model_name,prefix,se", [("resnet50_ferplus_dag", "", False), ("senet50_ferplus_dag", "se_", True)])
def test_ferplus_models_vs_reference_golden(cuda, tmp_path, model_name, prefix, se):
    """FER+ ResNet-50 / SENet-50 through the table-driven CNN executor (Resize(256) / CenterCrop(224) on the device, 52
    BN-folded convolutions on BF16X3 GEMMs) against outputs of the unmodified reference functions, plus the
    mirrored script's files."""
    import importlib.util
    import types

    import numpy as np

    from mertools_b200 import synthetic as S
    from mertools_b200.encoders import FerplusResnet50Encoder
    from mertools_b200.extract import ferplus
    gdir = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    spec = importlib.util.spec_from_file_location("make_golden_ferplus", os.path.join(gdir, "make_golden_ferplus.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    g = np.load(os.path.join(gdir, "ferplus_golden.npz"))
    sd = S.ferplus_resnet50_state_dict(int(g["seed"]), se=se)
    enc = FerplusResnet50Encoder(sd, device=cuda)
    clips = mod.golden_clips()
    for vid, frames in clips.items():
        got = enc.frame_features(torch.from_numpy(frames).to(cuda), max_frames=2).cpu().numpy()
        ref = g[f"{prefix}fra_{vid}"]
        assert got.shape == ref.shape and np.abs(got - ref).max() / np.abs(ref).max() < 1e-3, vid
    face = tmp_path / "face"
    for vid, frames in clips.items():
        os.makedirs(face / vid)
        np.save(face / vid / f"{vid}.npy", frames)
    cfg = types.SimpleNamespace(PATH_TO_RAW_FACE={"D": str(face)}, PATH_TO_FEATURES={"D": str(tmp_path / "feat")})
    for level, key in (("UTTERANCE", "utt"), ("FRAME", "fra")):
        args = ferplus.build_parser().parse_args(["--dataset=D", f"--feature_level={level}",
                                                  f"--model_name={model_name}", "--gpu=0"])
        ferplus.main(args, config=cfg, state_dict=sd)
        for vid in clips:
            got = np.load(tmp_path / "feat" / f"{model_name.split('_')[0]}face_{level[:3]}" / f"{vid}.npy")
            ref = g[f"{prefix}{key}_{vid}"]
            assert got.shape == ref.shape and np.abs(got - ref).max() / np.abs(ref).max() < 1e-3, (vid, level)


@pytest.mark.parametrize("large", [False, True])
def test_hubert_ragged_batch_equals_per_clip_forwards(cuda, large):
    """mer_hubert_forward_ragged: clips of different lengths in one pass (per-clip normalisation / GroupNorm
    statistics, zero-padded positional conv at each clip's end, varlen attention) against one forward per clip."""
    import numpy as np

    from mertools_b200 import synthetic as S
    from mertools_b200.encoders import HubertEncoder
    sd = S.hubert_state_dict(seed=1, layers=4, large=large)
    enc = HubertEncoder(sd, device=cuda)
    lens = [16000, 4321, 40000, 16000, 777, 25013]
    waves = [(S.synth_waves(1, n, seed=30 + i)[0].astype(np.float64) / 32768.0).astype(np.float32)
             for i, n in enumerate(lens)]
    rows = torch.zeros(len(lens), max(lens))
    for r, w in enumerate(waves):
        rows[r, :len(w)] = torch.from_numpy(w)
    rows[1, lens[1]:] = 1e3   # the tail of a row must not matter when the kernel normalises
    utt, frames = enc.forward_ragged(rows.to(cuda), lens, normalize=True, want_frames=True)
    torch.cuda.synchronize()
    for r, w in enumerate(waves):
        u1, f1 = enc.forward(torch.from_numpy(w)[None].to(cuda), normalize=True, want_frames=True)
        scale = float(f1.abs().max())
        assert frames[r].shape == f1[0].shape, (r, frames[r].shape, f1.shape)
        assert float((frames[r] - f1[0]).abs().max()) / scale < 2e-4, r
        assert float((utt[r] - u1[0]).abs().max()) / float(u1.abs().max()) < 2e-4, r


def test_audio_extractor_ragged_mode_matches_default(cuda):
    import numpy as np

    from mertools_b200 import synthetic as S
    from mertools_b200.extract.audio import AudioExtractor
    sd = S.hubert_state_dict(seed=1, layers=4)
    waves = [S.synth_waves(1, n, seed=40 + i)[0].astype(np.float64) / 32768.0 for i, n in enumerate([8000, 12345, 8000, 30000])]
    a = AudioExtractor(sd, device="cuda:0", ragged=False)
    b = AudioExtractor(sd, device="cuda:0", ragged=True)
    for level in ("UTTERANCE", "FRAME"):
        ra, rb = a.extract_waves(waves, level), b.extract_waves(waves, level)
        for x, y in zip(ra, rb):
            assert x.shape == y.shape and np.abs(x - y).max() / np.abs(x).max() < 2e-4


def test_manet_vs_reference_golden(cuda, tmp_path):
    """MA-Net through the CNN executor (crop / slice / CBAM / ranged average-pool ops) against outputs of the
    unmodified reference model, plus the mirrored script's files."""
    import importlib.util
    import types

    import numpy as np

    from mertools_b200 import synthetic as S
    from mertools_b200.encoders import ManetEncoder
    from mertools_b200.extract import manet
    gdir = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    spec = importlib.util.spec_from_file_location("make_golden_manet", os.path.join(gdir, "make_golden_manet.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    g = np.load(os.path.join(gdir, "manet_golden.npz"))
    sd = S.manet_state_dict(int(g["seed"]))
    enc = ManetEncoder(sd, device=cuda)
    clips = mod.golden_clips()
    for vid, frames in clips.items():
        got = enc.frame_features(torch.from_numpy(frames).to(cuda), max_frames=2).cpu().numpy()
        ref = g[f"fra_{vid}"]
        assert got.shape == ref.shape and np.abs(got - ref).max() / np.abs(ref).max() < 1e-3, vid
    face = tmp_path / "face"
    for vid, frames in clips.items():
        os.makedirs(face / vid)
        np.save(face / vid / f"{vid}.npy", frames)
    cfg = types.SimpleNamespace(PATH_TO_RAW_FACE={"D": str(face)}, PATH_TO_FEATURES={"D": str(tmp_path / "feat")})
    for level, key in (("UTTERANCE", "utt"), ("FRAME", "fra")):
        manet.main(manet.build_parser().parse_args(["--dataset=D", f"--feature_level={level}", "--gpu=0"]),
                   config=cfg, state_dict=sd)
        for vid in clips:
            got = np.load(tmp_path / "feat" / f"manet_{level[:3]}" / f"{vid}.npy")
            ref = g[f"{key}_{vid}"]
            assert got.shape == ref.shape and np.abs(got - ref).max() / np.abs(ref).max() < 1e-3, (vid, level)


def test_msceleb_extractor_vs_reference_classes_golden(cuda, tmp_path):
    """extract_msceleb_embedding mirror (the GPU-verified ResNet-18 path with another checkpoint / directory name)
    against outputs of the reference script's own classes."""
    import importlib.util
    import types

    import numpy as np

    from mertools_b200 import synthetic as S
    from mertools_b200.extract import msceleb
    gdir = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    spec = importlib.util.spec_from_file_location("make_golden_msceleb", os.path.join(gdir, "make_golden_msceleb.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    g = np.load(os.path.join(gdir, "msceleb_golden.npz"))
    sd = S.resnet18_state_dict(int(g["seed"]))
    face = tmp_path / "face"
    for vid, frames in mod.golden_clips().items():
        os.makedirs(face / vid)
        np.save(face / vid / f"{vid}.npy", frames)
    cfg = types.SimpleNamespace(PATH_TO_RAW_FACE={"D": str(face)}, PATH_TO_FEATURES={"D": str(tmp_path / "feat")})
    for level, key in (("UTTERANCE", "utt"), ("FRAME", "fra")):
        msceleb.main(msceleb.build_parser().parse_args(["--dataset=D", f"--feature_level={level}", "--gpu=0"]),
                     config=cfg, state_dict=sd)
        for vid in mod.golden_clips():
            got = np.load(tmp_path / "feat" / f"msceleb_{level[:3]}" / f"{vid}.npy")
            ref = g[f"{key}_{vid}"]
            assert got.shape == ref.shape and np.abs(got - ref).max() / np.abs(ref).max() < 1e-3, (vid, level)


def test_cv2_resize_kernel_is_bit_exact(cuda):
    cv2 = pytest.importorskip("cv2")
    import ctypes as C

    import numpy as np
    fn = L.declare("mer_resize_cv2_linear_u8", [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                                C.c_void_p])
    for hw in [(112, 112), (300, 300), (224, 224), (100, 180), (512, 512), (31, 47)]:
        frames = np.random.default_rng(hw[0]).integers(0, 256, (2, hw[0], hw[1], 3), dtype=np.uint8)
        dev = torch.from_numpy(frames).to(cuda)
        out = torch.empty(2, 256, 256, 3, dtype=torch.uint8, device=cuda)
        L.check(fn(L.ptr(dev), 2, hw[0], hw[1], L.ptr(out), 256, 256, L.stream_ptr()))
        ref = np.stack([cv2.resize(f, (256, 256)) for f in frames])
        assert np.array_equal(out.cpu().numpy(), ref), hw


def test_emonet_vs_reference_golden(cuda, tmp_path):
    """EmoNet through the CNN executor (affine / slice / upsample-add / mask-multiply ops, cv2-exact resize) against
    outputs of the unmodified reference model + augmentor, plus the mirrored script's files."""
    import importlib.util
    import types

    import numpy as np

    from mertools_b200 import synthetic as S
    from mertools_b200.encoders import EmonetEncoder
    from mertools_b200.extract import emonet
    gdir = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    spec = importlib.util.spec_from_file_location("make_golden_emonet", os.path.join(gdir, "make_golden_emonet.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    g = np.load(os.path.join(gdir, "emonet_golden.npz"))
    sd = S.emonet_state_dict(int(g["seed"]))
    enc = EmonetEncoder(sd, device=cuda)
    clips = mod.golden_clips()
    for vid, frames in clips.items():
        got = enc.frame_features(torch.from_numpy(frames).to(cuda), max_frames=2).cpu().numpy()
        ref = g[f"fra_{vid}"]
        assert got.shape == ref.shape and np.abs(got - ref).max() / np.abs(ref).max() < 1e-3, vid
    face = tmp_path / "face"
    for vid, frames in clips.items():
        os.makedirs(face / vid)
        np.save(face / vid / f"{vid}.npy", frames)
    cfg = types.SimpleNamespace(PATH_TO_RAW_FACE={"D": str(face)}, PATH_TO_FEATURES={"D": str(tmp_path / "feat")})
    for level, key in (("UTTERANCE", "utt"), ("FRAME", "fra")):
        emonet.main(emonet.build_parser().parse_args(["--dataset=D", f"--feature_level={level}", "--gpu=0"]),
                    config=cfg, state_dict=sd)
        for vid in clips:
            got = np.load(tmp_path / "feat" / f"emonet_{level[:3]}" / f"{vid}.npy")
            ref = g[f"{key}_{vid}"]
            assert got.shape == ref.shape and np.abs(got - ref).max() / np.abs(ref).max() < 1e-3, (vid, level)


def test_data2vec_audio_vs_reference_golden_and_oracle(cuda):
    """data2vec-audio-base (chain of five k = 19 positional convs as block-diagonal GEMMs + affine-free LayerNorm +
    GELU, LayerNorm feature encoder without biases, post-LN stack): hidden states against the oracle, the extractor
    against outputs of the unmodified reference extract()."""
    import numpy as np

    from mertools_b200 import synthetic as S
    from mertools_b200.encoders import HubertEncoder
    from mertools_b200.extract.audio import AudioExtractor
    from oracle import encoders as E
    from oracle import pipeline as P
    gdir = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    g = np.load(os.path.join(gdir, "audio_data2vec_golden.npz"))
    layers = int(g["layers"])
    sd = S.hubert_state_dict(seed=int(g["seed"]), layers=layers, data2vec=True)
    wav = (S.synth_waves(2, 16000, seed=25).astype(np.float64) / 32768.0).astype(np.float32)
    utt, frames, hidden = HubertEncoder(sd, device=cuda).forward(torch.from_numpy(wav).to(cuda), normalize=True,
                                                                 want_frames=True, return_hidden=True)
    ref_hs = E.hubert_hidden_states(sd, torch.from_numpy(np.stack([P.wav2vec2_normalize(w) for w in wav])), layers=layers)
    for l in range(layers + 1):
        assert float((hidden[l].cpu() - ref_hs[l]).abs().max() / ref_hs[l].abs().max()) < 4e-3, l
    waves = [S.synth_waves(1, int(n), seed=int(g["seed0"]) + i)[0].astype(np.float64) / 32768.0 for i, n in enumerate(g["lens"])]
    ext = AudioExtractor(sd, device="cuda:0")
    u, f = ext.extract_waves(waves, "UTTERANCE"), ext.extract_waves(waves, "FRAME")
    for i in range(len(waves)):
        assert np.abs(u[i] - g[f"utt{i}"]).max() / np.abs(g[f"utt{i}"]).max() < 1e-3, i
        assert np.abs(f[i][::16] - g[f"fra{i}"]).max() / np.abs(g[f"fra{i}"]).max() < 2e-3, i


def test_data2vec_audio_large_vs_oracle(cuda):
    """data2vec-audio-large: the data2vec graph at hidden 1024 / 16 heads (64-channel positional conv groups)."""
    import numpy as np

    from mertools_b200 import synthetic as S
    from mertools_b200.encoders import HubertEncoder
    from oracle import encoders as E
    from oracle import pipeline as P
    layers = 4
    sd = S.hubert_state_dict(seed=4, layers=layers, data2vec=True, large=True)
    wav = (S.synth_waves(2, 16000, seed=26).astype(np.float64) / 32768.0).astype(np.float32)
    utt, frames, hidden = HubertEncoder(sd, device=cuda).forward(torch.from_numpy(wav).to(cuda), normalize=True,
                                                                 want_frames=True, return_hidden=True)
    ref_hs = E.hubert_hidden_states(sd, torch.from_numpy(np.stack([P.wav2vec2_normalize(w) for w in wav])), layers=layers,
                                    heads=16)
    for l in range(layers + 1):
        assert float((hidden[l].cpu() - ref_hs[l]).abs().max() / ref_hs[l].abs().max()) < 4e-3, l
    ref = torch.stack(ref_hs)[-4:].sum(dim=0)
    assert float((frames.cpu().view_as(ref) - ref).abs().max() / ref.abs().max()) < 1e-3


def test_clip_l14_with_fp16_linear_layers(cuda):
    """CLIP L/14 (257 tokens) with precision="f16": fp16 linear layers around the fp32-operand flash attention
    (the hybrid branch of mer_run_stack) against the oracle, like the TF32 default."""
    import numpy as np

    from mertools_b200 import synthetic as S
    from mertools_b200.encoders import ClipVisionEncoder
    from oracle import encoders as E
    from oracle import pipeline as P
    c = S.CLIP_CFGS["l14"]
    sd = S.clip_vision_state_dict(seed=4, variant="l14", layers=2)
    frames = np.random.default_rng(31).integers(0, 256, (3, 224, 224, 3), dtype=np.uint8)
    enc = ClipVisionEncoder(sd, device=cuda, precision="f16")
    assert enc.tokens == 257 and enc.precision == "f16"
    emb = enc.frame_features(torch.from_numpy(frames).to(cuda))
    ref_emb, _ = E.clip_image_features({k: torch.from_numpy(v) for k, v in sd.items()}, P.clip_preprocess(frames),
                                       layers=2, heads=c["heads"])
    assert float((emb.cpu() - ref_emb).abs().max() / ref_emb.abs().max()) < 1e-3


def test_wav2vec2_large_960h_family(cuda):
    """hidden 1024 / 16 heads on the GroupNorm feature extractor with post-LN layers (wav2vec2-large-960h): a
    combination of paths that exist (conv0 GroupNorm kernels, 64-channel-group positional conv GEMM, post-LN BF16X3
    stack at runtime dims) but had never been run together."""
    import numpy as np

    from mertools_b200 import synthetic as S
    from mertools_b200.encoders import HubertEncoder
    from oracle import encoders as E
    from oracle import pipeline as P
    sd = S.hubert_state_dict(seed=5, layers=4, large=True, group_norm=True)
    wav = (S.synth_waves(2, 16000, seed=27).astype(np.float64) / 32768.0).astype(np.float32)
    enc = HubertEncoder(sd, device=cuda)
    assert enc.hidden == 1024 and not enc.model.stable_layer_norm and not enc.model.feat_norm_layer
    utt, frames, hidden = enc.forward(torch.from_numpy(wav).to(cuda), normalize=True, want_frames=True, return_hidden=True)
    ref_hs = E.hubert_hidden_states(sd, torch.from_numpy(np.stack([P.wav2vec2_normalize(w) for w in wav])), layers=4, heads=16)
    for l in range(5):
        assert float((hidden[l].cpu() - ref_hs[l]).abs().max() / ref_hs[l].abs().max()) < 4e-3, l
    ref = torch.stack(ref_hs)[[-4, -3, -2, -1]].sum(dim=0)
    assert float((frames.cpu() - ref).abs().max() / ref.abs().max()) < 2e-3


@pytest.mark.parametrize("roberta", [False, True])
def test_bert_large_hidden_states_and_readout(cuda, roberta):
    """bert-large / roberta-large shape (1024 / 16 heads / 4096) through mer_bert_forward: templated embedding
    kernel, post-LN BF16X3 stack at runtime dims, last-four readout."""
    from mertools_b200 import synthetic as S
    from mertools_b200.encoders import BertEncoder
    from oracle import encoders as E
    layers, off = 4, (2 if roberta else 0)
    sd = S.bert_state_dict(400, seed=6, layers=layers, large=True, max_pos=64)
    enc = BertEncoder(sd, device=cuda, ln_eps=1e-5 if roberta else 1e-12, position_offset=off)
    assert enc.hidden == 1024
    sents = [[2, 17, 250, 99, 42, 7, 3], [2, 5, 3], [2] + list(range(10, 40)) + [3]]
    utt, toks, hidden, cu = enc.forward(sents, start=1, end=-1, want_tokens=True, return_hidden=True)
    tsd = {k: torch.from_numpy(v) for k, v in sd.items()}
    for i, ids in enumerate(sents):
        ref_hs = E.bert_hidden_states(tsd, torch.tensor([ids]), layers=layers, heads=16, eps=1e-5 if roberta else 1e-12,
                                      position_offset=off)
        a, b = int(cu[i]), int(cu[i + 1])
        for l in range(layers + 1):
            assert float((hidden[l, a:b].cpu() - ref_hs[l][0]).abs().max() / ref_hs[l].abs().max()) < 4e-3, (i, l)
        ref = torch.stack(ref_hs)[[-4, -3, -2, -1]].sum(dim=0)[0]
        assert float((toks[a:b].cpu() - ref).abs().max() / ref.abs().max()) < 2e-3, i
        assert float((utt[i].cpu() - ref[1:-1].mean(dim=0)).abs().max() / ref.abs().max()) < 1e-3, i


def test_whisper_branch_vs_reference_golden(cuda):
    """Whisper branch: mer_whisper_logmel against the oracle front-end, then the whole WhisperNet on CudaOps (3-tap
    GEMM convolutions, TF32 linears, flash attention over 1500 frames, mer_small_attention in the decoder) against
    outputs of the unmodified reference extract()."""
    import numpy as np

    from mertools_b200 import synthetic as S
    from mertools_b200.extract.whisper import CudaOps, WhisperExtractor
    from oracle import pipeline as P
    gdir = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    g = np.load(os.path.join(gdir, "audio_whisper_golden.npz"))
    layers = int(g["layers"])
    waves = [S.synth_waves(1, int(n), seed=int(g["seed0"]) + i)[0].astype(np.float64) / 32768.0 for i, n in enumerate(g["lens"])]
    mel = CudaOps("cuda:0").logmel(waves).cpu().numpy()
    for i, w in enumerate(waves):
        ref = P.whisper_log_mel(w).T
        assert np.abs(mel[i, :, :80] - ref).max() < 2e-3 and not mel[i, :, 80:].any()   # TF32-rounded values in [-1.5, 1.5]
    ext = WhisperExtractor(S.whisper_state_dict(seed=int(g["seed"]), enc_layers=layers, dec_layers=layers), int(g["start"]),
                           device="cuda:0")
    utt, fra = ext.extract_waves(waves, "UTTERANCE"), ext.extract_waves(waves, "FRAME")
    for i in range(len(waves)):
        assert fra[i].shape == (2, 512) and np.abs(fra[i] - g[f"fra{i}"]).max() / np.abs(g[f"fra{i}"]).max() < 2e-3, i
        assert np.abs(utt[i] - g[f"utt{i}"]).max() / np.abs(g[f"utt{i}"]).max() < 2e-3, i


def test_load_video_from_npy_device_path(cuda):
    """load_video_from_npy mirror on the device (gather, cv2-exact resize kernel, BGR->RGB) against the golden of the
    reference's own function source, all four readtypes."""
    import importlib.util

    import numpy as np

    from mertools_b200.extract.visual import load_video_from_npy
    gdir = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    spec = importlib.util.spec_from_file_location("make_golden_video_npy", os.path.join(gdir, "make_golden_video_npy.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    g = np.load(os.path.join(gdir, "video_npy_golden.npz"))
    for ci, (readtype, n_frms, vlen, size) in enumerate(mod.CASES):
        np.random.seed(1000 + ci)
        x = load_video_from_npy(mod.golden_clip(vlen, size, 200 + ci), n_frms=n_frms, readtype=readtype, device=cuda).cpu().numpy()
        assert list(x.shape) == list(g[f"shape{ci}"])
        assert np.array_equal(x[:, :, ::16, ::16].astype(np.uint8), g[f"probe{ci}"]) and float(x.sum(dtype=np.float64)) == float(g[f"sum{ci}"][0])


def test_videomae_extractor_vs_oracle(cuda):
    """VideoMAE branch (extract_vision_huggingface.py:147-159): tubelet patch gather + host-orchestrated encoder."""
    import numpy as np

    from mertools_b200 import synthetic as S
    from oracle import pipeline as P
    TOL = 1e-3
    _rel = lambda a, b: float(np.abs(np.asarray(a, np.float64) - b).max() / np.abs(b).max())  # noqa: E731
    from mertools_b200.extract.videomae import VideoMaeExtractor
    sd = S.videomae_state_dict(seed=15, layers=3, final_norm=True)
    frames = np.random.default_rng(31).integers(0, 256, (21, 120, 160, 3), dtype=np.uint8)
    ext = VideoMaeExtractor(sd, device=cuda)
    pre = ext.preprocess(frames).cpu().numpy()
    sel = frames[P.resample_frames_uniform_indices(len(frames), 16)]
    ref_px = P.pil_resize_bilinear_u8(sel, 224, 298)[:, :, 37:261]
    np.testing.assert_array_equal(pre, ref_px)                                          # geometry bit-exact
    for level in ("UTTERANCE", "FRAME"):
        got, ref = ext.extract_clip(frames, level), P.videomae_clip_features(sd, frames, level)
        assert got.shape == ref.shape and _rel(got, ref) < TOL


def test_dinov2_extractor_vs_oracle(cuda):
    """DINOv2 branch (extract_vision_huggingface.py:135-145) on the CLIP L/14 tower kernels (MER_VISION_DINOV2)."""
    import numpy as np

    from mertools_b200 import synthetic as S
    from oracle import pipeline as P
    TOL = 1e-3
    _rel = lambda a, b: float(np.abs(np.asarray(a, np.float64) - b).max() / np.abs(b).max())  # noqa: E731
    from mertools_b200.extract.visual import VisualExtractor
    sd = S.dinov2_state_dict(seed=17, layers=3)
    frames = np.random.default_rng(3).integers(0, 256, (5, 120, 160, 3), dtype=np.uint8)
    ext = VisualExtractor(sd, device=cuda)
    assert ext.feature_dim == 1024
    for level in ("UTTERANCE", "FRAME"):
        got = ext.extract_clips([frames], level, nframe=8)[0]
        ref = P.dinov2_clip_features(sd, frames, level, nframe=8)
        assert got.shape == ref.shape and _rel(got, ref) < TOL


@pytest.mark.parametrize("large", [False, True])
def test_wavlm_encoder_vs_oracle(cuda, large):
    """WavLM branch: mer_hubert_frontend + mer_wavlm_gate + mer_biased_attention under the host orchestration."""
    import numpy as np

    from mertools_b200 import synthetic as S
    from mertools_b200.extract.audio import AudioExtractor
    from mertools_b200.extract.wavlm import WavLmEncoder
    from oracle import encoders as E
    from oracle import pipeline as P
    layers, heads = 4, 16 if large else 12
    sd = S.hubert_state_dict(seed=6, layers=layers, wavlm=True, large=large)
    wav = (S.synth_waves(2, 16000, seed=27).astype(np.float64) / 32768.0).astype(np.float32)
    utt, frames, hidden = WavLmEncoder(sd, device=cuda).forward(torch.from_numpy(wav).to(cuda), normalize=True,
                                                               want_frames=True, return_hidden=True)
    ref = E.hubert_hidden_states({k: torch.from_numpy(v) for k, v in sd.items()},
                                 torch.from_numpy(np.stack([P.wav2vec2_normalize(w) for w in wav])), layers=layers, heads=heads)
    for l in range(layers + 1):
        assert float((hidden[l].cpu() - ref[l]).abs().max() / ref[l].abs().max()) < 4e-3, l
    want = torch.stack(ref)[-4:].sum(dim=0)
    assert float((frames.cpu() - want).abs().max() / want.abs().max()) < 2e-3
    waves = [S.synth_waves(1, n, seed=40 + i)[0].astype(np.float64) / 32768.0 for i, n in enumerate((9000, 16000, 9000))]
    got = AudioExtractor(sd, device="cuda:0").extract_waves(waves, "UTTERANCE")
    for w, g in zip(waves, got):
        r = E.hubert_hidden_states({k: torch.from_numpy(v) for k, v in sd.items()},
                                   torch.from_numpy(P.wav2vec2_normalize(w))[None], layers=layers, heads=heads)
        r = torch.stack(r)[-4:].sum(dim=0)[0].mean(dim=0).numpy()
        assert g.shape == r.shape and np.abs(g - r).max() / np.abs(r).max() < 2e-3


def test_data2vec_vision_extractor_vs_oracle(cuda):
    """data2vec-vision branch: MER_VISION_EMBED_ONLY embeddings + host-orchestrated BEiT layers (mer_biased_attention)."""
    import numpy as np

    from mertools_b200 import synthetic as S
    from mertools_b200.extract.visual import VisualExtractor
    from oracle import pipeline as P
    sd = S.data2vec_vision_state_dict(seed=19, layers=3)
    frames = np.random.default_rng(8).integers(0, 256, (5, 112, 112, 3), dtype=np.uint8)
    ext = VisualExtractor(sd, device=cuda)
    assert ext.feature_dim == 768
    for level in ("UTTERANCE", "FRAME"):
        got = ext.extract_clips([frames], level)[0]
        ref = P.visual_clip_features(sd, frames, feature_level=level)
        assert got.shape == ref.shape and np.abs(got - ref).max() / np.abs(ref).max() < 1e-3


def test_dinov2_giant_extractor_vs_oracle(cuda):
    """dinov2-giant branch: embed-only patch embedding at 1536 columns + host-orchestrated SwiGLU layers."""
    import numpy as np

    from mertools_b200 import synthetic as S
    from mertools_b200.extract.visual import VisualExtractor
    from oracle import pipeline as P
    sd = S.dinov2_state_dict(seed=21, layers=2, hidden=1536, swiglu=True)
    frames = np.random.default_rng(3).integers(0, 256, (3, 120, 160, 3), dtype=np.uint8)
    ext = VisualExtractor(sd, device=cuda)
    assert ext.feature_dim == 1536
    got = ext.extract_clips([frames], "FRAME", nframe=4)[0]
    ref = P.dinov2_clip_features(sd, frames, "FRAME", heads=24, nframe=4)
    assert got.shape == ref.shape and np.abs(got - ref).max() / np.abs(ref).max() < 1e-3
