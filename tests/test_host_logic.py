"""CPU tests of the host-side logic and of the C-ABI surface (no GPU compute)."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from mertools_b200 import shard
from mertools_b200 import synthetic as S
from oracle import encoders as E
from oracle import pipeline as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_frame_sampling_is_bit_exact_with_the_reference_rule():
    from mertools_b200.extract.visual import resample_frames_uniform
    for n in (8, 16, 64):
        for vlen in list(range(1, 400)) + [999, 1000, 1999, 4097]:
            got = resample_frames_uniform(np.arange(vlen), n).tolist()
            assert got == P.resample_frames_uniform_indices(vlen, n), (n, vlen)
            assert len(got) == n and max(got) < vlen


def test_split_into_batch_matches_reference_rule():
    from mertools_b200.extract import audio, visual
    x = list(range(70))
    assert visual.split_into_batch(x, 32) == P.split_into_batch(x, 32)
    assert [len(b) for b in visual.split_into_batch(x, 32)] == [32, 32, 6]
    for n in (1000, 160000, 160001, 170000, 320000, 320001):
        w = torch.arange(n, dtype=torch.float32)[None]
        a, b = audio.split_into_batch(w), P.audio_split_into_batch(w)
        assert a.shape == b.shape and torch.equal(a, b)


def test_feature_file_contract(tmp_path):
    from mertools_b200.extract.common import save_feature
    f = str(tmp_path / "x.npy")
    e = save_feature(f, np.ones((5, 768), np.float32), "UTTERANCE", 768)
    assert e.shape == (768,) and np.load(f).dtype == np.float32
    e = save_feature(f, np.ones((768,), np.float32), "FRAME", 768)
    assert np.load(f).shape == (1, 768)
    e = save_feature(f, [], "UTTERANCE", 768)
    assert e.shape == (768,) and e.dtype == np.float64 and not e.any()   # np.zeros fallback of the reference
    e = save_feature(f, [], "FRAME", 768)
    assert e.shape == (1, 768)


def test_config_mirror_has_the_reference_keys():
    from mertools_b200 import config
    for k in ("PATH_TO_RAW_AUDIO", "PATH_TO_RAW_FACE", "PATH_TO_TRANSCRIPTIONS", "PATH_TO_FEATURES",
              "PATH_TO_LABEL"):
        assert "MER2023" in getattr(config, k)
    assert isinstance(config.PATH_TO_PRETRAINED_MODELS, str)


def test_shared_library_exports_every_declared_symbol():
    """The C ABI loads without a GPU and exports what include/mer_b200.h declares."""
    lib_path = os.path.join(ROOT, "mertools_b200", "lib", "libmer_b200.so")
    if not os.path.exists(lib_path):
        import __graft_entry__
        __graft_entry__.build()
    dll = ctypes.CDLL(lib_path)
    hdr = open(os.path.join(ROOT, "include", "mer_b200.h")).read()
    names = sorted(set(re.findall(r"MER_API[^;(]*?\b(mer_[a-z0-9_]+)\s*\(", hdr)))
    assert len(names) >= 20
    for n in names:
        assert hasattr(dll, n), f"missing export {n}"
    assert dll.mer_abi_version() == 4
    dll.mer_last_error.restype = ctypes.c_char_p
    assert isinstance(dll.mer_last_error(), bytes)


def test_no_cpu_fallback_without_a_device():
    """Without a GPU the product path must fail loudly, never fall back to the oracle/CPU."""
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from mertools_b200 import _lib
    rc = _lib.lib().mer_check_device()
    assert rc != 0 and _lib.lib().mer_last_error()
    from mertools_b200.encoders import VitEncoder
    with pytest.raises(_lib.MerError):
        VitEncoder(S.vit_state_dict(layers=1))


def test_product_package_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "mertools_b200")
    for d, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(d, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, re.M), f"{f} imports oracle"


def test_fusion_parameter_layout_matches_reference_state_dict_order():
    from mertools_b200.fusion import param_names, param_shapes
    names = param_names()
    assert names == list(S.fusion_state_dict().keys())
    shapes = param_shapes(768, 768, 768, 128, 6, 1)
    assert sum(int(np.prod(s)) for s in shapes.values()) == 477962  # SURVEY.md §2


def test_shard_helpers():
    assert shard.shard_indices(10, 1, 4) == [1, 5, 9]
    cover = sorted(i for r in range(8) for i in shard.shard_indices(1000, r, 8))
    assert cover == list(range(1000))
    sl = [shard.batch_slice(70, r, 4) for r in range(4)]
    assert sl[0][0] == 0 and sl[-1][1] == 70 and all(a[1] == b[0] for a, b in zip(sl, sl[1:]))
    assert sorted(h - l for l, h in sl) == [17, 17, 18, 18]


def _dp_worker(rank, world, port, q):
    import torch.distributed as dist
    from oracle import fusion as OF
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    sd = S.fusion_state_dict(seed=3)
    a, t, v, emo, val = S.synth_fusion_features(50, seed=5)
    lo, hi = shard.batch_slice(50, rank, world)
    T = torch.from_numpy
    psd = {k: torch.tensor(x, requires_grad=True) for k, x in sd.items()}
    _, eo, vo = OF.attention_forward(psd, T(a[lo:hi]), T(t[lo:hi]), T(v[lo:hi]))
    # per-rank loss = sum of per-sample losses / GLOBAL batch (loss_inv_batch of mer_fusion_fwd_bwd)
    ce, mse = OF.losses(eo, vo, T(emo[lo:hi]), T(val[lo:hi]).view(-1, 1))
    ((ce + mse) * (hi - lo) / 50.0).backward()
    flat = torch.cat([p.grad.reshape(-1) for p in psd.values()])
    shard.allreduce_grads_(flat, world)
    q.put((rank, flat.numpy()))
    dist.destroy_process_group()


def test_data_parallel_gradient_equals_full_batch_gradient_gloo():
    """world_size-2 gloo run of the N>1 fusion path semantics: all-reduce(SUM) of per-rank gradients
    scaled by 1/global_batch == the reference's gradient on the concatenated batch."""
    import torch.multiprocessing as mp
    from oracle import fusion as OF
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_dp_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    outs = dict(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    sd = S.fusion_state_dict(seed=3)
    a, t, v, emo, val = S.synth_fusion_features(50, seed=5)
    T = torch.from_numpy
    tr = OF.Trainer(sd)
    grads = tr.step(T(a), T(t), T(v), T(emo), T(val).view(-1, 1))[5]
    full = torch.cat([grads[k].reshape(-1) for k in sd]).numpy()
    for r in (0, 1):
        assert np.abs(outs[r] - full).max() <= 1e-5 * np.abs(full).max()
    assert np.array_equal(outs[0], outs[1])


def test_frame_level_shaping_is_bit_identical_to_the_reference_functions():
    """feature_scale_compress / align_to_text / pad_to_maxlen_pre_modality (read_data.py:72-125) in
    Data_Feat's order, against arrays produced by the reference's own functions."""
    import os
    import numpy as np
    from mertools_b200 import frame_features as FF
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "frame_shaping_golden.npz"))
    n, dim = int(g["n"]), int(g["dim"])

    def ragged(seed):
        rng = np.random.default_rng(seed)
        lens = rng.integers(1, 60, (3, n))
        return [[rng.standard_normal((int(t), dim)).astype(np.float32) for t in lens[m]] for m in range(3)]

    for feat_type, scale in (("frm_align", 6), ("frm_unalign", 12), ("frm_unalign", 1)):
        a, t, v = FF.shape_split(*ragged(int(g["seed"])), feat_type, scale)
        for name, x in (("a", a), ("t", t), ("v", v)):
            ref = g[f"{feat_type}_{scale}_{name}"]
            got = np.array(x)
            assert got.shape == ref.shape and got.dtype == ref.dtype and np.array_equal(got, ref), (feat_type, scale, name)


def test_c_abi_host_side_contract():
    """Pure host answers of the C ABI (no GPU work): sizes, counts, and argument validation that fails with a
    message before anything is launched."""
    import ctypes as C
    from mertools_b200 import _lib
    from mertools_b200.fusion import MerFusionDims
    dll = _lib.lib()
    dll.mer_last_error.restype = C.c_char_p
    assert dll.mer_hubert_num_frames(80000) == 249 and dll.mer_hubert_num_frames(160000) == 499
    assert dll.mer_logmel_num_frames(80000) == 498 and dll.mer_logmel_num_frames(399) == 0
    dims = MerFusionDims(768, 768, 768, 128, 6, 1)
    for fn in (dll.mer_fusion_param_count, dll.mer_fusion_frm_param_count):
        fn.restype = C.c_longlong
        fn.argtypes = [C.POINTER(MerFusionDims)]
    assert dll.mer_fusion_param_count(C.byref(dims)) == 477962           # SURVEY.md §8 a10
    lstm = 3 * (512 * 768 + 512 * 128 + 512 + 512 + 128 * 128 + 128)
    head = 128 * 384 + 128 + 2 * (128 * 128 + 128) + 3 * 128 + 3 + 6 * 128 + 6 + 128 + 1
    assert dll.mer_fusion_frm_param_count(C.byref(dims)) == lstm + head
    dll.mer_vit_workspace_bytes.restype = C.c_longlong
    assert dll.mer_vit_workspace_bytes(32) > 32 * 197 * (768 * 2 + 2304 + 3072) * 4
    # validation errors: non-zero status + message, nothing launched
    rc = dll.mer_layernorm(None, None, None, None, None, None, 4, 768, C.c_float(1e-5), 0, None)
    assert rc != 0 and b"null operand" in dll.mer_last_error()
    desc = _lib.MerGemmDesc()
    rc = dll.mer_gemm(C.byref(desc), None)
    assert rc != 0 and b"null operand" in dll.mer_last_error()
    dll.mer_resize_u8.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                  C.c_void_p, C.c_void_p]
    rc = dll.mer_resize_u8(None, 1, 10, 10, None, 224, 224, 0, None, None)
    assert rc != 0 and b"bad arguments" in dll.mer_last_error()


@pytest.mark.parametrize("hidden", [768, 1024])
def test_block_diagonal_pos_conv_weights_reproduce_the_grouped_conv(hidden):
    """The windowed block-diagonal matrix that lets the positional conv run as one GEMM
    (encoders.block_diagonal_pos_conv_weight + MerGemmDesc.a_row0 / a_col_group semantics, emulated here in
    torch) against F.conv1d(groups=16, k=128, padding=64) minus its last frame."""
    import torch.nn.functional as F
    from mertools_b200.encoders import block_diagonal_pos_conv_weight
    g = torch.Generator().manual_seed(hidden)
    gch, T, taps = hidden // 16, 37, 128
    window = 320 if gch == 48 else 256
    w = torch.randn(hidden, gch, taps, generator=g, dtype=torch.float64) * 0.05
    x = torch.randn(T, hidden, generator=g, dtype=torch.float64)
    ref = F.conv1d(x.t()[None], w, None, padding=64, groups=16)[0, :, :-1].t()              # [T, hidden]
    wbd = torch.from_numpy(block_diagonal_pos_conv_weight(w.numpy().astype(np.float32), window=window, group=gch)).double()
    xp = torch.zeros(T + taps, hidden + window, dtype=torch.float64)                          # zero rows / columns = TMA fill
    xp[64:64 + T, :hidden] = x
    out = torch.empty(T, hidden, dtype=torch.float64)
    for j in range(hidden // 256):                                                            # one 256-column output block
        win0 = (256 * j // gch) * gch
        a = torch.stack([xp[t:t + taps, win0:win0 + window].reshape(-1) for t in range(T)])  # row t: taps x window
        out[:, 256 * j:256 * (j + 1)] = a @ wbd[256 * j:256 * (j + 1)].t()
    assert float((out - ref).abs().max() / ref.abs().max()) < 1e-6


def test_clip_geometry_and_bn_folding_helpers():
    from mertools_b200.encoders import clip_preprocess_geometry, fold_conv_bn
    assert clip_preprocess_geometry(112, 112) == (224, 224, 0, 0)
    assert clip_preprocess_geometry(150, 100) == (336, 224, 56, 0)
    assert clip_preprocess_geometry(100, 151) == (224, 338, 0, 57)
    rng = np.random.default_rng(1)
    w = rng.standard_normal((8, 4, 3, 3)).astype(np.float32)
    gamma, beta = rng.uniform(0.5, 1.5, 8), rng.standard_normal(8)
    mean, var = rng.standard_normal(8), rng.uniform(0.5, 1.5, 8)
    x = torch.from_numpy(rng.standard_normal((2, 4, 9, 9)))
    ref = torch.nn.functional.batch_norm(torch.nn.functional.conv2d(x, torch.from_numpy(w).double(), None, padding=1),
                                         torch.from_numpy(mean), torch.from_numpy(var), torch.from_numpy(gamma),
                                         torch.from_numpy(beta), False, 0.0, 1e-5)
    wf, bf = fold_conv_bn(w, gamma, beta, mean, var)
    got = torch.nn.functional.conv2d(x, torch.from_numpy(wf), torch.from_numpy(bf), padding=1)
    assert float((got - ref).abs().max()) < 1e-10


@pytest.mark.slow
def test_bench_reference_arm_prints_the_contract_line():
    """`bench.py --impl reference` (the CPU arm the driver runs beside ours): one JSON line with the contract keys."""
    import json
    import subprocess
    import sys
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1",
                        "--warmup", "1", "--cpu-clips", "1"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
              "scaling", "vs_baseline", "dtype", "data", "config", "e2e", "cpu_baseline"):
        assert k in line, k
    assert line["impl"] == "reference" and line["unit"] == "clips/s" and line["value"] > 0
    assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] >= 1
    assert line["e2e"]["h2d_bytes_per_step"] == 0 and "workload" in line["config"]


def test_vggish_save_rules_match_reference_script():
    """extract_vggish_embedding.py:52-59: UTTERANCE squeezes and averages over segments, FRAME saves [segments, 128]."""
    from mertools_b200.extract import vggish
    one, many = np.arange(128.0)[None], np.stack([np.arange(128.0), np.ones(128)])
    assert vggish.save_embeddings(None, one, "UTTERANCE").shape == (128,)
    assert np.array_equal(vggish.save_embeddings(None, many, "UTTERANCE"), many.mean(0))
    assert vggish.save_embeddings(None, one, "FRAME").shape == (1, 128)
    args = vggish.build_parser().parse_args([])
    assert (args.gpu, args.feature_level, args.dataset) == (0, "FRAME", "MER2023")


def test_cnn_executor_plans_the_ferplus_tables_without_a_gpu():
    """mer_cnn_workspace_bytes walks the op table on the host (shape inference, buffer extents, table checks):
    52 convolutions, ceil-mode max-pool 112 -> 56, caffe-style strides down to 7 x 7 x 512."""
    from mertools_b200 import encoders as En
    from mertools_b200 import synthetic as S
    m, _keep = En.ferplus_resnet50_tables(S.ferplus_resnet50_state_dict(9), lambda wp, bp: (1, 1))
    assert m.n_convs == 52 and m.ops[m.n_ops - 1].kind == En.CNN_GAP
    import ctypes as C

    from mertools_b200 import _lib
    dll = _lib.lib()
    dll.mer_cnn_workspace_bytes.restype = C.c_longlong
    dll.mer_cnn_workspace_bytes.argtypes = [C.POINTER(En.MerCnnModel), C.c_int]
    one, two = dll.mer_cnn_workspace_bytes(C.byref(m), 1), dll.mer_cnn_workspace_bytes(C.byref(m), 2)
    # stem output 112*112*128 fp32 + stream / shortcut 56*56*256 fp32 each + 56*56*128 + the stem's split operand
    expect = 4 * (112 * 112 * 128 + 2 * 56 * 56 * 256 + 56 * 56 * 128) + 112 * 112 * 160 * 4
    assert expect <= one <= expect + 8 * 256 and 2 * expect <= two <= 2 * expect + 8 * 256
    m.ops[3].res = 2   # 56 x 56 x 128 residual for a 256-channel output
    assert dll.mer_cnn_workspace_bytes(C.byref(m), 1) == -1 and b"residual shape" in dll.mer_last_error()
    m.ops[3].res = -1
    m.ops[1].ceil_mode = 0   # floor mode: 55 x 55 maps, 4 x 4 at the end -> still a valid chain
    assert dll.mer_cnn_workspace_bytes(C.byref(m), 1) > 0
    # senet50_ferplus_dag: 15 squeeze-and-excitation ops with their 30 dense layers
    m, _keep = En.ferplus_resnet50_tables(S.ferplus_resnet50_state_dict(9, se=True), lambda wp, bp: (1, 1))
    assert m.n_convs == 82 and sum(m.ops[i].kind == En.CNN_SE for i in range(m.n_ops)) == 15
    assert dll.mer_cnn_workspace_bytes(C.byref(m), 1) >= one + 2 * 2048 * 4
    se_op = next(i for i in range(m.n_ops) if m.ops[i].kind == En.CNN_SE)
    m.ops[se_op].res = 2   # 64-channel map as the shortcut of a 256-channel block
    assert dll.mer_cnn_workspace_bytes(C.byref(m), 1) == -1 and b"SE shortcut shape" in dll.mer_last_error()


def test_cnn_planner_refuses_tables_the_executor_cannot_run():
    """mer_cnn_workspace_bytes (the planning pass mer_cnn_forward also runs before its first launch) returns -1 with a
    message for convolution geometry the im2col gather or the GEMM cannot run, a stem whose output width is no GEMM
    column block, and a 3x3 / 2 max-pool whose window does not fit the map (torch raises for those sizes).  The same
    tables with the defect removed plan normally."""
    import ctypes as C

    from mertools_b200 import _lib
    from mertools_b200 import encoders as En
    dll = _lib.lib()
    dll.mer_cnn_workspace_bytes.restype = C.c_longlong
    dll.mer_cnn_workspace_bytes.argtypes = [C.POINTER(En.MerCnnModel), C.c_int]
    import _kernel_refs as R
    for name, m, _keep, msg in R.cnn_refused_tables():
        assert dll.mer_cnn_workspace_bytes(C.byref(m), 2) == -1, name
        err = dll.mer_last_error().decode()
        assert msg in err, (name, err)
    # controls: the f16 conv at 64 channels (K 576), split at 8 channels 2x2 (K 32), pad 0 ceil-mode pool of 2 x 2
    fake = 0x7F0000000000
    conv = lambda cin, k, kpad: dict(w=fake, b=fake, cin=cin, cout=128, cout_pad=128, k=k, stride=1, pad=1,  # noqa
                                     kpad=kpad)
    for mode, c, ch in ((_lib.MER_GEMM_F16, conv(64, 3, 576), 64), (_lib.MER_GEMM_BF16X3, conv(8, 2, 32), 8)):
        stem = dict(conv(3, 7, 192 if mode == _lib.MER_GEMM_F16 else 160), stride=2, pad=3)
        m, _k = R.cnn_model([stem, c], [dict(kind=0, conv=0, dst=0), dict(kind=6, src=0, dst=1, p=(ch,)),
                                        dict(kind=1, conv=1, src=1, dst=2), dict(kind=3, src=2)], mode, (3, 3), 128)
        assert dll.mer_cnn_workspace_bytes(C.byref(m), 2) == R.cnn_plan(m, 2)[0]["total"]
    m, _k = R.cnn_model([dict(conv(3, 7, 192), stride=2, pad=3)],
                        [dict(kind=0, conv=0, dst=0), dict(kind=2, src=0, dst=1, k=3, stride=2, pad=0, ceil_mode=1),
                         dict(kind=3, src=1)], _lib.MER_GEMM_F16, (3, 3), 128)
    assert dll.mer_cnn_workspace_bytes(C.byref(m), 1) == R.cnn_plan(m, 1)[0]["total"]
    assert R.cnn_plan(m, 1)[1][1][:2] == (1, 1)


def test_pool_output_size_matches_torch():
    """The planner's MaxPool2d(3, 2) output size (mirrored by _kernel_refs.pool_out_size) against torch's own, including
    the sizes torch refuses."""
    import _kernel_refs as R
    import torch.nn.functional as F
    for pad in (0, 1):
        for ceil in (0, 1):
            for h in range(1, 120):
                try:
                    want = F.max_pool2d(torch.zeros(1, 1, h, 1 + 2 * pad + 2), 3, 2, pad, ceil_mode=bool(ceil)).shape[2]
                except RuntimeError:
                    want = 0
                assert max(R.pool_out_size(h, pad, ceil), 0) == want, (h, pad, ceil)


def _interpret(m, store, frames_bgr):
    """out_feats of the float64 interpreter of the op semantics (tests/_kernel_refs.py), every column written."""
    import _kernel_refs as R
    out, _ = R.interpret_cnn_tables(m, store, frames_bgr, dtype=torch.float64)
    assert not torch.isnan(out).any(), "some output columns were never written"
    return out.numpy()


@pytest.mark.parametrize("se,prefix", [(False, ""), (True, "se_")])
def test_ferplus_op_tables_reproduce_the_reference_golden_on_a_cpu_interpreter(se, prefix):
    """The conv / op tables FerplusResnet50Encoder hands to mer_cnn_forward (BN folding, (ky, kx, c) weight layout,
    channel padding, caffe-style strides, shortcut wiring, SE layer indices), run by a torch interpreter of the op
    semantics, against outputs of the unmodified reference extractor.  Checks the host side of the CUDA path; the
    kernels themselves are compared with the same interpreter op by op in tests/test_cnn_kernels_gpu.py."""
    import importlib.util
    from mertools_b200 import encoders as En
    from oracle import pipeline as P
    gdir = os.path.join(ROOT, "tests", "golden")
    spec = importlib.util.spec_from_file_location("make_golden_ferplus", os.path.join(gdir, "make_golden_ferplus.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    g = np.load(os.path.join(gdir, "ferplus_golden.npz"))
    store = {}

    def pack(w, b):
        store[len(store) + 1] = np.asarray(w, np.float32)
        store[len(store) + 1] = np.asarray(b, np.float32)
        return len(store) - 1, len(store)
    m, _keep = En.ferplus_resnet50_tables(S.ferplus_resnet50_state_dict(int(g["seed"]), se=se), pack)
    frames = mod.golden_clips()["vidA"][:2]                       # 256 x 256: Resize(256) is the identity
    crop = frames[:, 16:240, 16:240]                              # CenterCrop(224), as frame_features slices it
    got = _interpret(m, store, crop)
    ref = g[f"{prefix}fra_vidA"][:2]
    assert got.shape == ref.shape and np.abs(got - ref).max() / np.abs(ref).max() < 1e-4
    enc_geom = En.FerplusResnet50Encoder.preprocess_geometry(None, 200, 300)
    assert En.ManetEncoder.preprocess_geometry(None, 200, 300) == (224, 224, 0, 0)
    assert enc_geom == (256, 384, 16, 80) and P.ferplus_preprocess(mod.golden_clips()["vidC"]).shape == (1, 3, 224, 224)


def test_vggish_tables_reproduce_the_oracle_on_a_cpu_interpreter():
    """The packed VGGish weights (HWIO -> [cout_pad, (ky, kx, c)], conv1 padded to 32 columns, FC matrices transposed
    to [N, K]) run through the op sequence of mer_vggish_forward (resnet.cu) in torch, against the oracle."""
    import torch.nn.functional as F
    from mertools_b200 import encoders as En
    from oracle import encoders as E
    sd = S.vggish_state_dict(seed=8)
    store = {}

    def pack(w, b):
        store[len(store) + 1] = np.asarray(w, np.float32)
        store[len(store) + 1] = np.asarray(b, np.float32)
        return len(store) - 1, len(store)
    m = En.vggish_tables(sd, pack)
    x = torch.from_numpy(np.random.default_rng(2).normal(-2.0, 2.0, (2, 96, 64, 1)).astype(np.float32))  # NHWC
    pool_after = (0, 1, 3, 5)
    for i in range(6):
        c = m.convs[i]
        kk = 9 * c.cin
        assert (c.k, c.stride, c.pad) == (3, 1, 1) and c.kpad == (32 if i == 0 else kk)
        wt = torch.from_numpy(store[c.w][:, :kk]).reshape(c.cout_pad, 3, 3, c.cin).permute(0, 3, 1, 2)
        y = F.conv2d(x[..., :c.cin].permute(0, 3, 1, 2), wt, torch.from_numpy(store[c.b]), padding=1)
        x = torch.relu(y).permute(0, 2, 3, 1)
        if i in pool_after:
            x = F.max_pool2d(x.permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
    assert x.shape == (2, 6, 4, 512)
    h = x.reshape(2, -1)                                            # the NHWC buffer as it lies
    for i in range(3):
        h = torch.relu(h @ torch.from_numpy(store[m.fc_w[i]]).T + torch.from_numpy(store[m.fc_b[i]]))
    ref = E.vggish_embeddings({k: torch.from_numpy(v) for k, v in sd.items()},
                              torch.from_numpy(np.random.default_rng(2).normal(-2.0, 2.0, (2, 96, 64, 1)).astype(np.float32))[..., 0])
    assert h.shape == (2, 128) and float((h - ref).abs().max() / ref.abs().max()) < 1e-5


def test_manet_op_tables_reproduce_the_reference_golden_on_a_cpu_interpreter():
    """The 136 layers / 184 ops MA-Net hands to mer_cnn_forward (trunk, four cropped CBAM branches accumulated into
    columns 0..511, the multi-scale branch assembled from channel slices into columns 512..1023), run by the torch
    interpreter of the op semantics, against outputs of the unmodified reference model."""
    import ctypes as C
    import importlib.util

    from mertools_b200 import _lib
    from mertools_b200 import encoders as En
    gdir = os.path.join(ROOT, "tests", "golden")
    spec = importlib.util.spec_from_file_location("make_golden_manet", os.path.join(gdir, "make_golden_manet.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    g = np.load(os.path.join(gdir, "manet_golden.npz"))
    store = {}

    def pack(w, b):
        store[len(store) + 1] = np.asarray(w, np.float32)
        store[len(store) + 1] = np.asarray(b, np.float32)
        return len(store) - 1, len(store)
    m, _keep = En.manet_tables(S.manet_state_dict(int(g["seed"])), pack)
    got = _interpret(m, store, mod.golden_clips()["vidA"][:2])
    ref = g["fra_vidA"][:2]
    assert got.shape == ref.shape and np.abs(got - ref).max() / np.abs(ref).max() < 1e-4
    dll = _lib.lib()
    dll.mer_cnn_workspace_bytes.restype = C.c_longlong
    dll.mer_cnn_workspace_bytes.argtypes = [C.POINTER(En.MerCnnModel), C.c_int]
    assert m.n_convs == 136 and dll.mer_cnn_workspace_bytes(C.byref(m), 2) > 0   # the C++ planner accepts the table


def test_emonet_op_tables_reproduce_the_reference_golden_on_a_cpu_interpreter():
    """The 222 layers / 367 ops EmoNet hands to mer_cnn_forward (folded stem, AFFINE -> CONV pre-activation triples
    written into channel slices, the two depth-4 hourglasses with their skip / low buffers, heat-map mask,
    emotion tower), run by the torch interpreter, against outputs of the unmodified reference model."""
    import ctypes as C
    import importlib.util

    from mertools_b200 import _lib
    from mertools_b200 import encoders as En
    gdir = os.path.join(ROOT, "tests", "golden")
    spec = importlib.util.spec_from_file_location("make_golden_emonet", os.path.join(gdir, "make_golden_emonet.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    g = np.load(os.path.join(gdir, "emonet_golden.npz"))
    store = {}

    def pack(w, b):
        store[len(store) + 1] = np.asarray(w, np.float32)
        store[len(store) + 1] = np.asarray(b, np.float32)
        return len(store) - 1, len(store)
    m, _keep = En.emonet_tables(S.emonet_state_dict(int(g["seed"])), pack)
    got = _interpret(m, store, mod.golden_clips()["vidA"][:1])                      # 256 x 256: no resize needed
    ref = g["fra_vidA"][:1]
    assert got.shape == ref.shape and np.abs(got - ref).max() / np.abs(ref).max() < 1e-4
    dll = _lib.lib()
    dll.mer_cnn_workspace_bytes.restype = C.c_longlong
    dll.mer_cnn_workspace_bytes.argtypes = [C.POINTER(En.MerCnnModel), C.c_int]
    assert dll.mer_cnn_workspace_bytes(C.byref(m), 2) > 0


def test_ctypes_struct_layouts_match_the_header(tmp_path):
    """Every struct the Python side passes by pointer is mirrored by hand in ctypes: compile a C probe against
    include/mer_b200.h and compare sizes and the offsets of the trailing fields."""
    import ctypes as C
    import shutil
    import subprocess

    from mertools_b200 import _lib, fusion, weights
    from mertools_b200 import encoders as En
    if shutil.which("gcc") is None:
        pytest.skip("no C compiler")
    probes = [("MerHubertModel", En.MerHubertModel, ["pos_window", "layers_f16", "n_pos_layers", "pos_layers_w", "ln_zeros", "conv_w_f16"]),
              ("MerCnnOp", En.MerCnnOp, ["relu", "ceil_mode", "p"]),
              ("MerCnnModel", En.MerCnnModel, ["ops", "scale", "mean", "feat_dim"]),
              ("MerVggishModel", En.MerVggishModel, ["fc_w", "fc_b"]),
              ("MerResnetConv", En.MerResnetConv, ["b", "kpad"]),
              ("MerResnet18Model", En.MerResnet18Model, ["mean", "std"]),
              ("MerClipVisionModel", En.MerClipVisionModel, []),
              ("MerVitModel", En.MerVitModel, []),
              ("MerBertModel", En.MerBertModel, ["layers"]),
              ("MerGemmDesc", _lib.MerGemmDesc, ["a_row0", "a_col_group", "ep"]),
              ("MerGemmEpilogue", _lib.MerGemmEpilogue, []),
              ("MerLayerWeights", weights.MerLayerWeights, []),
              ("MerFusionDims", fusion.MerFusionDims, []),
              ("MerFusionTopnDims", fusion.MerFusionTopnDims, [])]
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{os.path.join(ROOT, "include", "mer_b200.h")}"',
             "int main(void) {"]
    for name, _cls, fields in probes:
        lines.append(f'  printf("{name} %zu", sizeof({name}));')
        for f in fields:
            lines.append(f'  printf(" %zu", offsetof({name}, {f}));')
        lines.append('  printf("\\n");')
    lines += ["  return 0;", "}"]
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-o", str(exe), str(src)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.strip().splitlines()
    for (name, cls, fields), line in zip(probes, out):
        want = [int(v) for v in line.split()[1:]]
        got = [C.sizeof(cls)] + [getattr(cls, f).offset for f in fields]
        assert got == want, f"{name}: ctypes {got} != C {want}"


def test_ctypes_declarations_have_the_arity_of_the_header_prototypes():
    """Every ``_lib.declare("mer_...", [argtypes])`` in the package against the parameter count of the MER_API
    prototype in include/mer_b200.h (a wrong count would only show up as garbage arguments on a GPU)."""
    import glob
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "mer_b200.h")).read(), flags=re.S)
    protos = {}
    for m in re.finditer(r"MER_API\s+[\w\s\*]+?\b(mer_\w+)\s*\(([^;]*?)\)\s*;", hdr, flags=re.S):
        args = m.group(2).strip()
        protos[m.group(1)] = 0 if args in ("", "void") else len(args.split(","))
    assert len(protos) >= 40
    checked = 0
    for f in glob.glob(os.path.join(ROOT, "mertools_b200", "**", "*.py"), recursive=True) + [os.path.join(ROOT, "bench.py")]:
        src = open(f).read()
        for m in re.finditer(r'declare\(\s*"(mer_\w+)"\s*,\s*\[', src):
            i = j = m.end()
            depth = 1
            while depth:
                depth += (src[j] == "[") - (src[j] == "]")
                j += 1
            body, d, n = src[i:j - 1].strip().rstrip(","), 0, 1
            for ch in body:
                d += (ch in "([") - (ch in ")]")
                n += ch == "," and d == 0
            assert m.group(1) in protos, (f, m.group(1))
            assert protos[m.group(1)] == n, (os.path.basename(f), m.group(1), n, protos[m.group(1)])
            checked += 1
    assert checked >= 20


class _TorchWhisperOps:
    """CPU stand-in for mertools_b200.extract.whisper.CudaOps with the same op semantics (test infrastructure): lets the
    backend-agnostic orchestration run against the reference golden without a GPU."""

    def tensor(self, a):
        return torch.from_numpy(np.ascontiguousarray(a, np.float32))

    weight = tensor

    def logmel(self, waves):
        out = torch.zeros(len(waves), 3000, 96)
        for i, w in enumerate(waves):
            out[i, :, :80] = torch.from_numpy(P.whisper_log_mel(w)).T          # time-major, K padded to 96
        return out

    def conv1(self, mel, w, b):
        B, T, K = mel.shape
        d = w.shape[0]
        xp = torch.zeros(B, T + 2, K)
        xp[:, 1:T + 1] = mel                                                    # a_row0 = -1: one zero row before / after
        y = sum(xp[:, k:k + T] @ w[:, k * K:(k + 1) * K].T for k in range(3)) + b
        out = torch.zeros(B, T + 2, d)
        out[:, 1:T + 1] = torch.nn.functional.gelu(y)
        return out

    def conv2(self, xpad, w, b, pos):
        B, rows, d = xpad.shape
        T = 1500
        y = sum(xpad[:, k:k + 2 * T:2] @ w[:, k * d:(k + 1) * d].T for k in range(3)) + b
        return pos + torch.nn.functional.gelu(y).reshape(B * T, d)

    def layernorm(self, x, g, b, operand):
        return torch.nn.functional.layer_norm(x, (x.shape[-1],), g, b, 1e-5)

    def linear(self, x, w, b, gelu=False, res=None, operand=False):
        y = x @ w.T + b
        y = torch.nn.functional.gelu(y) if gelu else y
        return y if res is None else res + y

    def _att(self, q, k, v, heads, causal):
        B, nq, d = q.shape
        hd = d // heads
        q, k, v = (t.reshape(B, -1, heads, hd).transpose(1, 2) for t in (q, k, v))
        s = q @ k.transpose(-1, -2) / 8.0
        if causal:
            s = s + torch.full(s.shape[-2:], float("-inf")).triu(1)
        return (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B * nq, d)

    def self_attention(self, qkv, B, T, heads):
        d = qkv.shape[1] // 3
        q, k, v = (qkv[:, i * d:(i + 1) * d].reshape(B, T, d) for i in range(3))
        return self._att(q, k, v, heads, False)

    def small_attention(self, q, q0, k, k0, v, v0, B, heads, nq, nk, causal):
        d = heads * 64
        return self._att(q[:, q0:q0 + d].reshape(B, nq, d), k[:, k0:k0 + d].reshape(B, nk, d),
                         v[:, v0:v0 + d].reshape(B, nk, d), heads, causal)


def test_whisper_orchestration_reproduces_the_reference_golden_with_a_cpu_backend():
    """mertools_b200.extract.whisper.WhisperNet (weight packing: tap-major conv matrices with the mel axis padded to 96,
    fused q|k|v with a zero k bias, fused cross k|v; op order, residuals, position tables, decoder start tokens) run
    with a torch backend of the same op semantics, against outputs of the unmodified reference extract()."""
    from mertools_b200.extract.whisper import WhisperNet, whisper_mel_filters
    g = np.load(os.path.join(ROOT, "tests", "golden", "audio_whisper_golden.npz"))
    layers = int(g["layers"])
    net = WhisperNet(S.whisper_state_dict(seed=int(g["seed"]), enc_layers=layers, dec_layers=layers), _TorchWhisperOps())
    waves = [S.synth_waves(1, int(n), seed=int(g["seed0"]) + i)[0].astype(np.float64) / 32768.0 for i, n in enumerate(g["lens"])]
    with torch.no_grad():
        out = net.last_hidden_state(waves, int(g["start"])).numpy()
    for i in range(len(waves)):
        ref = g[f"fra{i}"]
        assert out[i].shape == ref.shape and np.abs(out[i] - ref).max() / np.abs(ref).max() < 1e-4, i
        assert np.abs(out[i].mean(0) - g[f"utt{i}"]).max() / np.abs(g[f"utt{i}"]).max() < 1e-4
    assert np.array_equal(whisper_mel_filters(), P.whisper_mel_filters().astype(np.float32))


def test_encoder_constructors_run_with_the_device_layer_stubbed(monkeypatch):
    """Every encoder's __init__ (checkpoint inspection, weight re-layout, ctypes model structs) executed on CPU with
    only the device-touching calls stubbed: tensors stay on the host, rounding / splitting kernels become identities.
    Catches host-side mistakes in constructor paths that the GPU tests of this round have not exercised yet."""
    from mertools_b200 import _lib
    from mertools_b200 import encoders as En
    from mertools_b200 import weights as Wt
    monkeypatch.setattr(_lib, "check", lambda rc: None)
    monkeypatch.setattr(_lib, "round_tf32_", lambda t: t)
    monkeypatch.setattr(_lib, "split_bf16", lambda t: t.clone())
    monkeypatch.setattr(Wt, "_dev", lambda x, device: (torch.from_numpy(np.ascontiguousarray(x)) if isinstance(x, np.ndarray)
                                                        else x).detach().to(dtype=torch.float32).contiguous())
    made = {
        "vit": En.VitEncoder(S.vit_state_dict(seed=0, layers=2)),
        "clip_b32": En.ClipVisionEncoder(S.clip_vision_state_dict(variant="b32", layers=2)),
        "clip_l14_f16": En.ClipVisionEncoder(S.clip_vision_state_dict(variant="l14", layers=1), precision="f16"),
        "dinov2": En.Dinov2Encoder(S.dinov2_state_dict(layers=1)),
        "resnet18": En.ResNet18Encoder(S.resnet18_state_dict()),
        "ferplus": En.FerplusResnet50Encoder(S.ferplus_resnet50_state_dict()),
        "senet": En.FerplusResnet50Encoder(S.ferplus_resnet50_state_dict(se=True)),
        "manet": En.ManetEncoder(S.manet_state_dict()),
        "emonet": En.EmonetEncoder(S.emonet_state_dict()),
        "vggish": En.VggishEncoder(S.vggish_state_dict()),
        "hubert": En.HubertEncoder(S.hubert_state_dict(layers=4)),
        "hubert_large": En.HubertEncoder(S.hubert_state_dict(layers=4, large=True)),
        "wav2vec2_large_960h": En.HubertEncoder(S.hubert_state_dict(layers=4, large=True, group_norm=True)),
        "data2vec": En.HubertEncoder(S.hubert_state_dict(layers=4, data2vec=True)),
        "data2vec_large": En.HubertEncoder(S.hubert_state_dict(layers=4, data2vec=True, large=True)),
        # WavLM checkpoints: the front-end of the WavLM branch is this struct (mer_hubert_frontend)
        "wavlm": En.HubertEncoder(S.hubert_state_dict(layers=4, wavlm=True)),
        "wavlm_large": En.HubertEncoder(S.hubert_state_dict(layers=4, wavlm=True, large=True)),
        "bert": En.BertEncoder(S.bert_state_dict(100, layers=4)),
        "bert_large": En.BertEncoder(S.bert_state_dict(100, layers=4, large=True)),
    }
    assert made["clip_l14_f16"].precision == "f16" and made["clip_l14_f16"].tokens == 257
    d = made["dinov2"]
    assert (d.precision, d.tokens, d.proj_dim, d.model.variant, bool(d.model.pre_ln_g), d.model.kpad) == ("tf32", 257, 1024, 1, False, 608)
    assert d.preprocess_geometry(120, 160) == (256, 341, 16, 58) and made["clip_b32"].preprocess_geometry(120, 160) == (224, 298, 0, 37)
    assert (made["ferplus"].model.n_convs, made["senet"].model.n_convs, made["manet"].model.n_convs,
            made["emonet"].model.n_convs) == (52, 82, 136, 222)
    h = made["data2vec"].model
    assert (h.n_pos_layers, h.pos_taps, h.feat_norm_layer, h.stable_layer_norm, bool(h.conv_b[1])) == (5, 19, 1, 0, False)
    h = made["wavlm_large"].model
    assert (h.hidden, h.feat_norm_layer, h.stable_layer_norm, bool(h.conv_b[1]), made["wavlm"].model.stable_layer_norm) == (1024, 1, 1, False, 0)
    h = made["data2vec_large"].model
    assert (h.hidden, h.heads, h.n_pos_layers, h.pos_window, h.stable_layer_norm, bool(h.conv_b[1])) == (1024, 16, 5, 256, 0, False)
    h = made["wav2vec2_large_960h"].model
    assert (h.hidden, h.heads, h.feat_norm_layer, h.stable_layer_norm, h.pos_window) == (1024, 16, 0, 0, 256)
    h = made["hubert_large"].model
    assert (h.hidden, h.feat_norm_layer, h.stable_layer_norm, bool(h.conv_b[1])) == (1024, 1, 1, True)
    b = made["bert_large"].model
    assert (made["bert_large"].hidden, b.hidden, b.ffn, b.heads) == (1024, 1024, 4096, 16) and made["bert"].model.hidden == 768


def _videomae_frames(n=21, h=120, w=160, seed=31):
    return np.random.default_rng(seed).integers(0, 256, (n, h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize("final_norm", [False, True])
def test_videomae_oracle_is_pinned_to_the_hf_model_and_processor(final_norm):
    """extract_vision_huggingface.py:147-159 restated in oracle/: VideoMAEImageProcessor (shortest edge 224 bilinear,
    centre crop, rescale, normalise) and VideoMAEModel (use_mean_pooling=True: no final LayerNorm) on a synthetic
    checkpoint that strict-loads into the HF class."""
    transformers = pytest.importorskip("transformers")
    # final_norm: the self-supervised checkpoints (use_mean_pooling=False, what `videomae-base` is) end with a LayerNorm
    sd = S.videomae_state_dict(seed=15, layers=2, final_norm=final_norm)
    cfg = transformers.VideoMAEConfig(num_hidden_layers=2, use_mean_pooling=not final_norm)
    model = transformers.VideoMAEModel(cfg).eval()
    missing = model.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=False)
    assert not missing.unexpected_keys and all("position" in k for k in missing.missing_keys), missing
    # the Pillow-backed processor = the transformers-4.x one the reference ran (5.x's default is torchvision-backed and
    # differs from Pillow by one grey level on ~1 % of the upscaled pixels)
    proc = transformers.VideoMAEImageProcessorPil()
    frames = _videomae_frames()
    sel = [frames[i] for i in P.resample_frames_uniform_indices(len(frames), 16)]
    inputs = proc([f[:, :, ::-1].copy() for f in sel], return_tensors="pt")["pixel_values"]
    mine = P.videomae_preprocess(frames, proc.image_mean, proc.image_std)
    assert tuple(inputs.shape) == tuple(mine.shape) == (1, 16, 3, 224, 224)
    assert float((inputs - mine).abs().max()) < 2e-6
    with torch.no_grad():
        ref = model(inputs).last_hidden_state
    got = E.videomae_last_hidden_state(sd, mine)
    assert float((got - ref).abs().max() / ref.abs().max()) < 1e-5
    utt = P.videomae_clip_features(sd, frames, "UTTERANCE", mean=proc.image_mean, std=proc.image_std)
    fra = P.videomae_clip_features(sd, frames, "FRAME", mean=proc.image_mean, std=proc.image_std)
    assert utt.shape == (768,) and fra.shape == (8, 768)
    np.testing.assert_allclose(fra, ref.view(8, 196, -1).mean(1).numpy(), rtol=0, atol=1e-5 * float(ref.abs().max()))


class _TorchVideoMaeOps(_TorchWhisperOps):
    """CPU stand-in for the VideoMAE product backend: the patch gather in the layout mer_videomae_patchify writes
    (rows = (clip, tubelet, patch row, patch column); K = (channel RGB, frame-in-tubelet, dy, dx))."""

    def patchify(self, frames, mean, std):
        from _kernel_refs import videomae_patches   # the one definition, shared with the kernel's own GPU test
        return videomae_patches(torch.from_numpy(np.ascontiguousarray(np.asarray(frames))), mean, std).float()

    def layernorm(self, x, g, b, operand, eps=1e-5):
        return torch.nn.functional.layer_norm(x, (x.shape[-1],), g, b, eps)


@pytest.mark.parametrize("final_norm", [False, True])
def test_videomae_orchestration_matches_the_oracle_with_a_cpu_backend(final_norm):
    """mertools_b200.extract.videomae.VideoMaeNet (Conv3d weight flattened to the patch-gather K order, fused q|k|v with
    the zero key bias, fixed sinusoid positions, pre-LN layers, no final LayerNorm) run over a torch backend."""
    from mertools_b200.extract.videomae import VideoMaeNet, sinusoid_table
    sd = S.videomae_state_dict(seed=16, layers=2, final_norm=final_norm)
    np.testing.assert_allclose(sinusoid_table(1568, 768), E.videomae_sinusoid_table(1568, 768).numpy(), atol=1e-6)
    frames = _videomae_frames(n=16, h=224, w=224, seed=32)
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    net = VideoMaeNet(sd, _TorchVideoMaeOps())
    assert net.heads == 12 and len(net.layers) == 2
    got = net.last_hidden_state(frames, mean, std)
    ref = E.videomae_last_hidden_state(sd, P.videomae_preprocess(frames, mean, std))
    assert tuple(got.shape) == tuple(ref.shape) == (1, 1568, 768)
    assert float((got - ref).abs().max() / ref.abs().max()) < 1e-5
    two = net.last_hidden_state(np.concatenate([frames, frames[::-1]]), mean, std)     # clip-major rows for B > 1
    assert float((two[0] - ref[0]).abs().max() / ref.abs().max()) < 1e-5


def test_dinov2_oracle_is_pinned_to_hf_and_the_clip_layout_conversion_reproduces_it():
    """extract_vision_huggingface.py:135-145 (DINOv2 branch).  (1) oracle restatement vs HF Dinov2Model and the
    Pillow-backed BitImageProcessor on a synthetic dinov2-large-shaped checkpoint that strict-loads; (2) the product's
    weight re-layout (dinov2_to_clip_layout: interpolated positions, folded patch bias and LayerScale) run through a
    torch emulation of what mer_clip_vision_forward computes for MER_VISION_DINOV2 (no pre_layrnorm, erf GELU, token
    sum of the last layer's output)."""
    transformers = pytest.importorskip("transformers")
    from PIL import Image

    from mertools_b200.encoders import dinov2_to_clip_layout
    sd = S.dinov2_state_dict(seed=17, layers=2)
    cfg = transformers.Dinov2Config(hidden_size=1024, num_hidden_layers=2, num_attention_heads=16, image_size=518, patch_size=14)
    model = transformers.Dinov2Model(cfg).eval()
    model.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    proc = transformers.BitImageProcessorPil(do_resize=True, size={"shortest_edge": 256}, resample=3, do_center_crop=True,
                                             crop_size={"height": 224, "width": 224}, do_rescale=True, do_normalize=True,
                                             image_mean=[0.485, 0.456, 0.406], image_std=[0.229, 0.224, 0.225], do_convert_rgb=True)
    frames = np.random.default_rng(3).integers(0, 256, (3, 120, 160, 3), dtype=np.uint8)
    inputs = proc(images=[Image.fromarray(f[:, :, ::-1].copy()) for f in frames], return_tensors="pt")["pixel_values"]
    mine = P.dinov2_preprocess(frames)
    assert float((inputs - mine).abs().max()) < 2e-6
    with torch.no_grad():
        ref = model(inputs, output_hidden_states=True).hidden_states[-1]
    got = E.dinov2_hidden_states(sd, mine)[-1]
    assert float((got - ref).abs().max() / ref.abs().max()) < 1e-5
    fra = P.dinov2_clip_features(sd, frames, "FRAME", nframe=4)
    assert fra.shape == (4, 1024)                                       # 3 frames resampled to 4 (last one repeated)
    np.testing.assert_allclose(fra[:3], ref.sum(dim=1).numpy(), rtol=0, atol=2e-5 * float(ref.sum(dim=1).abs().max()))
    # (2) the CLIP-layout tensors through the tower as the kernels walk it
    c = {k: torch.from_numpy(np.asarray(v, np.float32)) for k, v in dinov2_to_clip_layout(sd).items()}
    v = "vision_model."
    pw = c[v + "embeddings.patch_embedding.weight"]
    x = torch.nn.functional.conv2d(mine, pw, None, stride=14).flatten(2).transpose(1, 2)
    pos = c[v + "embeddings.position_embedding.weight"]
    assert tuple(pos.shape) == (257, 1024)
    x = torch.cat([(c[v + "embeddings.class_embedding"] + pos[0]).expand(len(x), 1, -1), x + pos[1:]], dim=1)
    lin = lambda t, n: torch.nn.functional.linear(t, c[n + ".weight"], c[n + ".bias"])  # noqa: E731
    ln = lambda t, n: torch.nn.functional.layer_norm(t, (1024,), c[n + ".weight"], c[n + ".bias"], 1e-6)  # noqa: E731
    for i in range(2):
        p = f"{v}encoder.layers.{i}."
        y = ln(x, p + "layer_norm1")
        q, k, vv = (lin(y, p + f"self_attn.{n}_proj").reshape(len(x), 257, 16, 64).transpose(1, 2) for n in "qkv")
        ctx = (torch.softmax(q @ k.transpose(-1, -2) / 8.0, -1) @ vv).transpose(1, 2).reshape(len(x), 257, 1024)
        x = x + lin(ctx, p + "self_attn.out_proj")
        x = x + lin(torch.nn.functional.gelu(lin(ln(x, p + "layer_norm2"), p + "mlp.fc1")), p + "mlp.fc2")
    assert float((x.sum(dim=1) - ref.sum(dim=1)).abs().max() / ref.sum(dim=1).abs().max()) < 1e-5


class _TorchWavLmOps(_TorchWhisperOps):
    """CPU stand-in for the WavLM product backend, with the semantics of mer_wavlm_gate / mer_biased_attention."""

    def operand(self, x):
        return x

    def layernorm(self, x, g, b, operand, eps=1e-5):
        return torch.nn.functional.layer_norm(x, (x.shape[-1],), g, b, eps)

    def gate(self, x, heads, w, b, c):
        proj = (x.reshape(x.shape[0], heads, 64) @ w.T + b).reshape(x.shape[0], heads, 2, 4).sum(-1)
        ga, gb = torch.sigmoid(proj[..., 0]), torch.sigmoid(proj[..., 1])
        return ga * (gb * c - 1.0) + 2.0                                            # [tokens, heads]

    def swiglu(self, x):
        a, b = x.chunk(2, dim=-1)
        return torch.nn.functional.silu(a) * b

    def biased_attention(self, qkv, bias, gate, B, T, heads):
        d = qkv.shape[1] // 3
        q, k, v = (qkv[:, i * d:(i + 1) * d].reshape(B, T, heads, 64).transpose(1, 2) for i in range(3))
        g = 1.0 if gate is None else gate.reshape(B, T, heads).permute(0, 2, 1)[..., None]
        s = (q * 0.125) @ k.transpose(-1, -2) + g * bias[None]
        return (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B * T, d)


@pytest.mark.parametrize("large", [False, True])
def test_wavlm_orchestration_matches_the_oracle_with_a_cpu_backend(large):
    """mertools_b200.extract.wavlm.WavLmNet (fused q|k|v, bucketed relative position bias built on the host, per-layer
    gate, post-LN base / pre-LN large layer order, hidden-state tuple) over a torch backend, against the oracle's
    WavLM restatement (itself pinned to HF WavLMModel in tests/test_oracle.py)."""
    from mertools_b200.extract.wavlm import WavLmNet, relative_buckets
    assert np.array_equal(relative_buckets(300), E.wavlm_relative_buckets(300).numpy())
    layers, heads = 4, 16 if large else 12
    sd = S.hubert_state_dict(seed=6, layers=layers, wavlm=True, large=large)
    x = torch.randn(2, 8000, generator=torch.Generator().manual_seed(5))
    ref = E.hubert_hidden_states({k: torch.from_numpy(v) for k, v in sd.items()}, x, layers=layers, heads=heads)
    B, T, D = ref[0].shape
    net = WavLmNet(sd, _TorchWavLmOps())
    assert (net.heads, net.stable, len(net.layers)) == (heads, large, layers)
    got = net.hidden_states(ref[0].reshape(B * T, D), B, T)
    assert len(got) == len(ref) == layers + 1
    for a, b in zip(got, ref):
        assert float((a.reshape(B, T, D) - b).abs().max() / b.abs().max()) < 2e-5


def test_data2vec_vision_oracle_is_pinned_to_hf_and_the_orchestration_reproduces_it():
    """extract_vision_huggingface.py:124-133 (data2vec-vision-base-ft1k = the BEiT graph).  (1) oracle restatement vs HF
    Data2VecVisionModel on a synthetic checkpoint that strict-loads (relative position bias on); (2) BeitNet (fused
    q|k|v with the zero key bias, per-layer bias tables gathered on the host, folded LayerScale) over a torch backend."""
    transformers = pytest.importorskip("transformers")
    from mertools_b200.extract.data2vec_vision import BeitNet, relative_position_index
    assert np.array_equal(relative_position_index(14), E.beit_relative_position_index(14).numpy())
    sd = S.data2vec_vision_state_dict(seed=19, layers=2)
    model = transformers.Data2VecVisionModel(
        transformers.Data2VecVisionConfig(num_hidden_layers=2, use_relative_position_bias=True), add_pooling_layer=False).eval()
    model.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    frames = np.random.default_rng(8).integers(0, 256, (2, 112, 112, 3), dtype=np.uint8)
    x = P.vit_preprocess(frames)
    with torch.no_grad():
        ref = model(x, output_hidden_states=True).hidden_states
    got = E.data2vec_vision_hidden_states(sd, x)
    assert len(got) == len(ref) == 3
    for a, b in zip(got, ref):
        assert float((a - b).abs().max() / b.abs().max()) < 1e-5
    fra = P.visual_clip_features(sd, frames, feature_level="FRAME")
    np.testing.assert_allclose(fra, ref[-1].sum(dim=1).numpy(), rtol=0, atol=2e-5 * float(ref[-1].sum(dim=1).abs().max()))
    net = BeitNet(sd, _TorchWavLmOps())
    assert (net.heads, net.tokens, len(net.layers)) == (12, 197, 2)
    out = net.last_hidden(ref[0].reshape(2 * 197, 768), 2).reshape(2, 197, 768)
    assert float((out - ref[-1]).abs().max() / ref[-1].abs().max()) < 1e-5
    # the other two configurations of the HF class: one table shared by all layers, and no relative bias at all
    shared = {k: v for k, v in sd.items() if "relative_position_bias" not in k}
    shared["encoder.relative_position_bias.relative_position_bias_table"] = \
        sd["encoder.layer.0.attention.attention.relative_position_bias.relative_position_bias_table"]
    plain = {k: v for k, v in shared.items() if "relative_position" not in k}
    for d, kw in ((shared, dict(use_shared_relative_position_bias=True)), (plain, {})):
        model = transformers.Data2VecVisionModel(transformers.Data2VecVisionConfig(num_hidden_layers=2, **kw),
                                                 add_pooling_layer=False).eval()
        model.load_state_dict({k: torch.from_numpy(v) for k, v in d.items()}, strict=True)
        with torch.no_grad():
            r = model(x[:1], output_hidden_states=True).hidden_states
        o = E.data2vec_vision_hidden_states(d, x[:1])[-1]
        assert float((o - r[-1]).abs().max() / r[-1].abs().max()) < 1e-5
        o = BeitNet(d, _TorchWavLmOps()).last_hidden(r[0].reshape(197, 768), 1).reshape(1, 197, 768)
        assert float((o - r[-1]).abs().max() / r[-1].abs().max()) < 1e-5


def test_host_orchestrated_encoder_constructors_run_with_the_device_layer_stubbed(monkeypatch):
    """The WavLM / data2vec-vision / VideoMAE encoder classes (checkpoint inspection, weight folding, the embed-only
    model struct) constructed on CPU: device ops replaced by the torch backends of the orchestration tests."""
    from mertools_b200 import _lib
    from mertools_b200 import weights as Wt
    from mertools_b200.extract import data2vec_vision as DV
    from mertools_b200.extract import videomae as VM
    from mertools_b200.extract import wavlm as WL
    monkeypatch.setattr(_lib, "check", lambda rc: None)
    monkeypatch.setattr(_lib, "round_tf32_", lambda t: t)
    monkeypatch.setattr(_lib, "split_bf16", lambda t: t.clone())
    monkeypatch.setattr(Wt, "_dev", lambda x, device: (torch.from_numpy(np.ascontiguousarray(x)) if isinstance(x, np.ndarray)
                                                        else x).detach().to(dtype=torch.float32).contiguous())

    def torch_ops(cls):
        def make(device):
            ops = cls()
            ops.device = torch.device("cpu")
            return ops
        return make
    from mertools_b200.extract import dinov2_giant as DG
    monkeypatch.setattr(DG, "_cuda_ops", torch_ops(_TorchWavLmOps))
    monkeypatch.setattr(WL, "_cuda_ops", torch_ops(_TorchWavLmOps))
    monkeypatch.setattr(VM, "_cuda_ops", torch_ops(_TorchVideoMaeOps))
    w = WL.WavLmEncoder(S.hubert_state_dict(layers=4, wavlm=True, large=True))
    assert (w.hidden, w.n_layers, w.net.stable, w.net.heads, w.front.model.stable_layer_norm) == (1024, 4, True, 16, 1)
    d = DV.Data2VecVisionEncoder(S.data2vec_vision_state_dict(layers=2))
    m = d.embed.model
    assert (d.hidden, d.tokens, m.variant, m.kpad, m.patch, m.image, m.n_layers, bool(m.pre_ln_g)) == (768, 197, 2, 768, 16, 224, 0, False)
    assert len(d.net.layers) == 2 and tuple(d.net.layers[0]["bias"].shape) == (12, 197, 197)
    gi = DG.Dinov2GiantEncoder(S.dinov2_state_dict(layers=1, hidden=1536, swiglu=True))
    m = gi.embed.model
    assert (gi.hidden, gi.tokens, gi.net.heads, m.variant, m.kpad, m.patch, m.heads) == (1536, 257, 24, 2, 608, 14, 24)
    assert tuple(gi.net.layers[0]["w_in"].shape) == (8192, 1536) and tuple(gi.net.layers[0]["w_out"].shape) == (1536, 4096)
    v = VM.VideoMaeExtractor(S.videomae_state_dict(layers=1))
    assert (v.net.d, v.net.heads, len(v.net.layers)) == (768, 12, 1)


def test_dinov2_swiglu_oracle_is_pinned_to_hf_and_the_orchestration_reproduces_it():
    """dinov2-giant's graph (Dinov2Model with use_swiglu_ffn) at a small width: oracle vs HF; Dinov2SwigluNet (fused
    q|k|v, folded LayerScale, silu(x1) * x2 of the fused input projection) over a torch backend vs HF."""
    transformers = pytest.importorskip("transformers")
    from mertools_b200.encoders import dinov2_embedding_rows
    from mertools_b200.extract.dinov2_giant import Dinov2SwigluNet
    sd = S.dinov2_state_dict(seed=21, layers=2, hidden=384, swiglu=True)
    cfg = transformers.Dinov2Config(hidden_size=384, num_hidden_layers=2, num_attention_heads=6, image_size=518, patch_size=14,
                                    use_swiglu_ffn=True)
    model = transformers.Dinov2Model(cfg).eval()
    model.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    x = torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        ref = model(x, output_hidden_states=True).hidden_states
    got = E.dinov2_hidden_states(sd, x, heads=6)
    for a, b in zip(got, ref):
        assert float((a - b).abs().max() / b.abs().max()) < 1e-5
    # the embedding rows the device patch embedder is given reproduce hidden_states[0]
    pw, cls, pos = dinov2_embedding_rows(sd, 224)
    patches = torch.nn.functional.conv2d(x, torch.from_numpy(pw), None, stride=14).flatten(2).transpose(1, 2)
    h0 = torch.cat([torch.from_numpy(cls + pos[0]).expand(2, 1, -1), patches + torch.from_numpy(pos[1:])], dim=1)
    assert float((h0 - ref[0]).abs().max() / ref[0].abs().max()) < 1e-5
    net = Dinov2SwigluNet(sd, _TorchWavLmOps())
    assert (net.heads, len(net.layers)) == (6, 2)
    out = net.last_hidden(h0.reshape(2 * 257, 384), 2, 257).reshape(2, 257, 384)
    assert float((out - ref[-1]).abs().max() / ref[-1].abs().max()) < 1e-5
