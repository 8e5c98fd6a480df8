"""Golden fixture of MER2024's VideoMAE face-clip extractor: the UNMODIFIED driver
(feature_extraction/visual/extract_sun_videomae.py, ``main(get_args())``) and videomae package, run on CPU with the
stand-ins of timm_shim.py registered, on synthetic pretraining checkpoints and synthetic face videos.

    python tests/golden/make_golden_sun_videomae.py --reference <checkout of MERTools>/MER2024

The models keep their factories' widths (vit_base_patch16_160 / _224, vit_large_patch16_224) with fewer blocks: the
factories are called through a VisionTransformer whose ``depth`` is overridden, so that the CPU run stays short.  On
this CPU-only run ``torch.cuda.amp.autocast()`` is inactive, so every forward is plain fp32.

Stored (tests/golden/sun_videomae_golden.npz):
  feat/<case>/<level>/<n>   the saved .npy (float64 in the reference; stored as float32)
  idx/<level>/<n>           int16 [items, 16]: the source frame of every clip frame of every dataset item, decoded from
                            a video whose frame k is the constant k; fid/<level>/<n> the items' frame ids
  clip/<name>               fp32 dataset_test[i][0][:, :2, :32, :] (the first tubelet, first two patch rows) of the
                            items listed in CLIPS (image size, video length, level, item index)
"""
import argparse
import glob
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import _sun_videomae_ref as R  # noqa: E402
import timm_shim  # noqa: E402

LENGTHS = (1, 5, 12, 16, 17, 19, 40, 64, 65, 150)
NONSQUARE = {40: (120, 100)}   # n -> (h, w); every other video is 112 x 112
# case -> (model, blocks, checkpoint seed, {level: lengths})
CASES = {
    "base160": ("vit_base_patch16_160", 2, 11, {"UTTERANCE": LENGTHS, "FRAME": (1, 5, 12, 16, 17, 19, 40)}),
    "base224": ("vit_base_patch16_224", 2, 12, {"UTTERANCE": (1, 17, 65, 150), "FRAME": (5, 19)}),
    "large224": ("vit_large_patch16_224", 1, 13, {"UTTERANCE": (17, 65), "FRAME": (12,)}),
}
CLIPS = {"sq160": (160, 65, "UTTERANCE", 3), "ns224": (224, 40, "FRAME", 37), "wrap160": (160, 12, "FRAME", 10)}


def video(n):
    h, w = NONSQUARE.get(n, (112, 112))
    return R.synth_video(n, h, w, seed=100 + n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", required=True, help="the MER2024 directory of a MERTools checkout")
    ap.add_argument("--out", default=os.path.join(HERE, "sun_videomae_golden.npz"))
    a = ap.parse_args()
    timm_shim.install()
    cfg = types.ModuleType("config")
    sys.modules["config"] = cfg
    sys.path.insert(0, os.path.join(a.reference, "feature_extraction", "visual"))
    import videomae.modeling_finetune as mf
    from videomae.datasets import build_dataset

    import extract_sun_videomae as drv
    full = mf.VisionTransformer
    depth = {"n": None}
    mf.VisionTransformer = lambda **kw: full(**{**kw, "depth": depth["n"]})

    store = {}
    with tempfile.TemporaryDirectory() as tmp:
        face_dir = os.path.join(tmp, "face")
        for n in LENGTHS:
            os.makedirs(os.path.join(face_dir, f"v{n:03d}"))
            np.save(os.path.join(face_dir, f"v{n:03d}", f"v{n:03d}.npy"), video(n))
        for case, (model, blocks, seed, levels) in CASES.items():
            S, dim, _ = R.SHAPES[model]
            depth["n"] = blocks
            ck_dir = os.path.join(tmp, f"videomae-{case}")
            os.makedirs(ck_dir)
            ckpt = os.path.join(ck_dir, "checkpoint-99.pth")
            torch.save(R.synth_checkpoint(dim, blocks, seed), ckpt)
            for level, lengths in levels.items():
                sel = os.path.join(tmp, f"sel-{case}-{level}")
                os.makedirs(sel)
                for n in lengths:
                    os.symlink(os.path.join(face_dir, f"v{n:03d}"), os.path.join(sel, f"v{n:03d}"))
                feats = os.path.join(tmp, f"feat-{case}-{level}")
                cfg.PATH_TO_RAW_FACE, cfg.PATH_TO_FEATURES = {"MER2023": sel}, {"MER2023": feats}
                sys.argv = ["extract_sun_videomae.py", "--dataset", "MER2023", "--feature_level", level,
                            "--model", model, "--input_size", str(S), "--short_side_size", str(S),
                            "--finetune", ckpt, "--device", "cpu", "--num_workers", "0", "--no_pin_mem"]
                drv.main(drv.get_args())
                for f in glob.glob(os.path.join(feats, "*", "*.npy")):
                    n = int(os.path.basename(f)[1:4])
                    store[f"feat/{case}/{level}/{n}"] = np.load(f).astype(np.float32)

        # the dataset's index decisions, read back from index-coded videos
        for level in ("UTTERANCE", "FRAME"):
            for n in LENGTHS:
                coded = np.repeat(np.arange(n, dtype=np.uint8)[:, None, None, None], 3, axis=3)
                coded = np.ascontiguousarray(np.broadcast_to(coded, (n, 16, 16, 3)))
                p = os.path.join(tmp, f"coded-{level}-{n}.npy")
                np.save(p, coded)
                ns = argparse.Namespace(num_frames=16, sampling_rate=4, test_num_segment=2, test_num_crop=2,
                                        input_size=160, short_side_size=160, feature_level=level, debug=False)
                ds = build_dataset(ns, p)
                idx, fid = [], []
                for i in range(len(ds)):
                    x, f = ds[i]
                    v = x[0, :, 0, 0].double() * R.STD[0] + R.MEAN[0]
                    idx.append(np.rint(v.numpy() * 255).astype(np.int16))
                    fid.append(int(f))
                store[f"idx/{level}/{n}"] = np.stack(idx)
                store[f"fid/{level}/{n}"] = np.array(fid, np.int32)

        # a few transformed clips, bit for bit
        for name, (S, n, level, item) in CLIPS.items():
            ns = argparse.Namespace(num_frames=16, sampling_rate=4, test_num_segment=2, test_num_crop=2,
                                    input_size=S, short_side_size=S, feature_level=level, debug=False)
            ds = build_dataset(ns, os.path.join(face_dir, f"v{n:03d}", f"v{n:03d}.npy"))
            x, _ = ds[item]
            store[f"clip/{name}"] = x[:, :2, :32, :].numpy().copy()
    np.savez_compressed(a.out, **store)
    print(f"wrote {a.out}: {len(store)} arrays")


if __name__ == "__main__":
    main()
