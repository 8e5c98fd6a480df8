"""Golden fixture of the visual extractor's EVACLIP_VIT branch: the UNMODIFIED
feature_extraction/visual/extract_vision_huggingface.py, run as ``__main__`` with ``--gpu -1`` and the stand-ins of
timm_eva_shim.py registered, on synthetic eva02 checkpoints and synthetic face ``.npy``s.

    python tests/golden/make_golden_eva02.py --reference <checkout of MERTools>/MER2024

The model keeps the tag's widths with 2 blocks (timm_eva_shim.DEPTH).  Checkpoints: synthetic.eva02_state_dict(seed,
layers=2, scale) for each case of CASES.  Faces: _eva02_ref.synth_faces(n, h, w, seed=n) for each (n, h, w) of CLIPS.

Stored (tests/golden/eva02_golden.npz):  feat/<case>/<level>/<vid>  the saved .npy (float64 in the reference; stored
as float32).
"""
import argparse
import glob
import os
import runpy
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import _eva02_ref as R  # noqa: E402
import timm_eva_shim  # noqa: E402
from mertools_b200 import synthetic as S  # noqa: E402

BLOCKS = 2
CASES = {"default": (27, 1.0), "x5": (28, 5.0)}   # case -> (checkpoint seed, matrix scale)
# vid -> (frames, h, w): 33 frames cross the reference's batch of 32; 137 x 112 resizes to 303 x 248, whose row offset
# int(round(79 / 2.0)) = 40 rounds half-even upward (the floor rule gives 39)
CLIPS = {"v01": (1, 112, 112), "v05": (5, 112, 112), "v33": (33, 112, 112), "r03": (3, 137, 112)}


def faces(vid):
    n, h, w = CLIPS[vid]
    return R.synth_faces(n, h, w, seed=n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", required=True, help="the MER2024 directory of a MERTools checkout")
    ap.add_argument("--out", default=os.path.join(HERE, "eva02_golden.npz"))
    a = ap.parse_args()
    timm_eva_shim.install()
    timm_eva_shim.DEPTH = BLOCKS
    cfg = types.ModuleType("config")
    sys.modules["config"] = cfg
    script = os.path.join(a.reference, "feature_extraction", "visual", "extract_vision_huggingface.py")
    from safetensors.numpy import save_file

    store = {}
    with tempfile.TemporaryDirectory() as tmp:
        face_dir = os.path.join(tmp, "face")
        for vid in CLIPS:
            os.makedirs(os.path.join(face_dir, vid))
            np.save(os.path.join(face_dir, vid, f"{vid}.npy"), faces(vid))
        for case, (seed, scale) in CASES.items():
            models = os.path.join(tmp, f"models-{case}")
            ck = os.path.join(models, "timm", timm_eva_shim.MODEL)
            os.makedirs(ck)
            save_file(S.eva02_state_dict(seed, layers=BLOCKS, scale=scale), os.path.join(ck, "model.safetensors"))
            feats = os.path.join(tmp, f"feat-{case}")
            cfg.PATH_TO_RAW_FACE, cfg.PATH_TO_FEATURES = {"MER2023": face_dir}, {"MER2023": feats}
            cfg.PATH_TO_PRETRAINED_MODELS = models
            for level in ("UTTERANCE", "FRAME"):
                sys.argv = [script, "--dataset", "MER2023", "--model_name", timm_eva_shim.MODEL, "--feature_level",
                            level, "--gpu", "-1"]
                runpy.run_path(script, run_name="__main__")
            for f in glob.glob(os.path.join(feats, "*", "*.npy")):
                level = "UTTERANCE" if os.path.basename(os.path.dirname(f)).endswith("UTT") else "FRAME"
                assert os.path.basename(os.path.dirname(f)) == f"eva02_base_patch14_224-{level[:3]}", f
                store[f"feat/{case}/{level}/{os.path.basename(f)[:-4]}"] = np.load(f).astype(np.float32)
    np.savez_compressed(a.out, **store)
    print(f"wrote {a.out}: {len(store)} arrays")


if __name__ == "__main__":
    main()
