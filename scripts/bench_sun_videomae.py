"""Videos/s of the MER2024 VideoMAE face-clip extractor (mertools_b200/extract/sun_videomae.py) against the reference's
way of running the same model: every one of the 4 views per frame id, PIL resize + ClipToTensor + Normalize on the host,
the model in torch under torch.autocast('cuda', float16) in batches of 64 (extract_sun_videomae.py, final_test), here
the CPU restatement's torch module (tests/_sun_videomae_ref.py) moved to the device.

Workload: MER2023-like face tracks, 30 .. 150 frames of 112 x 112, full-depth models with synthetic weights, at
UTTERANCE and FRAME level, S = 160 (vit_base_patch16_160) and 224 (vit_base_patch16_224).  Prints one JSON line per
(model, level) with videos/s and view-forwards/s of both arms and the largest |difference| between their outputs, plus
the card's name and power limit read in the same run.

    python scripts/bench_sun_videomae.py [--utt-videos 32] [--frame-videos 3] [--repeats 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import _sun_videomae_ref as R  # noqa: E402
from mertools_b200.extract import sun_videomae as SV  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def baseline(params, videos, model, level, dev, batch=64):
    """The reference's loop: all items of every video, host preprocessing, fp16 autocast forward, float64 readout."""
    S, _, heads = R.SHAPES[model]
    out, forwards = [], 0
    for v in videos:
        rs = R.resize(v, S)
        items = R.views(len(v), level)
        feats = []
        for s in range(0, len(items), batch):
            x = torch.stack([R.clip_tensor(rs, r) for _, r in items[s:s + batch]]).to(dev, non_blocking=True)
            with torch.no_grad(), torch.autocast("cuda", torch.float16):
                feats.append(R.view_features(params, x, heads).float().cpu().numpy())
            forwards += x.shape[0]
        out.append(R.final_test(items, np.concatenate(feats), level))
    return out, forwards


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utt-videos", type=int, default=32)
    ap.add_argument("--frame-videos", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=2)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    name = card()
    for model in ("vit_base_patch16_160", "vit_base_patch16_224"):
        S, dim, _ = R.SHAPES[model]
        ck = R.synth_checkpoint(dim, 12, seed=1)
        params = {k: v.to(dev) for k, v in R.model_params(ck).items()}
        ext = SV.SunVideoMae(SV.model_state_dict(ck, model), model, device=dev)
        for level, nv in (("UTTERANCE", a.utt_videos), ("FRAME", a.frame_videos)):
            lengths = rng.integers(30, 151, nv)
            videos = [R.synth_video(int(n), seed=int(i)) for i, n in enumerate(lengths)]
            ext.extract_videos(videos[:2], level)               # warm-up: module load, workspace
            baseline(params, videos[:1], model, level, dev)
            t_ours, t_base = [], []
            for _ in range(a.repeats):                           # alternate the arms
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                ours = ext.extract_videos(videos, level)
                torch.cuda.synchronize()
                t_ours.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                base, forwards = baseline(params, videos, model, level, dev)
                torch.cuda.synchronize()
                t_base.append(time.perf_counter() - t0)
            ours_fw = sum(len({r for _, r in SV.plan_views(len(v), level)}) for v in videos)
            diff = max(float(np.abs(o - b).max() / np.abs(b).max()) for o, b in zip(ours, base))
            to, tb = min(t_ours), min(t_base)
            print(json.dumps(dict(model=model, level=level, videos=nv, frames=int(lengths.sum()),
                                  ours_videos_per_s=round(nv / to, 2), ours_view_forwards_per_s=round(ours_fw / to, 1),
                                  base_videos_per_s=round(nv / tb, 2), base_view_forwards_per_s=round(forwards / tb, 1),
                                  ours_view_forwards=ours_fw, base_view_forwards=forwards,
                                  speedup=round(tb / to, 2), max_abs_over_max_ref=diff, card=name)), flush=True)


if __name__ == "__main__":
    main()
