"""Frames/s of the EVA02 branch of the visual extractor (Eva02Encoder, eva02_base_patch14_224, 12 blocks) against the
reference's way of running it: the timm stand-in (tests/golden/timm_eva_shim.py, what timm's Eva computes) in torch
eager fp32 on the same GPU, fed by the host path of extract_vision_huggingface.py:202-210 (cv2 BGR -> RGB -> PIL ->
timm eval transform per frame, batches of 32); and against the same stand-in fed device tensors already transformed
(the model alone).

Workload: OpenFace-sized 112 x 112 face clips (synthetic frames and weights), 32 clips of 30 .. 150 frames, FRAME
features.  Every arm runs --repeats times, alternating; the JSON line reports the best and the spread.  The linears'
TFLOP/s come from the shapes (2 M N K per GEMM, M = frames x 257).  A separate torch.profiler run of our arm gives the
kernel time shares.  The card's name and power limit are read in the same run.

    python scripts/bench_eva02.py [--clips 32] [--repeats 3] [--out results.json]
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
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import _eva02_ref as R  # noqa: E402
import timm_eva_shim as T  # noqa: E402
from mertools_b200 import synthetic as S  # noqa: E402
from mertools_b200.extract import visual as V  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def linear_flops(frames, D=768, F=2048):
    M = frames * 257
    return 2.0 * M * 12 * (D * 3 * D + D * D + D * 2 * F + F * D)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=32)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    name = card()
    sd = S.eva02_state_dict(27, layers=12)
    ext = V.VisualExtractor(sd, device=dev)
    model = T.Eva(depth=12)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    model = model.to(dev).eval()
    tf = T.create_transform(**T.resolve_model_data_config(model))
    lengths = np.random.default_rng(0).integers(30, 151, a.clips)
    clips = [R.synth_faces(int(n), seed=i) for i, n in enumerate(lengths)]
    frames = int(lengths.sum())

    def ours():
        out = ext.extract_clips(clips, "FRAME")
        torch.cuda.synchronize()
        return out

    def reference():   # host transforms per frame, batches of 32, eager fp32
        out = []
        with torch.no_grad():
            for c in clips:
                x = R.pixels_from_frames(c, tf).to(dev)
                out.append(torch.cat([model(x[s:s + 32]) for s in range(0, len(x), 32)]).cpu().numpy())
        return out

    pix = [R.pixels_from_frames(c, tf).to(dev) for c in clips]

    def model_only():
        with torch.no_grad():
            out = [torch.cat([model(x[s:s + 32]) for s in range(0, len(x), 32)]) for x in pix]
        torch.cuda.synchronize()
        return out

    ours(), model_only()                      # warm-up: module load, workspace, cuDNN / cuBLAS choices
    times = {"ours": [], "reference": [], "model_only": []}
    res = {}
    for _ in range(a.repeats):
        for k, f in (("ours", ours), ("reference", reference), ("model_only", model_only)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res[k] = f()
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
    diff = max(float(np.abs(o - b).max() / np.abs(b).max()) for o, b in zip(res["ours"], res["reference"]))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ours()
    ev = [e for e in prof.key_averages() if e.self_device_time_total > 0]
    tot = sum(e.self_device_time_total for e in ev) or 1.0
    shares = sorted(((e.key[:60], round(e.self_device_time_total / tot, 3)) for e in ev), key=lambda x: -x[1])[:10]
    t = {k: min(v) for k, v in times.items()}
    line = dict(model="eva02_base_patch14_224", blocks=12, clips=a.clips, frames=frames, frame_size="112x112",
                ours_frames_per_s=round(frames / t["ours"], 1),
                reference_frames_per_s=round(frames / t["reference"], 1),
                model_only_frames_per_s=round(frames / t["model_only"], 1),
                speedup_vs_reference=round(t["reference"] / t["ours"], 2),
                speedup_vs_model_only=round(t["model_only"] / t["ours"], 2),
                ours_linear_tflops_end_to_end=round(linear_flops(frames) / t["ours"] / 1e12, 1),
                spread={k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
                kernel_time_shares=shares, max_abs_over_max_ref=diff, card=name)
    print(json.dumps(line), flush=True)
    if a.out:
        if os.path.dirname(a.out):
            os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    main()
