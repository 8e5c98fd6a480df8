"""Throughput of MER2023's audio extractor (extract/audio_mer2023.py) on whole clips of mixed length.

Workload: 64 seeded clips of 1 .. 40 s (uniform), a seeded HuBERT-base checkpoint (12 layers), UTTERANCE readout
hidden_states[-1].  Arms, in one process on one GPU:
  ours  Mer2023AudioExtractor.extract_waves over the whole set (ragged launches, default operand formats)
  hf    the reference's loop: batch-1 fp32 HF HubertModel(output_hidden_states=True), hidden_states[-1].mean(1), per
        clip, on the same GPU (the first 16 clips: it is the slow arm)
Each arm is warmed up once and timed --repeats times (host clock around work that ends in a device synchronise);
the spread is reported.  Then the attention share at 1,249 frames: torch.profiler over one launch of 8 clips of 25 s,
kernel time of the attention kernels over all kernel time.  Prints one JSON line (GPU name and power limit included).
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
from mertools_b200 import synthetic as S  # noqa: E402
from mertools_b200.extract.audio_mer2023 import LAST, Mer2023AudioExtractor  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, check=True).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except (OSError, subprocess.CalledProcessError, IndexError, ValueError):
        return torch.cuda.get_device_name(), "unknown"


def timed(fn, repeats):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t0)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--hf-clips", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", type=str, default=None, help="also write the JSON result here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    rng = np.random.default_rng(5)
    secs = rng.uniform(1.0, 40.0, args.clips)
    waves = [S.synth_waves(1, int(s * 16000), seed=1000 + i)[0].astype(np.float64) / 32768.0 for i, s in enumerate(secs)]
    sd = S.hubert_state_dict(seed=1, layers=12)
    ext = Mer2023AudioExtractor(sd, layer_ids=LAST, device="cuda")
    t_ours = timed(lambda: ext.extract_waves(waves, "UTTERANCE"), args.repeats)

    from transformers import HubertConfig, HubertModel
    from oracle import pipeline as P
    hf = HubertModel(HubertConfig(num_hidden_layers=12)).eval()
    hf.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=False)
    hf = hf.cuda()
    hf_in = [torch.from_numpy(P.wav2vec2_normalize(w))[None].cuda() for w in waves[:args.hf_clips]]

    def run_hf():
        with torch.no_grad():
            return [hf(x, output_hidden_states=True).hidden_states[-1][0].mean(0).cpu() for x in hf_in]
    t_hf = timed(run_hf, args.repeats)

    # attention share at 1,249 frames (25 s clips)
    from torch.profiler import ProfilerActivity, profile
    long_waves = [S.synth_waves(1, 400000, seed=2000 + i)[0].astype(np.float64) / 32768.0 for i in range(8)]
    ext.extract_waves(long_waves, "UTTERANCE")
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ext.extract_waves(long_waves, "UTTERANCE")
        torch.cuda.synchronize()
    att = tot = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if e.device_type is not None and str(e.device_type).endswith("CUDA") and t > 0:
            tot += t
            if "attention" in e.key:
                att += t
    name, power = gpu_info()
    res = dict(gpu=name, power_limit=power, clips=args.clips, seconds_min_max=[float(secs.min()), float(secs.max())],
               ours_clips_per_s=[args.clips / t for t in t_ours], hf_batch1_clips_per_s=[args.hf_clips / t for t in t_hf],
               attention_share_at_1249_frames=att / tot if tot else None)
    res["speedup_median"] = float(np.median(res["ours_clips_per_s"]) / np.median(res["hf_batch1_clips_per_s"]))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
