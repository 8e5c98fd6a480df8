"""Stand-alone timing of the attention kernels at the bench shapes (CUDA events).

fp16 operands (q | k rows + V^T), the kernels of the fp16 stacks, timed alternately in the same process:
  short : attention_short.cu, one CTA per (sequence, head), rows of <= 249 tokens (MER_ATT_SHORT=1)
  tile  : the 64 x 64-tile kernel of attention_f16.cu (MER_ATT_SHORT=0)
at ViT 2,048 x 197 tokens x 12 heads, HuBERT 256 x 249 x 12 and BERT 256 ragged rows of <= 32 tokens x 12.
Per shape and kernel: median ms over the rounds, algorithmic TFLOP/s (4 s^2 64 flop per (sequence, head)) and GB/s
on compulsory bytes (q, k and V^T read once, ctx written once: 4 x 128 bytes per token and head).  The first line
names the card and its power limit.  --with-long adds the long-row and TF32-operand kernels (one timing each)."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mertools_b200 import _lib as L  # noqa: E402


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        info["nvidia_smi"] = q
    except (OSError, subprocess.SubprocessError) as e:
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def operands(lens, heads, dtype=torch.float16, seed=3):
    dev = torch.device("cuda:0")
    tokens = sum(lens)
    g = torch.Generator(device=dev).manual_seed(seed)
    qkv = (torch.randn(tokens, 3 * heads * 64, generator=g, device=dev) * 1.5).to(dtype)
    if dtype == torch.float32:
        L.round_tf32_(qkv)
    align = 8 if dtype == torch.float16 else 4
    vt = torch.zeros(heads * 64, (tokens + align - 1) // align * align, dtype=dtype, device=dev)
    vt[:, :tokens] = qkv[:, 2 * heads * 64:].T
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0).tolist()), dtype=torch.int32, device=dev)
    ctx = torch.empty(tokens, heads * 64, dtype=dtype, device=dev)
    return qkv, vt, cu, ctx


def time_launches(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def f16_ab(name, lens, heads, iters, rounds):
    qkv, vt, cu, ctx = operands(lens, heads)
    S = max(lens)
    arms = {"short": "1", "tile": "0"}  # forced either way, whatever the default for the shape
    run = lambda: L.attention(qkv, ctx, cu, S, heads, vt=vt)  # noqa: E731
    for v in arms.values():  # warm-up: module load, one-time attributes
        os.environ["MER_ATT_SHORT"] = v
        for _ in range(3):
            run()
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, v in arms.items():
            os.environ["MER_ATT_SHORT"] = v
            ms[k].append(time_launches(run, iters))
    os.environ.pop("MER_ATT_SHORT", None)
    flops = 4.0 * 64 * heads * sum(s * s for s in lens)
    nbytes = 4.0 * 128 * heads * sum(lens)
    out = []
    for k in arms:
        m = statistics.median(ms[k])
        out.append(dict(shape=name, kernel=k, n_seq=len(lens), max_len=S, tokens=sum(lens), heads=heads,
                        ms=round(m, 4), ms_min=round(min(ms[k]), 4), ms_max=round(max(ms[k]), 4),
                        tflops=round(flops / m / 1e9, 1), gbs=round(nbytes / m / 1e6, 1)))
    out.append(dict(shape=name, ratio_short_over_tile=round(statistics.median(ms["short"]) /
                                                           statistics.median(ms["tile"]), 3)))
    return out


def single(name, lens, heads, dtype, iters, **kw):
    qkv, vt, cu, ctx = operands(lens, heads, dtype)
    if kw.pop("no_vt", False):
        vt = None
    run = lambda: L.attention(qkv, ctx, cu, max(lens), heads, vt=vt, **kw)  # noqa: E731
    for _ in range(2):
        run()
    torch.cuda.synchronize()
    m = time_launches(run, iters)
    return dict(shape=name, n_seq=len(lens), max_len=max(lens), heads=heads, ms=round(m, 4),
                tflops=round(4.0 * 64 * heads * sum(s * s for s in lens) / m / 1e9, 1))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20, help="launches per timing")
    ap.add_argument("--rounds", type=int, default=5, help="alternating timings per kernel")
    ap.add_argument("--with-long", action="store_true", help="also time the long-row and TF32-operand kernels")
    a = ap.parse_args()
    print(json.dumps(dict(card=card())), flush=True)
    g = torch.Generator().manual_seed(5)
    bert = torch.randint(8, 33, (256,), generator=g).tolist()  # sentences of 8 .. 32 tokens
    for name, lens in (("vit", [197] * 2048), ("hubert", [249] * 256), ("bert", bert)):
        for r in f16_ab(name, lens, 12, a.iters, a.rounds):
            print(json.dumps(r), flush=True)
    if a.with_long:
        # fp16 V^T operands of long rows (10 s audio, 7 s, CLIP L/14) on the tile kernel; TF32 operands <= 253 tokens
        for n, S, heads in ((256, 499, 12), (256, 349, 12), (512, 257, 16)):
            print(json.dumps(single(f"f16_long_{S}", [S] * n, heads, torch.float16, a.iters)), flush=True)
        print(json.dumps(single("tf32_vt_249", [249] * 256, 12, torch.float32, a.iters, round_out=True)), flush=True)
        print(json.dumps(single("tf32_legacy_499", [499] * 256, 12, torch.float32, max(2, a.iters // 4),
                                round_out=True, no_vt=True)), flush=True)
