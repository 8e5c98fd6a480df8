"""Stand-alone timing of gemm_kernel's two epilogues at the bench shapes (CUDA events).

The register epilogue (MER_GEMM_EPI_TMA=0: bias / activation / residual applied in the consumer warpgroups' registers
and stored straight to global memory) against the default, which stages each 64-row sub-tile of an output without
residual or activation (qkv below) in shared memory and stores it with TMA; the residual and activation forms (proj,
fc1) keep the register epilogue by default and are timed to show that they are unchanged.  The two arms alternate in
the same process; each result line names the epilogue that ran ("path").

Shapes (fp16 operands, MER_GEMM_F16), each timed at K = 768, 1536 and 3072 so that a straight line through
(K, ms) gives the fixed cost at K = 0 -- what the epilogue and the pipeline fill add per launch, whatever K is:
  qkv     ViT QKV      N 2304, fp16 out, V^T side output of columns >= 1536
  proj    ViT out-proj N 768,  fp32 out + in-place residual   (FC2 at K = 3072)
  fc1     ViT FC1      N 3072, erf-GELU, fp16 out
at M = 2,048 frames x 197 tokens = 403,456 rows, plus the HuBERT / BERT layers (f16_small class: fewer than 2^17 rows)
and a BF16X3 feature projection.  Per shape and arm: median ms, TFLOP/s (2 M N K), and GB/s of compulsory bytes (A, W
and the output once, the residual once).  The first line names the card and its power limit."""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mertools_b200 import _lib as L  # noqa: E402
from scripts.bench_attention import card, time_launches  # noqa: E402

ARMS = {"reg": "0", "default": "1"}


def problem(form, M, K, mode, seed):
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(seed)
    N = {"qkv": 2304, "proj": 768, "fc1": 3072}[form]
    if mode == L.MER_GEMM_F16:
        a = (torch.randn(M, K, generator=g, device=dev) * 0.5).half()
        w = (torch.randn(N, K, generator=g, device=dev) * K ** -0.5).half()
    else:  # BF16X3: split rows
        a = L.split_bf16(torch.randn(M, K, generator=g, device=dev))
        w = L.split_bf16(torch.randn(N, K, generator=g, device=dev) * K ** -0.5)
    bias = torch.randn(N, generator=g, device=dev)
    kw = dict(bias=bias, mode=mode)
    out_bytes = 4
    if form == "qkv":
        out = torch.empty(M, N, dtype=torch.float16, device=dev)
        vt = torch.empty(N - 1536, (M + 7) // 8 * 8, dtype=torch.float16, device=dev)
        kw.update(f16_out=True, vt=vt, vt_col0=1536)
        out_bytes = 2
    elif form == "proj":
        out = torch.randn(M, N, generator=g, device=dev)
        kw.update(res=out)
    else:
        out = torch.empty(M, N, dtype=torch.float16, device=dev)
        kw.update(gelu=True, f16_out=True)
        out_bytes = 2
    nbytes = a.numel() * a.element_size() + w.numel() * w.element_size() + M * N * out_bytes
    if form == "proj":
        nbytes += M * N * 4
    return (lambda: L.gemm(a, w, out, **kw)), 2.0 * M * N * K, nbytes


def ab(name, form, M, K, iters, rounds, mode=L.MER_GEMM_F16):
    run, flops, nbytes = problem(form, M, K, mode, seed=K + M)
    count = L.gemm_epilogue_launches
    paths = {}
    for k, v in ARMS.items():  # warm-up: module load, one-time attributes; which epilogue each arm runs
        os.environ["MER_GEMM_EPI_TMA"] = v
        c0 = count()
        for _ in range(3):
            run()
        c1 = count()
        paths[k] = "tma" if c1[1] > c0[1] else "reg"
    torch.cuda.synchronize()
    ms = {k: [] for k in ARMS}
    for _ in range(rounds):
        for k, v in ARMS.items():
            os.environ["MER_GEMM_EPI_TMA"] = v
            ms[k].append(time_launches(run, iters))
    os.environ.pop("MER_GEMM_EPI_TMA", None)
    rows = []
    for k in ARMS:
        m = statistics.median(ms[k])
        rows.append(dict(shape=name, form=form, arm=k, path=paths[k], M=M, K=K, ms=round(m, 4),
                         ms_min=round(min(ms[k]), 4), ms_max=round(max(ms[k]), 4),
                         tflops=round(flops / m / 1e9, 1), gbs=round(nbytes / m / 1e6, 1)))
    rows.append(dict(shape=name, ratio_default_over_reg=round(statistics.median(ms["default"]) /
                                                              statistics.median(ms["reg"]), 4)))
    return rows


def intercept(points):
    """Least-squares line through [(K, ms)] -> (ms at K = 0, ms per 1000 K)."""
    n = len(points)
    mk = sum(k for k, _ in points) / n
    mt = sum(t for _, t in points) / n
    slope = sum((k - mk) * (t - mt) for k, t in points) / sum((k - mk) ** 2 for k, _ in points)
    return mt - slope * mk, slope * 1000


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50, help="launches per timing (after warm-up)")
    ap.add_argument("--rounds", type=int, default=3, help="alternating timings per arm")
    ap.add_argument("--M", type=int, default=2048 * 197)
    a = ap.parse_args()
    print(json.dumps(dict(card=card())), flush=True)
    sweep = {}
    for form in ("qkv", "proj", "fc1"):
        for K in (768, 1536, 3072):
            name = {("proj", 3072): "vit_fc2", ("qkv", 768): "vit_qkv", ("proj", 768): "vit_out_proj",
                    ("fc1", 768): "vit_fc1"}.get((form, K), f"{form}_K{K}")
            for r in ab(name, form, a.M, K, a.iters, a.rounds):
                print(json.dumps(r), flush=True)
                if "arm" in r:
                    sweep.setdefault((form, r["arm"]), []).append((K, r["ms"]))
    for (form, arm), pts in sweep.items():
        t0, per_k = intercept(pts)
        at768 = dict(pts)[768]
        print(json.dumps(dict(fixed_cost=form, arm=arm, ms_at_K0=round(t0, 4), ms_per_1000K=round(per_k, 4),
                              share_of_K768=round(t0 / at768, 3))), flush=True)
    # the other classes must not regress: HuBERT (256 clips x 249 frames) and BERT (256 x ~20 tokens) layers in F16,
    # and the BF16X3 class at the HuBERT feature projection's rows
    for tag, M in (("hubert", 256 * 249), ("bert", 256 * 20)):
        for form, K in (("qkv", 768), ("proj", 768), ("fc1", 768), ("proj", 3072)):
            for r in ab(f"{tag}_{form}_K{K}", form, M, K, max(a.iters, 200), a.rounds):
                print(json.dumps(r), flush=True)
    for r in ab("bf16x3_proj_K512", "proj", 256 * 249, 512, max(a.iters, 200), a.rounds, mode=L.MER_GEMM_BF16X3):
        print(json.dumps(r), flush=True)
