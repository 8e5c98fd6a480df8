"""GPU probe: correctness + timing of the kernel-level entry points, with verbose diagnostics.

Run on the GPU box:  timeout 300 python scripts/gpu_probe.py [section ...]
Writes one JSON line per check to stdout (and gpurun_out/probe.jsonl).
"""
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mertools_b200 import _lib as L  # noqa: E402

OUT = None


def emit(**kw):
    line = json.dumps(kw)
    print(line, flush=True)
    if OUT:
        OUT.write(line + "\n")
        OUT.flush()


def tf32(x):
    i = x.contiguous().view(torch.int32)
    r = (i + 0xFFF + ((i >> 13) & 1)) & ~0x1FFF
    return r.view(torch.float32)


def time_cuda(fn, iters=20, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def gelu(x):
    return torch.nn.functional.gelu(x)


def check_gemm(name, M, N, K, bias=False, use_gelu=False, res=False, rnd=False, ints=False,
               force=0, cluster=0):
    g = torch.Generator(device="cuda").manual_seed(1)
    if ints:
        A = torch.randint(-3, 4, (M, K), device="cuda", generator=g).float()
        W = torch.randint(-3, 4, (N, K), device="cuda", generator=g).float()
    else:
        A = tf32(torch.randn(M, K, device="cuda", generator=g))
        W = tf32(torch.randn(N, K, device="cuda", generator=g) * 0.05)
    b = torch.randn(N, device="cuda", generator=g) if bias else None
    R = torch.randn(M, N, device="cuda", generator=g) if res else None
    out = torch.full((M, N), float("nan"), device="cuda")
    try:
        L.gemm_tf32(A, W, out, bias=b, res=R, gelu=use_gelu, round_out=rnd, force_block_n=force,
                    cluster=cluster)
        torch.cuda.synchronize()
    except Exception as e:  # noqa: BLE001
        emit(check=name, ok=False, error=str(e)[:500])
        return False
    ref = A.double() @ W.double().t()
    if bias:
        ref = ref + b.double()
    if use_gelu:
        ref = gelu(ref)
    if res:
        ref = ref + R.double()
    if rnd:
        ref = tf32(ref.float()).double()
    err = (out.double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    nan = int(torch.isnan(out).sum().item())
    ok = nan == 0 and err <= 2e-5 * max(scale, 1.0) * (8 if rnd else 1) + (1e-3 * scale if rnd else 0)
    info = dict(check=name, ok=bool(ok), M=M, N=N, K=K, max_err=err, ref_max=scale, nan=nan)
    if not ok:
        bad = ((out.double() - ref).abs() > 1e-3 * max(scale, 1.0)) | torch.isnan(out)
        rows = bad.any(1).nonzero().flatten()[:8].tolist()
        cols = bad.any(0).nonzero().flatten()[:8].tolist()
        info.update(bad_frac=bad.float().mean().item(), bad_rows=rows, bad_cols=cols,
                    sample_out=out[:2, :4].tolist(), sample_ref=ref[:2, :4].tolist())
    emit(**info)
    return ok


def sec_gemm():
    ok = True
    ok &= check_gemm("gemm_int_1tile_k32", 128, 128, 32, ints=True)
    ok &= check_gemm("gemm_int_1tile_k128", 128, 128, 128, ints=True)
    ok &= check_gemm("gemm_int_n256", 128, 256, 64, ints=True, force=256)
    ok &= check_gemm("gemm_tail_m300", 300, 256, 768)
    ok &= check_gemm("gemm_bias_gelu", 1000, 3072, 768, bias=True, use_gelu=True, rnd=True)
    ok &= check_gemm("gemm_bias_res", 1000, 768, 3072, bias=True, res=True)
    ok &= check_gemm("gemm_big_256", 20000, 2304, 768, bias=True, force=256)
    ok &= check_gemm("gemm_big_128", 20000, 768, 768, bias=True, force=128)
    # transposed side output (V^T of the QKV GEMM)
    g = torch.Generator(device="cuda").manual_seed(3)
    A = tf32(torch.randn(1000, 768, device="cuda", generator=g))
    W = tf32(torch.randn(2304, 768, device="cuda", generator=g) * 0.05)
    bq = torch.randn(2304, device="cuda", generator=g)
    out = torch.full((1000, 2304), float("nan"), device="cuda")
    vt = torch.full((768, 1000), float("nan"), device="cuda")
    L.gemm(A, W, out, bias=bq, round_out=True, vt=vt, vt_col0=1536)
    torch.cuda.synchronize()
    ref = tf32((A.double() @ W.double().t() + bq.double()).float())
    e1 = (out[:, :1536] - ref[:, :1536]).abs().max().item()
    e2 = (vt - ref[:, 1536:].t()).abs().max().item()
    good = e1 < 2e-2 and e2 < 2e-2 and bool(torch.isnan(out[:, 1536:]).all())
    emit(check="gemm_vt_side_output", ok=bool(good), err_qk=e1, err_vt=e2)
    ok &= good
    # CTA pairs with multicast weight tiles (odd and even numbers of row tiles, residual in place)
    ok &= check_gemm("gemm_pair_int", 256, 256, 64, ints=True, force=256, cluster=2)
    ok &= check_gemm("gemm_pair_odd_tiles", 128 * 5 + 7, 768, 768, bias=True, res=True, force=256, cluster=2)
    ok &= check_gemm("gemm_pair_big", 40000, 2304, 768, bias=True, rnd=True, cluster=2)
    ok &= check_gemm("gemm_pair_fc2", 40000, 768, 3072, bias=True, res=True, cluster=2)
    return ok


def sec_gemm_x3():
    """BF16X3 mode: split operands, 3 MMAs per K step, ~fp32 accuracy; also split outputs."""
    ok = True
    for (name, M, N, K, force) in [("x3_1tile", 128, 128, 64, 0), ("x3_tail", 300, 256, 768, 256),
                                   ("x3_fc1", 5000, 3072, 768, 0), ("x3_fc2", 5000, 768, 3072, 0)]:
        g = torch.Generator(device="cuda").manual_seed(7)
        A = torch.randn(M, K, device="cuda", generator=g)
        W = torch.randn(N, K, device="cuda", generator=g) * 0.05
        b = torch.randn(N, device="cuda", generator=g)
        As, Ws = L.split_bf16(A), L.split_bf16(W)
        rt = (L.unsplit_bf16(As) - A).abs().max().item() / A.abs().max().item()
        out = torch.full((M, N), float("nan"), device="cuda")
        L.gemm(As, Ws, out, bias=b, mode=L.MER_GEMM_BF16X3, force_block_n=force)
        outs = torch.full((M, N), float("nan"), device="cuda")
        L.gemm(As, Ws, outs, bias=b, gelu=True, split_out=True, mode=L.MER_GEMM_BF16X3, force_block_n=force)
        torch.cuda.synchronize()
        ref = A.double() @ W.double().t() + b.double()
        err = (out.double() - ref).abs().max().item() / ref.abs().max().item()
        refg = gelu(ref)
        errs = (L.unsplit_bf16(outs).double() - refg).abs().max().item() / refg.abs().max().item()
        good = err < 5e-5 and errs < 5e-5 and rt < 2e-5
        emit(check=name, ok=bool(good), M=M, N=N, K=K, rel_err=err, rel_err_split_out=errs, split_roundtrip=rt)
        ok &= good
    M, N, K = 100864, 3072, 768
    A = L.split_bf16(torch.randn(M, K, device="cuda"))
    W = L.split_bf16(torch.randn(N, K, device="cuda") * 0.02)
    b = torch.randn(N, device="cuda")
    out = torch.empty(M, N, device="cuda")
    for cl in (1, 2):
        ms = time_cuda(lambda: L.gemm(A, W, out, bias=b, gelu=True, split_out=True, mode=L.MER_GEMM_BF16X3,
                                      cluster=cl), iters=10)
        emit(perf=f"x3_fc1_cluster{cl}", M=M, N=N, K=K, ms=ms, tflops_useful=2.0 * M * N * K / ms / 1e9)
    return ok


def sec_gelu_ab():
    """A/B in one process: polynomial vs libdevice erf in the FC1 epilogue, interleaved repeats."""
    M, N, K = 403456, 3072, 768
    A = tf32(torch.randn(M, K, device="cuda"))
    W = tf32(torch.randn(N, K, device="cuda") * 0.02)
    b = torch.randn(N, device="cuda")
    out = torch.empty(M, N, device="cuda")
    for rep in range(3):
        r = {}
        for name, kw in (("poly", {}), ("libm", dict(gelu_libm=True)), ("nogelu", None)):
            if kw is None:
                fn = lambda: L.gemm(A, W, out, bias=b, round_out=True)  # noqa: E731
            else:
                fn = lambda kw=kw: L.gemm(A, W, out, bias=b, gelu=True, round_out=True, **kw)  # noqa: E731
            r[name] = 2.0 * M * N * K / time_cuda(fn, iters=8) / 1e9
        emit(perf="fc1_full_gelu_ab", rep=rep, **r)
    return True


def sec_conv():
    """Conv1d(k=3,s=2) and (k=2,s=2) over time-major activations through the tap-aware A map."""
    ok = True
    for (k, s, T) in [(3, 2, 1001), (2, 2, 499), (3, 2, 15999)]:
        B, Cin, Cout = 3, 512, 512
        g = torch.Generator(device="cuda").manual_seed(2)
        x = tf32(torch.randn(B, T + 2, Cin, device="cuda", generator=g))  # +2 rows of slack
        w = tf32(torch.randn(Cout, Cin, k, device="cuda", generator=g) * 0.03)
        Tout = (T - k) // s + 1
        Wg = w.permute(0, 2, 1).contiguous().view(Cout, k * Cin)  # [out, tap, in]
        out = torch.full((B, Tout, Cout), float("nan"), device="cuda")
        try:
            L.gemm_tf32(x, Wg, out, gelu=True, rows_per_batch=Tout, batches=B,
                        a_rows_dim=(T + 2) // s, K_inner=Cin, taps=k, P=s,
                        a_phase_stride=Cin, a_row_stride=s * Cin, a_batch_stride=(T + 2) * Cin,
                        out_bstride=Tout, ld_out=Cout)
            torch.cuda.synchronize()
        except Exception as e:  # noqa: BLE001
            emit(check=f"conv_k{k}s{s}_T{T}", ok=False, error=str(e)[:500])
            ok = False
            continue
        ref = torch.nn.functional.conv1d(x[:, :T].double().transpose(1, 2), w.double(), stride=s)
        ref = gelu(ref).transpose(1, 2)
        err = (out.double() - ref).abs().max().item()
        good = err < 1e-4 and not torch.isnan(out).any().item()
        emit(check=f"conv_k{k}s{s}_T{T}", ok=bool(good), max_err=err, ref_max=ref.abs().max().item())
        ok &= good
    return ok


def sec_gemm_perf():
    """ViT-B/16 linear shapes at the bench's M (2,048 frames x 197 tokens); default dispatch."""
    M = 403456
    for (name, N, K, kw) in [
        ("qkv", 2304, 768, dict(bias=True, rnd=True)),
        ("outproj", 768, 768, dict(bias=True, res=True)),
        ("fc1", 3072, 768, dict(bias=True, gelu=True, rnd=True)),
        ("fc2", 768, 3072, dict(bias=True, res=True)),
    ]:
        A = tf32(torch.randn(M, K, device="cuda"))
        W = tf32(torch.randn(N, K, device="cuda") * 0.02)
        b = torch.randn(N, device="cuda")
        R = torch.randn(M, N, device="cuda") if kw.get("res") else None
        out = torch.empty(M, N, device="cuda")
        fn = lambda: L.gemm_tf32(A, W, out, bias=b, res=R, gelu=kw.get("gelu", False),  # noqa: E731
                                 round_out=kw.get("rnd", False))
        try:
            ms = time_cuda(fn, iters=10)
        except Exception as e:  # noqa: BLE001
            emit(perf=name, error=str(e)[:300])
            continue
        torch.backends.cuda.matmul.allow_tf32 = True
        ms_t = time_cuda(lambda: torch.matmul(A, W.t(), out=out), iters=5)
        emit(perf=name, M=M, N=N, K=K, ms=ms, tflops=2.0 * M * N * K / ms / 1e9,
             torch_tf32_ms=ms_t, torch_tflops=2.0 * M * N * K / ms_t / 1e9)
        del A, W, out, R
    return True


def sec_gemm_f16():
    """F16 mode: fp16 operands, fp32 accumulate; fp32 / tf32 / fp16 outputs, residual, V^T side output."""
    ok = True
    for (name, M, N, K, force, cl) in [("f16_1tile", 128, 128, 64, 0, 0), ("f16_tail", 300, 256, 768, 256, 0),
                                       ("f16_fc1", 45000, 3072, 768, 0, 0), ("f16_fc2", 45000, 768, 3072, 0, 0),
                                       ("f16_qkv_1cta", 5000, 2304, 768, 0, 1)]:
        g = torch.Generator(device="cuda").manual_seed(11)
        A = torch.randn(M, K, device="cuda", generator=g).half()
        W = (torch.randn(N, K, device="cuda", generator=g) * 0.05).half()
        b = torch.randn(N, device="cuda", generator=g)
        R = torch.randn(M, N, device="cuda", generator=g)
        ref = A.double() @ W.double().t() + b.double()
        out = torch.full((M, N), float("nan"), device="cuda")
        L.gemm(A, W, out, bias=b, res=R, mode=L.MER_GEMM_F16, force_block_n=force, cluster=cl)
        out16 = torch.full((M, N), float("nan"), device="cuda", dtype=torch.float16)
        L.gemm(A, W, out16, bias=b, gelu=True, f16_out=True, mode=L.MER_GEMM_F16, force_block_n=force, cluster=cl)
        torch.cuda.synchronize()
        e1 = (out.double() - (ref + R.double())).abs().max().item() / ref.abs().max().item()
        refg = gelu(ref)
        e2 = (out16.double() - refg).abs().max().item() / refg.abs().max().item()
        good = e1 < 2e-5 and e2 < 6e-4 and not torch.isnan(out16).any().item()
        info = dict(check=name, ok=bool(good), M=M, N=N, K=K, rel_err_f32_res=e1, rel_err_gelu_f16=e2)
        if N == 2304:  # QKV shape: tf32-rounded output + transposed V
            ld = (M + 3) // 4 * 4
            vt = torch.zeros(768, ld, device="cuda")
            q = torch.full((M, N), float("nan"), device="cuda")
            L.gemm(A, W, q, bias=b, round_out=True, mode=L.MER_GEMM_F16, vt=vt, vt_col0=1536, cluster=cl)
            torch.cuda.synchronize()
            rq = tf32(ref.float()).double()
            e3 = (q[:, :1536].double() - rq[:, :1536]).abs().max().item() / rq.abs().max().item()
            e4 = (vt[:, :M].double() - rq[:, 1536:].t()).abs().max().item() / rq.abs().max().item()
            info.update(rel_err_qk=e3, rel_err_vt=e4)
            good = good and e3 < 1e-3 and e4 < 1e-3
            info["ok"] = bool(good)
        emit(**info)
        ok &= good
    M = 403456
    for (name, N, K, kw) in [("qkv", 2304, 768, dict(round_out=True)), ("outproj", 768, 768, dict(res=True)),
                             ("fc1", 3072, 768, dict(gelu=True, f16_out=True)), ("fc2", 768, 3072, dict(res=True))]:
        A = torch.randn(M, K, device="cuda").half()
        W = (torch.randn(N, K, device="cuda") * 0.02).half()
        b = torch.randn(N, device="cuda")
        R = torch.randn(M, N, device="cuda") if kw.pop("res", False) else None
        out = torch.empty(M, N, device="cuda", dtype=torch.float16 if kw.get("f16_out") else torch.float32)
        ms = time_cuda(lambda: L.gemm(A, W, out, bias=b, res=R, mode=L.MER_GEMM_F16, **kw), iters=10)
        o2 = torch.empty(M, N, device="cuda", dtype=torch.float16)
        ms_t = time_cuda(lambda: torch.matmul(A, W.t(), out=o2), iters=5)
        emit(perf="f16_" + name, M=M, N=N, K=K, ms=ms, tflops=2.0 * M * N * K / ms / 1e9, torch_f16_ms=ms_t,
             torch_tflops=2.0 * M * N * K / ms_t / 1e9)
        del A, W, out, R, o2
    return ok


def sec_one():
    """One ViT GEMM shape, a few launches (for ncu): MER_PROBE_SHAPE = qkv | outproj | fc1 | fc2."""
    M = 403456
    shapes = dict(qkv=(2304, 768, dict(rnd=True)), outproj=(768, 768, dict(res=True)),
                  fc1=(3072, 768, dict(gelu=True, rnd=True)), fc2=(768, 3072, dict(res=True)))
    name = os.environ.get("MER_PROBE_SHAPE", "fc1")
    N, K, kw = shapes[name]
    A = tf32(torch.randn(M, K, device="cuda"))
    W = tf32(torch.randn(N, K, device="cuda") * 0.02)
    b = torch.randn(N, device="cuda")
    R = torch.randn(M, N, device="cuda") if kw.get("res") else None
    out = torch.empty(M, N, device="cuda")
    for _ in range(3):
        L.gemm_tf32(A, W, out, bias=b, res=R, gelu=kw.get("gelu", False), round_out=kw.get("rnd", False))
    torch.cuda.synchronize()
    return True


def sec_ln():
    ok = True
    for dim, eps in [(768, 1e-12), (512, 1e-5), (768, 1e-5)]:
        rows = 5003
        x = torch.randn(rows, dim, device="cuda") * 3 + 1
        g = torch.randn(dim, device="cuda")
        b = torch.randn(dim, device="cuda")
        y = torch.empty_like(x)
        acc = torch.zeros_like(x)
        L.layernorm(x, g, b, y, eps=eps, acc=acc, flags=L.MER_LN_ACC_INIT)
        L.layernorm(x, g, b, y, eps=eps, acc=acc, flags=L.MER_LN_ACC_ADD)
        torch.cuda.synchronize()
        ref = torch.nn.functional.layer_norm(x.double(), (dim,), g.double(), b.double(), eps)
        e1 = (y.double() - ref).abs().max().item()
        e2 = (acc.double() - 2 * ref).abs().max().item()
        good = e1 < 2e-5 and e2 < 4e-5
        emit(check=f"layernorm_{dim}", ok=bool(good), err=e1, err_acc=e2)
        ok &= good
    rows = 403456
    x = torch.randn(rows, 768, device="cuda")
    y = torch.empty_like(x)
    g = torch.ones(768, device="cuda")
    b = torch.zeros(768, device="cuda")
    ms = time_cuda(lambda: L.layernorm(x, g, b, y, eps=1e-12, flags=L.MER_LN_ROUND_TF32))
    emit(perf="layernorm_768", rows=rows, ms=ms, gbs=rows * 768 * 8 / ms / 1e6)
    return ok


def sec_attn():
    ok = True
    heads = 12
    for lens in [[197] * 5, [249] * 3, [7, 64, 65, 1, 130, 499], [7, 64, 65, 1, 130, 256, 200, 128, 129], [16] * 40]:
        cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32, device="cuda")
        tot = sum(lens)
        qkv = tf32(torch.randn(tot, 3 * heads * 64, device="cuda") * 1.5)
        ctx = torch.full((tot, heads * 64), float("nan"), device="cuda")
        ld = (tot + 3) // 4 * 4
        vt = torch.zeros(heads * 64, ld, device="cuda")
        vt[:, :tot] = qkv[:, 2 * heads * 64:].t()
        L.attention(qkv, ctx, cu, max(lens), heads, vt=vt)
        torch.cuda.synchronize()
        err = 0.0
        s0 = 0
        for n in lens:
            q, k, v = qkv[s0:s0 + n].double().view(n, 3, heads, 64).permute(1, 2, 0, 3)
            p = torch.softmax(q @ k.transpose(-1, -2) / 8.0, -1)
            ref = (p @ v).permute(1, 0, 2).reshape(n, heads * 64)
            err = max(err, (ctx[s0:s0 + n].double() - ref).abs().max().item())
            s0 += n
        good = err < 2e-3 and not torch.isnan(ctx).any().item()
        emit(check=f"attention_{lens[0]}x{len(lens)}", ok=bool(good), max_err=err)
        ok &= good
    n_seq = 2048
    cu = (torch.arange(n_seq + 1, device="cuda", dtype=torch.int32) * 197)
    qkv = torch.randn(n_seq * 197, 2304, device="cuda")
    ctx = torch.empty(n_seq * 197, 768, device="cuda")
    vt = qkv[:, 1536:].t().contiguous()
    ms = time_cuda(lambda: L.attention(qkv, ctx, cu, 197, heads, round_out=True, vt=vt), iters=5)
    flops = n_seq * heads * 4.0 * 197 * 197 * 64
    emit(perf="attention_vit_2048x197", ms=ms, tflops=flops / ms / 1e9)
    return ok


def sec_attn_f16():
    """All-fp16 V^T attention (fp16 q | k | v^T in, fp16 ctx out) against fp64 softmax attention."""
    ok = True
    heads = 12
    for lens in [[197] * 5, [249] * 3, [7, 64, 65, 1, 130, 240], [7, 64, 65, 1, 130, 200, 128, 129, 3], [16] * 40]:
        cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32, device="cuda")
        tot = sum(lens)
        qkv = (torch.randn(tot, 3 * heads * 64, device="cuda") * 1.5).half()
        ctx = torch.full((tot, heads * 64), float("nan"), device="cuda", dtype=torch.float16)
        ld = (tot + 7) // 8 * 8
        vt = torch.zeros(heads * 64, ld, device="cuda", dtype=torch.float16)
        vt[:, :tot] = qkv[:, 2 * heads * 64:].t()
        L.attention(qkv, ctx, cu, max(lens), heads, vt=vt)
        torch.cuda.synchronize()
        err = 0.0
        s0 = 0
        for n in lens:
            q, k, v = qkv[s0:s0 + n].double().view(n, 3, heads, 64).permute(1, 2, 0, 3)
            p = torch.softmax(q @ k.transpose(-1, -2) / 8.0, -1)
            ref = (p @ v).permute(1, 0, 2).reshape(n, heads * 64)
            err = max(err, (ctx[s0:s0 + n].double() - ref).abs().max().item())
            s0 += n
        good = err < 3e-3 and not torch.isnan(ctx).any().item()
        emit(check=f"attention_f16_{lens[0]}x{len(lens)}", ok=bool(good), max_err=err)
        ok &= good
    n_seq = 2048
    cu = (torch.arange(n_seq + 1, device="cuda", dtype=torch.int32) * 197)
    qkv = torch.randn(n_seq * 197, 2304, device="cuda").half()
    ctx = torch.empty(n_seq * 197, 768, device="cuda", dtype=torch.float16)
    vt = qkv[:, 1536:].t().contiguous()
    ms = time_cuda(lambda: L.attention(qkv, ctx, cu, 197, heads, vt=vt), iters=5)
    flops = n_seq * heads * 4.0 * 197 * 197 * 64
    emit(perf="attention_f16_vit_2048x197", ms=ms, tflops=flops / ms / 1e9)
    return ok


def sec_vit():
    from mertools_b200 import synthetic as S
    from mertools_b200.encoders import VitEncoder
    enc = VitEncoder(S.vit_state_dict(seed=0, layers=12), device="cuda")
    for n in (256, 2048):
        frames = torch.randint(0, 256, (n, 224, 224, 3), dtype=torch.uint8, device="cuda")
        ms = time_cuda(lambda: enc.frame_features(frames), iters=3, warmup=2)
        emit(perf=f"vit_forward_{n}frames", ms=ms, clips_per_s=n / 8 / ms * 1e3,
             tflops=35.13e9 * n / ms / 1e9)
    return True


SECTIONS = dict(attn_f16=sec_attn_f16, one=sec_one, gemm_f16=sec_gemm_f16, vit=sec_vit, gemm_x3=sec_gemm_x3, gelu_ab=sec_gelu_ab, gemm=sec_gemm, conv=sec_conv, gemm_perf=sec_gemm_perf, ln=sec_ln, attn=sec_attn)

if __name__ == "__main__":
    os.makedirs("gpurun_out", exist_ok=True)
    OUT = open("gpurun_out/probe.jsonl", "a")
    L.check(L.lib().mer_check_device())
    emit(device=torch.cuda.get_device_name(0), abi=L.lib().mer_abi_version())
    names = sys.argv[1:] or list(SECTIONS)
    for n in names:
        t0 = time.time()
        try:
            r = SECTIONS[n]()
        except Exception as e:  # noqa: BLE001
            emit(section=n, crashed=str(e)[:800])
            # a sticky CUDA error poisons the context: stop here
            break
        emit(section=n, ok=r, seconds=round(time.time() - t0, 1))
