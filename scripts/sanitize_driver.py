"""Small launches of every hand-synchronised kernel family, for compute-sanitizer (scripts/sanitize.sh):
the wgmma GEMM in its three operand modes and both tile widths, every tensor-core attention route
on ragged batches, the LLaMA kernels (causal head-dim-128 attention, RoPE, RMSNorm, SwiGLU), the BLOOM / OPT / GPT-2
kernels (ALiBi attention, causal attention at head_dim 64 / 96 / 128, wide LayerNorm, tanh-GELU / fp16 ReLU epilogues), LayerNorm, the HuBERT front-end (conv0 + GroupNorm, positional conv) through a 2-layer forward, the
fused fusion step (cluster kernel with DSMEM exchange + weight-gradient kernel).  Sizes are tiny: racecheck is slow."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from mertools_b200 import _lib as L  # noqa: E402
from mertools_b200 import synthetic as S  # noqa: E402

dev = torch.device("cuda:0")
torch.manual_seed(0)


def gemms():
    for M, N, K in ((300, 256, 128), (1000, 768, 256)):
        a = torch.randn(M, K, device=dev)
        w = torch.randn(N, K, device=dev) * 0.05
        bias = torch.randn(N, device=dev)
        out = torch.empty(M, N, device=dev)
        L.gemm(L.round_tf32_(a.clone()), L.round_tf32_(w.clone()), out, bias=bias)
        L.gemm(L.split_bf16(a), L.split_bf16(w), out, bias=bias, gelu=True, mode=L.MER_GEMM_BF16X3)
        o16 = torch.empty(M, N, dtype=torch.float16, device=dev)
        L.gemm(a.half(), w.half(), o16, bias=bias, mode=L.MER_GEMM_F16, f16_out=True)
    torch.cuda.synchronize()
    print("gemm ok")


def attention():
    """One small launch per route of tests/test_attention_tc_gpu.py (the short kernel, the fp16 / tf32 tiled kernel,
    mer_attention_hd, mer_attention_long, the causal, ALiBi and multi-query kernels), on ragged rows with an empty
    sequence and unaligned starts, in the fp32 and fp16 ctx formats."""
    import _kernel_refs as R
    from test_attention_tc_gpu import _device_operands, _run
    for name in R.ATT_TC_CASES:
        c = R.att_tc_case(name)
        c["lens"] = [5, 0, 17, 600 if c["entry"] == "long" else min(max(c["lens"]), 300)]
        ops = R.att_tc_operands(c, 1.5)
        qkv, vt, cu = _device_operands(c, ops, dev)
        slopes = None if ops["slopes"] is None else ops["slopes"].to(dev)
        for fmt in ("f16",) if c["causal"] else ("fp32", "f16"):
            _run(c, qkv, vt, cu, fmt, slopes)
    torch.cuda.synchronize()
    print("attention ok")


def llama():
    """The LLaMA kernels: causal head-dim-128 attention on ragged rows with unaligned starts, RoPE (both position
    sources), RMSNorm in both output modes, the fp16 SwiGLU, then a 3-layer LlamaNet forward."""
    from mertools_b200.extract import llama_text as LT
    heads, lens = 2, [5, 70, 1, 129, 17]
    tokens, D = sum(lens), heads * 128
    qkv = torch.randn(tokens, 3 * D, device=dev).half()
    vt = torch.zeros(D, (tokens + 7) // 8 * 8, dtype=torch.float16, device=dev)
    vt[:, :tokens] = qkv[:, 2 * D:].T
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=dev)
    ops = LT.CudaOps(dev)
    cos, sin = (t.to(dev) for t in LT.rope_tables(256, 10000.0))
    b = ops.batch(lens)
    L.check(ops._rope(L.ptr(qkv), 3 * D, tokens, heads, L.ptr(cu), len(lens), None, L.ptr(cos), L.ptr(sin), 256,
                      L.stream_ptr()))
    pos = torch.cat([torch.arange(n) for n in lens]).to(torch.int32).to(dev)
    L.check(ops._rope(L.ptr(qkv), 3 * D, tokens, heads, None, 0, L.ptr(pos), L.ptr(cos), L.ptr(sin), 256, L.stream_ptr()))
    ctx = torch.empty(tokens, D, dtype=torch.float16, device=dev)
    L.check(ops._att(L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(ctx), L.ptr(cu), len(lens), tokens, max(lens), heads,
                     L.stream_ptr()))
    x = torch.randn(tokens, 512, device=dev)
    w = torch.ones(512, device=dev)
    ops.rmsnorm(x, w, 1e-6)
    ops.rmsnorm(x, w, 1e-6, acc=torch.zeros_like(x))
    L.check(ops._swiglu(L.ptr(torch.randn(tokens, 2 * 512, device=dev)), L.ptr(torch.empty(tokens, 512, dtype=torch.float16,
                                                                                            device=dev)), tokens, 512,
                        L.stream_ptr()))
    sd = {k: torch.from_numpy(v) for k, v in S.llama_state_dict(seed=21, vocab=300, layers=3).items()}
    LT.LlamaNet(sd, ops, 3, 4, 1e-6, 10000.0, 256).forward(np.arange(3, 3 + tokens) % 300, lens)
    torch.cuda.synchronize()
    print("llama ok")


def ln_decoders():
    """The BLOOM / OPT / GPT-2 kernels: causal attention with ALiBi, and without at head_dim 64, 96 and 128, on ragged
    rows with unaligned starts, the wide LayerNorm in its three output modes, the tanh-GELU and fp16 ReLU GEMM
    epilogues, then a 3-layer LnDecoderNet forward per family."""
    from mertools_b200.extract import ln_decoder_text as LD
    heads, lens = 3, [5, 70, 1, 129, 17]
    tokens, D = sum(lens), heads * 128
    qkv = torch.randn(tokens, 3 * D, device=dev).half()
    vt = torch.zeros(D, (tokens + 7) // 8 * 8, dtype=torch.float16, device=dev)
    vt[:, :tokens] = qkv[:, 2 * D:].T
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=dev)
    ops = LD.CudaOps(dev)
    ctx = torch.empty(tokens, D, dtype=torch.float16, device=dev)
    L.check(ops._att_alibi(L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(ctx), L.ptr(cu), len(lens), tokens, max(lens),
                           heads, L.ptr(LD.alibi_slopes(heads).to(dev)), L.stream_ptr()))
    for hd in LD.GPT2_HEAD_DIMS:
        Dh = heads * hd
        qkv_h = torch.randn(tokens, 3 * Dh, device=dev).half()
        vt_h = torch.zeros(Dh, (tokens + 7) // 8 * 8, dtype=torch.float16, device=dev)
        vt_h[:, :tokens] = qkv_h[:, 2 * Dh:].T
        L.check(ops._att(L.ptr(qkv_h), L.ptr(vt_h), vt_h.shape[1], L.ptr(torch.empty(tokens, Dh, dtype=torch.float16,
                                                                                     device=dev)),
                         L.ptr(cu), len(lens), tokens, max(lens), heads, hd, L.stream_ptr()))
    x = torch.randn(tokens, 512, device=dev)
    g, b = torch.ones(512, device=dev), torch.zeros(512, device=dev)
    ops.layernorm(x, g, b, 1e-5)
    ops.layernorm(x, g, b, 1e-5, out="f32")
    ops.layernorm(x, g, b, 1e-5, acc=torch.zeros_like(x))
    a, w, bias = torch.randn(tokens, 256, device=dev).half(), torch.randn(384, 256, device=dev).half(), torch.randn(384, device=dev)
    for f16 in (False, True):
        out = torch.empty(tokens, 384, dtype=torch.float16 if f16 else torch.float32, device=dev)
        L.gemm(a, w, out, bias=bias, mode=L.MER_GEMM_F16, f16_out=f16, gelu_tanh=True)
    L.gemm(a, w, torch.empty(tokens, 384, dtype=torch.float16, device=dev), bias=bias, mode=L.MER_GEMM_F16,
           f16_out=True, relu=True)
    ids = np.arange(4, 4 + tokens) % 300
    bsd = {LD._strip(k, "bloom"): torch.from_numpy(v) for k, v in S.bloom_state_dict(vocab=300, layers=3).items()}
    LD.LnDecoderNet(bsd, ops, "bloom", 3, 4, 1e-5).forward(ids, lens)
    osd = {LD._strip(k, "opt"): torch.from_numpy(v) for k, v in S.opt_state_dict(vocab=300, layers=3, max_pos=256).items()}
    LD.LnDecoderNet(osd, ops, "opt", 3, 4, 1e-5, 256).forward(ids, lens)
    gsd = {LD._strip(k, "gpt2"): (torch.from_numpy(v).T if k.endswith(LD.GPT2_CONV1D) else torch.from_numpy(v))
           for k, v in S.gpt2_state_dict(vocab=300, layers=3, max_pos=256).items()}
    LD.LnDecoderNet(gsd, ops, "gpt2", 3, 4, 1e-5, 256).forward(ids, lens, token_types=np.zeros_like(ids))
    torch.cuda.synchronize()
    print("ln_decoders ok")


def encoders():
    from mertools_b200.encoders import BertEncoder, HubertEncoder, VitEncoder
    sd = S.hubert_state_dict(seed=1, layers=4)
    wav = (S.synth_waves(2, 16000, seed=2).astype(np.float64) / 32768.0).astype(np.float32)
    for prec in ("f16", "bf16x3"):
        HubertEncoder(sd, device=dev, stack_precision=prec).forward(torch.from_numpy(wav).to(dev))
    BertEncoder(S.bert_state_dict(300, seed=2, layers=4), device=dev).forward([[2, 17, 250, 99, 3], [2, 5, 3]])
    VitEncoder(S.vit_state_dict(seed=0, layers=2), device=dev).frame_features(torch.from_numpy(S.synth_frames(1, 2, seed=1)[0]).to(dev))
    torch.cuda.synchronize()
    print("encoders ok")


def fusion():
    from mertools_b200.fusion import FusionNet
    for B, hidden in ((32, 128), (130, 64)):
        net = FusionNet(hidden_dim=hidden, dropout=0.3, device=dev, seed=1).load_state_dict(S.fusion_state_dict(seed=3, hidden=hidden))
        a, t, v, emo, val = S.synth_fusion_features(B, seed=4)
        T = torch.from_numpy
        for _ in range(2):
            net.train_step(T(a).to(dev), T(t).to(dev), T(v).to(dev), T(emo).to(dev), T(val).view(-1, 1).to(dev),
                           weight_decay=1e-5, use_graph=False)
    torch.cuda.synchronize()
    print("fusion ok")


def fusion_mlp():
    """The MER2023 baseline nets: both kinds, an input chunked through the staging buffer, a ragged last cluster."""
    from mertools_b200.fusion_mlp import MlpFusionNet, reference_init
    for kind, layers, dims, B in (("mlp", "256,128", (1582, 88, 1500), 33), ("attention", "130,3", (10, 12, 7), 6)):
        net = MlpFusionNet(kind, *dims, layers, device=dev, max_batch=64, seed=1)
        net.load_state_dict(reference_init(kind, *dims, layers))
        g = torch.Generator().manual_seed(5)
        x = [torch.randn(B, d, generator=g).to(dev) for d in dims]
        emo, val = torch.randint(0, 6, (B,), generator=g).to(dev), torch.randn(B, 1, generator=g).to(dev)
        for _ in range(2):
            net.train_step(*x, emo, val, use_graph=False)
        net(*x)
    torch.cuda.synchronize()
    print("fusion_mlp ok")


if __name__ == "__main__":
    which = sys.argv[1:] or ["gemms", "attention", "llama", "ln_decoders", "encoders", "fusion", "fusion_mlp"]
    for w in which:
        globals()[w]()
