"""Throughput of the XLNet text-feature path at the published xlnet-base (12 x 768, 12 heads) and xlnet-large
(24 x 1024, 16 heads) shapes against the reference's loop, plus mer_xlnet_attention against mer_attention on the same
q | k | V^T.

Packed path: XlnetNet on the CUDA backend with BertEncoder's operand rule (f16 at 768, bf16x3 at 1024), sentences
packed up to --tokens per pass, with token types (the segment term on).  Reference loop (extract_text_huggingface.py,
the AutoModel branch): HF XLNetModel in fp32 at batch 1, output_hidden_states and the last-four sum.  Weights are seeded
random fp32 tensors generated on the device; sentence lengths are bench_llm_text.py's seeded draws.  Time shares of GEMM
/ attention / LayerNorm come from CUDA events around every launch, in a separate pass.

    python scripts/bench_xlnet_text.py [--shapes base,large] [--sentences 1024] [--ref-sentences 64]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_llm_text import card, packed_batches, sentence_lengths  # noqa: E402

from mertools_b200 import _lib as L  # noqa: E402
from mertools_b200.extract import xlnet_text as XT  # noqa: E402

SHAPES = {"base": dict(d_model=768, n_head=12, d_inner=3072, n_layer=12, ff_activation="gelu"),
          "large": dict(d_model=1024, n_head=16, d_inner=4096, n_layer=24, ff_activation="gelu")}
VOCAB = 32000


def hf_model(kw, dev):
    import transformers as tf
    cfg = tf.XLNetConfig(vocab_size=VOCAB, dropout=0.0, **kw)
    with torch.device(dev):
        m = tf.XLNetModel(cfg)
    return m.to(dev).eval(), cfg     # mask_emb is created on the host whatever the default device


def seeded_weights(m, seed):
    g = torch.Generator(device=next(m.parameters()).device).manual_seed(seed)
    with torch.no_grad():
        for k, p in m.named_parameters():
            if k.endswith("layer_norm.weight"):
                p.copy_(1 + 0.1 * torch.randn(p.shape, generator=g, device=p.device))
            else:
                p.copy_(torch.randn(p.shape, generator=g, device=p.device) * (0.5 if "embedding" in k else 0.02))
    return {k: v for k, v in m.state_dict().items()}


def types_of(x):
    return np.r_[np.zeros(len(x) - 1, np.int64), 2]


def reference_loop(m, ids, dev):
    with torch.no_grad():
        def fwd(x):
            t = torch.from_numpy(types_of(x))[None].to(dev)
            hs = m(torch.from_numpy(x)[None].to(dev), token_type_ids=t, output_hidden_states=True).hidden_states
            return torch.stack(hs)[[-4, -3, -2, -1]].sum(0)[0, :-2].cpu().numpy()
        for x in ids[:2]:
            fwd(x)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for x in ids:
            fwd(x)
        torch.cuda.synchronize()
        return time.perf_counter() - t0


def attention_vs_mer_attention(lens, heads, dev, reps=20):
    """fp16 operands, fp16 ctx, token types on: the new kernel and mer_attention on the same q | k | V^T."""
    T, D = sum(lens), heads * 64
    g = torch.Generator(device=dev).manual_seed(5)
    qkv = torch.randn(T, 3 * D, generator=g, device=dev).half()
    vt = torch.zeros(D, (T + 7) // 8 * 8, dtype=torch.float16, device=dev)
    vt[:, :T] = qkv[:, 2 * D:].T
    _, rows = XT.rel_table(D, max(lens))
    r = torch.randn(2 * max(lens) - 1, D, generator=g, device=dev).half()
    rows = torch.from_numpy(rows).to(dev)
    bias = [torch.randn(n, heads, 64, generator=g, device=dev) * 0.3 for n in (1, 1, 1, 2)]
    tt = torch.from_numpy(np.concatenate([types_of(np.zeros(n)) for n in lens]).astype(np.int32)).to(dev)
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=dev)
    ctx = torch.empty(T, D, dtype=torch.float16, device=dev)

    def new():
        L.check(L.lib().mer_xlnet_attention(
            L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(r), D, L.ptr(rows), *(L.ptr(b) for b in bias), L.ptr(tt), 0.125,
            L.ptr(ctx), L.ptr(cu), len(lens), T, max(lens), heads, L.MER_ATT_QKV_F16 | L.MER_EPI_OUT_F16,
            L.stream_ptr()))

    def old():
        L.attention(qkv, ctx, cu, max(lens), heads, vt=vt)
    out = {}
    for name, fn in (("mer_xlnet_attention", new), ("mer_attention", old)):
        for _ in range(3):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out[name] = e0.elapsed_time(e1) / reps
    out["ratio"] = out["mer_xlnet_attention"] / out["mer_attention"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="base,large")
    ap.add_argument("--sentences", type=int, default=1024)
    ap.add_argument("--ref-sentences", type=int, default=64)
    ap.add_argument("--tokens", type=int, default=16384, help="tokens per packed pass")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None, help="JSON file for the results")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda:0")
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}")
    lens = sentence_lengths(a.sentences, a.seed)
    rng = np.random.default_rng(a.seed + 1)
    ids = [np.concatenate([rng.integers(10, VOCAB, n - 2), [4, 3]]).astype(np.int64) for n in lens]
    results = dict(card=name, power=power, lengths=dict(n=len(lens), mean=float(np.mean(lens)), total=int(sum(lens))))
    for heads in (12, 16):
        r = attention_vs_mer_attention(lens[:256], heads, dev)
        results[f"attention_{heads}_heads"] = r
        print(f"attention, {heads} heads, 256 packed sentences: mer_xlnet_attention "
              f"{r['mer_xlnet_attention']:.3f} ms, mer_attention {r['mer_attention']:.3f} ms (x{r['ratio']:.2f})")
    for shape in a.shapes.split(","):
        kw = SHAPES[shape]
        m, cfg = hf_model(kw, dev)
        sd = seeded_weights(m, a.seed + 7)
        ref_ids = ids[:a.ref_sentences]
        ref_dt = reference_loop(m, ref_ids, dev)
        del m
        torch.cuda.empty_cache()
        ops = XT.CudaOps("f16" if kw["d_model"] == 768 else "bf16x3", dev)
        net = XT.XlnetNet(sd, ops, XT.XlnetDims(cfg))
        del sd

        def run():
            for batch in packed_batches(ids, a.tokens):
                net.forward(np.concatenate(batch), [len(x) for x in batch], np.concatenate([types_of(x) for x in batch]))
        with torch.no_grad():
            run()                                           # warm-up: every shape of the timed window
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                run()
            e1.record()
            torch.cuda.synchronize()
            dt = e0.elapsed_time(e1) / 1e3 / a.steps
            ops.timing = []
            run()
            torch.cuda.synchronize()
        shares = {}
        for klass, b, e in ops.timing:
            shares[klass] = shares.get(klass, 0.0) + b.elapsed_time(e)
        tot = sum(shares.values())
        r = dict(packed_sentences_per_s=len(ids) / dt, packed_tokens_per_s=sum(lens) / dt,
                 reference="HF fp32 batch 1", reference_sentences_per_s=len(ref_ids) / ref_dt,
                 speedup=(len(ids) / dt) / (len(ref_ids) / ref_dt), shares={k: v / tot for k, v in sorted(shares.items())})
        results[shape] = r
        print(f"{shape}: packed {r['packed_sentences_per_s']:.1f} sentences/s ({r['packed_tokens_per_s']:.0f} tokens/s); "
              f"HF fp32 batch-1 loop {r['reference_sentences_per_s']:.2f} sentences/s; x{r['speedup']:.1f}")
        print(f"{shape}: time shares (per-launch events) " + ", ".join(f"{k} {v:.3f}" for k, v in r["shares"].items()))
        del net, ops
        torch.cuda.empty_cache()
    print(json.dumps(results))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
