"""Throughput of the DeBERTa text-feature path at the published deberta-large (24 x 1024, 16 heads, v1) and
deberta-v2-xxlarge (48 x 1536, 24 heads, log buckets, conv layer) shapes against the reference's loop, plus
mer_disentangled_attention against mer_attention on the same q | k | V^T.

Packed path: DebertaNet on the CUDA backend with BertEncoder's operand rule (bf16x3 at these widths), sentences packed
up to --tokens per pass.  Reference loop (extract_text_huggingface.py:193-231): HF DebertaModel / DebertaV2Model in fp32
at batch 1, output_hidden_states and the last-four sum.  Weights are seeded random fp32 tensors generated on the device;
sentence lengths are bench_llm_text.py's seeded draws.  Time shares of GEMM / attention / LayerNorm come from CUDA
events around every launch, in a separate pass.

    python scripts/bench_deberta_text.py [--shapes large,xxlarge] [--sentences 1024] [--ref-sentences 64]
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
from mertools_b200.extract import deberta_text as DT  # noqa: E402

BASE = dict(max_position_embeddings=512, max_relative_positions=-1, relative_attention=True,
            pos_att_type=["c2p", "p2c"], position_biased_input=False, type_vocab_size=0, layer_norm_eps=1e-7)
SHAPES = {"large": (False, dict(BASE, hidden_size=1024, num_attention_heads=16, intermediate_size=4096,
                                num_hidden_layers=24)),
          "xxlarge": (True, dict(BASE, hidden_size=1536, num_attention_heads=24, intermediate_size=6144,
                                 num_hidden_layers=48, position_buckets=256, norm_rel_ebd="layer_norm",
                                 share_att_key=True, conv_kernel_size=3, conv_act="gelu"))}
VOCAB = 21128


def hf_model(v2, kw, dev):
    import transformers as tf
    cfg = (tf.DebertaV2Config if v2 else tf.DebertaConfig)(vocab_size=VOCAB, **kw)
    with torch.device(dev):
        return (tf.DebertaV2Model if v2 else tf.DebertaModel)(cfg).eval(), cfg


def seeded_weights(m, seed):
    g = torch.Generator(device=next(m.parameters()).device).manual_seed(seed)
    with torch.no_grad():
        for k, p in m.named_parameters():
            if k.endswith("LayerNorm.weight"):
                p.copy_(1 + 0.1 * torch.randn(p.shape, generator=g, device=p.device))
            else:
                p.copy_(torch.randn(p.shape, generator=g, device=p.device) * (0.5 if "embeddings" in k else 0.02))
    return {k: v for k, v in m.state_dict().items()}


def reference_loop(m, ids, dev):
    with torch.no_grad():
        def fwd(x):
            hs = m(torch.from_numpy(x)[None].to(dev), output_hidden_states=True).hidden_states
            return torch.stack(hs)[[-4, -3, -2, -1]].sum(0)[0, 1:-1].cpu().numpy()
        for x in ids[:2]:
            fwd(x)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for x in ids:
            fwd(x)
        torch.cuda.synchronize()
        return time.perf_counter() - t0


def attention_vs_mer_attention(lens, heads, dev, reps=20):
    """fp16 operands, fp16 ctx: the new kernel (span 256, v2 rows) and mer_attention on the same q | k | V^T."""
    T, D, span = sum(lens), heads * 64, 256
    g = torch.Generator(device=dev).manual_seed(5)
    qkv = torch.randn(T, 3 * D, generator=g, device=dev).half()
    vt = torch.zeros(D, (T + 7) // 8 * 8, dtype=torch.float16, device=dev)
    vt[:, :T] = qkv[:, 2 * D:].T
    pos = torch.randn(2 * span, 2 * D, generator=g, device=dev).half()
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=dev)
    import transformers as tf
    dims = DT.DebertaDims(tf.DebertaV2Config(hidden_size=D, num_attention_heads=heads, position_buckets=span,
                                             max_relative_positions=512, relative_attention=True))
    rows = torch.from_numpy(DT.rel_rows(dims, max(lens))).to(dev)
    ops = DT.CudaOps("f16", dev)
    b = dict(cu=cu, n=len(lens), max_len=max(lens), rows=rows)
    ctx = torch.empty(T, D, dtype=torch.float16, device=dev)

    def new():
        L.check(ops._att(L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(pos), L.ptr(pos[:, D:]), 2 * D, span, L.ptr(rows),
                         0.0722, L.ptr(ctx), L.ptr(cu), b["n"], T, b["max_len"], heads,
                         L.MER_ATT_QKV_F16 | L.MER_EPI_OUT_F16, L.stream_ptr()))

    def old():
        L.attention(qkv, ctx, cu, max(lens), heads, vt=vt)
    out = {}
    for name, fn in (("mer_disentangled_attention", new), ("mer_attention", old)):
        for _ in range(3):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out[name] = e0.elapsed_time(e1) / reps
    out["ratio"] = out["mer_disentangled_attention"] / out["mer_attention"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="large,xxlarge")
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
    ids = [np.concatenate([[2], rng.integers(5, VOCAB, n - 2), [3]]).astype(np.int64) for n in lens]
    results = dict(card=name, power=power, lengths=dict(n=len(lens), mean=float(np.mean(lens)), total=int(sum(lens))))
    for heads in (16, 24):
        r = attention_vs_mer_attention(lens[:256], heads, dev)
        results[f"attention_{heads}_heads"] = r
        print(f"attention, {heads} heads, 256 packed sentences: mer_disentangled_attention "
              f"{r['mer_disentangled_attention']:.3f} ms, mer_attention {r['mer_attention']:.3f} ms (x{r['ratio']:.2f})")
    for shape in a.shapes.split(","):
        v2, kw = SHAPES[shape]
        m, cfg = hf_model(v2, kw, dev)
        sd = seeded_weights(m, a.seed + 7)
        ref_ids = ids[:a.ref_sentences]
        ref_dt = reference_loop(m, ref_ids, dev)
        del m
        torch.cuda.empty_cache()
        ops = DT.CudaOps("f16" if kw["hidden_size"] == 768 else "bf16x3", dev)
        net = DT.DebertaNet(sd, ops, DT.DebertaDims(cfg))
        del sd
        with torch.no_grad():
            for batch in packed_batches(ids, a.tokens):                     # warm-up: every shape of the timed window
                net.forward(np.concatenate(batch), [len(x) for x in batch])
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                for batch in packed_batches(ids, a.tokens):
                    net.forward(np.concatenate(batch), [len(x) for x in batch])
            e1.record()
            torch.cuda.synchronize()
            dt = e0.elapsed_time(e1) / 1e3 / a.steps
            ops.timing = []
            for batch in packed_batches(ids, a.tokens):
                net.forward(np.concatenate(batch), [len(x) for x in batch])
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
