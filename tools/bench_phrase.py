"""Phrase encoding on one GPU: Encoder.forward(input_ids=..., return_phrase=True) (phrase tower over every token + filter head) on
synthetic ragged contexts (real lengths spread over [S/2, S], padded to S), in every precision mode.
Workloads: B = 32 at S = 384 (max_seq_length, options.py:33) and B = 16 at S = 512 (the reference's dump recipe).
Reports contexts/s, tokens/s (padded tokens, as computed), algorithmic TFLOP/s and the tensor pipe's share of its TF32 peak
(Encoder.mma_multiplier), the attention kernels' share of the forward (torch.profiler, a separate run), the SIMT attention at
S = 384 for comparison, and the reference's torch path on the same GPU (tests/phrase_ref.py on oracle/encoder_ref.py): fp32 with
TF32 off, and fp16 autocast (the reference dumps with --fp16).
    python tools/bench_phrase.py [--reps 10] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

TF32_PEAK = 494.7e12            # H100 SXM data sheet, dense TF32 tensor-core rate (bf16: twice that)
H, FF, LAYERS = 768, 3072, 12
WORKLOADS = ((32, 384), (16, 512))
SEED, VOCAB = 11, 28996


def gemm_flop_per_token():
    """QKV, attention output, FFN in, FFN out: 2 * (768*2304 + 768*768 + 768*3072 + 3072*768) * 12 = 169.9 MFLOP."""
    return 2 * (H * 3 * H + H * H + H * FF + FF * H) * LAYERS


def flop_per_context(S):
    """GEMMs over S tokens + attention (QK^T and PV: 2 * 2 * S^2 * 768 per layer); the filter head (2 x 768 per token) is noise."""
    return gemm_flop_per_token() * S + LAYERS * 4 * S * S * H


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q}


def time_ms(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def attention_share(fn, reps=3):
    """(attention kernels' ms per call, share of all kernel time) from a torch.profiler run of fn."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    total = attn = 0.0
    for ev in prof.key_averages():
        t = ev.self_device_time_total
        total += t
        if "attention" in ev.key:
            attn += t
    return attn / reps / 1e3, attn / total if total else float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_phrase needs a GPU")
    from densephrases_b200.encoder import BertGeometry, Encoder, random_phrase_state_dict, synthetic_context_batch
    from tests import phrase_ref
    info = gpu_info()
    print(info, flush=True)
    geo = BertGeometry(vocab_size=VOCAB)
    sd = random_phrase_state_dict(geo, SEED)
    enc = Encoder(geo, state_dict=sd, phrase_only=True)
    sd_gpu = {k: v.cuda() for k, v in sd.items()}
    rows = []
    for B, S in WORKLOADS:
        ids, mask, tt = (t.cuda() for t in synthetic_context_batch(B, S, VOCAB, SEED + S))
        flop = B * flop_per_context(S)
        r = {"B": B, "S": S, "real_tokens": int(mask.sum()), "gflop_per_batch": flop / 1e9,
             "attention_flop_share": B * LAYERS * 4 * S * S * H / flop, **info}

        def run():
            return enc(input_ids=ids, attention_mask=mask, token_type_ids=tt, return_phrase=True)
        for mode in enc.precision_modes():
            enc.set_precision(mode)
            for tc in ((True, False) if S <= 384 else (True,)):
                enc.set_attention(tc)
                ms = time_ms(run, a.reps)
                attn_ms, attn_frac = attention_share(run)
                tflops = flop / ms / 1e9
                key = mode if tc else f"{mode}_simt_attention"
                r[key] = {"ms": ms, "contexts_per_s": B / ms * 1e3, "tokens_per_s": B * S / ms * 1e3, "algorithmic_tflops": tflops,
                          "tensor_pipe_frac_of_tf32_peak": tflops * 1e12 * enc.mma_multiplier(mode) / TF32_PEAK,
                          "attention_ms": attn_ms, "attention_frac_of_kernel_time": attn_frac}
            enc.set_attention(True)
        for name, fp16 in (("torch_fp32", False), ("torch_fp16_autocast", True)):
            torch.backends.cuda.matmul.allow_tf32 = False
            torch.backends.cudnn.allow_tf32 = False

            def ref():
                with torch.autocast("cuda", dtype=torch.float16, enabled=fp16):
                    return phrase_ref.embed_phrase(sd_gpu, ids, mask, tt)
            ms = time_ms(ref, max(2, a.reps // 3), warm=1)
            r[name] = {"ms": ms, "contexts_per_s": B / ms * 1e3, "tokens_per_s": B * S / ms * 1e3, "algorithmic_tflops": flop / ms / 1e9}
        rows.append(r)
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()
    print(f"\n{info}")
    print(f"{'B x S':>9} {'arm':>28} {'ms':>8} {'ctx/s':>8} {'tok/s':>9} {'TFLOP/s':>8} {'pipe/TF32pk':>11} {'attn ms':>8} {'attn share':>10}")
    for r in rows:
        for key, v in r.items():
            if not isinstance(v, dict):
                continue
            pk = f"{100 * v['tensor_pipe_frac_of_tf32_peak']:>10.1f}%" if "tensor_pipe_frac_of_tf32_peak" in v else f"{'':>11}"
            at = f"{v['attention_ms']:>8.2f} {100 * v['attention_frac_of_kernel_time']:>9.1f}%" if "attention_ms" in v else f"{'':>8} {'':>10}"
            print(f"{r['B']:>3} x {r['S']:<3} {key:>28} {v['ms']:>8.2f} {v['contexts_per_s']:>8.1f} {v['tokens_per_s']:>9.0f} "
                  f"{v['algorithmic_tflops']:>8.1f} {pk} {at}")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_phrase.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
