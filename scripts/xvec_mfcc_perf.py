"""XVectorMFCC embeddings: times (CUDA events, after warm-up) the workloads of xvec_perf.py on one GPU and the fp32
eager-CUDA oracle (tests/oracle_xvector_mfcc.py: torchaudio MFCC + TDNN, TF32 off) on the same input.

  (a) 512 utterances of 8 s in one b200_xvec_mfcc_forward call
  (b) one 30 min file, Inference(window="whole")
  (c) Inference(window="sliding", duration=3.0, step=1.0) over a 10 min file

Prints ms per call, audio-hours/s, TDNN TFLOP/s from a FLOP model of the five TDNN layers (2 x C_in x kernel x C_out
per output frame; 4.27 GFLOP per 10 s), and the card's name and power limit.  Then, in a separate torch.profiler run of
workload (a), the MFCC front end's share of the kernel time (its three kernels and the DFT GEMM, which is the
gemm_tc_split launch with N = 512 and 2 taps: counted as the first GEMM after each mfcc_rows_kernel).  Synthetic
weights and audio (seeded).

    python scripts/xvec_mfcc_perf.py [--iters 5] [--no-oracle] [--no-profile] [--flop-model-only]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from emb_utt_perf import card, time_ms  # noqa: E402

SR = 16000
TDNN = ((40, 512, 5, 1), (512, 512, 3, 2), (512, 512, 3, 3), (512, 512, 1, 1), (512, 1500, 1, 1))


def tdnn_flop(num_samples: int) -> float:
    """Multiply-adds x 2 of the five TDNN layers on one utterance (the MFCC front end and the Linear left out)."""
    n = 1 + num_samples // 200
    flop = 0.0
    for cin, cout, k, d in TDNN:
        n -= d * (k - 1)
        flop += 2.0 * cin * k * cout * n
    return flop


def front_end_share(ctx, wav, off, N):
    """(front-end kernel ms, all kernel ms) of one call under torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    ctx.xvec_mfcc_forward(wav, off, N)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ctx.xvec_mfcc_forward(wav, off, N)
        torch.cuda.synchronize()
    kernels = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                      and "memcpy" not in e.name.lower() and "memset" not in e.name.lower()),
                     key=lambda e: e.time_range.start)
    total = front = 0.0
    after_rows = False
    for e in kernels:
        us = e.time_range.end - e.time_range.start
        total += us
        if "mfcc_" in e.name:
            front += us
            after_rows = "mfcc_rows_kernel" in e.name
        elif after_rows and "gemm_tc_split" in e.name:
            front += us                                   # the DFT GEMM right after the rows kernel
            after_rows = False
    return front / 1e3, total / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--no-oracle", action="store_true")
    ap.add_argument("--no-profile", action="store_true")
    ap.add_argument("--flop-model-only", action="store_true")
    args = ap.parse_args()
    print(f"TDNN FLOP model: {tdnn_flop(160000) / 1e9:.2f} GFLOP per 10 s")
    if args.flop_model_only:
        return
    import warnings

    import numpy as np
    import torch

    from oracle_xvector_mfcc import XVectorMFCC as OracleXVector
    from pyannote_audio_b200 import synthetic as syn
    from pyannote_audio_b200.inference import Inference, chunk_layout
    from pyannote_audio_b200.models import XVectorMFCC

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures on the GPU only")
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda:0")
    print(f"card: {card()}")
    sd = syn.make_xvector_mfcc_state_dict(5)
    model = XVectorMFCC()
    model.load_state_dict(sd)
    model.to(dev)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        oracle = OracleXVector()
    oracle.load_state_dict(sd)
    oracle = oracle.to(dev).eval()
    ctx = model._ctx()
    g = torch.Generator().manual_seed(0)

    def report(name, ms, audio_s, flop, oracle_ms):
        line = (f"{name}: {ms:.2f} ms/call, {audio_s / 3600 / (ms / 1e3):.2f} audio-h/s, "
                f"TDNN {flop / (ms / 1e3) / 1e12:.1f} TFLOP/s")
        if oracle_ms is not None:
            line += f" | fp32 eager oracle {oracle_ms:.1f} ms/call ({oracle_ms / ms:.1f}x)"
        print(line, flush=True)

    def oracle_ms(fn):
        if args.no_oracle:
            return None
        with torch.inference_mode():
            return time_ms(fn, 1, warmup=1)

    # (a) 512 utterances x 8 s, one call
    n, N = 512, 8 * SR
    wav = (torch.rand(n * N, generator=g) * 0.2 - 0.1).to(dev)
    off = np.arange(n, dtype=np.int64) * N
    ms = time_ms(lambda: ctx.xvec_mfcc_forward(wav, off, N), args.iters)
    batches = wav.view(n, 1, N).split(64)
    report("(a) 512 x 8 s utterances", ms, n * N / SR, n * tdnn_flop(N), oracle_ms(lambda: [oracle(b) for b in batches]))
    if not args.no_profile:
        front, total = front_end_share(ctx, wav, off, N)
        print(f"(a) under torch.profiler: MFCC front end {front:.2f} ms of {total:.2f} ms kernel time "
              f"({100 * front / total:.1f}%)", flush=True)

    # (b) one 30 min file, window="whole"
    N = 30 * 60 * SR
    file = {"waveform": (torch.rand(1, N, generator=g) * 0.2 - 0.1), "sample_rate": SR}
    whole = Inference(model, window="whole")
    ms = time_ms(lambda: whole(file), args.iters)
    report("(b) 30 min file, whole", ms, N / SR, tdnn_flop(N), oracle_ms(lambda: oracle(file["waveform"][None].to(dev))))

    # (c) sliding 3 s / 1 s over 10 min
    N = 10 * 60 * SR
    file = {"waveform": (torch.rand(1, N, generator=g) * 0.2 - 0.1), "sample_rate": SR}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sliding = Inference(model, window="sliding", duration=3.0, step=1.0)
    off, _, _, _ = chunk_layout(N, 3 * SR, SR)
    ms = time_ms(lambda: sliding(file), args.iters)
    padded = torch.zeros(int(off[-1]) + 3 * SR)
    padded[:N] = file["waveform"][0]
    chunks = torch.stack([padded[o: o + 3 * SR] for o in off])[:, None].to(dev)
    report(f"(c) sliding 3 s / 1 s over 10 min ({len(off)} windows)", ms, N / SR, len(off) * tdnn_flop(3 * SR),
           oracle_ms(lambda: [oracle(c) for c in chunks.split(256)]))


if __name__ == "__main__":
    main()
