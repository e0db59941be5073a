"""Segmentation of audio of any length: times (CUDA events, after warm-up) three workloads on one GPU and the fp32
eager-CUDA oracle (oracle/nets.py, TF32 off) on the same input.

  (a) 512 windows of 5 s in one b200_seg_forward_window call
  (b) one 30 min file, Inference(window="whole"): one window, so the BiLSTM runs one 2-CTA cluster per direction over
      106 k frames (latency-bound); the oracle runs torch's native CUDA LSTM here, cuDNN rejects the sequence
  (c) Inference(window="sliding", duration=5.0, step=0.5) over a 10 min file

Prints ms per call, audio-hours/s (seconds of input audio per wall second, overlap not counted twice) and the card's
name and power limit.  Synthetic weights and audio (seeded).

    python scripts/seg_utt_perf.py [--iters 5] [--no-oracle]
"""
import argparse
import os
import subprocess
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SR = 16000


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:                                                   # noqa: BLE001
        return f"unknown ({e})"


def time_ms(fn, iters, warmup=2):
    import torch

    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--no-oracle", action="store_true")
    args = ap.parse_args()
    import numpy as np
    import torch

    from oracle import nets
    from pyannote_audio_b200 import synthetic as syn
    from pyannote_audio_b200.inference import Inference, chunk_layout
    from pyannote_audio_b200.models import PyanNet

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures on the GPU only")
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda:0")
    print(f"card (name, power limit, max SM clock): {card()}")
    sd = syn.make_segmentation_state_dict(0)
    seg = PyanNet()
    seg.load_state_dict(sd)
    seg.to(dev)
    oseg = nets.PyanNet()
    oseg.load_state_dict(sd)
    oseg = oseg.to(dev).eval()
    ctx = seg._ctx()
    g = torch.Generator().manual_seed(0)

    def report(name, ms, audio_s, oracle_ms):
        line = f"{name}: {ms:.2f} ms/call, {audio_s / 3600 / (ms / 1e3):.2f} audio-h/s"
        if oracle_ms is not None:
            line += f" | fp32 eager oracle {oracle_ms:.1f} ms/call ({oracle_ms / ms:.1f}x)"
        print(line, flush=True)

    def oracle_ms(fn):
        if args.no_oracle:
            return None
        with torch.inference_mode():
            return time_ms(fn, 1, warmup=1)

    # (a) 512 windows x 5 s, one call
    n, N = 512, 5 * SR
    wav = (torch.rand(n * N, generator=g) * 0.2 - 0.1).to(dev)
    off = np.arange(n, dtype=np.int64) * N
    valid = np.full(n, N, dtype=np.int32)
    ms = time_ms(lambda: ctx.seg_forward(wav, off, valid, window=N), args.iters)
    batches = wav.view(n, 1, N).split(64)
    report("(a) 512 x 5 s windows", ms, n * N / SR, oracle_ms(lambda: [oseg(b) for b in batches]))

    # (b) one 30 min file, window="whole"
    N = 30 * 60 * SR
    file = {"waveform": (torch.rand(1, N, generator=g) * 0.2 - 0.1), "sample_rate": SR}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")                                     # "whole" with a frame-based model
        whole = Inference(seg, window="whole")
    ms = time_ms(lambda: whole(file), args.iters, warmup=1)

    def oracle_whole():                     # cuDNN rejects this 106 k-step sequence: torch's native CUDA LSTM
        with torch.backends.cudnn.flags(enabled=False):
            return oseg(file["waveform"][None].to(dev))

    report(f"(b) 30 min file, whole ({seg.num_frames(N)} frames)", ms, N / SR, oracle_ms(oracle_whole))

    # (c) sliding 5 s / 0.5 s over 10 min
    N = 10 * 60 * SR
    file = {"waveform": (torch.rand(1, N, generator=g) * 0.2 - 0.1), "sample_rate": SR}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")                                     # trained on 10 s chunks
        sliding = Inference(seg, window="sliding", duration=5.0, step=0.5, skip_aggregation=True)
    W, S = 5 * SR, SR // 2
    off, _, _, _ = chunk_layout(N, W, S)
    ms = time_ms(lambda: sliding(file), args.iters)
    padded = torch.zeros(int(off[-1]) + W)
    padded[:N] = file["waveform"][0]
    chunks = torch.stack([padded[o: o + W] for o in off])[:, None].to(dev)
    report(f"(c) sliding 5 s / 0.5 s over 10 min ({len(off)} windows)", ms, N / SR,
           oracle_ms(lambda: [oseg(c) for c in chunks.split(256)]))


if __name__ == "__main__":
    main()
