"""Speaker embeddings of audio of any length: times (CUDA events, after warm-up) three workloads on one GPU and the
fp32 eager-CUDA oracle (oracle/nets.py, TF32 off) on the same input.

  (a) 512 utterances of 8 s in one b200_emb_forward_utt call
  (b) one 30 min file, Inference(window="whole")
  (c) Inference(window="sliding", duration=3.0, step=1.0) over a 10 min file

Prints ms per call, audio-hours/s, trunk TFLOP/s from a FLOP model of the conv widths of each layer (45.18 GFLOP per
10 s segment, as bench.py counts), and the card's name and power limit.  Synthetic weights and audio (seeded).

    python scripts/emb_utt_perf.py [--iters 5] [--no-oracle] [--flop-model-only]
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SR = 16000


def trunk_flop(num_samples: int) -> float:
    """Multiply-adds x 2 of the 32 3x3 block convs and the 3 1x1 shortcuts of ResNet34 on one utterance (the 1 -> 32
    stem is left out, as bench.py counts)."""
    W = 1 + (num_samples - 400) // 160
    H, cin, flop = 80, 32, 0.0
    for planes, n, stride in ((32, 3, 1), (64, 4, 2), (128, 6, 2), (256, 3, 2)):
        for i in range(n):
            s = stride if i == 0 else 1
            Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
            flop += 2.0 * 9 * cin * planes * Ho * Wo                      # conv1
            flop += 2.0 * 9 * planes * planes * Ho * Wo                   # conv2
            if s != 1 or cin != planes:
                flop += 2.0 * cin * planes * Ho * Wo                      # 1x1 shortcut
            H, W, cin = Ho, Wo, planes
    return flop


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=20).stdout.strip()
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
    ap.add_argument("--flop-model-only", action="store_true")
    args = ap.parse_args()
    print(f"trunk FLOP model: {trunk_flop(160000) / 1e9:.2f} GFLOP per 10 s segment")
    if args.flop_model_only:
        return
    import numpy as np
    import torch

    from oracle import nets
    from pyannote_audio_b200 import synthetic as syn
    from pyannote_audio_b200.inference import Inference, chunk_layout
    from pyannote_audio_b200.models import WeSpeakerResNet34

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures on the GPU only")
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda:0")
    print(f"card: {card()}")
    sd = syn.make_embedding_state_dict(1)
    emb = WeSpeakerResNet34()
    emb.load_state_dict(sd)
    emb.to(dev)
    oemb = nets.WeSpeakerResNet34()
    oemb.load_state_dict(sd)
    oemb = oemb.to(dev).eval()
    ctx = emb._ctx()
    g = torch.Generator().manual_seed(0)

    def report(name, ms, audio_s, flop, oracle_ms):
        line = (f"{name}: {ms:.2f} ms/call, {audio_s / 3600 / (ms / 1e3):.2f} audio-h/s, "
                f"trunk {flop / (ms / 1e3) / 1e12:.1f} TFLOP/s")
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
    ms = time_ms(lambda: ctx.emb_forward_utt(wav, off, N), args.iters)
    batches = wav.view(n, 1, N).split(64)
    report("(a) 512 x 8 s utterances", ms, n * N / SR, n * trunk_flop(N),
           oracle_ms(lambda: [oemb(b) for b in batches]))

    # (b) one 30 min file, window="whole"
    N = 30 * 60 * SR
    file = {"waveform": (torch.rand(1, N, generator=g) * 0.2 - 0.1), "sample_rate": SR}
    whole = Inference(emb, window="whole")
    ms = time_ms(lambda: whole(file), args.iters)
    report("(b) 30 min file, whole", ms, N / SR, trunk_flop(N), oracle_ms(lambda: oemb(file["waveform"][None].to(dev))))

    # (c) sliding 3 s / 1 s over 10 min
    N = 10 * 60 * SR
    file = {"waveform": (torch.rand(1, N, generator=g) * 0.2 - 0.1), "sample_rate": SR}
    import warnings

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")                                     # trained on 10 s chunks
        sliding = Inference(emb, window="sliding", duration=3.0, step=1.0)
    off, _, _, _ = chunk_layout(N, 3 * SR, SR)
    ms = time_ms(lambda: sliding(file), args.iters)
    padded = torch.zeros(int(off[-1]) + 3 * SR)
    padded[:N] = file["waveform"][0]
    chunks = torch.stack([padded[o: o + 3 * SR] for o in off])[:, None].to(dev)
    report(f"(c) sliding 3 s / 1 s over 10 min ({len(off)} windows)", ms, N / SR, len(off) * trunk_flop(3 * SR),
           oracle_ms(lambda: [oemb(c) for c in chunks.split(256)]))


if __name__ == "__main__":
    main()
