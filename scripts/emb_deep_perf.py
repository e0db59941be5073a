"""WeSpeaker ResNet34 and the bottleneck ResNet152 / 221 / 293: times (CUDA events, after warm-up) two workloads per
model on one GPU and the fp32 eager-CUDA oracle (TF32 off) on the same input.

  (a) b200_emb_forward on 264 x 10 s chunks with binary masks (3 local speakers), one call
  (b) one 30 min file, Inference(window="whole")

Prints ms per call, audio-hours/s, trunk TFLOP/s from the FLOP model below, and the card's name and power limit.
Synthetic weights and audio (seeded).

    python scripts/emb_deep_perf.py [--iters 5] [--no-oracle] [--flop-model-only] [--models 34,152,221,293]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))                   # the bottleneck oracle lives with the tests

from emb_utt_perf import card, time_ms, trunk_flop as resnet34_flop  # noqa: E402

SR = 16000
BLOCKS = {152: (3, 8, 36, 3), 221: (6, 16, 48, 3), 293: (10, 20, 64, 3)}


def trunk_flop(depth: int, num_samples: int) -> float:
    """Multiply-adds x 2 of the block convs (and shortcuts) of one utterance; the 1 -> 32 stem is left out."""
    if depth == 34:
        return resnet34_flop(num_samples)
    W = 1 + (num_samples - 400) // 160
    H, cin, flop = 80, 32, 0.0
    for p, n, stride in zip((32, 64, 128, 256), BLOCKS[depth], (1, 2, 2, 2)):
        for i in range(n):
            s = stride if i == 0 else 1
            Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
            flop += 2.0 * cin * p * H * W                               # conv1 1x1
            flop += 2.0 * 9 * p * p * Ho * Wo                           # conv2 3x3
            flop += 2.0 * p * 4 * p * Ho * Wo                           # conv3 1x1
            if s != 1 or cin != 4 * p:
                flop += 2.0 * cin * 4 * p * Ho * Wo                     # 1x1 shortcut
            H, W, cin = Ho, Wo, 4 * p
    return flop


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--no-oracle", action="store_true")
    ap.add_argument("--flop-model-only", action="store_true")
    ap.add_argument("--models", default="34,152,221,293")
    args = ap.parse_args()
    depths = [int(d) for d in args.models.split(",")]
    for d in depths:
        print(f"ResNet{d} trunk FLOP model: {trunk_flop(d, 160000) / 1e9:.2f} GFLOP per 10 s chunk")
    if args.flop_model_only:
        return
    import numpy as np
    import torch

    from oracle import nets
    from pyannote_audio_b200 import models, synthetic as syn
    from pyannote_audio_b200.inference import Inference
    from oracle_bottleneck import WeSpeakerBottleneck

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures on the GPU only")
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda:0")
    print(f"card: {card()}")
    g = torch.Generator().manual_seed(0)
    n = 264
    wav = syn.make_conversation(10.0 + (n - 1), seed=264)[0]
    buf = wav.to(dev).contiguous()
    off = np.arange(n, dtype=np.int64) * SR
    valid = np.full(n, 10 * SR, dtype=np.int32)
    masks = torch.from_numpy((np.random.default_rng(0).uniform(size=(n, 3, 589)) < 0.6).astype(np.uint8)).to(dev)
    chunks = torch.stack([wav[o: o + 10 * SR] for o in off])[:, None]
    N = 30 * 60 * SR
    file = {"waveform": (torch.rand(1, N, generator=g) * 0.2 - 0.1), "sample_rate": SR}

    print("| model | workload | ms per call | audio-h/s | trunk TFLOP/s | fp32 eager oracle |")
    print("|---|---|---|---|---|---|")
    for d in depths:
        if d == 34:
            emb, oemb, sd = models.WeSpeakerResNet34(), nets.WeSpeakerResNet34(), syn.make_embedding_state_dict(1)
        else:
            emb, oemb, sd = getattr(models, f"WeSpeakerResNet{d}")(), WeSpeakerBottleneck(d), \
                syn.make_bottleneck_state_dict(d, 1)
        emb.load_state_dict(sd)
        emb.to(dev)
        oemb.load_state_dict(sd)
        oemb = oemb.to(dev).eval()
        ctx = emb._ctx()

        def row(name, ms, audio_s, flop, oracle):
            o = "not measured" if oracle is None else f"{oracle:.1f} ms ({oracle / ms:.1f}x)"
            print(f"| ResNet{d} | {name} | {ms:.2f} | {audio_s / 3600 / (ms / 1e3):.2f} | "
                  f"{flop / (ms / 1e3) / 1e12:.1f} | {o} |", flush=True)

        def oracle_ms(fn):
            if args.no_oracle:
                return None
            with torch.inference_mode():
                return time_ms(fn, 1, warmup=1)

        ms = time_ms(lambda: ctx.emb_forward(buf, off, valid, masks), args.iters)
        fw = masks.float()
        row("264 x 10 s chunks, masks", ms, n * 10.0, n * trunk_flop(d, 10 * SR),
            oracle_ms(lambda: [oemb(c.to(dev), weights=w) for c, w in zip(chunks.split(24), fw.split(24))]))
        whole = Inference(emb, window="whole")
        ms = time_ms(lambda: whole(file), args.iters)
        row("30 min file, whole", ms, N / SR, trunk_flop(d, N), oracle_ms(lambda: oemb(file["waveform"][None].to(dev))))
        del emb, oemb, whole
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
