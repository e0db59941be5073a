"""PyanNet with sigmoid heads: times (CUDA events, after warm-up) three workloads on one GPU and the fp32 eager-CUDA
oracle (oracle/nets.py PyanNet with a sigmoid activation, TF32 off) on the same chunks.

  (a) sliding multi-label Inference (4 labels, duration 5 s, step 0.5 s, aggregated on the device) over a 10 min file
  (b) VoiceActivityDetection with a binary head (1 class, 5 s / 0.5 s) on a 1 h file: the fused per-frame maximum,
      the device overlap-add and Binarize
  (c) MultiLabelSegmentation (4 labels, 5 s / 0.5 s) on a 10 min file: (a) plus Binarize per label

The oracle times only its network over the same chunks (no aggregation, no binarisation), so its ratio is a lower
bound.  Prints ms per call, audio-hours/s (seconds of input audio per wall second, overlap not counted twice) and the
card's name and power limit.  Synthetic weights and audio (seeded).

    python scripts/seg_heads_perf.py [--iters 5] [--no-oracle]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from seg_utt_perf import card, time_ms  # noqa: E402

SR = 16000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--no-oracle", action="store_true")
    args = ap.parse_args()
    import torch

    from oracle import nets
    from pyannote_audio_b200.core import Problem, Resolution, Specifications
    from pyannote_audio_b200.inference import Inference, chunk_layout
    from pyannote_audio_b200.models import PyanNet
    from pyannote_audio_b200.multilabel import MultiLabelSegmentation
    from pyannote_audio_b200.testing import synthetic as syn
    from pyannote_audio_b200.vad import VoiceActivityDetection

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures on the GPU only")
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda:0")
    print(f"card (name, power limit, max SM clock): {card()}")
    g = torch.Generator().manual_seed(0)

    def models(k):
        problem = Problem.BINARY_CLASSIFICATION if k == 1 else Problem.MULTI_LABEL_CLASSIFICATION
        sd = syn.make_segmentation_state_dict(0, num_classes=k)
        seg = PyanNet()
        seg.specifications = Specifications(problem, Resolution.FRAME, 5.0, classes=[f"label#{i}" for i in range(k)])
        seg.load_state_dict(sd)
        oseg = nets.PyanNet(num_classes=k)
        oseg.activation = torch.nn.Sigmoid()
        oseg.load_state_dict(sd)
        return seg.to(dev), oseg.to(dev).eval()

    def report(name, ms, audio_s, oracle_ms):
        line = f"{name}: {ms:.2f} ms/call, {audio_s / 3600 / (ms / 1e3):.2f} audio-h/s"
        if oracle_ms is not None:
            line += f" | fp32 eager oracle network only {oracle_ms:.1f} ms/call ({oracle_ms / ms:.1f}x)"
        print(line, flush=True)

    def oracle_ms(oseg, file):
        if args.no_oracle:
            return None
        W, S = 5 * SR, SR // 2
        N = file["waveform"].shape[1]
        off, _, _, _ = chunk_layout(N, W, S)
        padded = torch.zeros(int(off[-1]) + W)
        padded[:N] = file["waveform"][0]
        chunks = torch.stack([padded[o: o + W] for o in off])[:, None].to(dev)
        with torch.inference_mode():
            return time_ms(lambda: [oseg(c) for c in chunks.split(256)], 1, warmup=1)

    def noise_file(seconds):
        return {"waveform": torch.rand(1, int(seconds * SR), generator=g) * 0.2 - 0.1, "sample_rate": SR}

    seg4, oseg4 = models(4)
    file = noise_file(600)
    sliding = Inference(seg4, duration=5.0, step=0.5)
    report("(a) sliding multi-label Inference, 4 labels, 10 min", time_ms(lambda: sliding(file), args.iters),
           600, oracle_ms(oseg4, file))

    seg1, oseg1 = models(1)
    hour = noise_file(3600)
    vad = VoiceActivityDetection(seg1, device=dev)
    vad.instantiate({"onset": 0.6, "offset": 0.4, "min_duration_on": 0.1, "min_duration_off": 0.1})
    report("(b) VoiceActivityDetection, binary head, 1 h", time_ms(lambda: vad(hour), args.iters, warmup=1),
           3600, oracle_ms(oseg1, hour))

    pipe = MultiLabelSegmentation(seg4, device=dev)
    report("(c) MultiLabelSegmentation, 4 labels, 10 min", time_ms(lambda: pipe(file), args.iters), 600,
           oracle_ms(oseg4, file))


if __name__ == "__main__":
    main()
