"""SSeRiouSS (WavLM Base front end) on the GPU against the fp32 eager oracle (tests/oracle_sseriouss.py, TF32 off) on
the same card: per-window forward at several batch sizes, sliding 10 s windows with a 1 s step over 10 minutes, and
one whole multi-minute window.  Prints the card and its power limit, times (CUDA-synchronised wall clock, best of
--repeat after a warm-up) and achieved TFLOP/s from the FLOP model below, and with --out writes them there as JSON.

    python scripts/sseriouss_perf.py [--repeat 3] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from pyannote_audio_b200.inference import Inference, chunk_layout  # noqa: E402
from pyannote_audio_b200.models import SSeRiouSS  # noqa: E402
from pyannote_audio_b200.testing import synthetic as syn  # noqa: E402

import oracle_sseriouss as oracle  # noqa: E402

SR = 16000


def flops(num_samples: int) -> dict:
    """Multiply-adds x 2 of one window, by part (the convs, the positional conv, the transformer GEMMs, attention's
    QK^T and PV, and the LSTM head's GEMMs; the recurrence and elementwise work are left out)."""
    n, lens = num_samples, []
    n = 1 + (n - 10) // 5
    lens.append(n)
    for k in (3, 3, 3, 3, 2, 2):
        n = 1 + (n - k) // 2
        lens.append(n)
    T = lens[-1]
    convs = 2 * lens[0] * 512 * 10 + sum(2 * lens[i + 1] * 512 * 512 * k for i, k in enumerate((3, 3, 3, 3, 2, 2)))
    convs += 2 * T * 512 * 768                                   # feature projection
    pos = 2 * T * 768 * 48 * 128
    gemms = 12 * 2 * T * 768 * (3 * 768 + 768 + 2 * 3072)
    attention = 12 * 2 * 2 * T * T * 768
    head = 2 * T * 1024 * (768 + 3 * 256) + 2 * T * 128 * (256 + 128)
    return {"convs": convs, "pos_conv": pos, "transformer_gemms": gemms, "attention": attention, "lstm_head": head,
            "total": convs + pos + gemms + attention + head}


def timed(fn, repeat):
    fn()
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(repeat):
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t)
    return best


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:           # the query is informative only
        q = f"unavailable ({e})"
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--out", default=None, help="JSON file for the results (optional)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sseriouss_perf.py measures the GPU path: no CUDA device is visible")
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda:0")
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}")
    sd = syn.make_sseriouss_state_dict(5)
    m = SSeRiouSS()
    m.load_state_dict(sd)
    m.to(dev).eval()
    results = {"card": name, "power_limit_max_sm_clock": power, "workloads": []}

    def record(label, seconds, oracle_seconds, total_flops):
        row = {"workload": label, "ms": seconds * 1e3, "tflops": total_flops / seconds / 1e12,
               "oracle_ms": None if oracle_seconds is None else oracle_seconds * 1e3,
               "speedup": None if oracle_seconds is None else oracle_seconds / seconds}
        results["workloads"].append(row)
        extra = "" if oracle_seconds is None else f", fp32 eager oracle {oracle_seconds * 1e3:9.1f} ms " \
                                                  f"(x{oracle_seconds / seconds:.1f})"
        print(f"{label:42s} {seconds * 1e3:9.2f} ms, {row['tflops']:6.1f} TFLOP/s{extra}")

    f10 = flops(160000)
    print("FLOP model of one 10 s window (GFLOP):", {k: round(v / 1e9, 2) for k, v in f10.items()})
    results["flops_10s_window"] = f10
    for batch in (1, 8, 32):
        wav = torch.cat([syn.make_conversation(10.0, seed=s) for s in range(batch)])[:, None, :160000].to(dev)
        t = timed(lambda: m(wav), args.repeat)
        to = timed(lambda: oracle.sseriouss(sd, wav[:, 0], device=dev), 1) if batch <= 8 else None
        record(f"forward, batch {batch} x 10 s", t, to, batch * f10["total"])

    wav = syn.make_conversation(600.0, seed=7)
    inf = Inference(m, skip_aggregation=True)
    file = {"waveform": wav, "sample_rate": SR}
    off, _, _, _ = chunk_layout(wav.shape[1], 160000, 16000)
    t = timed(lambda: inf(file), args.repeat)

    def oracle_sliding():
        padded = torch.zeros(int(off[-1]) + 160000)
        padded[: wav.shape[1]] = wav[0]
        for i in range(0, len(off), 32):
            oracle.sseriouss(sd, torch.stack([padded[o: o + 160000] for o in off[i: i + 32]]), device=dev)

    record(f"sliding 10 s / 1 s over 10 min ({len(off)} windows)", t, timed(oracle_sliding, 1),
           len(off) * f10["total"])

    n = 180 * SR
    whole = syn.make_conversation(180.0, seed=9)[:, :n]
    x = whole[:, None].to(dev)
    t = timed(lambda: m(x), args.repeat)
    record("whole 180 s window", t, timed(lambda: oracle.sseriouss(sd, whole, device=dev), 1), flops(n)["total"])
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
