"""The WavLM Base front end of SSeRiouSS (csrc/ssl_wavlm.cu) on its own: the features it hands to the LSTM head
(Context.ssl_features) against tests/oracle_sseriouss.py run in float64 on the CPU.

The end-to-end tests (test_sseriouss.py) see these features only through four LSTM layers, two Linears and a
classifier, at three window lengths.  Here every layer output is compared directly, at the window lengths where the
front end's geometry changes: the attention's 64-frame tiles (T = 63 .. 65, 127 .. 129), the relative-position clamp
at +-1023 frames (T = 1023 .. 1030), and n = 400 + 320 (T - 1) + r samples for r in {0, 1, 5, 319}, which moves
n mod 5, the lengths of the six strided convs and the conv-0 row padding ceil64(len0) - len0.  Batches mix full,
partial, 1-sample and empty windows at odd offsets, split into sub-batches whose rows cross the GEMMs' 128-row tiles;
the input edges are silence, a DC offset, a full-scale square wave and speech at 1e-4.

CPU: the fp64 oracle against the fp32 one, and the relative-position buckets the attention kernel reads against the
oracle's, offsets clamped to +-1023.
"""
import os
import sys

import pytest
import torch

from pyannote_audio_b200 import ops
from pyannote_audio_b200.testing import synthetic as syn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import oracle_sseriouss as oracle  # noqa: E402

SR = 16000
# Max |GPU - fp64 oracle| on an H100 80GB HBM3, synthetic weights (seed 5): layer outputs reach max |x| ~ 5, the
# layer average ~ 2.5.  Measured at most, per group (layer outputs / layer average):
#   every layer, T = 130          1.48e-4 / 5.1e-5
#   window-length sweep           1.52e-4 / 6.0e-5
#   mixed batch                   -       / 6.2e-5
#   input edges                   1.29e-4 / 5.5e-5
# That is ~20x the fp32 oracle's own error (<= 6.3e-6 against fp64), and the fp64 oracle with every GEMM operand
# rounded to its fp16 (hi, lo) pair moves by at most 1.5e-5: the rest is already there at layer 1 and hardly grows
# over the 12 layers.  The bars are 2x the maxima, an order of magnitude under the end-to-end ones.
LAYER_ATOL = 3e-4
AVG_ATOL = 1.2e-4
# the head on the GPU's features against the forward, at the end-to-end bars of test_sseriouss.py: measured at most
# 7.3e-5 (log-probabilities) and 1.2e-5 (sigmoid scores)
LOGP_ATOL, SCORE_ATOL = 2e-3, 1e-3


def _n(T, r=0):
    """Window samples of T frames plus r (< 320) samples that add no frame."""
    return 400 + 320 * (T - 1) + r


def _speech(n, seed):
    return syn.make_conversation(max(n, SR) / SR, seed=seed)[0, :n]


@pytest.fixture(scope="module")
def sd():
    return syn.make_sseriouss_state_dict(5, wav2vec_layer=-1, num_classes=7)


@pytest.fixture(scope="module")
def sd64(sd):
    return {k: v.double() for k, v in sd.items()}


def _oracle(sd64, windows):
    """(B, n) zero-padded windows -> the 12 layer outputs (B, T, 768), float64 on the CPU."""
    with torch.no_grad():
        return oracle.wavlm_layers(sd64, windows.double())


def _average(sd64, layers):
    return torch.stack(layers, dim=-1) @ torch.softmax(sd64["wav2vec_weights"], dim=0)


def _padded(buf, off, valid, n):
    """The windows buf[off : off + valid] zero-padded to n samples, as the kernels read them."""
    out = torch.zeros(len(off), n, dtype=torch.float64)
    for i, (o, v) in enumerate(zip(off, valid)):
        out[i, :v] = buf[o: o + v]
    return out


def _check(name, got, ref, atol):
    assert tuple(got.shape) == tuple(ref.shape), (name, tuple(got.shape), tuple(ref.shape))
    err = float((got.cpu().double() - ref).abs().max())
    print(f"[wavlm] {name}: max |d| {err:.2e} (max |x| {float(ref.abs().max()):.2f})")
    assert err <= atol, (name, err)


# ---- CPU -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T,r", [(1, 319), (74, 7)])
def test_fp64_oracle_matches_the_fp32_oracle(sd, sd64, T, r):
    n = _n(T, r)
    wav = torch.stack([_speech(n, 41), _speech(n, 42)])
    with torch.no_grad():
        lo = oracle.wavlm_layers(sd, wav)
    hi = _oracle(sd64, wav)
    assert all(x.dtype == torch.float64 for x in hi)
    for layer, (a, b) in enumerate(zip(lo, hi), start=1):
        assert a.shape == (2, T, 768)
        torch.testing.assert_close(a.double(), b, atol=2e-5, rtol=0, msg=f"layer {layer}")


def test_relative_buckets_match_the_oracle_with_offsets_clamped():
    table = ops.wavlm_relative_buckets().long()            # what b200_ssl_load turns into the attention's bias rows
    assert table.shape == (2 * ops.SSL_REL_SPAN + 1,)
    d = torch.arange(-4095, 4096)
    clamped = d.clamp(-ops.SSL_REL_SPAN, ops.SSL_REL_SPAN) + ops.SSL_REL_SPAN
    assert torch.equal(oracle.relative_bucket(d), table[clamped])
    T = 1030
    pos = torch.arange(T)
    rel = (pos[None, :] - pos[:, None]).clamp(-ops.SSL_REL_SPAN, ops.SSL_REL_SPAN) + ops.SSL_REL_SPAN
    assert torch.equal(oracle.relative_buckets(T), table[rel])


# ---- GPU ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def no_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def _context(dev, sd, layer, specifications=None):
    c = ops.Context(dev)
    c.load_sseriouss(sd, specifications, wav2vec_layer=layer)
    return c


@pytest.fixture(scope="module")
def ctx_avg(dev, sd):
    return _context(dev, sd, -1)


@pytest.fixture(scope="module")
def ctx_last(dev, sd):
    return _context(dev, sd, 12)


@pytest.mark.gpu
def test_every_layer(dev, sd, sd64):
    # two windows of T = 130; the second keeps 29999 of its samples, and the buffer holds speech after them
    n = _n(130, 37)
    buf = torch.cat([_speech(n, 41), _speech(n, 42)])
    off, valid = [0, n], [n, 29999]
    ref = _oracle(sd64, _padded(buf, off, valid, n))
    wav = buf.to(dev)
    c = ops.Context(dev)
    for layer in range(1, 13):
        c.load_sseriouss(sd, wav2vec_layer=layer)
        _check(f"layer {layer}", c.ssl_features(wav, off, valid, window=n), ref[layer - 1], LAYER_ATOL)
    c.load_sseriouss(sd, wav2vec_layer=-1)
    _check("layer average", c.ssl_features(wav, off, valid, window=n), _average(sd64, ref), AVG_ATOL)


# every (T, r) below the attention's second tile edge; T = 499 (10 s) and the relative-position clamp with one r each
GEOMETRY = [(T, r) for T in (1, 2, 63, 64, 65, 127, 128, 129) for r in (0, 1, 5, 319)] + \
    [(499, 0), (499, 319), (1023, 0), (1024, 5), (1025, 319), (1030, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("T,r", GEOMETRY, ids=[f"T{T}-r{r}" for T, r in GEOMETRY])
def test_window_geometry(ctx_avg, ctx_last, sd64, T, r):
    n = _n(T, r)
    assert ops.ssl_num_frames(n) == T and ops.ssl_num_frames(n - r - 1) == T - 1
    buf = _speech(n, 43 + T)
    ref = _oracle(sd64, buf[None])
    wav = buf.to(ctx_avg.device)
    _check(f"T {T} r {r} average", ctx_avg.ssl_features(wav, [0], [n], window=n), _average(sd64, ref), AVG_ATOL)
    _check(f"T {T} r {r} layer 12", ctx_last.ssl_features(wav, [0], [n], window=n), ref[11], LAYER_ATOL)


@pytest.mark.gpu
def test_mixed_batch_matches_alone_and_split(ctx_avg, sd64):
    # T = 249: window boundaries fall inside the 128-row tiles of the GEMMs (rows 249, 498, ...) and of the positional
    # conv (rows 377, 754, ...), whose taps then read the next window's zero rows
    n = _n(249, 3)
    off = [0, 3, 7777, 11, 101]
    valid = [n, n - 12345, 1, 0, n]
    buf = _speech(max(off) + n, 44)
    ref = _average(sd64, _oracle(sd64, _padded(buf, off, valid, n)))
    wav = buf.to(ctx_avg.device)
    batched = ctx_avg.ssl_features(wav, off, valid, window=n).cpu()
    for i in range(len(off)):
        _check(f"batch window {i} (valid {valid[i]}, offset {off[i]})", batched[i], ref[i], AVG_ATOL)
        alone = ctx_avg.ssl_features(wav, off[i: i + 1], valid[i: i + 1], window=n).cpu()
        assert torch.equal(alone[0], batched[i]), i
    ctx_avg.set_option("ssl_max_batch", 1)                 # 160000 samples: sub-batches of 2, 2 and 1 windows
    try:
        split = ctx_avg.ssl_features(wav, off, valid, window=n).cpu()
    finally:
        ctx_avg.set_option("ssl_max_batch", 32)
    assert torch.equal(split, batched)


@pytest.mark.gpu
def test_input_edges(ctx_avg, ctx_last, sd64):
    n = _n(130)
    speech = _speech(n, 45)
    t = torch.arange(n)
    inputs = {"silence": torch.zeros(n),                         # the conv-0 GroupNorm's variance is 0
              "DC offset 0.5": speech + 0.5,                     # its mean dominates the variance
              "square wave +-1": torch.where((t // 40) % 2 == 0, 1.0, -1.0),
              "speech at 1e-4": speech * 1e-4}                   # the GroupNorm eps dominates the variance
    buf = torch.stack(list(inputs.values())).float()
    ref = _oracle(sd64, buf.double())
    avg = _average(sd64, ref)
    wav = buf.reshape(-1).contiguous().to(ctx_avg.device)
    off, valid = [i * n for i in range(len(inputs))], [n] * len(inputs)
    got_avg = ctx_avg.ssl_features(wav, off, valid, window=n)
    got_last = ctx_last.ssl_features(wav, off, valid, window=n)
    for i, name in enumerate(inputs):
        _check(f"{name} average", got_avg[i], avg[i], AVG_ATOL)
        _check(f"{name} layer 12", got_last[i], ref[11][i], LAYER_ATOL)


@pytest.mark.gpu
@pytest.mark.parametrize("layer", [-1, 3])
def test_launch_counts(dev, sd, layer):
    # per sub-batch, 30 launches before the first layer (conv 0, GroupNorm statistics and apply, 6 conv GEMMs, the
    # projection's LayerNorm and GEMM, the positional pack, 16 group GEMMs and residual add, the encoder LayerNorm) and
    # 8 per layer; the forward adds the head's 12 (log-softmax with log-probabilities)
    c = _context(dev, sd, layer)
    num_layers = 12 if layer < 0 else layer
    wav = _speech(2 * 160000, 46).to(dev)
    off, valid = [0, 16000, 160000], [160000, 160000, 159993]

    def launches(call):
        call()
        n0 = c.launch_count
        call()
        return c.launch_count - n0

    for max_batch, sub_batches in ((32, 1), (1, 3)):
        c.set_option("ssl_max_batch", max_batch)
        try:
            features = launches(lambda: c.ssl_features(wav, off, valid))
            forward = launches(lambda: c.ssl_forward(wav, off, valid, return_logp=True))
        finally:
            c.set_option("ssl_max_batch", 32)
        assert features == sub_batches * (30 + 8 * num_layers), (max_batch, features)
        assert forward - features == sub_batches * 12, (max_batch, forward, features)


@pytest.mark.gpu
@pytest.mark.parametrize("layer,sigmoid", [(-1, False), (6, True)])
def test_features_are_what_the_head_reads(dev, layer, sigmoid):
    from pyannote_audio_b200.core import Problem, Resolution, Specifications

    sd = syn.make_sseriouss_state_dict(5, wav2vec_layer=layer, num_classes=4 if sigmoid else 7)
    specs = Specifications(Problem.MULTI_LABEL_CLASSIFICATION, Resolution.FRAME, 10.0,
                           classes=["speech", "music", "noise", "laughter"]) if sigmoid else None
    c = _context(dev, sd, layer, specs)
    n = 160000
    wav = torch.cat([_speech(n, 41), _speech(n, 42)]).to(dev)
    off, valid = [0, n], [n, 99999]
    x = c.ssl_features(wav, off, valid, window=n)
    ref = oracle.head({k: v.float().to(dev) for k, v in sd.items()}, x, sigmoid)
    if sigmoid:
        _check("head on the features, sigmoid scores", c.ssl_forward(wav, off, valid, window=n).cpu(),
               ref.double(), SCORE_ATOL)
    else:
        _, logp = c.ssl_forward(wav, off, valid, return_logp=True, window=n)
        _check("head on the features, log-probabilities", logp.cpu(), ref.double(), LOGP_ATOL)
