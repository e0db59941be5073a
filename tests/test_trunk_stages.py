"""The WeSpeaker trunk, stage by stage, against a float64 reference that rounds where the kernels round.

Every trunk conv reads fp16 values and writes fp16 values, so the exact result of each stage on the GPU's own input is
known: BatchNorm folded as the library folds it (float32 scale, fp16 weights; the stem keeps fp32 weights), each conv
summed in float64 on those values, ReLU, and fp16 round-to-nearest-even where the kernels store.  The GPU may differ
from it by one fp16 ulp of the output plus fp32 accumulation in any order:

    |gpu - ref| <= ulp16(y) + C_ACC * 2^-23 * (|b'| + sum |x| |w| (+ |residual|))

and, where an intermediate of the block (conv1's output, the shortcut) may round one ulp away from the GPU, the next
conv adds sum |w| * (ulp16(h) + h's own accumulation term).  The magnitude sums are float64 convs over absolute values.
The bound is per element: a wrong tap, a border column read as padding or a residual from the wrong row shows however
large the rest of the tensor is.

Each GPU case prints max(|d| / bound) and the fraction of bit-identical outputs (`pytest -s`).
"""
import hashlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pyannote_audio_b200 import synthetic as syn

U32 = 2.0 ** -23              # float32 epsilon
C_ACC = 8                     # fp32 accumulation, any order (wgmma's accumulator included)
STAGE_WIDTHS = [1, 2, 3, 125, 126, 127, 128, 129, 135, 136, 137, 252, 253, 256, 257]


# ---- the reference ---------------------------------------------------------------------------------------------
def _ulp16(y):
    """Spacing of fp16 above |y| (y float64 holding fp16 values): the larger of the two at a binade edge."""
    a = y.abs()
    _, e = torch.frexp(a)
    ulp = torch.pow(2.0, (e - 1).clamp_min(-14).double() - 10)
    return torch.where(a == 0, torch.full_like(a, 2.0 ** -24), ulp)


def _fold(sd, conv, bn, rounding, fp16=True):
    """(w', b') of a conv with its eval BatchNorm folded, as make_conv / load_stem fold it (float32 arithmetic, fp16
    weights unless ``fp16`` is False), or exactly in float64 with ``rounding`` off."""
    w, g, beta, mean, var = (sd[conv + ".weight"], sd[bn + ".weight"], sd[bn + ".bias"], sd[bn + ".running_mean"],
                             sd[bn + ".running_var"])
    dt = torch.float32 if rounding else torch.float64
    w, g, beta, mean, var = (t.to(dt) for t in (w, g, beta, mean, var))
    s = g / torch.sqrt(var + 1e-5)
    wf = w * s.view(-1, 1, 1, 1)
    if rounding and fp16:
        wf = wf.half()
    return wf.double(), (beta - mean * s).double()


class TrunkRef:
    """Stage k of the WeSpeaker trunk in float64 on NCHW float64 inputs: k = 0 the stem, k >= 1 block k - 1 (a
    BasicBlock, or a Bottleneck when the state dict has conv3).  ``rounding`` off: exact float64 folding, no fp16
    rounding, and the bound is meaningless."""

    def __init__(self, sd, rounding=True):
        self.rounding = rounding
        self.stem = _fold(sd, "resnet.conv1", "resnet.bn1", rounding, fp16=False)
        self.bottleneck = "resnet.layer1.0.conv3.weight" in sd
        self.blocks = []
        for li in range(1, 5):
            i = 0
            while f"resnet.layer{li}.{i}.conv1.weight" in sd:
                p = f"resnet.layer{li}.{i}"
                convs = ("conv1", "conv2", "conv3") if self.bottleneck else ("conv1", "conv2")
                blk = {c: _fold(sd, f"{p}.{c}", f"{p}.bn{c[-1]}", rounding) for c in convs}
                blk["shortcut"] = (_fold(sd, p + ".shortcut.0", p + ".shortcut.1", rounding)
                                   if p + ".shortcut.0.weight" in sd else None)
                blk["stride"] = 2 if i == 0 and li > 1 else 1
                self.blocks.append(blk)
                i += 1

    def _round(self, z, relu):
        if relu:
            z = z.clamp_min(0)
        return z.half().double() if self.rounding else z

    def _conv(self, x, wb, stride, relu, res=None, d_res=None, d_in=None):
        """One conv as the kernels run it -> (y, bound on |gpu - y|).  d_in: the bound on the input's own error."""
        w, b = wb
        pad = w.shape[-1] // 2
        z = F.conv2d(x, w, stride=stride, padding=pad) + b.view(1, -1, 1, 1)
        m = F.conv2d(x.abs(), w.abs(), stride=stride, padding=pad) + b.abs().view(1, -1, 1, 1)
        if res is not None:
            z, m = z + res, m + res.abs()
        y = self._round(z, relu)
        bound = _ulp16(y) + C_ACC * U32 * m
        if d_in is not None:
            bound = bound + F.conv2d(d_in, w.abs(), stride=stride, padding=pad)
        if d_res is not None:
            bound = bound + d_res
        return y, bound

    def stem_forward(self, fbank, fmean):
        """fbank (B, W, 80), fmean (B, 80) -> NCHW (B, 32, 80, W): the stem on fp32(fbank - fmean) as conv1_kernel
        forms it."""
        x = fbank.float() - fmean.float()[:, None, :] if self.rounding else fbank.double() - fmean.double()[:, None, :]
        return self._conv(x.double().permute(0, 2, 1).unsqueeze(1), self.stem, 1, True)

    def block_forward(self, k, x):
        """Block k on NCHW float64 x -> (y, bound)."""
        blk = self.blocks[k]
        s = blk["stride"]
        res, d_res = x, None
        if blk["shortcut"] is not None:
            res, d_res = self._conv(x, blk["shortcut"], s, False)
        if self.bottleneck:
            h1, d1 = self._conv(x, blk["conv1"], 1, True)
            h2, d2 = self._conv(h1, blk["conv2"], s, True, d_in=d1)
            return self._conv(h2, blk["conv3"], 1, True, res=res, d_res=d_res, d_in=d2)
        h, dh = self._conv(x, blk["conv1"], s, True)
        return self._conv(h, blk["conv2"], 1, True, res=res, d_res=d_res, d_in=dh)

    def forward(self, k, x, fmean=None):
        return self.stem_forward(x, fmean) if k == 0 else self.block_forward(k - 1, x)


def _nchw(t):
    return t.permute(0, 3, 1, 2).double().cpu()


def _activations(shape, seed):
    """Random non-negative fp16 NHWC activations: about 40 % exact zeros and a few values 30 times the rest."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g).abs()
    x[torch.rand(shape, generator=g) < 0.4] = 0
    big = torch.rand(shape, generator=g) < 1e-3
    x[big] = x[big] * 30 + 4
    return x.half()


# ---- CPU: the reference is the network, and its bound admits fp32 arithmetic -----------------------------------
def _basic_block_sd(sd, p):
    return {k[len(p) + 1:]: v for k, v in sd.items() if k.startswith(p + ".")}


@pytest.mark.parametrize("depth", [34, 152])
def test_reference_without_rounding_is_the_network(depth):
    from oracle import nets

    from oracle_bottleneck import Bottleneck

    sd = syn.make_embedding_state_dict(1) if depth == 34 else syn.make_bottleneck_state_dict(152, 1)
    ref = TrunkRef(sd, rounding=False)
    g = torch.Generator().manual_seed(5)
    fb, fm = torch.randn((2, 21, 80), generator=g, dtype=torch.float64), torch.randn((2, 80), generator=g,
                                                                                      dtype=torch.float64)
    stem = torch.nn.Sequential(torch.nn.Conv2d(1, 32, 3, padding=1, bias=False), torch.nn.BatchNorm2d(32)).double()
    stem.load_state_dict({"0.weight": sd["resnet.conv1.weight"], **{"1." + k[len("resnet.bn1."):]: v for k, v in
                                                                     sd.items() if k.startswith("resnet.bn1.")}})
    want = F.relu(stem.eval()((fb - fm[:, None, :]).permute(0, 2, 1).unsqueeze(1)))
    got, _ = ref.stem_forward(fb, fm)
    assert (got - want).abs().max() <= 1e-12 * want.abs().max()
    # every block of the first two layers and the first of layers 3 and 4: strides, shortcuts and all channel counts
    H, C, k = 80, 32, 0
    for li in range(1, 5):
        i = 0
        while f"resnet.layer{li}.{i}.conv1.weight" in sd:
            p, blk = f"resnet.layer{li}.{i}", ref.blocks[k]
            cout = sd[p + (".conv3.weight" if ref.bottleneck else ".conv2.weight")].shape[0]
            if li <= 2 or i == 0:
                mod = (Bottleneck if ref.bottleneck else nets.BasicBlock)(C, cout // 4 if ref.bottleneck else cout,
                                                                         blk["stride"])
                mod.load_state_dict(_basic_block_sd(sd, p))
                x = torch.rand((2, C, H, 9), generator=g, dtype=torch.float64)
                want = mod.double().eval()(x)
                got, _ = ref.block_forward(k, x)
                assert got.shape == want.shape
                assert (got - want).abs().max() <= 1e-12 * want.abs().max(), p
            H, C, k, i = (H - 1) // blk["stride"] + 1, cout, k + 1, i + 1


def _fp32_conv(x, wb, stride, relu, res=None):
    w, b = wb
    z = F.conv2d(x.float(), w.float(), stride=stride, padding=w.shape[-1] // 2) + b.float().view(1, -1, 1, 1)
    if res is not None:
        z = z + res.float()
    return (z.clamp_min(0) if relu else z).half().double()


@pytest.mark.parametrize("depth,k,W", [(34, 1, 40), (34, 3, 40), (34, 7, 33), (34, 13, 17),
                                       (152, 0, 30), (152, 3, 30), (152, 12, 17)])
def test_fp32_block_is_within_the_bound(depth, k, W):
    """The same fp16-rounded block computed honestly in fp32 (conv2d in float32, fp16 stores between convs) stays
    inside the bound: the bound is not tighter than fp32 arithmetic allows."""
    sd = syn.make_embedding_state_dict(1) if depth == 34 else syn.make_bottleneck_state_dict(152, 1)
    ref = TrunkRef(sd)
    blk = ref.blocks[k]
    C_in = (blk["conv1"][0].shape[1])
    H = 80 >> sum(b["stride"] == 2 for b in ref.blocks[:k])
    x = _nchw(_activations((2, H, W, C_in), seed=k))
    s = blk["stride"]
    res = x if blk["shortcut"] is None else _fp32_conv(x, blk["shortcut"], s, False)
    if ref.bottleneck:
        h = _fp32_conv(_fp32_conv(x, blk["conv1"], 1, True), blk["conv2"], s, True)
        got = _fp32_conv(h, blk["conv3"], 1, True, res)
    else:
        got = _fp32_conv(_fp32_conv(x, blk["conv1"], s, True), blk["conv2"], 1, True, res)
    want, bound = ref.block_forward(k, x)
    r = ((got - want).abs() / bound).max().item()
    assert r <= 1.0, f"fp32 block {k}: max |d| / bound = {r:.3f}"
    assert (got != want).any(), "fp32 rounding never moved an output: the case does not test the bound"


# ---- GPU ---------------------------------------------------------------------------------------------------------
def _check(name, gpu, want, bound):
    """gpu: the GPU's NCHW (or any) float64 CPU tensor; prints max |d| / bound and the bit-identical fraction."""
    assert torch.isfinite(gpu).all(), f"{name}: non-finite outputs"
    assert gpu.shape == want.shape, f"{name}: shape {tuple(gpu.shape)}, expected {tuple(want.shape)}"
    r = (gpu - want).abs() / bound
    worst = int(r.argmax())
    same = (gpu == want).double().mean().item()
    print(f"{name}: max|d|/bound {r.max().item():.3f}  bit-identical {same:.4f}")
    idx = np.unravel_index(worst, tuple(r.shape))
    assert r.max() <= 1.0, (f"{name}: max |d| / bound {r.max().item():.3f} at {idx}: gpu {gpu[idx].item()!r}, "
                            f"reference {want[idx].item()!r}, bound {bound[idx].item():.3g}")
    return r.max().item(), same


class _Cache:
    """Reference results keyed by stage and input bytes: conv_impl 1 and 2 give the same stage outputs, so a
    teacher-forced chain computes each reference once."""

    def __init__(self, ref):
        self.ref, self.d = ref, {}

    def __call__(self, k, x, fmean=None):
        h = hashlib.sha1(x.cpu().numpy().tobytes() + (b"" if fmean is None else fmean.cpu().numpy().tobytes()))
        h = h.hexdigest()
        if (k, h) not in self.d:
            self.d[(k, h)] = self.ref.forward(k, x.cpu() if k == 0 else _nchw(x),
                                              None if fmean is None else fmean.cpu())
        return self.d[(k, h)]


def _stage(ctx, impl, k, x, fmean=None):
    ctx.set_option("conv_impl", impl)
    try:
        return ctx.emb_trunk_stage(k, x, fmean)
    finally:
        ctx.set_option("conv_impl", 1)


IMPLS = [1, 2, 0]


@pytest.fixture(scope="module")
def ctx34():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from pyannote_audio_b200 import ops

    c = ops.Context(torch.device("cuda:0"))
    c.load_embedding(syn.make_embedding_state_dict(1))
    return c


@pytest.fixture(scope="module")
def ref34():
    return _Cache(TrunkRef(syn.make_embedding_state_dict(1)))


@pytest.fixture(scope="module")
def ctx152():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from pyannote_audio_b200 import ops

    c = ops.Context(torch.device("cuda:0"))
    c.load_embedding(syn.make_bottleneck_state_dict(152, 1))
    return c


@pytest.fixture(scope="module")
def ref152():
    return _Cache(TrunkRef(syn.make_bottleneck_state_dict(152, 1)))


def _speech_fbank(ctx, n):
    wav = syn.make_conversation(10.0 * n + 1.0, seed=21)[0].cuda()
    off = np.arange(n, dtype=np.int64) * 160000 + 7
    return ctx.emb_fbank(wav, off, np.full(n, 160000, dtype=np.int32))


def _teacher_forced(ctx, ref, impl, x0, label):
    x, n = x0, len(ctx.emb_blocks) + 1
    for k in range(n):
        y = _stage(ctx, impl, k, x)
        want, bound = ref(k, x, torch.zeros(x.shape[0], 80) if k == 0 else None)
        kind = "stem" if k == 0 else f"block {k - 1}"
        _check(f"{label} impl {impl} stage {k} ({kind}, W {x.shape[-2 if k else 1]})", _nchw(y), want, bound)
        x = y
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
def test_resnet34_every_stage_teacher_forced(ctx34, ref34, impl):
    fb = _speech_fbank(ctx34, 2)
    out = _teacher_forced(ctx34, ref34, impl, fb, "resnet34 speech")
    assert out.shape == (2, 10, 125, 256)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", [1, 2])
def test_chained_stages_are_emb_trunk(ctx34, impl):
    g = torch.Generator().manual_seed(77)
    fb = (torch.randn((3, 998, 80), generator=g) * 2.0 + 0.5).cuda()
    ctx34.set_option("conv_impl", impl)
    try:
        x = fb
        for k in range(len(ctx34.emb_blocks) + 1):
            x = ctx34.emb_trunk_stage(k, x)
        want = ctx34.emb_trunk(fb)
    finally:
        ctx34.set_option("conv_impl", 1)
    assert torch.equal(x.permute(0, 3, 1, 2).float(), want)


# the first block of layers 2-4 (stride 2, 1x1 shortcut) and one stride-1 block of each layer (under conv_impl 1:
# the fused block, the row kernel, the chunk-row kernel on row pairs, the chunk-row kernel on single rows)
SWEEP_STAGES = [4, 8, 14, 2, 5, 9, 15]


@pytest.mark.gpu
@pytest.mark.parametrize("k", SWEEP_STAGES)
def test_resnet34_block_at_widths(ctx34, ref34, k):
    C_in = ctx34.emb_blocks[k - 1][0]
    H = 80 >> sum(b[2] == 2 for b in ctx34.emb_blocks[:k - 1])
    for W in STAGE_WIDTHS:
        x = _activations((2, H, W, C_in), seed=1000 * k + W).cuda()
        for impl in IMPLS:
            want, bound = ref34(k, x)
            _check(f"resnet34 stage {k} W {W} impl {impl}", _nchw(_stage(ctx34, impl, k, x)), want, bound)


@pytest.mark.gpu
@pytest.mark.parametrize("W", [1, 2, 127, 128, 129, 998])
def test_stem_at_widths(ctx34, ref34, W):
    g = torch.Generator().manual_seed(W)
    fb = torch.randn((2, W, 80), generator=g) * 3.0 - 6.0
    fm = torch.randn((2, 80), generator=g) * 2.0 - 6.0
    want, bound = ref34(0, fb, fm)
    for impl in IMPLS:
        _check(f"stem W {W} impl {impl}", _nchw(_stage(ctx34, impl, 0, fb.cuda(), fm.cuda())), want, bound)


@pytest.mark.gpu
@pytest.mark.parametrize("B,W", [(1, 998), (20, 998), (264, 128)])
def test_band_plans(ctx34, ref34, B, W):
    """Short bands (one segment), two bands per column strip (20 segments at 10 s) and full-height bands (a sub-batch
    of 264 short segments) in a stride-1 block of layers 1 and 2.  Segments are independent: the reference covers the
    first, a middle and the last."""
    segs = sorted({0, B // 2, B - 1})
    for k, w in ((2, W), (5, (W - 1) // 2 + 1)):
        C_in = ctx34.emb_blocks[k - 1][0]
        H = 80 >> (k > 4)
        x = _activations((B, H, w, C_in), seed=B * 7 + k).cuda()
        want, bound = ref34(k, x[segs])
        for impl in IMPLS:
            y = _nchw(_stage(ctx34, impl, k, x)[segs])
            _check(f"bands B {B} W {w} stage {k} impl {impl}", y, want, bound)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
def test_bottleneck_every_stage_teacher_forced(ctx152, ref152, impl):
    fb = _speech_fbank(ctx152, 2)[:, 400:530].contiguous()
    out = _teacher_forced(ctx152, ref152, impl, fb, "resnet152 W 130")
    assert out.shape == (2, 10, 17, 1024)


@pytest.mark.gpu
def test_bottleneck_blocks_at_10s(ctx152, ref152):
    """The first block of each layer and one layer-3 block at the widths of a 10 s chunk: 1x1 convs up to 1024
    output channels on 256-wide column tiles, and the chunk-row conv2."""
    blocks = ctx152.emb_blocks
    first = [i for i, b in enumerate(blocks) if i == 0 or b[0] != b[1]]
    for k in [i + 1 for i in first] + [first[2] + 2]:
        C_in = blocks[k - 1][0]
        strides = sum(b[2] == 2 for b in blocks[:k - 1])
        H, W = 80 >> strides, 998
        for _ in range(strides):
            W = (W - 1) // 2 + 1
        x = _activations((1, H, W, C_in), seed=k).cuda()
        want, bound = ref152(k, x)
        for impl in IMPLS:
            _check(f"resnet152 stage {k} W {W} impl {impl}", _nchw(_stage(ctx152, impl, k, x)), want, bound)


# ---- the fbank ---------------------------------------------------------------------------------------------------
K_EPS = float(np.finfo(np.float32).eps)   # the log floor: torchaudio's EPSILON in the input's dtype, the kernel's kEps
FBANK_VALID = [0, 1, 399, 400, 401, 559, 560, 561, 16000, 159999, 160000]
FBANK_A = 1.0        # per-bin spectral error of the fp32 fbank, in float32 eps per unit of the frame's L2 norms


def _mel_banks():
    """(torchaudio's mel bank, the library's): kaldi.get_mel_banks builds its triangles in float32 whatever the input's
    dtype, the library in float64 rounded once to float32 (build_fbank_constants).  Near the triangles' edges they
    differ by up to 1.4e-5 per weight, 8e-4 of a small weight, which moves a weak mel bin next to a loud one by many
    float32 eps: the oracle's own error, not the kernel's.  Both (80, 257), zero Nyquist column."""
    import torchaudio.compliance.kaldi as kaldi

    def mel(f):
        return 1127.0 * torch.log1p(f / 700.0)

    ml, mh = mel(torch.tensor(20.0, dtype=torch.float64)), mel(torch.tensor(8000.0, dtype=torch.float64))
    delta = (mh - ml) / 81
    left = ml + torch.arange(80, dtype=torch.float64)[:, None] * delta
    m = mel(16000.0 / 512 * torch.arange(256, dtype=torch.float64))[None]
    lib = torch.clamp(torch.minimum((m - left) / delta, (left + 2 * delta - m) / delta), min=0).float().double()
    ta = kaldi.get_mel_banks(80, 512, 16000.0, 20.0, 0.0, 100.0, -500.0, 1.0)[0].double()
    return F.pad(ta, (0, 1)), F.pad(lib, (0, 1))


def _fbank_ref(chunk, mel):
    """compute_fbank's steps in float64 on one 160000-sample chunk with the mel bank ``mel`` -> (centred log mel
    (998, 80), mel energies E, power spectrum P (998, 257), per-frame spectral error scale dX (998, 1): the L2 norms
    of the frame as scaled and as windowed).  With torchaudio's bank this is the oracle's compute_fbank
    (test_fbank_reference_is_the_oracle)."""
    import math

    x = chunk.double() * 32768.0
    fr = x.unfold(0, 400, 160)                                        # (998, 400) snip_edges frames
    v = fr - fr.mean(1, keepdim=True)
    v = torch.cat([v[:, :1] - 0.97 * v[:, :1], v[:, 1:] - 0.97 * v[:, :-1]], 1)
    n = torch.arange(400, dtype=torch.float64)
    v = v * (0.54 - 0.46 * torch.cos(2 * math.pi * n / 399))
    P = torch.fft.rfft(v, n=512).abs() ** 2                           # (998, 257)
    E = P @ mel.T
    lm = torch.log(E.clamp_min(K_EPS))
    return lm - lm.mean(0, keepdim=True), E, P, (v.norm(dim=1) + fr.norm(dim=1)).unsqueeze(1)


def _fbank_bound(E, P, dX, mel, a=FBANK_A, dmel=None):
    """Bound on |gpu - ref| of the centred fbank.  A spectral error e = a eps32 dX per bin moves E by at most
    sum_i w_i (2 |X_i| e + e^2) (+ sum_i |dmel_i| P_i for a different mel bank); the bound is the width of that
    interval in the log domain, with the floor exact, plus float32 rounding of the mel sum and the log, and the same
    over the frame mean for the centring.  The e^2 term is the fp32 residue of a frame whose exact energy is zero
    (a DC offset: the fp32 frame mean is not exact)."""
    e = a * U32 * dX
    dE = 2 * (P.sqrt() @ mel.T) * e + (e ** 2) * mel.sum(1) + 4 * U32 * E
    if dmel is not None:
        dE = dE + P @ dmel.abs().T
    lo, hi = torch.log((E - dE).clamp_min(K_EPS)), torch.log((E + dE).clamp_min(K_EPS))
    b = (hi - lo) + 2 * U32 * (1 + hi.abs())
    return b + b.mean(0, keepdim=True)


def test_fbank_reference_is_the_oracle():
    from oracle import nets

    g = torch.Generator().manual_seed(3)
    chunk = torch.randn(160000, generator=g, dtype=torch.float64) * 0.1
    chunk[100000:] = 0
    want = nets.WeSpeakerResNet34.compute_fbank(chunk[None, None])[0]
    ta, lib = _mel_banks()
    got, *_ = _fbank_ref(chunk, ta)
    assert (got - want).abs().max() <= 1e-9
    assert 1e-6 < (ta - lib).abs().max() < 2e-5          # the two banks differ as _mel_banks says


def _fbank_inputs(n):
    """Five signals of n samples: speech, silence, a DC offset, a +-1 square wave and speech at 1e-4."""
    sp = syn.make_conversation(n / 16000.0 + 0.1, seed=5)[0][:n]
    t = torch.arange(n)
    return {"speech": sp, "silence": torch.zeros(n), "dc": torch.full((n,), 0.3),
            "square": torch.where((t // 37) % 2 == 0, 1.0, -1.0), "quiet": sp * 1e-4}


@pytest.mark.gpu
def test_fbank_against_float64_oracle(ctx34):
    """ctx.emb_fbank (centred) against the fbank in float64: chunks whose valid samples end around one frame (400),
    the second frame (560), 1 s and the full 10 s, at odd offsets.  A silent chunk and an empty one are exactly zero
    after centring (the kernel's fp64 mean of 998 equal frames is exact).  Every other chunk is held to the bound of
    _fbank_bound against the float64 fbank with the library's mel bank, and to that bound plus the two banks'
    difference against the oracle's compute_fbank itself."""
    from oracle import nets

    ta, lib = _mel_banks()
    off = np.arange(len(FBANK_VALID), dtype=np.int64) * 160037 + 13
    valid = np.array(FBANK_VALID, dtype=np.int32)
    report = []
    for name, wav in _fbank_inputs(int(off[-1]) + 160000 + 1).items():
        got = ctx34.emb_fbank(wav.float().cuda(), off, valid).double().cpu()
        for i, (o, v) in enumerate(zip(off, valid)):
            if name == "silence" or v == 0:
                assert torch.equal(got[i], torch.zeros_like(got[i])), f"{name} valid {v}: not exactly zero"
                continue
            chunk = torch.zeros(160000, dtype=torch.float64)
            chunk[:v] = wav[o:o + v].double()
            want, E, P, dX = _fbank_ref(chunk, lib)
            oracle = nets.WeSpeakerResNet34.compute_fbank(chunk[None, None])[0]
            r = ((got[i] - want).abs() / _fbank_bound(E, P, dX, lib)).max().item()
            ro = ((got[i] - oracle).abs() / _fbank_bound(E, P, dX, lib, dmel=ta - lib)).max().item()
            report.append((r, ro, (got[i] - want).abs().max().item(), (got[i] - oracle).abs().max().item(), name,
                           int(v)))
    for name in ("speech", "dc", "square", "quiet"):
        rs = [r for r in report if r[4] == name]
        print(f"fbank {name}: max|d|/bound {max(r[0] for r in rs):.3f} (vs the oracle {max(r[1] for r in rs):.3f}), "
              f"max|d| {max(r[2] for r in rs):.3g} (vs the oracle {max(r[3] for r in rs):.3g}), "
              f"valid lengths with |d| >= 1e-3: {[r[5] for r in rs if r[3] >= 1e-3]}")
    assert max(r[0] for r in report) <= 1.0 and max(r[1] for r in report) <= 1.0
