"""PyanNet's segmentation stack, stage by stage, against a float64 reference that rounds where the kernels round.

The end-to-end tests see the SincNet front end only through four BiLSTM layers and a log-softmax, and a recurrence
error only through the layers after it, where saturated gates compress it.  Here every stage the kernels hand to the
next one (Context.seg_stages, Context.seg_head_stages) is compared with a float64 reference fed the GPU's own input of
that stage (teacher forcing), so a fault shows in the stage that makes it.

The reference uses the weights as loaded: the float32 sinc bank of ops.sinc_filter_bank, b_g = fl32(b_ih + b_hh), and
under the split-precision kernels (impl 1 and 2) every tensor-core operand as the fp16 pair hi = rn16(v),
lo = rn16(fl32(v - hi)), with the lo * lo product dropped.  Under the fp32 twins (impl 0) it uses the float32 values.
It sums in float64, and the GPU may differ from it by

    |gpu - ref| <= ulp32(y) + C * 2^-23 * (|b| + sum |x| |w|)

per element (a maximum of three such terms where MaxPool 3 picks one).  C is 8 for the fp32 twins.  The tensor cores
add each of a K-long sum's 3 * K / 16 split products into the fp32 accumulator with truncation (SegRef.acc), so there
C is 8 + 3 * ceil(K / 16).  With C = 8 alone the sinc layer failed on the H100, by up to 1.86 x the bound.  That
happened only where one product dominates the sum: an impulse, or the sample where a window's valid part ends.  At
the worst element of every failing case the GPU's |P0| was below the reference's, as truncation makes it.  Where the
GPU stores an fp16 (hi, lo) pair, the bound adds the pair's own representation error 2^-25 + 2^-22 |y|, because lo is
subnormal once |y| < 1/8.

* Affines (wav_norm1d, norm1d.0-2) are (scale, shift) pairs.  They must lie within two roundings of the float64
  statistics of the GPU's own stage output (zero padding counts, eps 1e-5): |d scale| <= 2^-23 |scale| and
  |d shift| <= ulp32(shift) + 2^-22 |mean scale|.  The next stage then reads the GPU's affine.
* Conv stages read leaky_relu(fmaf(P, scale, shift)) in float32, split, then apply |.| (sinc only), MaxPool 3 and the
  bias.
* x0 must be within one ulp of leaky_relu(fmaf(P2, affine)), and its 4 pad columns exactly 0.
* Gx_l is the GPU's input (x0 split, or Y_{l-1} as stored) times W_ih, plus b_g.
* The recurrence is teacher-forced per step.  Step t takes the GPU's h_{t-1} from Y_l as stored, the GPU's Gx_l and
  the reference's own float64 cell state.  The cell state's error is carried as e_c(t) = |f| e_c(t-1) + local(t).
  local(t) covers the fp32 gate sums, the fp32 transcendentals (4 * 2^-23 relative, and 2^-126 absolute where a gate
  underflows) and sigmoid' / tanh' at the reference's values.  Each GPU h_t must lie within
  |o| (1 - tanh^2 c) e_c(t) + local_h(t).  h errors are not propagated through sum |W_hh|: that bound grows
  geometrically over 1775 steps.
* Linears and classifier: Z1 comes from the GPU's Y_last, Z2 from the GPU's Z1, and the classifier runs on the GPU's
  Z2.  cls must be the reference's argmax, except where the top two reference logits are within twice the logit
  bound.

CPU tests:
* With rounding off, the reference equals oracle.nets.PyanNet's SincNet, each nn.LSTM layer and the head in float64,
  to 1e-12 relative.
* An honest float32 computation of the same operands stays inside every bound.  Its max |d| / bound (median), for
  synthetic weights (seed 0), split operands / float32 operands:
      sinc 0.07 (0.001) / 0.54 (0.01)    conv1 0.02 (0.001) / 0.15 (0.01)    conv2 0.04 (0.002) / 0.25 (0.02)
      Gx 0.19 (0.007) / 0.42 (0.02)      h, T = 1775: 0.08 (0.007) / 0.76 (0.004), and 0.91 (0.02) with
      ih_gain = hh_gain = 1.
* On 10 s of speech, 95.7 % of the gate pre-activations have |z| < 2 with the default synthetic gains, and 99.99 %
  with ih_gain = hh_gain = 1.  The GPU recurrence cases run both weight sets.

GPU: `pytest -s` prints max |d| / bound, its median and the bit-identical fraction per stage.  Measured on an NVIDIA
H100 80GB HBM3 at a 700 W power limit, worst case over every window, input, sequence count and length; tensor cores
(impl 1 and 2, bit-identical to each other) / fp32 twins (impl 0):
    af_wav  0.75 / 0.75     af0-af2  0.95 / 0.95
    P0      0.29 / 0.56     P1       0.15 / 0.57     P2   0.15 / 0.44     x0   0 / 0 (bit-identical: 1.0000)
    Gx      0.24 / 0.48     z1       0.09 / 0.35     z2   0.14 / 0.40
    h, default gains 1.00 / 0.93    h, ih_gain = hh_gain = 1: 1.00 / 0.68    h, SSeRiouSS: 0.84 / 0.36
    logp    0.06 / 0.06     sigmoid scores 0.05 / 0.07
The medians of |d| / bound are at most 0.25 (affines), 0.02 (every other stage) and 0.04 (h).  Under the tensor cores,
h reaches 1.00 only where |h| < 1/8: the stored pair is then off by half the fp16 subnormal spacing of lo, 2^-25, which
is the whole bound when the arithmetic error is far smaller.  Bit-identical fractions: x0 1.0 under every impl; P0
0.16-0.19 under impl 0 and at most 0.002 under the tensor cores; affine shifts in up to 40 % of the windows; the
log-probabilities of the K = 1 head (exactly 0) and the dominant class of the K = 7 head; every other stage 0.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pyannote_audio_b200 import ops
from pyannote_audio_b200.testing import synthetic as syn

U32 = 2.0 ** -23              # float32 epsilon
C_ACC = 8                     # fp32 accumulation, any order
FLT_MIN = 2.0 ** -126         # float32 gates below this underflow (expf overflows past |z| ~ 88)
C_TR = 4                      # fp32 expf / tanhf / division, relative
SLOPE = float(np.float32(0.01))   # leaky_relu's slope as the kernels multiply it (0.01f)
SR = 16000


# ---- rounding helpers ----------------------------------------------------------------------------------------------
def fl32(x):
    return x.float().double()


def rn16(x):
    """fp16 round-to-nearest-even of float64 tensors holding float32 values (exact through float32)."""
    return x.float().half().double()


def split(v, mode):
    """(hi, lo) of float32 values v as split_f16 / the staging loops form them; mode "fp32": (v, 0); None: (v, 0)."""
    if mode == "split":
        hi = rn16(v)
        return hi, rn16(fl32(v - hi))
    return v, torch.zeros_like(v)


def ulp32(y):
    """Spacing of float32 at |y| (float64 y): the larger of the two at a binade edge."""
    a = y.abs()
    _, e = torch.frexp(a)
    ulp = torch.pow(2.0, (e - 1).clamp_min(-126).double() - 23)
    return torch.where(a == 0, torch.full_like(a, 2.0 ** -149), ulp)


def store_err(y, mode):
    """Representation error of an fp16 (hi, lo) store of y (lo may be subnormal), or 0 for float32 stores."""
    return 2.0 ** -25 + 2.0 ** -22 * y.abs() if mode == "split" else torch.zeros_like(y)


def mm3(a, w, mode):
    """a @ w^T as the kernels multiply: split operands, lo * lo dropped; and sum |a| |w| for the bound."""
    ah, al = a if isinstance(a, tuple) else split(a, mode)
    wh, wl = split(w, mode)
    y = ah @ wh.T + ah @ wl.T + al @ wh.T if mode == "split" else ah @ wh.T
    return y, (ah.abs() + al.abs()) @ w.abs().T


def leaky32(v, mode):
    """leaky_relu of float32 values as the kernels form it (v > 0 ? v : 0.01f * v); exact for mode None."""
    if mode is None:
        return torch.where(v > 0, v, 0.01 * v)
    return torch.where(v > 0, v, fl32(v * SLOPE))


def fma32(p, sc, sh, mode):
    """fmaf(p, sc, sh) in float32 (p * sc is exact in float64), or exactly for mode None."""
    z = p * sc + sh
    return z if mode is None else fl32(z)


# ---- the reference -------------------------------------------------------------------------------------------------
def affine(x, gamma, beta):
    """InstanceNorm over the last axis (zero padding included) as float64 (scale, shift) and their bounds."""
    mean = x.mean(-1)
    var = (x * x).mean(-1) - mean * mean
    var = var.clamp_min(0)
    sc = gamma / torch.sqrt(var + 1e-5)
    sh = beta - mean * sc
    return sc, sh, 2.0 ** -23 * sc.abs(), ulp32(sh) + 2.0 ** -22 * (mean * sc).abs()


class SegRef:
    """PyanNet's stages in float64 on the weights as loaded.  mode: "split" (fp16 pairs, impl 1 and 2), "fp32"
    (impl 0) or None (exact, the network itself)."""

    def __init__(self, sd, mode="split"):
        self.mode = mode
        d = lambda k: sd[k].detach().double()          # noqa: E731
        p = "sincnet.conv1d.0.filterbank."
        self.bank = ops.sinc_filter_bank(sd[p + "low_hz_"], sd[p + "band_hz_"], sd.get(p + "window_"),
                                         sd.get(p + "n_")).double()
        self.wav_gb = (float(sd["sincnet.wav_norm1d.weight"].reshape(-1)[0]),
                       float(sd["sincnet.wav_norm1d.bias"].reshape(-1)[0]))
        self.norm = [(d(f"sincnet.norm1d.{i}.weight"), d(f"sincnet.norm1d.{i}.bias")) for i in range(3)]
        self.conv = [(d(f"sincnet.conv1d.{i}.weight"), d(f"sincnet.conv1d.{i}.bias")) for i in (1, 2)]
        self.layers = 0
        while f"lstm.weight_ih_l{self.layers}" in sd:
            self.layers += 1
        self.lstm = []
        for layer in range(self.layers):
            per_dir = []
            for suffix in ("", "_reverse"):
                w_ih, w_hh = d(f"lstm.weight_ih_l{layer}{suffix}"), d(f"lstm.weight_hh_l{layer}{suffix}")
                b_ih, b_hh = d(f"lstm.bias_ih_l{layer}{suffix}"), d(f"lstm.bias_hh_l{layer}{suffix}")
                b = b_ih + b_hh if mode is None else fl32(b_ih + b_hh)
                per_dir.append((w_ih, w_hh, b))
            self.lstm.append(per_dir)
        self.lin = [(d(f"linear.{i}.weight"), d(f"linear.{i}.bias")) for i in range(2)]
        self.cls = (d("classifier.weight"), d("classifier.bias"))

    def acc(self, K):
        """Accumulation constant of a K-long sum.  The fp32 twins: C_ACC.  wgmma: each K = 16 step adds three products
        (lo * hi, hi * lo, hi * hi) into the fp32 accumulator, and the tensor cores align and truncate (round toward
        zero) at every such addition (Fasi, Higham, Mikaitis, Pranesh, "Numerical behavior of NVIDIA tensor cores",
        PeerJ CS 2021): up to one ulp of the partial sum per addition, 3 * ceil(K / 16) of them, plus C_ACC."""
        return C_ACC + (3 * -(-K // 16) if self.mode == "split" else 0)

    # -- SincNet --
    def wav_affine(self, windows):
        return affine(windows, *self.wav_gb)

    def sinc(self, windows, sc, sh):
        """windows (n, W) raw samples as the kernels read them (zeros past valid), GPU affine -> P0 (n, 80, pool0)."""
        x = fma32(windows, sc[:, None], sh[:, None], self.mode)
        pool0 = (1 + (x.shape[1] - 251) // 10) // 3
        ys, ms = [], []
        for b in range(x.shape[0]):              # one window at a time: the unfolded input is 251 x larger
            xu = x[b].unfold(0, 251, 10)[:3 * pool0]
            y, m = mm3(xu, self.bank, self.mode)
            ys.append(y.abs().view(pool0, 3, 80).amax(1).T)
            ms.append(m.view(pool0, 3, 80).amax(1).T)
        y, m = torch.stack(ys), torch.stack(ms)
        return y, ulp32(y) + self.acc(256) * U32 * m

    def conv_stage(self, i, P, sc, sh):
        """Conv1d i (0, 1) on the GPU's P (n, C, L) and affine -> (n, 60, pool)."""
        w, b = self.conv[i]
        x = leaky32(fma32(P, sc[..., None], sh[..., None], self.mode), self.mode)
        n, C, L = x.shape
        pool = (L - 4) // 3
        xu = x.unfold(2, 5, 1).permute(0, 2, 1, 3).reshape(n, L - 4, C * 5)[:, :3 * pool]
        y, m = mm3(xu, w.reshape(60, C * 5), self.mode)
        y = y.view(n, pool, 3, 60).amax(2).transpose(1, 2) + b[:, None]
        m = m.view(n, pool, 3, 60).amax(2).transpose(1, 2) + b.abs()[:, None]
        return y, ulp32(y) + self.acc(5 * (80 if C == 80 else 64)) * U32 * m

    def x0(self, P2, sc, sh):
        return leaky32(fma32(P2, sc[..., None], sh[..., None], self.mode), self.mode).transpose(1, 2)

    # -- head --
    def gx(self, layer, inp):
        """inp: (rows, k) values or an (hi, lo) pair as the GPU stored them -> per direction (rows, 512) in PyTorch
        gate order, with the bound."""
        out = []
        for w_ih, _, b in self.lstm[layer]:
            if not isinstance(inp, tuple) and inp.shape[-1] > w_ih.shape[1]:
                inp = inp[..., :w_ih.shape[1]]          # x0's pad columns: zero weights in the kernels
            if isinstance(inp, tuple) and inp[0].shape[-1] > w_ih.shape[1]:
                inp = (inp[0][..., :w_ih.shape[1]], inp[1][..., :w_ih.shape[1]])
            y, m = mm3(inp, w_ih, self.mode)
            y = y + b
            out.append((y, ulp32(y) + self.acc(w_ih.shape[1]) * U32 * (m + b.abs())))
        return out

    def recurrence(self, layer, d, gx, y_prev):
        """Teacher-forced direction d of a layer on one batch of sequences.  gx (n, T, 512) the GPU's projection in
        PyTorch gate order, y_prev the GPU's layer output of this direction (n, T, 128): values, or an (hi, lo) pair.
        Returns (h reference (n, T, 128), bound)."""
        _, w_hh, _ = self.lstm[layer][d]
        if isinstance(y_prev, tuple):
            hp = [torch.zeros_like(y_prev[0]), torch.zeros_like(y_prev[1])]
            src = y_prev
        else:
            hp = [torch.zeros_like(y_prev)]
            src = (y_prev,)
        # h_{t-1} of every step: the previous step in the direction of travel, zero at the first
        for k, s in enumerate(src):
            if d == 0:
                hp[k][:, 1:] = s[:, :-1]
            else:
                hp[k][:, :-1] = s[:, 1:]
        z, m = mm3(tuple(hp) if len(hp) == 2 else hp[0], w_hh, self.mode)
        z = gx + z
        ez = self.acc(128) * U32 * (gx.abs() + m)
        zi, zf, zg, zo = z.split(128, -1)
        ei, ef, eg, eo = ez.split(128, -1)
        i, f, g, o = torch.sigmoid(zi), torch.sigmoid(zf), torch.tanh(zg), torch.sigmoid(zo)
        e_i = i * (1 - i) * ei + C_TR * U32 * i + FLT_MIN
        e_f = f * (1 - f) * ef + C_TR * U32 * f + FLT_MIN
        e_o = o * (1 - o) * eo + C_TR * U32 * o + FLT_MIN
        e_g = (1 - g * g) * eg + C_TR * U32 * g.abs() + FLT_MIN
        ig = (i * g).numpy()
        fn = f.numpy()
        T = z.shape[1]
        c = np.zeros_like(ig)
        ec = np.zeros_like(ig)
        cprev = np.zeros(ig[:, 0].shape)
        eprev = np.zeros_like(cprev)
        e_f_, e_i_, e_g_, i_, g_ = (t.numpy() for t in (e_f, e_i, e_g, i, g))
        order = range(T) if d == 0 else range(T - 1, -1, -1)
        for t in order:
            local = (np.abs(cprev) * e_f_[:, t] + np.abs(g_[:, t]) * e_i_[:, t] + np.abs(i_[:, t]) * e_g_[:, t]
                     + 2 * U32 * (np.abs(fn[:, t] * cprev) + np.abs(ig[:, t])))
            cprev = fn[:, t] * cprev + ig[:, t]
            eprev = fn[:, t] * eprev + local
            c[:, t], ec[:, t] = cprev, eprev
        c, ec = torch.from_numpy(c), torch.from_numpy(ec)
        tc = torch.tanh(c)
        h = o * tc
        bound = (tc.abs() * e_o + o * (1 - tc * tc) * ec + C_TR * U32 * h.abs() + U32 * h.abs() + FLT_MIN
                 + store_err(h, self.mode))
        return h, bound

    def linear(self, i, inp):
        w, b = self.lin[i]
        y, m = mm3(inp, w, self.mode)
        y = y + b
        y = torch.where(y > 0, y, y * (0.01 if self.mode is None else SLOPE))
        return y, ulp32(y) + self.acc(w.shape[1]) * U32 * (m + b.abs())

    def logits(self, z2):
        w, b = self.cls
        v = z2 @ w.T + b
        return v, C_ACC * U32 * (z2.abs() @ w.abs().T + b.abs())


# ---- GPU output in reference layouts -------------------------------------------------------------------------------
def _val(t):
    """A captured tensor as float64 values: fp32 as is, an (hi, lo) pair as hi + lo."""
    if isinstance(t, tuple):
        return t[0].double().cpu() + t[1].double().cpu()
    return t.double().cpu()


def _pair(t):
    return (t[0].double().cpu(), t[1].double().cpu()) if isinstance(t, tuple) else t.double().cpu()


def _sel(t, seqs):
    return tuple(x[seqs] for x in t) if isinstance(t, tuple) else t[seqs]


def _gates_torch_order(gx):
    """GPU Gx (n, T, 1024), column dir * 512 + unit * 4 + gate -> (n, T, 2, 512) in PyTorch's gate * 128 + unit."""
    n, T, _ = gx.shape
    return gx.view(n, T, 2, 128, 4).transpose(3, 4).reshape(n, T, 2, 512)


def _half(t, d):
    """Direction d's 128 units of a layer output (values or an (hi, lo) pair)."""
    if isinstance(t, tuple):
        return tuple(x[..., 128 * d: 128 * (d + 1)] for x in t)
    return t[..., 128 * d: 128 * (d + 1)]


# ---- checks --------------------------------------------------------------------------------------------------------
def _check(name, gpu, want, bound, log=None):
    gpu, want, bound = gpu.double(), want.double(), bound.double()
    assert gpu.shape == want.shape, f"{name}: shape {tuple(gpu.shape)}, expected {tuple(want.shape)}"
    assert torch.isfinite(gpu).all(), f"{name}: non-finite outputs"
    r = (gpu - want).abs() / bound
    same = (gpu == want).double().mean().item()
    worst = int(r.argmax())
    idx = np.unravel_index(worst, tuple(r.shape))
    print(f"{name}: max|d|/bound {r.max().item():.3f}  median {r.median().item():.3f}  bit-identical {same:.4f}")
    if log is not None:
        log.setdefault(name.split("[")[0], []).append((r.max().item(), same))
    assert r.max() <= 1.0, (f"{name}: max |d| / bound {r.max().item():.3f} at {idx}: gpu {gpu[idx].item()!r}, "
                            f"reference {want[idx].item()!r}, bound {bound[idx].item():.3g}")
    return r


def check_head(ref, x0, cap, seqs, tag="", log=None):
    """Every head stage of a capture (Context.seg_head_stages / seg_stages) on the sequences ``seqs``, teacher-forced
    from the GPU's own inputs."""
    mode = ref.mode
    inp = _sel(x0.double().cpu(), seqs)
    if mode == "split":
        inp = split(inp, "split")
    for layer in range(ref.layers):
        gx_gpu = _gates_torch_order(cap["gx"][layer][seqs].double().cpu())
        for d, (want, bound) in enumerate(ref.gx(layer, inp)):
            _check(f"gx{layer}.{d}{tag}", gx_gpu[:, :, d], want, bound, log)
        y = _pair(_sel(cap["y"][layer], seqs))
        for d in range(2):
            yd = _half(y, d)
            h, bound = ref.recurrence(layer, d, gx_gpu[:, :, d], yd)
            _check(f"h{layer}.{d}{tag}", _val(yd), h, bound, log)
        inp = y
    z1, bz1 = ref.linear(0, inp)
    z1_gpu = _pair(_sel(cap["z1"], seqs))
    _check(f"z1{tag}", _val(z1_gpu), z1, bz1 + store_err(z1, mode), log)
    z2, bz2 = ref.linear(1, z1_gpu)
    z2_gpu = cap["z2"][seqs].double().cpu()
    _check(f"z2{tag}", z2_gpu, z2, bz2, log)
    v, ev = ref.logits(z2_gpu)
    K = v.shape[-1]
    if "scores" in cap:
        s = torch.sigmoid(v)
        bound = s * (1 - s) * ev + C_TR * U32 * s + ulp32(s)
        sc = cap["scores"][seqs].double().cpu()
        _check(f"scores{tag}", sc, s, bound, log)
        assert torch.equal(cap["max_scores"][seqs].cpu(), cap["scores"][seqs].amax(-1).cpu()), "max_scores"
        return
    lp = v - torch.logsumexp(v, -1, keepdim=True)
    emax = ev.amax(-1, keepdim=True)
    bound = ev + emax + (K + 4) * U32 + ulp32(v - v.amax(-1, keepdim=True)) + ulp32(lp)
    _check(f"logp{tag}", cap["logp"][seqs].double().cpu(), lp, bound, log)
    cls = cap["cls"][seqs].long().cpu()
    top = v.amax(-1)
    picked = v.gather(-1, cls[..., None])[..., 0]
    bad = picked < top - 2 * emax[..., 0]
    assert not bad.any(), f"cls{tag}: {int(bad.sum())} frames pick a class below the reference's top"


# ---- CPU: the reference is the network, and its bounds admit fp32 arithmetic -----------------------------------
def _speech(n, seed):
    return syn.make_conversation(max(n, SR) / SR, seed=seed)[0, :n].double()


def test_reference_without_rounding_is_the_network():
    from oracle import nets

    sd = syn.make_segmentation_state_dict(0)
    net = nets.PyanNet()
    net.load_state_dict(sd, strict=False)
    net = net.double().eval()
    ref = SegRef(sd, mode=None)
    ref.bank = net.sincnet.conv1d[0].filterbank.filters()[:, 0].detach()   # the bank in float64, not float32
    wav = torch.stack([_speech(20000, 3), torch.cat([_speech(15000, 4), torch.zeros(5000, dtype=torch.float64)])])
    with torch.no_grad():
        s = net.sincnet
        want = [s.wav_norm1d(wav[:, None])]
        x = want[0]
        for c in range(3):
            x = s.conv1d[c](x)
            if c == 0:
                x = x.abs()
            x = s.pool1d[c](x)
            want.append(x)
            x = F.leaky_relu(s.norm1d[c](x))
        want_x0 = x.transpose(1, 2)
        sc, sh, _, _ = ref.wav_affine(wav)
        assert (sc[:, None] * wav + sh[:, None] - want[0][:, 0]).abs().max() <= 1e-12 * want[0].abs().max()
        P0, _ = ref.sinc(wav, sc, sh)
        assert (P0 - want[1]).abs().max() <= 1e-12 * want[1].abs().max()
        P = P0
        for i in range(2):
            sc, sh, _, _ = affine(P, *ref.norm[i])
            P, _ = ref.conv_stage(i, P, sc, sh)
            assert (P - want[i + 2]).abs().max() <= 1e-12 * want[i + 2].abs().max()
        sc, sh, _, _ = affine(P, *ref.norm[2])
        x0 = ref.x0(P, sc, sh)
        assert (x0 - want_x0).abs().max() <= 1e-12 * want_x0.abs().max()

        # each LSTM layer against nn.LSTM in double, teacher-forced from nn.LSTM's own outputs
        inp = want_x0
        for layer in range(ref.layers):
            lstm = torch.nn.LSTM(60 if layer == 0 else 256, 128, batch_first=True, bidirectional=True).double()
            lstm.load_state_dict({k[5:].replace(f"_l{layer}", "_l0"): v.double() for k, v in sd.items()
                                  if k.startswith("lstm.") and f"_l{layer}" in k})
            out, _ = lstm(inp)
            for d, (gx, _) in enumerate(ref.gx(layer, inp)):
                h, _ = ref.recurrence(layer, d, gx, out[..., 128 * d: 128 * (d + 1)])
                assert (h - out[..., 128 * d: 128 * (d + 1)]).abs().max() <= 1e-12
            inp = out
        z1, _ = ref.linear(0, inp)
        z2, _ = ref.linear(1, z1)
        v, _ = ref.logits(z2)
        lp = v - torch.logsumexp(v, -1, keepdim=True)
        want_lp = net(wav[:, None])
        assert (lp - want_lp).abs().max() <= 1e-12 * want_lp.abs().max()


def _fp32_mm(a, w, mode):
    """a @ w^T in float32 on the split operands (each product a float32 matmul, summed in float32)."""
    ah, al = a if isinstance(a, tuple) else split(a, mode)
    wh, wl = split(w, mode)
    f = lambda x, y: x.float() @ y.float().T     # noqa: E731
    y = (f(al, wh) + f(ah, wl)) + f(ah, wh) if mode == "split" else f(ah, wh)
    return y.double()


def _fp32_store(y, mode):
    return split(fl32(y), "split") if mode == "split" else fl32(y)


def _fp32_recurrence(ref, layer, d, gx, mode):
    """An honest float32 run of one direction: fp32 gates and cell, h stored as the kernels store it."""
    _, w_hh, _ = ref.lstm[layer][d]
    n, T, _ = gx.shape
    c = torch.zeros((n, 128))
    h = _fp32_store(torch.zeros((n, 128), dtype=torch.float64), mode)
    out = [None] * T
    for t in (range(T) if d == 0 else range(T - 1, -1, -1)):
        z = (gx[:, t].float() + _fp32_mm(h, w_hh, mode).float())
        zi, zf, zg, zo = z.split(128, -1)
        c = torch.sigmoid(zf) * c + torch.sigmoid(zi) * torch.tanh(zg)
        hv = torch.sigmoid(zo) * torch.tanh(c)
        h = _fp32_store(hv.double(), mode)
        out[t] = h
    if mode == "split":
        return torch.stack([o[0] for o in out], 1), torch.stack([o[1] for o in out], 1)
    return torch.stack(out, 1)


@pytest.mark.parametrize("mode", ["split", "fp32"])
def test_fp32_computation_is_within_the_bounds(mode):
    """The same stages computed honestly in float32 on the same (split) operands stay inside every bound: the bounds
    are not tighter than float32 arithmetic allows."""
    sd = syn.make_segmentation_state_dict(0)
    ref = SegRef(sd, mode)
    W = 20000
    wav = torch.stack([fl32(_speech(W, 5)), torch.cat([fl32(_speech(7777, 6)), torch.zeros(W - 7777).double()])])
    sc, sh, _, _ = ref.wav_affine(wav)
    sc, sh = fl32(sc), fl32(sh)
    x = fma32(wav, sc[:, None], sh[:, None], mode)
    pool0 = (1 + (W - 251) // 10) // 3
    got = torch.stack([_fp32_mm(x[b].unfold(0, 251, 10)[:3 * pool0], ref.bank, mode).abs().view(pool0, 3, 80)
                       .amax(1).T for b in range(2)])
    want, bound = ref.sinc(wav, sc, sh)
    _check("fp32 sinc", got, want, bound)
    P = fl32(got)
    for i in range(2):
        sc, sh, _, _ = affine(P, *ref.norm[i])
        sc, sh = fl32(sc), fl32(sh)
        w, b = ref.conv[i]
        xx = leaky32(fma32(P, sc[..., None], sh[..., None], mode), mode)
        n, C, L = xx.shape
        pool = (L - 4) // 3
        xu = xx.unfold(2, 5, 1).permute(0, 2, 1, 3).reshape(n, L - 4, C * 5)[:, :3 * pool]
        y = _fp32_mm(xu, w.reshape(60, C * 5), mode).view(n, pool, 3, 60).amax(2).transpose(1, 2)
        got = fl32(y + b[:, None])
        want, bound = ref.conv_stage(i, P, sc, sh)
        _check(f"fp32 conv{i + 1}", got, want, bound)
        P = got
    # the head on random SincNet-like inputs, T = 1775, for both weight sets
    for gains in ({}, {"ih_gain": 1.0, "hh_gain": 1.0}):
        ref = SegRef(syn.make_segmentation_state_dict(0, **gains), mode)
        g = torch.Generator().manual_seed(9)
        x0 = fl32(leaky32(torch.randn((2, 1775, 60), generator=g, dtype=torch.float64), None))
        inp = split(x0, mode) if mode == "split" else x0
        for layer in range(2):
            ys = []
            for d, (want, bound) in enumerate(ref.gx(layer, inp)):
                w_ih, _, b = ref.lstm[layer][d]
                gx = fl32(_fp32_mm(inp, w_ih, mode) + b)
                _check(f"fp32 gx{layer}.{d}", gx, want, bound)
                y = _fp32_recurrence(ref, layer, d, gx, mode)
                h, hb = ref.recurrence(layer, d, gx, y)
                _check(f"fp32 h{layer}.{d} {gains}", _val(y), h, hb)
                ys.append(y)
            inp = (torch.cat([ys[0][0], ys[1][0]], -1), torch.cat([ys[0][1], ys[1][1]], -1)) if mode == "split" \
                else torch.cat(ys, -1)


def test_gate_sensitivity_of_the_synthetic_weights():
    """Share of gate pre-activations with |z| < 2 on 10 s of speech: the default synthetic gains saturate many gates,
    ih_gain = hh_gain = 1 keeps most of them sensitive, so the GPU recurrence cases run both."""
    from oracle import nets

    wav = syn.make_conversation(10.0, seed=11)[None]
    shares = []
    for gains in ({}, {"ih_gain": 1.0, "hh_gain": 1.0}):
        sd = syn.make_segmentation_state_dict(0, **gains)
        net = nets.PyanNet()
        net.load_state_dict(sd, strict=False)
        with torch.no_grad():
            x = net.sincnet(wav).transpose(1, 2).double()
            ref = SegRef(sd, None)
            small = total = 0
            for layer in range(ref.layers):
                lstm = torch.nn.LSTM(x.shape[-1], 128, batch_first=True, bidirectional=True).double()
                lstm.load_state_dict({k[5:].replace(f"_l{layer}", "_l0"): v.double() for k, v in sd.items()
                                      if k.startswith("lstm.") and f"_l{layer}" in k})
                out, _ = lstm(x)
                for d, (gx, _) in enumerate(ref.gx(layer, x)):
                    _, w_hh, _ = ref.lstm[layer][d]
                    hp = torch.zeros_like(out[..., :128])
                    o = out[..., 128 * d: 128 * (d + 1)]
                    if d == 0:
                        hp[:, 1:] = o[:, :-1]
                    else:
                        hp[:, :-1] = o[:, 1:]
                    z = gx + hp @ w_hh.T
                    small += int((z.abs() < 2).sum())
                    total += z.numel()
                x = out
        shares.append(small / total)
    print(f"gate pre-activations with |z| < 2: default gains {shares[0]:.3f}, ih_gain = hh_gain = 1 {shares[1]:.3f}")
    assert shares[1] > shares[0]


# ---- GPU -----------------------------------------------------------------------------------------------------------
IMPLS_CONV = [1, 2, 0]
IMPLS_HEAD = [(1, 1), (1, 2), (0, 0)]
WINDOWS = [1261, 20000, 30000, 34000, 160000, 160001, 246030, 246031, 491790, 491791, 480000]


def _mode(gemm_impl):
    return "split" if gemm_impl else "fp32"


def _ctx(sd, specifications=None, conv=1, gemm=1, rec=1):
    ctx = ops.Context("cuda:0")
    ctx.load_segmentation(sd, specifications)
    ctx.set_option("seg_conv_impl", conv)
    ctx.set_option("seg_gemm_impl", gemm)
    ctx.set_option("seg_rec_impl", rec)
    return ctx


def _inputs(W, n_max):
    """Windows of W samples at odd offsets in one buffer: speech (full, ending mid-tile, 1 sample, empty), silence,
    a DC offset, a +-1 square wave, speech at 1e-4 and a single impulse.
    -> (buffer, offsets, valid, padded windows)."""
    mid = min(W, 30 * 64 * 3 * 5 + 7)          # inside the sixth stage-0 tile (or the whole of a short window)
    sp = fl32(_speech(W, 21))
    sq = torch.where((torch.arange(W) // 37) % 2 == 0, 1.0, -1.0).double()
    imp = torch.zeros(W, dtype=torch.float64)
    imp[W // 3] = 0.75
    kinds = [(sp, W), (fl32(_speech(W, 22)), mid), (sp, 1), (sp, 0), (torch.zeros(W, dtype=torch.float64), W),
             (torch.full((W,), 0.3125, dtype=torch.float64), W), (sq, W), (fl32(_speech(W, 23) * 1e-4), W), (imp, W)]
    kinds = kinds[:n_max]
    off, pos = [], 0
    for i in range(len(kinds)):
        pos += 2 * (i % 3) + 1                    # odd gaps: odd and even offsets
        off.append(pos)
        pos += W
    buf = torch.zeros(pos + 16, dtype=torch.float32)
    valid = [v for _, v in kinds]
    windows = torch.zeros((len(off), W), dtype=torch.float64)
    for i, ((x, v), o) in enumerate(zip(kinds, off)):
        buf[o: o + W] = x.float()
        windows[i, :v] = buf[o: o + v].double()
    return buf, off, valid, windows


@pytest.fixture(scope="module")
def sd():
    return syn.make_segmentation_state_dict(0)


@pytest.fixture(scope="module")
def sd_soft():
    return syn.make_segmentation_state_dict(0, ih_gain=1.0, hh_gain=1.0)


@pytest.mark.gpu
@pytest.mark.parametrize("conv", IMPLS_CONV)
@pytest.mark.parametrize("W", WINDOWS)
def test_sincnet_stages(sd, conv, W):
    """Every SincNet stage, teacher-forced from the GPU's previous stage, and its InstanceNorm affine."""
    ctx = _ctx(sd, conv=conv)
    ref = SegRef(sd, "split" if conv else "fp32")
    n = 9 if W < 246030 else 5
    buf, off, valid, windows = _inputs(W, n)
    cap = ctx.seg_stages(buf.cuda(), off, valid, W)
    tag = f"[W={W} conv={conv}]"
    # wav_norm1d
    sc, sh, bsc, bsh = ref.wav_affine(windows)
    af = cap["af_wav"].double().cpu()
    _check("af_wav.scale" + tag, af[:, 0], sc, bsc)
    _check("af_wav.shift" + tag, af[:, 1], sh, bsh)
    P0, b0 = ref.sinc(windows, af[:, 0], af[:, 1])
    _check("P0" + tag, cap["P0"].double().cpu(), P0, b0)
    P = cap["P0"].double().cpu()
    for i, (name, nxt) in enumerate((("af0", "P1"), ("af1", "P2"))):
        sc, sh, bsc, bsh = affine(P, *ref.norm[i])
        af = cap[name].double().cpu()
        _check(f"{name}.scale" + tag, af[..., 0], sc, bsc)
        _check(f"{name}.shift" + tag, af[..., 1], sh, bsh)
        want, bound = ref.conv_stage(i, P, af[..., 0], af[..., 1])
        P = cap[nxt].double().cpu()
        _check(nxt + tag, P, want, bound)
    sc, sh, bsc, bsh = affine(P, *ref.norm[2])
    af = cap["af2"].double().cpu()
    _check("af2.scale" + tag, af[..., 0], sc, bsc)
    _check("af2.shift" + tag, af[..., 1], sh, bsh)
    x0 = cap["x0"].double().cpu()
    assert torch.equal(x0[..., 60:], torch.zeros_like(x0[..., 60:])), "x0 pad columns"
    want = ref.x0(P, af[..., 0], af[..., 1])
    _check("x0" + tag, x0[..., :60], want, ulp32(want))


def _heads_equal(a, b, what):
    for k in ("cls", "logp", "scores", "max_scores", "z2"):
        if k in a:
            assert torch.equal(a[k], b[k]), f"{what}: {k} differs"


@pytest.mark.gpu
@pytest.mark.parametrize("gemm,rec", IMPLS_HEAD)
@pytest.mark.parametrize("W", [34000, 160000])
def test_stages_chain_is_the_forward(sd, gemm, rec, W):
    """seg_stages runs the forward: the same outputs bit for bit and the same launches; seg_head_stages on its x0
    reproduces them; a fresh Context gives the same bits on its first call as on its second."""
    buf, off, valid, _ = _inputs(W, 4)
    wav = buf.cuda()
    ctx = _ctx(sd, gemm=gemm, rec=rec)
    n0 = ctx.launch_count
    cls, logp = ctx.seg_forward(wav, off, valid, return_logp=True, window=W)
    n1 = ctx.launch_count
    cap = ctx.seg_stages(wav, off, valid, W)
    n2 = ctx.launch_count
    torch.cuda.synchronize()
    assert n2 - n1 == n1 - n0, f"seg_stages made {n2 - n1} launches, the forward {n1 - n0}"
    assert torch.equal(cap["cls"], cls) and torch.equal(cap["logp"], logp), "seg_stages differs from seg_forward"
    head = ctx.seg_head_stages("seg", cap["x0"])
    _heads_equal(cap, head, "seg_head_stages on the captured x0")
    fresh = _ctx(sd, gemm=gemm, rec=rec)
    first = fresh.seg_stages(wav, off, valid, W)
    second = fresh.seg_stages(wav, off, valid, W)
    for k in ("x0", "P0", "P2", "cls", "logp"):
        assert torch.equal(first[k], second[k]) and torch.equal(first[k], cap[k]), f"fresh Context: {k} differs"
    ctx.set_option("seg_max_batch", 1)              # one sub-batch: 160000 // W windows
    k = 160000 // W + 1
    with pytest.raises(ValueError, match="more than one segmentation sub-batch"):
        ctx.seg_stages(wav, [0] * k, [W] * k, W)


def _x0(kind, n, T, sd, seed):
    """Head inputs (n, T, 64): leaky_relu(randn) like SincNet's output, the same scaled by 1/16 so that |h| stays
    mostly below 1/8, or the GPU SincNet of speech (tiled over n with per-sequence gains)."""
    g = torch.Generator().manual_seed(seed)
    if kind == "sinc":
        W = {1775: 480000, 589: 160000, 2: 1261}[T]
        buf, off, valid, _ = _inputs(W, 3)
        x = _ctx(sd).seg_stages(buf.cuda(), off, valid, W)["x0"].cpu()
        reps = torch.arange(n) % 3
        x = x[reps] * (1 + 0.01 * torch.arange(n).float())[:, None, None]
        x[..., 60:] = 0
        return x.contiguous()
    x = F.leaky_relu(torch.randn((n, T, 64), generator=g))
    x[..., 60:] = 0
    return x / 16 if kind == "small" else x


HEAD_CASES = [(1, 1, "rand"), (129, 1, "rand"), (63, 2, "small"), (65, 2, "rand"), (64, 589, "sinc"),
              (65, 589, "small"), (1, 1775, "small"), (129, 1775, "sinc")]


def _seqs(n):
    return sorted({0, 62, 63, 64, 65, 127, 128, n - 1} & set(range(n)))


@pytest.mark.gpu
@pytest.mark.parametrize("gemm,rec", IMPLS_HEAD)
@pytest.mark.parametrize("n,T,kind", HEAD_CASES)
@pytest.mark.parametrize("weights", ["default", "sensitive"])
def test_head_stages(sd, sd_soft, gemm, rec, n, T, kind, weights):
    """Gx, both directions of every BiLSTM layer, the linears and the classifier, teacher-forced, at the recurrence's
    64-sequence tile edges, T = 1 and 2, and with |h| mostly below 1/8 (lo halves subnormal)."""
    w = sd if weights == "default" else sd_soft
    x0 = _x0(kind, n, T, sd, seed=n * 7 + T)
    ctx = _ctx(w, gemm=gemm, rec=rec)
    cap = ctx.seg_head_stages("seg", x0)
    check_head(SegRef(w, _mode(gemm)), x0, cap, _seqs(n), f"[{weights} n={n} T={T} {kind} {gemm}{rec}]")


def _specs(K):
    from pyannote_audio_b200.core import Problem, Resolution, Specifications

    return Specifications(Problem.MULTI_LABEL_CLASSIFICATION, Resolution.FRAME, 10.0,
                          classes=[f"label#{i}" for i in range(K)])


@pytest.mark.gpu
@pytest.mark.parametrize("gemm,rec", IMPLS_HEAD)
@pytest.mark.parametrize("K,act", [(1, "logsoftmax"), (7, "dominant"), (32, "logsoftmax"), (4, "sigmoid")])
def test_classifier_heads(gemm, rec, K, act):
    """Log-softmax heads at both ends of the classifier table (K = 1 and 32), a K = 7 head whose last class leads by
    more than float32's exp range (a max taken over fewer than K classes overflows), and a K = 4 sigmoid head."""
    w = syn.make_segmentation_state_dict(0, num_classes=K, fitted_classifier=False)
    if act == "dominant":
        w["classifier.bias"] = w["classifier.bias"].clone()
        w["classifier.bias"][K - 1] += 100.0
    ctx = _ctx(w, _specs(K) if act == "sigmoid" else None, gemm=gemm, rec=rec)
    x0 = _x0("rand", 3, 40, w, seed=K)
    cap = ctx.seg_head_stages("seg", x0)
    check_head(SegRef(w, _mode(gemm)), x0, cap, [0, 1, 2], f"[K={K} {act} {gemm}{rec}]")


@pytest.mark.gpu
@pytest.mark.parametrize("gemm,rec", IMPLS_HEAD)
def test_sseriouss_head_stages(gemm, rec):
    """The SSeRiouSS head (K = 768 input projection) on the GPU's WavLM features."""
    sd = syn.make_sseriouss_state_dict(5, wav2vec_layer=-1, num_classes=7)
    ctx = ops.Context("cuda:0")
    ctx.load_sseriouss(sd)
    ctx.set_option("seg_gemm_impl", gemm)
    ctx.set_option("seg_rec_impl", rec)
    buf, off, valid, _ = _inputs(48000, 3)
    x0 = ctx.ssl_features(buf.cuda(), off, valid, 48000)
    cap = ctx.seg_head_stages("ssl", x0)
    head = {k: v for k, v in sd.items() if k.startswith(("lstm.", "linear.", "classifier."))}
    ref = SegRef({**syn.make_segmentation_state_dict(0, num_classes=7), **head}, _mode(gemm))
    check_head(ref, x0, cap, [0, 1, 2], f"[ssl {gemm}{rec}]")
    cls, logp = ctx.ssl_forward(buf.cuda(), off, valid, return_logp=True, window=48000)
    assert torch.equal(cap["cls"], cls) and torch.equal(cap["logp"], logp), "seg_head_stages differs from ssl_forward"
