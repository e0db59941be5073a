"""fp32 eager restatement of SSeRiouSS on WavLM Base (models/segmentation/SSeRiouSS.py over torchaudio's
wav2vec2 components and WavLMSelfAttention), from a state dict with the module's keys.  Pinned on the CPU against
the reference executed by path (tests/golden/reference_sseriouss_vectors.npz) and against torchaudio's wavlm_model;
the GPU tests compare the CUDA path with it (neither torchaudio nor the reference is needed there)."""
import math

import torch
import torch.nn.functional as F


def relative_buckets(T, num_buckets=320, max_distance=800):
    """(T, T) bucket of key j - query i, WavLM's bidirectional bucketing."""
    pos = torch.arange(T, dtype=torch.long)   # on the CPU: the float log rounds as in the reference
    return relative_bucket(pos[None, :] - pos[:, None], num_buckets, max_distance)


def relative_bucket(rel, num_buckets=320, max_distance=800):
    """Bucket of every offset key - query in the CPU long tensor ``rel``."""
    half = num_buckets // 2
    buckets = (rel > 0).to(torch.long) * half
    a = torch.abs(rel)
    max_exact = half // 2
    large = max_exact + (torch.log(a.float() / max_exact) / math.log(max_distance / max_exact)
                         * (half - max_exact)).to(torch.long)
    large = torch.min(large, torch.full_like(large, half - 1))
    return buckets + torch.where(a < max_exact, a, large)


def pos_conv_weight(sd, prefix):
    if prefix + "parametrizations.weight.original0" in sd:
        g, v = sd[prefix + "parametrizations.weight.original0"], sd[prefix + "parametrizations.weight.original1"]
    else:
        g, v = sd[prefix + "weight_g"], sd[prefix + "weight_v"]
    return torch._weight_norm(v, g, 2)        # in the state dict's dtype: the fp64 oracle runs the same code


def wavlm_layers(sd, wav, num_layers=12):
    """wav (B, S) -> list of the first ``num_layers`` layer outputs (B, T, 768): Wav2Vec2Model.extract_features."""
    fe, enc = "wav2vec.feature_extractor.conv_layers.", "wav2vec.encoder."
    x = F.conv1d(wav[:, None], sd[fe + "0.conv.weight"], stride=5)
    x = F.gelu(F.group_norm(x, 512, sd[fe + "0.layer_norm.weight"], sd[fe + "0.layer_norm.bias"]))
    for i, s in zip(range(1, 7), (2,) * 6):
        x = F.gelu(F.conv1d(x, sd[f"{fe}{i}.conv.weight"], stride=s))
    x = x.transpose(1, 2)
    fp = enc + "feature_projection."
    x = F.layer_norm(x, (512,), sd[fp + "layer_norm.weight"], sd[fp + "layer_norm.bias"])
    x = F.linear(x, sd[fp + "projection.weight"], sd[fp + "projection.bias"])
    tr = enc + "transformer."
    pc = tr + "pos_conv_embed.conv."
    p = F.conv1d(x.transpose(1, 2), pos_conv_weight(sd, pc), sd[pc + "bias"], padding=64, groups=16)[..., :-1]
    x = x + F.gelu(p).transpose(1, 2)
    # the post-LN encoder (encoder_layer_norm_first False) builds its Transformer with layer_norm_first True, whose
    # _preprocess normalises here, before layer 0
    x = F.layer_norm(x, (768,), sd[tr + "layer_norm.weight"], sd[tr + "layer_norm.bias"])
    B, T, _ = x.shape
    rel = sd[tr + "layers.0.attention.rel_attn_embed.weight"]
    bias = F.embedding(relative_buckets(T).to(rel.device), rel).permute(2, 0, 1)
    outs = []
    for layer in range(num_layers):
        lp = f"{tr}layers.{layer}."
        gates = F.linear(x.view(B, T, 12, 64).permute(0, 2, 1, 3), sd[lp + "attention.gru_rel_pos_linear.weight"],
                         sd[lp + "attention.gru_rel_pos_linear.bias"])
        gate_a, gate_b = torch.sigmoid(gates.view(B, 12, T, 2, 4).sum(-1)).chunk(2, dim=-1)
        gate = gate_a * (gate_b * sd[lp + "attention.gru_rel_pos_const"] - 1.0) + 2.0
        mask = gate.view(B, 12, T, 1) * bias[None]
        qkv = F.linear(x, sd[lp + "attention.attention.in_proj_weight"], sd[lp + "attention.attention.in_proj_bias"])
        q, k, v = (t.view(B, T, 12, 64).transpose(1, 2) for t in qkv.chunk(3, -1))
        a = F.scaled_dot_product_attention(q, k, v, attn_mask=mask).transpose(1, 2).reshape(B, T, 768)
        a = F.linear(a, sd[lp + "attention.attention.out_proj.weight"], sd[lp + "attention.attention.out_proj.bias"])
        x = F.layer_norm(x + a, (768,), sd[lp + "layer_norm.weight"], sd[lp + "layer_norm.bias"])
        h = F.gelu(F.linear(x, sd[lp + "feed_forward.intermediate_dense.weight"],
                            sd[lp + "feed_forward.intermediate_dense.bias"]))
        h = F.linear(h, sd[lp + "feed_forward.output_dense.weight"], sd[lp + "feed_forward.output_dense.bias"])
        x = F.layer_norm(x + h, (768,), sd[lp + "final_layer_norm.weight"], sd[lp + "final_layer_norm.bias"])
        outs.append(x)
    return outs


def features(sd, wav, wav2vec_layer=-1):
    """The LSTM input of SSeRiouSS.forward: softmax-weighted layer average, or the output of layer wav2vec_layer."""
    if wav2vec_layer < 0:
        return torch.stack(wavlm_layers(sd, wav), dim=-1) @ F.softmax(sd["wav2vec_weights"], dim=0)
    return wavlm_layers(sd, wav, wav2vec_layer)[-1]


@torch.no_grad()
def sseriouss(sd, wav, wav2vec_layer=-1, sigmoid=False, device="cpu"):
    """wav (B, S) fp32 -> (B, T, K) log-probabilities (or sigmoid scores) on the CPU, computed on ``device`` (fp32:
    callers on a GPU disable TF32)."""
    sd = {k: v.detach().float().to(device) for k, v in sd.items()}
    return head(sd, features(sd, wav.float().to(device), wav2vec_layer), sigmoid)


@torch.no_grad()
def head(sd, x, sigmoid=False):
    """The LSTM input x (B, T, 768) -> (B, T, K) log-probabilities (or sigmoid scores) on the CPU: the BiLSTM, the
    two Linears and the classifier of SSeRiouSS.forward, on x's device with the fp32 state dict ``sd`` there."""
    device = x.device
    layers = 0
    while f"lstm.weight_ih_l{layers}" in sd:
        layers += 1
    lstm = torch.nn.LSTM(768, 128, num_layers=layers, bidirectional=True, batch_first=True).to(device)
    lstm.load_state_dict({k[5:]: v for k, v in sd.items() if k.startswith("lstm.")})
    x, _ = lstm(x)
    for i in range(2):
        x = F.leaky_relu(F.linear(x, sd[f"linear.{i}.weight"], sd[f"linear.{i}.bias"]))
    logits = F.linear(x, sd["classifier.weight"], sd["classifier.bias"])
    return (torch.sigmoid(logits) if sigmoid else F.log_softmax(logits, dim=-1)).cpu()
