"""oracle/model.py — PyTorch fp32 restatement of the reference network.  TEST INFRASTRUCTURE.

Restates cchess_alphazero/agent/model.py:32-83 (CChessModel.build / _build_residual_block) with the Keras
defaults recorded in data/model/model_best_config.json: Conv2D channels_first, padding "same", no bias;
BatchNormalization(axis=1, epsilon=1e-3) in inference mode; Flatten over (C,H,W); Dense kernels (in,out);
softmax policy, tanh value.  TensorFlow/Keras are not installable here, so NN parity is pinned only by
this restatement ("parity unpinned" by any reference test, SURVEY.md §8c) with tolerance 1e-3.

Weights are exchanged as a dict of Keras-style names -> float32 arrays in Keras layouts
(conv HWIO, dense (in,out)), the same dict the product's `cz_nn_set_weights` consumes.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

BN_EPS = 1e-3
N_LABELS = 2086


def keras_names(filters, blocks):
    names = [f"input_conv-5-{filters}/kernel"] + [f"input_batchnorm/{w}" for w in ("gamma", "beta", "moving_mean", "moving_variance")]
    for i in range(1, blocks + 1):
        for j in (1, 2):
            names.append(f"res{i}_conv{j}-3-{filters}/kernel")
            names += [f"res{i}_batchnorm{j}/{w}" for w in ("gamma", "beta", "moving_mean", "moving_variance")]
    names += ["policy_conv-1-2/kernel"] + [f"policy_batchnorm/{w}" for w in ("gamma", "beta", "moving_mean", "moving_variance")]
    names += ["policy_out/kernel", "policy_out/bias"]
    names += ["value_conv-1-4/kernel"] + [f"value_batchnorm/{w}" for w in ("gamma", "beta", "moving_mean", "moving_variance")]
    names += ["value_dense/kernel", "value_dense/bias", "value_out/kernel", "value_out/bias"]
    return names


def _glorot(rng, shape, fan_in, fan_out):
    lim = math.sqrt(6.0 / (fan_in + fan_out))
    return rng.uniform(-lim, lim, size=shape).astype(np.float32)


def init_weights(filters, blocks, value_fc=256, seed=0, trained_like=False, spread=1.0, in_planes=14, policy_filters=4,
                 value_filters=2):
    """Keras-equivalent initialisation (glorot-uniform kernels, zero biases, BN gamma=1 beta=0 mean=0 var=1).
    trained_like=True perturbs the BN statistics and biases so that folding bugs cannot hide; `spread` scales the
    perturbation (1.0: gamma in [0.5,1.5], variance in [0.5,2] - a deep random net in that regime amplifies any
    perturbation of its inputs several-fold per 10 blocks; 0.3 keeps the conditioning close to a Keras-initialised net)."""
    rng = np.random.RandomState(seed)
    w = {}

    def conv(name, k, cin, cout):
        w[name + "/kernel"] = _glorot(rng, (k, k, cin, cout), k * k * cin, k * k * cout)

    def bn(name, c):
        if trained_like:
            w[name + "/gamma"] = rng.uniform(1 - 0.5 * spread, 1 + 0.5 * spread, c).astype(np.float32)
            w[name + "/beta"] = rng.uniform(-0.3 * spread, 0.3 * spread, c).astype(np.float32)
            w[name + "/moving_mean"] = rng.uniform(-0.2 * spread, 0.2 * spread, c).astype(np.float32)
            w[name + "/moving_variance"] = np.exp(rng.uniform(-0.7 * spread, 0.7 * spread, c)).astype(np.float32)
        else:
            w[name + "/gamma"] = np.ones(c, np.float32)
            w[name + "/beta"] = np.zeros(c, np.float32)
            w[name + "/moving_mean"] = np.zeros(c, np.float32)
            w[name + "/moving_variance"] = np.ones(c, np.float32)

    def dense(name, cin, cout):
        w[name + "/kernel"] = _glorot(rng, (cin, cout), cin, cout)
        w[name + "/bias"] = (rng.uniform(-0.1, 0.1, cout) if trained_like else np.zeros(cout)).astype(np.float32)

    conv(f"input_conv-5-{filters}", 5, in_planes, filters)     # 28 = the use_history variant (model_128_l1_config.json)
    bn("input_batchnorm", filters)
    for i in range(1, blocks + 1):
        for j in (1, 2):
            conv(f"res{i}_conv{j}-3-{filters}", 3, filters, filters)
            bn(f"res{i}_batchnorm{j}", filters)
    # agent/model.py:47-61 builds 4 policy and 2 value channels; the older JSON configs under data/model/ (128f, 256f,
    # 128_l1) still carry the head widths of earlier versions (policy 2 or 32, value 4) under the same layer names
    conv("policy_conv-1-2", 1, filters, policy_filters)
    bn("policy_batchnorm", policy_filters)
    dense("policy_out", 90 * policy_filters, N_LABELS)
    conv("value_conv-1-4", 1, filters, value_filters)
    bn("value_batchnorm", value_filters)
    dense("value_dense", 90 * value_filters, value_fc)
    dense("value_out", value_fc, 1)
    return w


def _array(w, layer, weight):
    for k, v in w.items():
        l, ww = k.split("/", 1)
        if ww.split(":")[0] == weight and (l == layer or l.startswith(layer + "-")):
            return np.asarray(v, dtype=np.float32)
    raise KeyError((layer, weight))


def _find(w, layer, weight, dtype=torch.float32, device="cpu"):
    return torch.as_tensor(_array(w, layer, weight), dtype=torch.float32).to(device=device, dtype=dtype)


def _conv(x, w, layer, pad):
    k = _find(w, layer, "kernel", x.dtype, x.device).permute(3, 2, 0, 1).contiguous()      # HWIO -> OIHW
    return F.conv2d(x, k, padding=pad)


def _bn(x, w, layer):
    g, b = _find(w, layer, "gamma", x.dtype, x.device), _find(w, layer, "beta", x.dtype, x.device)
    m, v = _find(w, layer, "moving_mean", x.dtype, x.device), _find(w, layer, "moving_variance", x.dtype, x.device)
    sh = (1, -1, 1, 1)
    return (x - m.view(sh)) / torch.sqrt(v.view(sh) + BN_EPS) * g.view(sh) + b.view(sh)


def forward_stages(w, planes, blocks, dtype=torch.float64, device="cpu"):
    """The network in `dtype` on `device` (float64 by default: the reference the GPU kernels are measured against), with
    every stage kept: first [B,C,10,9] (input conv + BN + ReLU), conv1[i] / out[i] (first conv + BN + ReLU / output of
    residual block i), pol_feat [B, policy channels * 90] (Keras Flatten of channels_first), logits [B,2086], policy
    (softmax), log_policy (log-softmax in `dtype`), value_pre [B] (before tanh), value [B]."""
    def dense(x, layer):
        return x @ _find(w, layer, "kernel", dtype, device) + _find(w, layer, "bias", dtype, device)

    x = torch.as_tensor(np.asarray(planes), dtype=torch.float32).to(device=device, dtype=dtype)
    st = {"conv1": [], "out": []}
    with torch.no_grad():
        x = F.relu(_bn(_conv(x, w, "input_conv", 2), w, "input_batchnorm"))
        st["first"] = x
        for i in range(1, blocks + 1):
            y = F.relu(_bn(_conv(x, w, f"res{i}_conv1", 1), w, f"res{i}_batchnorm1"))
            st["conv1"].append(y)
            y = _bn(_conv(y, w, f"res{i}_conv2", 1), w, f"res{i}_batchnorm2")
            x = F.relu(x + y)
            st["out"].append(x)
        p = F.relu(_bn(_conv(x, w, "policy_conv", 0), w, "policy_batchnorm")).flatten(1)
        st["pol_feat"] = p
        st["logits"] = dense(p, "policy_out")
        st["policy"] = torch.softmax(st["logits"], dim=1)
        st["log_policy"] = torch.log_softmax(st["logits"], dim=1)
        v = F.relu(_bn(_conv(x, w, "value_conv", 0), w, "value_batchnorm")).flatten(1)
        v = F.relu(dense(v, "value_dense"))
        st["value_pre"] = dense(v, "value_out")[:, 0]
        st["value"] = torch.tanh(st["value_pre"])
    return st


def forward(w, planes, blocks):
    """planes: float32 [B,14,10,9] -> (policy [B,2086] softmax, value [B]) in fp32 on the CPU."""
    st = forward_stages(w, planes, blocks, dtype=torch.float32)
    return st["policy"].numpy(), st["value"].numpy()


def _bn_fold(w, layer):
    """k_bn_fold in float32: scale = gamma / sqrt(var + eps), shift = beta - mean * scale; also |beta| + |mean * scale|, the
    magnitude of the shift's terms."""
    g, b = _array(w, layer, "gamma"), _array(w, layer, "beta")
    m, v = _array(w, layer, "moving_mean"), _array(w, layer, "moving_variance")
    s = g / np.sqrt(v + np.float32(BN_EPS))
    return s, b - m * s, np.abs(b) + np.abs(m * s)


def _split16(f):
    """f32 -> (hi, lo) fp16 with hi = RN(f), lo = RN(f - hi) (f - hi is exact in f32)."""
    hi = f.astype(np.float16)
    return hi, (f - hi.astype(np.float32)).astype(np.float16)


def folded_operands(w, in_planes=14):
    """The operands cz_nn.cu's weight preparation builds from a Keras weight dict, restated in float32 numpy:
      w_first     fp16 [5][5][in_planes][C]  input conv, HWIO, BN scale folded (k_prep_hwio)
      w_conv[l]   fp16 [9][C_out][C_in]       residual conv l = 2*block + j, tap-major, BN scale folded (k_prep_conv3)
      wh          f32  [pol_c + val_c][C]     policy then value 1x1 conv, BN scale folded (k_prep_1x1)
      w_pol       fp16 [2304][3 * pol_k1]     policy Dense split as [w_hi | w_hi | w_lo], zero padded (k_prep_policy)
      shift_first, shift_conv[l], shifth: BN shifts (f32); b_pol f32 [2304]; wv1, bv1, wv2, bv2: value Dense copies.
      shift_first_abs, shift_conv_abs[l], shifth_abs: |beta| + |mean * scale|, the magnitude of each shift's terms.
    Division and sqrt are correctly rounded on both sides, so the fp16 operands agree bit for bit with the GPU's.  A shift
    may differ where nvcc contracts beta - mean * scale into an FMA: by half an f32 ulp of mean * scale, which exceeds an
    ulp of the shift itself when the two terms cancel (hence the *_abs magnitudes)."""
    out = {}
    s, out["shift_first"], out["shift_first_abs"] = _bn_fold(w, "input_batchnorm")
    k = _array(w, "input_conv", "kernel")
    assert k.shape[2] == in_planes, (k.shape, in_planes)
    out["w_first"] = (k * s).astype(np.float16)
    blocks = sum(1 for key in w if key.startswith("res") and "_conv1" in key and key.endswith("/kernel"))
    out["w_conv"], out["shift_conv"], out["shift_conv_abs"] = [], [], []
    for i in range(1, blocks + 1):
        for j in (1, 2):
            s, sh, sha = _bn_fold(w, f"res{i}_batchnorm{j}")
            k = _array(w, f"res{i}_conv{j}", "kernel")                         # [3][3][ci][co]
            c = k.shape[3]
            out["w_conv"].append((k * s).astype(np.float16).reshape(9, c, c).transpose(0, 2, 1).copy())
            out["shift_conv"].append(sh)
            out["shift_conv_abs"].append(sha)
    heads, shifts, shifts_abs = [], [], []
    for conv, bn in (("policy_conv", "policy_batchnorm"), ("value_conv", "value_batchnorm")):
        s, sh, sha = _bn_fold(w, bn)
        heads.append((_array(w, conv, "kernel")[0, 0] * s).T)                 # [ci][co] -> [co][ci]
        shifts.append(sh)
        shifts_abs.append(sha)
    out["pol_c"], out["val_c"] = heads[0].shape[0], heads[1].shape[0]
    out["wh"], out["shifth"], out["shifth_abs"] = np.concatenate(heads), np.concatenate(shifts), np.concatenate(shifts_abs)
    pol_in = 90 * out["pol_c"]
    pol_k1 = (pol_in + 63) // 64 * 64
    f = np.zeros((2304, pol_k1), np.float32)
    f[:N_LABELS, :pol_in] = _array(w, "policy_out", "kernel").T
    hi, lo = _split16(f)
    out["pol_k1"], out["w_pol"] = pol_k1, np.concatenate([hi, hi, lo], axis=1)
    out["b_pol"] = np.zeros(2304, np.float32)
    out["b_pol"][:N_LABELS] = _array(w, "policy_out", "bias")
    for name, layer, weight in (("wv1", "value_dense", "kernel"), ("bv1", "value_dense", "bias"),
                                ("wv2", "value_out", "kernel"), ("bv2", "value_out", "bias")):
        out[name] = _array(w, layer, weight)
    return out


class TorchNet:
    """predict_on_batch-compatible wrapper (what api.py:63-64 calls on the Keras model)."""

    def __init__(self, weights, blocks):
        self.w, self.blocks = weights, blocks

    def predict_on_batch(self, data):
        p, v = forward(self.w, data, self.blocks)
        return p, v[:, None]
