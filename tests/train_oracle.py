"""Float64 restatement of one Keras 2.0.8 `Model.fit` batch for worker/optimize.py:108-136, on oracle/model.py's layers,
plus the host loop around it (validation split, per-epoch shuffle, batches, lr schedule).  TEST INFRASTRUCTURE.

TensorFlow / Keras cannot be installed next to this project, so these semantics are restated (DESIGN.md §11), not pinned:
  loss      w_p * CE + w_v * MSE + l2 * sum ||K||^2 over every conv kernel and the three Dense kernels
  CE        Keras categorical_crossentropy on the softmax output (TF backend): p / sum p, clipped to [eps, 1 - eps]
            with eps = 1e-7 in fp32, -sum t log p; a clipped term passes no gradient (torch.clamp's gradient)
  BN        batch statistics over (N, H, W), biased variance, eps 1e-3; moving stats m -= (m - batch) * (1 - 0.99)
            with the BIASED batch variance
  SGD       v = mu * v - lr * g, w = w + v (no Nesterov, decay 0)
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import model as om

BN_EPS = 1e-3
KERAS_EPS = float(np.float32(1e-7))
KERAS_HI = float(np.float32(1) - np.float32(1e-7))
MOMENTUM_BN = 0.99


def is_stat(name):
    return name.endswith("/moving_mean") or name.endswith("/moving_variance")


def is_reg(name):
    return name.endswith("/kernel")


def _name(w, layer, weight):
    for k in w:
        l, ww = k.split("/", 1)
        if ww == weight and (l == layer or l.startswith(layer + "-")):
            return k
    raise KeyError((layer, weight))


def _scaled16(g):
    m = g.abs().max().item()
    e = 0 if m == 0 else 14 - (int(np.frexp(m)[1]) - 1)
    return (g * 2.0 ** e).half().to(g.dtype) * 2.0 ** -e


class _Round16(torch.autograd.Function):
    """fp16 rounding of a tensor-core operand (activation or weight); the gradient passes unchanged."""
    @staticmethod
    def forward(ctx, x):
        return x.half().to(x.dtype)

    @staticmethod
    def backward(ctx, g):
        return g


class _GradRound16(torch.autograd.Function):
    """Identity forward; the gradient becomes the power-of-two-scaled fp16 operand the GPU feeds to dgrad and wgrad."""
    @staticmethod
    def forward(ctx, x):
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return _scaled16(g)


def forward_train(w, planes, blocks, dtype=torch.float64, device="cpu", fp16_operands=False):
    """Training-mode forward on tensors `w` (name -> tensor, may require grad).  Returns (logits, value_pre, stats, z):
    stats[bn layer] = (batch mean, biased batch var), z[bn layer] = that BN's input (retain_grad'ed: .grad = dz).
    fp16_operands: round the operands of the 3x3 convolutions where the GPU does (activations and weights to fp16, the
    conv-output gradient to scaled fp16), everything else stays float64 — the GPU's arithmetic without its fp32 sums."""
    stats, zs = {}, {}

    def conv(x, layer, pad):
        k = w[_name(w, layer, "kernel")].permute(3, 2, 0, 1)
        if fp16_operands and pad == 1:
            return _GradRound16.apply(F.conv2d(_Round16.apply(x), _Round16.apply(k), padding=pad))
        return F.conv2d(x, k, padding=pad)

    def bn(x, layer):
        if x.requires_grad:
            x.retain_grad()
        zs[layer] = x
        mean = x.mean(dim=(0, 2, 3))
        var = x.var(dim=(0, 2, 3), unbiased=False)
        stats[layer] = (mean.detach(), var.detach())
        sh = (1, -1, 1, 1)
        g, b = w[_name(w, layer, "gamma")], w[_name(w, layer, "beta")]
        return (x - mean.view(sh)) / torch.sqrt(var.view(sh) + BN_EPS) * g.view(sh) + b.view(sh)

    x = torch.as_tensor(np.asarray(planes), dtype=torch.float32).to(device=device, dtype=dtype)
    x = F.relu(bn(conv(x, "input_conv", 2), "input_batchnorm"))
    for i in range(1, blocks + 1):
        y = F.relu(bn(conv(x, f"res{i}_conv1", 1), f"res{i}_batchnorm1"))
        y = bn(conv(y, f"res{i}_conv2", 1), f"res{i}_batchnorm2")
        x = F.relu(x + y)
    p = F.relu(bn(conv(x, "policy_conv", 0), "policy_batchnorm")).flatten(1)
    logits = p @ w[_name(w, "policy_out", "kernel")] + w[_name(w, "policy_out", "bias")]
    v = F.relu(bn(conv(x, "value_conv", 0), "value_batchnorm")).flatten(1)
    v = F.relu(v @ w[_name(w, "value_dense", "kernel")] + w[_name(w, "value_dense", "bias")])
    v = v @ w[_name(w, "value_out", "kernel")] + w[_name(w, "value_out", "bias")]
    return logits, v[:, 0], stats, zs


def keras_ce(logits, target):
    p = torch.softmax(logits, dim=1)
    p = p / p.sum(dim=1, keepdim=True)
    return -(target * torch.log(torch.clamp(p, KERAS_EPS, KERAS_HI))).sum(dim=1)


def losses(w, planes, policy, value, blocks, w_p=1.0, w_v=1.0, l2=1e-4, dtype=torch.float64, device="cpu", fp16_operands=False):
    logits, vpre, stats, zs = forward_train(w, planes, blocks, dtype, device, fp16_operands)
    t = torch.as_tensor(np.asarray(policy), dtype=dtype, device=device)
    z = torch.as_tensor(np.asarray(value), dtype=dtype, device=device).reshape(-1)
    ce = keras_ce(logits, t).mean()
    mse = ((torch.tanh(vpre) - z) ** 2).mean()
    l2t = l2 * sum((v ** 2).sum() for k, v in w.items() if is_reg(k))
    return w_p * ce + w_v * mse, ce, mse, l2t, stats, zs


def fit_step(weights, planes, policy, value, blocks, lr, momentum=0.9, w_p=1.0, w_v=1.0, l2=1e-4, velocity=None,
             dtype=torch.float64, device="cpu", fp16_operands=False):
    """One Keras fit batch.  weights / velocity: name -> array (Keras layout).  Returns a dict:
      losses (total, policy, value, l2) before the update; grad[name] = gradient of the loss terms (without L2);
      weights / velocity after the update (moving statistics included); stats[bn layer] = (mean, var);
      dz[bn layer] = gradient at that BN's input (the conv output) [N, C, 10, 9]."""
    w = {k: torch.as_tensor(np.asarray(v), dtype=dtype, device=device).clone().requires_grad_(not is_stat(k))
         for k, v in weights.items()}
    data, ce, mse, l2t, stats, zs = losses(w, planes, policy, value, blocks, w_p, w_v, l2, dtype, device, fp16_operands)
    names = [k for k in w if not is_stat(k)]
    grads = torch.autograd.grad(data, [w[k] for k in names], retain_graph=True)
    dz = {layer: torch.autograd.grad(data, z, retain_graph=True)[0].detach() for layer, z in zs.items()}
    g = dict(zip(names, (x.detach() for x in grads)))
    new_w, new_v = {}, {}
    for k in w:
        x = w[k].detach()
        if is_stat(k):
            layer = k.split("/")[0]
            m, v = stats[layer]
            new_w[k] = x - (x - (m if k.endswith("moving_mean") else v)) * (1 - MOMENTUM_BN)
            continue
        gt = g[k] + (2 * l2 * x if is_reg(k) else 0)
        v0 = torch.zeros_like(x) if velocity is None else torch.as_tensor(np.asarray(velocity[k]), dtype=dtype, device=device)
        new_v[k] = momentum * v0 - lr * gt
        new_w[k] = x + new_v[k]
    total = (data + l2t).item()
    return {"losses": (total, ce.item(), mse.item(), l2t.item()), "grad": g, "weights": new_w, "velocity": new_v,
            "stats": stats, "dz": dz}


# ---------------------------------------------------------------------------------------------- the host loop of fit
def validation_split(n, split=0.02):
    """Keras 2.0.8 fit: split_at = int(n * (1 - split)); the LAST samples (before any shuffle) validate."""
    split_at = int(n * (1.0 - split))
    return np.arange(split_at), np.arange(split_at, n)


def make_batches(size, batch_size):
    """Keras _make_batches: ceil(size / batch_size) slices, the last one partial."""
    nb = int(np.ceil(size / float(batch_size)))
    return [(i * batch_size, min(size, (i + 1) * batch_size)) for i in range(nb)]


def epoch_order(n_train, rng):
    """shuffle=True: a fresh permutation of the training indices every epoch."""
    idx = np.arange(n_train)
    rng.shuffle(idx)
    return idx


def decide_learning_rate(schedules, total_steps):
    """optimize.py:194-200."""
    ret = None
    for step, lr in schedules:
        if total_steps >= step:
            ret = lr
    return ret
