"""Keras 2.0.8 Adam (keras/optimizers.py Adam.get_updates, decay 0) restated, on top of train_oracle's gradients.

    t = iterations + 1;  lr_t = lr * (sqrt(1 - b2^t) / (1 - b1^t))
    g = grad + 2 l2 K (kernels only);  m = b1 m + (1 - b1) g;  v = b2 v + (1 - b2) g^2;  w = w - lr_t m / (sqrt(v) + eps)

`adam_update` runs in float64 (torch or numpy arrays); `adam_update_f32` is the float32 restatement in the operation order
of csrc/cz_train.cu k_adam, which the GPU must match bit for bit.  `fit_step_adam` is one float64 fit batch.
"""
import numpy as np
import torch

from tests import train_oracle as to

B1, B2, EPS = 0.9, 0.999, 1e-8


class AdamState:
    def __init__(self, m, v, iterations=0):
        self.m, self.v, self.iterations = m, v, iterations

    @staticmethod
    def zeros_like(weights):
        z = {k: (torch.zeros_like(x) if torch.is_tensor(x) else np.zeros_like(np.asarray(x, np.float64)))
             for k, x in weights.items() if not to.is_stat(k)}
        return AdamState(z, {k: (x.clone() if torch.is_tensor(x) else x.copy()) for k, x in z.items()})


def lr_t(lr, iterations, b1=B1, b2=B2):
    t = iterations + 1
    return lr * (np.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t))


def adam_update(weights, grads, state, lr, l2=0.0, b1=B1, b2=B2, eps=EPS):
    """float64, in place on weights / state; grads are the loss-term gradients (without L2)."""
    a = lr_t(float(lr), state.iterations, b1, b2)
    for k, g in grads.items():
        w = weights[k]
        gt = g + 2 * l2 * w if to.is_reg(k) else g
        state.m[k] = b1 * state.m[k] + (1 - b1) * gt
        state.v[k] = b2 * state.v[k] + (1 - b2) * gt * gt
        sq = torch.sqrt(state.v[k]) if torch.is_tensor(state.v[k]) else np.sqrt(state.v[k])
        weights[k] = w - a * state.m[k] / (sq + eps)
    state.iterations += 1


def adam_update_f32(w, g, m, v, lr, iterations, l2x2, reg, b1=B1, b2=B2, eps=EPS):
    """float32 numpy restatement of k_adam for one tensor; returns (w, m, v).  lr_t is float64 rounded to fp32 once."""
    f = np.float32
    a = f(float(np.float32(lr)) * (np.sqrt(1.0 - b2 ** (iterations + 1)) / (1.0 - b1 ** (iterations + 1))))
    b1f, b2f = f(b1), f(b2)
    gt = (g + f(l2x2) * w).astype(np.float32) if reg else g
    m = (b1f * m + (f(1) - b1f) * gt).astype(np.float32)
    v = (b2f * v + (f(1) - b2f) * (gt * gt)).astype(np.float32)
    w = (w - (a * m) / (np.sqrt(v) + f(eps))).astype(np.float32)
    return w, m, v


def fit_step_adam(weights, state, planes, policy, value, blocks, lr, w_p=1.0, w_v=1.0, l2=1e-4, dtype=torch.float64,
                  device="cpu", fp16_operands=False):
    """One Keras fit batch with Adam: train_oracle's gradients and moving statistics, then the Adam update.  Returns
    (losses, new weights)."""
    r = to.fit_step(weights, planes, policy, value, blocks, 0.0, 0.0, w_p, w_v, l2, None, dtype, device, fp16_operands)
    # moving statistics updated; trainable weights unchanged (lr 0)
    new_w = {k: x.detach().cpu().numpy().astype(np.float64) for k, x in r["weights"].items()}
    adam_update(new_w, {k: g.cpu().numpy().astype(np.float64) for k, g in r["grad"].items()}, state, lr, l2)
    return r["losses"], new_w
