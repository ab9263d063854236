"""Training step of the policy-value network on the GPU: what Keras `Model.fit` runs per batch for worker/optimize.py.

`Trainer(model, batch_size, device, optimizer="sgd"|"adam")` owns the fp32 master weights, the SGD velocity (and, for Adam,
the moments m / v) and the trainer workspace as torch tensors; `step()` runs one batch through `cz_train_step`
(csrc/cz_train.cu: training-mode forward, backward and the SGD-momentum or fused Keras Adam update, all CUDA).
`validation_loss()` evaluates with the inference forward of the engine (`cz_nn_forward`, BatchNormalization on the
moving statistics) — the same network self-play serves.  `export()` hands the weights back in
Keras names for `CChessModel.save()`.
"""
import ctypes as C

import numpy as np
import torch

from .lib import CzTensorDesc, CzTrainConfig, CzTrainHparams, get_lib
from .model import engine_net_kwargs, head_channels

KERAS_EPS = np.float32(1e-7)


def _is_stat(name):
    return name.endswith("/moving_mean") or name.endswith("/moving_variance")


def _descs(tensors):
    arr = (CzTensorDesc * len(tensors))()
    for i, (k, t) in enumerate(tensors.items()):
        arr[i].name, arr[i].dev, arr[i].numel = k.encode(), t.data_ptr(), t.numel()
    return arr


def keras_policy_loss(policy, target):
    """Keras categorical_crossentropy on softmax outputs (float64): renormalise, clip to [eps, 1 - eps] in fp32, -sum t log p."""
    p = np.asarray(policy, np.float64)
    p = p / p.sum(axis=1, keepdims=True)
    hi = float(np.float32(1) - KERAS_EPS)
    return -(np.asarray(target, np.float64) * np.log(np.clip(p, float(KERAS_EPS), hi))).sum(axis=1)


class Trainer:
    def __init__(self, model, batch_size, device=None, lib=None, optimizer="sgd", beta_1=0.9, beta_2=0.999, epsilon=1e-8):
        """optimizer "sgd": Keras SGD with momentum (worker/optimize.py); "adam": Keras 2.0.8 Adam (worker/sl.py), whose
        moments m / v this object owns and whose `iterations` run on across every step of this trainer."""
        if optimizer not in ("sgd", "adam"):
            raise ValueError(f"optimizer must be 'sgd' or 'adam', not {optimizer!r}")
        self.optimizer = optimizer
        self.model = model
        self.config = model.config
        self.lib = lib or get_lib()
        self.device = torch.device(device or "cuda")
        if self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        mc = self.config.model
        self.batch_size = int(batch_size)
        self.weights = {k: torch.as_tensor(np.asarray(v, np.float32)).to(self.device).contiguous() for k, v in model.weights.items()}
        self.velocity = {k: torch.zeros_like(v) for k, v in self.weights.items() if not _is_stat(k)}
        first = next(v for k, v in self.weights.items() if k.startswith("input_conv") and k.endswith("/kernel"))
        pol_c, val_c = head_channels(mc)
        cfg = CzTrainConfig()
        cfg.struct_bytes = C.sizeof(CzTrainConfig)
        cfg.filters, cfg.blocks, cfg.in_planes = mc.cnn_filter_num, mc.res_layer_num, int(first.shape[2])
        cfg.policy_channels, cfg.value_channels, cfg.value_fc = pol_c, val_c, mc.value_fc_size
        cfg.max_batch = self.batch_size
        self.cfg = cfg
        self.in_planes = cfg.in_planes
        nbytes = C.c_uint64(0)
        self.lib.call("cz_train_workspace_bytes", C.byref(cfg), C.byref(nbytes))
        self.workspace = torch.zeros(nbytes.value, dtype=torch.uint8, device=self.device)
        self._h = C.c_void_p(0)
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        self.lib.call("cz_train_create", C.byref(cfg), C.c_void_p(self.workspace.data_ptr()), nbytes, stream, C.byref(self._h))
        self._pd, self._vd = _descs(self.weights), _descs(self.velocity)
        self.lib.call("cz_train_set_params", self._h, self._pd, len(self.weights), self._vd, len(self.velocity))
        self.adam_m = self.adam_v = None
        if optimizer == "adam":
            self.adam_m = {k: torch.zeros_like(v) for k, v in self.velocity.items()}
            self.adam_v = {k: torch.zeros_like(v) for k, v in self.velocity.items()}
            self._md, self._vvd = _descs(self.adam_m), _descs(self.adam_v)
            self.lib.call("cz_train_set_adam", self._h, self._md, len(self.adam_m), self._vvd, len(self.adam_v),
                          float(beta_1), float(beta_2), float(epsilon))
        self.losses = torch.zeros(4, dtype=torch.float32, device=self.device)
        self._engine = None

    def hparams(self, lr):
        tc, mc = self.config.trainer, self.config.model
        hp = CzTrainHparams()
        hp.struct_bytes = C.sizeof(CzTrainHparams)
        hp.lr = float(lr)
        hp.momentum = 0.0 if self.optimizer == "adam" else float(tc.momentum)      # Adam ignores it
        hp.w_policy, hp.w_value = (float(x) for x in tc.loss_weights)
        hp.l2 = float(mc.l2_reg)
        return hp

    def _dev(self, x):
        return torch.as_tensor(x, dtype=torch.float32).to(self.device).contiguous()

    def step_async(self, planes, policy, value, lr):
        """One SGD step on a batch (planes [B][in_planes][10][9], one-hot policy [B][2086], value [B]); returns the device
        tensor of losses {total, policy, value, l2} evaluated before the update, without synchronising."""
        planes, policy, value = self._dev(planes), self._dev(policy), self._dev(value).reshape(-1)
        n = planes.shape[0]
        self._keep = (planes, policy, value)
        hp = self.hparams(lr)
        self.lib.call("cz_train_step", self._h, C.c_void_p(planes.data_ptr()), C.c_void_p(policy.data_ptr()),
                      C.c_void_p(value.data_ptr()), n, C.byref(hp), C.c_void_p(self.losses.data_ptr()))
        return self.losses

    def step(self, planes, policy, value, lr):
        return self.step_async(planes, policy, value, lr).cpu().numpy().astype(np.float64)

    @property
    def iterations(self):
        """Adam's step counter (Keras `iterations`): steps run since this trainer was built."""
        it = C.c_int64(0)
        self.lib.call("cz_train_adam_iterations", self._h, C.byref(it))
        return it.value

    def grad(self, name):
        """The last step's gradient of one trainable weight (loss terms, without L2) — tests."""
        t = self.weights[name]
        out = torch.empty_like(t)
        self.lib.call("cz_train_read_grad", self._h, name.encode(), C.c_void_p(out.data_ptr()), t.numel())
        return out

    def export(self):
        """Keras-name dict of float32 arrays (what CChessModel.save() writes)."""
        return {k: v.detach().cpu().numpy().copy() for k, v in self.weights.items()}

    def l2_term(self):
        l2 = float(self.config.model.l2_reg)
        return l2 * sum(float((v.double() ** 2).sum()) for k, v in self.weights.items() if k.endswith("/kernel"))

    def validation_loss(self, planes, policy, value, chunk=1024):
        """Keras evaluates the validation split in inference mode: the engine's forward on the current weights (moving
        statistics).  Returns (total, policy CE, value MSE, l2) as floats."""
        from .engine import Engine
        mc = self.config.model
        if self._engine is None:
            self._engine = Engine(self.lib, self.device, n_games=min(chunk, 512), sims_per_move=1, leaves_per_round=1,
                                  max_nodes_per_game=16, max_edges_per_game=256, max_path=8, **engine_net_kwargs(mc),
                                  use_history=self.in_planes == 28)
        self._engine.set_weights(self.weights)
        ce, se = [], []
        for i in range(0, len(planes), chunk):
            pol, val = self._engine.nn_forward_planes(self._dev(planes[i:i + chunk]))
            ce.append(keras_policy_loss(pol.cpu().numpy(), policy[i:i + chunk]))
            se.append((val.cpu().numpy().astype(np.float64) - np.asarray(value[i:i + chunk], np.float64).reshape(-1)) ** 2)
        w_p, w_v = (float(x) for x in self.config.trainer.loss_weights)
        cem, msem, l2 = float(np.concatenate(ce).mean()), float(np.concatenate(se).mean()), self.l2_term()
        return w_p * cem + w_v * msem + l2, cem, msem, l2

    def close(self):
        if self._h:
            self.lib.raw("cz_train_destroy")(self._h)
            self._h = C.c_void_p(0)
        if self._engine is not None:
            self._engine.close()
            self._engine = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
