"""`CChessModel` drop-in (reference: cchess_alphazero/agent/model.py:22-126).

The reference object wraps a Keras model; here it is a plain container of the network weights in Keras names and
layouts (conv kernels HWIO, dense (in,out), BatchNormalization gamma/beta/moving_mean/moving_variance) plus the
geometry from `config.model`.  The forward pass itself is the tensor-core pipeline inside the engine
(`cz_nn_set_weights` / `cz_nn_forward`), reached through `get_pipes()` exactly like the reference reaches Keras
through CChessModelAPI.

Weight files: the reference's own Keras `.h5` (read by the pure-Python HDF5 subset reader in keras_h5.py; geometry is
inferred from the tensor names, so the Keras JSON config is not needed) or `.npz` (one array per Keras weight name)
next to a small JSON config, which is what `save()` writes.
"""
import hashlib
import json
import math
import os

import numpy as np

N_LABELS = 2086
BN_WEIGHTS = ("gamma", "beta", "moving_mean", "moving_variance")


def layer_names(filters, blocks, first=5, k=3):
    """Keras layer names the reference builds (model.py:37-62, 71-80)."""
    conv = [f"input_conv-{first}-{filters}"]
    bn = ["input_batchnorm"]
    for i in range(1, blocks + 1):
        conv += [f"res{i}_conv1-{k}-{filters}", f"res{i}_conv2-{k}-{filters}"]
        bn += [f"res{i}_batchnorm1", f"res{i}_batchnorm2"]
    conv += ["policy_conv-1-2", "value_conv-1-4"]
    bn += ["policy_batchnorm", "value_batchnorm"]
    return conv, bn, ["policy_out", "value_dense", "value_out"]


def head_channels(mc):
    """(policy, value) 1x1-convolution filters of a model config: agent/model.py:47-61 builds 4 / 2; the older configs under
    the reference's data/model/ have 2 / 4 (model_128f.json, model_256f.json) and 32 / 4 (model_128_l1_config.json)."""
    return int(getattr(mc, "policy_channels", 0) or 4), int(getattr(mc, "value_channels", 0) or 2)


def engine_net_kwargs(mc):
    """The network geometry arguments of `Engine(...)` for a model config."""
    pol_c, val_c = head_channels(mc)
    return dict(nn_filters=mc.cnn_filter_num, nn_blocks=mc.res_layer_num, nn_value_fc=mc.value_fc_size,
                nn_policy_channels=pol_c, nn_value_channels=val_c)


class CChessModel:
    def __init__(self, config):
        self.config = config
        self.weights = None          # dict: "<layer>/<weight>" -> np.float32 array (Keras layout)
        self.model = None            # attribute kept for callers that test `model.model is not None`
        self.digest = None
        self.n_labels = N_LABELS
        self.graph = None
        self.api = None

    # ---- model.py:32-66 — same topology, Keras default initialisers (glorot_uniform kernels, zero biases,
    #      BN gamma = 1, beta = 0, moving_mean = 0, moving_variance = 1)
    def build(self, seed=None):
        mc = self.config.model
        rng = np.random.RandomState(seed)
        f, blocks, vfc = mc.cnn_filter_num, mc.res_layer_num, mc.value_fc_size
        w = {}

        def glorot(shape, fan_in, fan_out):
            lim = math.sqrt(6.0 / (fan_in + fan_out))
            return rng.uniform(-lim, lim, size=shape).astype(np.float32)

        def conv(name, k, cin, cout):
            w[name + "/kernel"] = glorot((k, k, cin, cout), k * k * cin, k * k * cout)

        def bn(name, c):
            w[name + "/gamma"] = np.ones(c, np.float32)
            w[name + "/beta"] = np.zeros(c, np.float32)
            w[name + "/moving_mean"] = np.zeros(c, np.float32)
            w[name + "/moving_variance"] = np.ones(c, np.float32)

        def dense(name, cin, cout):
            w[name + "/kernel"] = glorot((cin, cout), cin, cout)
            w[name + "/bias"] = np.zeros(cout, np.float32)

        first = getattr(mc, "cnn_first_filter_size", 5)
        k = getattr(mc, "cnn_filter_size", 3)
        depth = getattr(mc, "input_depth", 14)        # 28 = the use_history network (data/model/model_128_l1_config.json)
        if first != 5 or k != 3 or depth not in (14, 28):
            raise NotImplementedError("the GPU path implements the 5x5 -> 3x3 residual tower on 14 or 28 input planes")
        conv(f"input_conv-{first}-{f}", first, depth, f)
        bn("input_batchnorm", f)
        for i in range(1, blocks + 1):
            for j in (1, 2):
                conv(f"res{i}_conv{j}-{k}-{f}", k, f, f)
                bn(f"res{i}_batchnorm{j}", f)
        pol_c, val_c = head_channels(mc)               # agent/model.py:47-61: 4 / 2 (the layer NAMES say "-1-2" / "-1-4")
        conv("policy_conv-1-2", 1, f, pol_c)
        bn("policy_batchnorm", pol_c)
        dense("policy_out", pol_c * 90, N_LABELS)
        conv("value_conv-1-4", 1, f, val_c)
        bn("value_batchnorm", val_c)
        dense("value_dense", val_c * 90, vfc)
        dense("value_out", vfc, 1)
        self.weights = w
        self.model = self
        return self

    @staticmethod
    def fetch_digest(weight_path):
        """model.py:85-92."""
        if os.path.exists(weight_path):
            m = hashlib.sha256()
            with open(weight_path, "rb") as f:
                m.update(f.read())
            return m.hexdigest()
        return None

    def load(self, config_path, weight_path):
        """model.py:95-107.  `weight_path` must be an .npz written by `save()`."""
        if not os.path.exists(weight_path):
            return False
        if weight_path.endswith(".h5") or open(weight_path, "rb").read(8) == b"\x89HDF\r\n\x1a\n":
            from .keras_h5 import read_keras_weights
            self.weights = read_keras_weights(weight_path)
            self._infer_geometry()
            self.digest = self.fetch_digest(weight_path)
            self.model = self
            return True
        if not os.path.exists(config_path):
            return False
        with open(config_path, "rt") as f:
            cfg = json.load(f)
        mc = self.config.model
        mc.cnn_filter_num, mc.res_layer_num = cfg["cnn_filter_num"], cfg["res_layer_num"]
        mc.value_fc_size = cfg.get("value_fc_size", 256)
        with np.load(weight_path) as z:
            self.weights = {k.replace("__", "/"): z[k].astype(np.float32) for k in z.files}
        self._infer_geometry()
        self.digest = self.fetch_digest(weight_path)
        self.model = self
        return True

    def _infer_geometry(self):
        """cnn_filter_num / res_layer_num / value_fc_size from the tensors themselves (a Keras .h5 carries no config)."""
        mc = self.config.model
        k = next(v for n, v in self.weights.items() if n.startswith("input_conv") and n.endswith("/kernel"))
        if k.shape[:2] != (5, 5) or k.shape[2] not in (14, 28):
            raise NotImplementedError(f"input convolution {k.shape}: only 5x5 on 14 or 28 planes is built")
        mc.input_depth = int(k.shape[2])
        mc.cnn_filter_num = int(k.shape[3])
        mc.res_layer_num = max(int(n[3:n.index("_")]) for n in self.weights if n.startswith("res"))
        mc.value_fc_size = int(self.weights["value_dense/bias"].shape[0])
        mc.policy_channels = int(next(v for n, v in self.weights.items() if n.startswith("policy_conv") and n.endswith("/kernel")).shape[3])
        mc.value_channels = int(next(v for n, v in self.weights.items() if n.startswith("value_conv") and n.endswith("/kernel")).shape[3])

    @property
    def use_history(self):
        """What load_model returns next to the model (worker/self_play.py:29-46): the network reads 28 planes."""
        if not self.weights:
            return getattr(self.config.model, "input_depth", 14) == 28
        k = next(v for n, v in self.weights.items() if n.startswith("input_conv") and n.endswith("/kernel"))
        return int(k.shape[2]) == 28

    def save(self, config_path, weight_path):
        """model.py:109-115."""
        mc = self.config.model
        os.makedirs(os.path.dirname(config_path) or ".", exist_ok=True)
        with open(config_path, "wt") as f:
            json.dump({"cnn_filter_num": mc.cnn_filter_num, "res_layer_num": mc.res_layer_num,
                       "value_fc_size": mc.value_fc_size, "format": "cczero-b200 npz, Keras weight names"}, f)
        with open(weight_path, "wb") as f:          # np.savez would append ".npz" to a bare path
            np.savez(f, **{k.replace("/", "__"): v for k, v in self.weights.items()})
        self.digest = self.fetch_digest(weight_path)

    def torch_weights(self, device=None):
        import torch
        return {k: torch.as_tensor(v).to(device) if device else torch.as_tensor(v) for k, v in self.weights.items()}

    # ---- model.py:117-126
    def get_pipes(self, num=1, api=None, need_reload=True):
        if self.api is None:
            from .api import CChessModelAPI
            self.api = CChessModelAPI(self.config, self)
            self.api.start(need_reload)
        return self.api.get_pipe(need_reload)

    def close_pipes(self):
        if self.api is not None:
            self.api.close()
            self.api = None
