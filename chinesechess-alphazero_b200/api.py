"""`CChessModelAPI` drop-in (reference: cchess_alphazero/agent/api.py:16-117): the batching prediction server.

Same wire protocol as the reference, so UNMODIFIED reference players can be served by the GPU network:
a client sends `list[np.float32[14,10,9]]` (`[28,10,9]` for a use_history network) on its pipe end, the server answers `list[(np.float32[2086], float)]`
in the same order (api.py:48-74 <-> player.py:118-120,131-140).  One daemon thread waits on every pipe, drains
what is ready, runs ONE batched forward (`cz_nn_forward`: tensor-core pipeline) and scatters the results.

Weight hot-reload: the reference re-reads the best-model file every 600 s when its digest changed
(api.py:42-44,76-88); `try_reload_model()` does the same against the `.npz` path in config.resource.
"""
from logging import getLogger
from multiprocessing import Pipe, connection
from threading import Thread
from time import time

import numpy as np
import torch

from .engine import Engine
from .model import engine_net_kwargs
from .lib import get_lib

logger = getLogger(__name__)


class CChessModelAPI:
    def __init__(self, config, agent_model, lib=None, device=None, max_batch=2048):
        self.agent_model = agent_model
        self.pipes = []
        self.config = config
        self.need_reload = True
        self.done = False
        self.lib = lib or get_lib()
        self.device = device or "cuda"
        self.max_batch = max_batch
        self.engine = None
        self.positions = 0
        self.batches = 0
        self.last_error = None
        self._last_check = time()

    def _ensure_engine(self):
        if self.engine is None:
            mc = self.config.model
            self.engine = Engine(self.lib, self.device, n_games=self.max_batch, sims_per_move=1, leaves_per_round=1,
                                 max_nodes_per_game=16, max_edges_per_game=256, max_path=8,
                                 **engine_net_kwargs(mc),
                                 use_history=bool(getattr(self.agent_model, "use_history", False)))
            self.engine.set_weights(self.agent_model.torch_weights())

    def start(self, need_reload=True):
        self.need_reload = need_reload
        self._ensure_engine()
        t = Thread(target=self.predict_batch_worker, name="prediction_worker", daemon=True)
        t.start()
        self.thread = t

    def get_pipe(self, need_reload=True):
        me, you = Pipe()
        self.pipes.append(me)
        self.need_reload = need_reload
        return you

    def predict_batch_worker(self):
        if self.engine.lib.is_cuda and self.engine.device.index is not None:
            torch.cuda.set_device(self.engine.device)
        while not self.done:
            try:
                self._serve_once()
            except Exception as e:           # keep serving: a dead prediction thread would block every player
                self.last_error = e
                logger.error(f"prediction worker: {e!r}")

    def _collect(self):
        """Every request waiting on any pipe, as (connection, list of planes), in arrival order per pipe."""
        requests = []
        for conn in connection.wait(self.pipes, timeout=0.001):
            try:
                while conn.poll():
                    requests.append((conn, conn.recv()))
            except EOFError:                             # the player went away
                conn.close()
                if conn in self.pipes:
                    self.pipes.remove(conn)
        return requests

    def _serve_once(self):
        now = time()
        if self.need_reload and now - self._last_check > 600:      # api.py:42-44
            self._last_check = now                                 # before the attempt: a failing reload is retried in 600 s, not every loop
            self.try_reload_model()
        requests = self._collect()
        if not requests:
            return
        batch = np.asarray([p for _, planes in requests for p in planes], dtype=np.float32)
        pol, val = self.engine.nn_forward_planes(torch.from_numpy(batch).to(self.engine.device))     # ONE forward for all of them
        policy, value = pol.cpu().numpy(), val.cpu().numpy()
        self.positions += len(batch)
        self.batches += 1
        offset = 0
        for conn, planes in requests:                    # one reply per request, same order (api.py:65-74)
            conn.send([(policy[offset + i], float(value[offset + i])) for i in range(len(planes))])
            offset += len(planes)

    def try_reload_model(self, config_file=None):
        rc = getattr(self.config, "resource", None)
        if rc is None:
            return
        path = rc.model_best_weight_path
        digest = self.agent_model.fetch_digest(path)
        if not digest or digest == self.agent_model.digest:
            return
        # Load into a scratch model first: the served model object (weights, digest, geometry) changes only after the
        # engine accepted the new weights, so a half-written file or a different geometry leaves the old network serving
        # AND the old digest in place (the next check tries again).
        import copy
        cand = type(self.agent_model)(copy.deepcopy(self.config))
        try:
            if not cand.load(rc.model_best_config_path, path):
                return
            cm, mc = cand.config.model, self.config.model
            geo = lambda m: (m.cnn_filter_num, m.res_layer_num, m.value_fc_size, getattr(m, "input_depth", 14))
            if geo(cm) != geo(mc):
                raise ValueError(f"new weight file has geometry {geo(cm)}, the serving engine was built for {geo(mc)}")
            self.engine.set_weights(cand.torch_weights())
        except Exception as e:
            logger.error(f"reload of {path} failed, keeping the current weights: {e!r}")
            return
        self.agent_model.weights, self.agent_model.digest = cand.weights, cand.digest

    def close(self):
        self.done = True
        if self.engine is not None and getattr(self, "thread", None) is not None:
            self.thread.join(timeout=2)
