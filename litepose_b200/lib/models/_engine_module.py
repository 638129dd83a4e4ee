"""Engine management shared by the drop-in LitePose modules (``pose_mobilenet``, ``pose_simplenet``).

``EngineModule`` is the ``nn.Module`` base of both: in eval mode on a CUDA tensor ``forward`` runs the hand-written
sm_90a kernels through a ``litepose_b200.engine.LitePoseEngine`` built from the module's state_dict and cached per
device; on CPU tensors and in training mode it runs the module tree (``_forward_modules`` of the subclass).  The
engine recognises which of the two heads the state_dict carries."""
import threading

import torch
import torch.nn as nn


class _EngineCache(object):
    """Per-device compiled state; deliberately not copied by deepcopy / pickling.  One object is shared by a module
    and its nn.DataParallel replicas (replicate() copies the module __dict__ shallowly), one engine per device, so
    lookups / builds take the lock (DataParallel runs the replicas on threads, reference valid.py:165)."""

    def __init__(self):
        self.engines = {}
        self.lock = threading.RLock()
        self.master_sig = None          # signature of the master module at the last DataParallel replication
        self.keys = None                # its state_dict keys (replicas resolve their tensors by attribute path)

    def clear(self):
        with self.lock:
            self.engines.clear()

    def __deepcopy__(self, memo):
        return _EngineCache()

    def __getstate__(self):
        return {}

    def __setstate__(self, state):
        self.__init__()


class EngineModule(nn.Module):
    """Subclasses set ``self.cfg_arch`` and ``self._lp_cache = _EngineCache()`` in their constructor and define
    ``_forward_modules(x)``, the module-tree forward."""

    def lp_invalidate(self):
        """Drop the packed-weight cache.  Not needed after the usual mutations: .to()/.half(), load_state_dict,
        train()/eval() switches, re-assignment, and any in-place update of a parameter or buffer itself (optimizer
        step, BN statistics, ``p.copy_`` / ``p.mul_`` under no_grad) are detected.  NOT detected: writes through a
        detached alias (``p.data.copy_(...)``, ``p.detach().mul_()``: the alias carries its own version counter) -
        call this after those."""
        self._lp_cache.clear()

    def _apply(self, fn, *args, **kwargs):      # .cuda() / .half() / .float() / .to()
        self._lp_cache.clear()
        return super()._apply(fn, *args, **kwargs)

    def load_state_dict(self, *args, **kwargs):
        self._lp_cache.clear()
        return super().load_state_dict(*args, **kwargs)

    def _load_from_state_dict(self, *args, **kwargs):   # when loaded as a child (network_to_half wrapper)
        self._lp_cache.clear()
        return super()._load_from_state_dict(*args, **kwargs)

    def train(self, mode=True):
        # training steps run the nn.Module tree and update parameters / BN statistics in place: the folded weights
        # of a previous eval phase are stale afterwards
        self._lp_cache.clear()
        return super().train(mode)

    def _lp_signature(self):
        """Hash over (identity, data pointer, autograd version counter) of every parameter and buffer: changes with
        every in-place update of the tensor itself (optimizer.step, running statistics, copy_/mul_ under no_grad) and with
        every re-assignment; writes through ``.data`` / ``.detach()`` aliases are invisible to it (lp_invalidate)."""
        return hash(tuple((id(t), t.data_ptr(), t._version)
                          for group in (self.parameters(), self.buffers()) for t in group))

    def _replicate_for_data_parallel(self):
        # nn.DataParallel replicates the master on every forward: publish the master's signature so that the replicas
        # (whose tensors are fresh broadcasts without history) can tell a stale per-device engine from a current one
        self._lp_cache.master_sig = self._lp_signature()
        self._lp_cache.keys = list(self.state_dict().keys())
        return super()._replicate_for_data_parallel()

    def _lp_state(self):
        """state_dict of this module; DataParallel replicas hold their (broadcast) tensors as plain attributes, not as
        registered parameters, so their entries are resolved by attribute path from the master's key list."""
        if not getattr(self, "_is_replica", False):
            return self.state_dict()
        out = {}
        for k in self._lp_cache.keys:
            obj = self
            for part in k.split("."):
                obj = getattr(obj, part)
            out[k] = obj
        return out

    def _lp_device_key(self, device):
        dev = torch.device(device) if device is not None else next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("the litepose_b200 engine needs the module on a CUDA device")
        return (dev.type, dev.index if dev.index is not None else torch.cuda.current_device())

    def _lp_cached(self, key, build, capacity=None):
        """The engine cached under ``key`` while the module's weights are those it was built from, else
        ``build(state_dict, device)``.  ``capacity``: keep at most that many engines, least recently used dropped."""
        # DataParallel replicas receive freshly broadcast tensors on every forward (version 0, new identity): they use
        # the signature the master published when it was replicated
        replica = getattr(self, "_is_replica", False)
        sig = self._lp_cache.master_sig if replica else self._lp_signature()
        with self._lp_cache.lock:
            engines = self._lp_cache.engines
            hit = engines.pop(key, None)
            if hit is not None and hit[1] == sig:
                engines[key] = hit              # most recently used last
                return hit[0]
            eng = build(self._lp_state(), torch.device("cuda", key[1]))
            engines[key] = (eng, sig)
            while capacity is not None and len(engines) > capacity:
                del engines[next(iter(engines))]
            return eng

    def lp_engine(self, device=None):
        from litepose_b200.engine import LitePoseEngine
        key = self._lp_device_key(device)
        return self._lp_cached(key, lambda state, dev: LitePoseEngine(state, self.cfg_arch, dev))

    def forward(self, x):
        if x.is_cuda and not self.training:
            # CUDA inference: hand-written sm_90a kernels only (raises if the library is missing)
            half_in = x.dtype == torch.float16
            return self.lp_engine(x.device).run(x, flip=False, out_fp32=not half_in, clone=True)
        return self._forward_modules(x)
