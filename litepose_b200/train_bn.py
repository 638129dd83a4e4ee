"""Training LitePose with its BatchNorm layers, and the ReLU / ReLU6 that follows each, on the sm_90a kernels
(csrc/bn_nchw_train.cu).

    model = convert_batchnorm(model)          # before the DDP / DataParallel wrap; independent of convert_depthwise

``convert_batchnorm(module)`` turns every eligible ``nn.BatchNorm2d`` (affine, tracking running statistics, a momentum
that is not None) into a ``BatchNormAct2d`` and every eligible ``SuperBatchNorm2d`` into a ``SuperBatchNormAct2d``, in
place, and returns ``module``.  The converted modules keep their ``Parameter`` objects, their state dict and their
``isinstance``; only ``forward`` changes: a train-mode forward on a CUDA tensor runs ``batch_norm_act``, anything else
(eval mode, CPU tensors) the unchanged ``F.batch_norm``.

Activation fusion: a ``nn.ReLU`` / ``nn.ReLU6`` that directly follows a converted BatchNorm in the same ``nn.Sequential``
becomes a ``FusedReLU`` / ``FusedReLU6`` (still an instance of its class), and the BatchNorm applies it in its kernel.
The fused output is tagged with the activation it had applied (and its version counter); the converted activation
returns a tensor so tagged unchanged and applies itself to anything else.  So the activation is applied exactly once
on every path: the fused one, the eval / CPU paths (untagged), and after the BatchNorm was replaced by a fresh module
(``nn.SyncBatchNorm.convert_sync_batchnorm``: untagged).  The residual add of ``InvBottleneck`` stays in torch.

``batch_norm_act(x, weight, bias, running_mean, running_var, momentum, eps, act)`` is the autograd function."""
import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from litepose_b200 import _lib
from litepose_b200.lib.models.pose_supermobilenet import SuperBatchNorm2d

_DTYPES = {torch.float32: _lib.LP_DT_F32, torch.float16: _lib.LP_DT_F16}
ACT_NONE, ACT_RELU, ACT_RELU6 = _lib.ACT_NONE, _lib.ACT_RELU, _lib.ACT_RELU6
_ACTS = {nn.ReLU: ACT_RELU, nn.ReLU6: ACT_RELU6}


def _check(x, weight, bias, running_mean, running_var, momentum, act):
    ts = (x, weight, bias, running_mean, running_var)
    if not all(torch.is_tensor(t) for t in ts):
        raise ValueError("batch_norm_act takes tensors x, weight, bias, running_mean and running_var")
    if not all(t.is_cuda and t.device == x.device for t in ts):
        raise ValueError("batch_norm_act runs on the sm_90a kernels: every tensor must be a CUDA tensor on x's device "
                         "(got %s)" % ", ".join(str(t.device) for t in ts))
    if x.dtype not in _DTYPES:
        raise ValueError("batch_norm_act: x is %s; the kernels take fp32 and fp16 (bf16 and fp64 are not implemented)"
                         % x.dtype)
    if any(t.dtype != torch.float32 for t in ts[1:]):
        raise ValueError("batch_norm_act: weight, bias and the running statistics must be fp32 (got %s); keep "
                         "BatchNorm in fp32 as network_to_half does" % ", ".join(str(t.dtype) for t in ts[1:]))
    if x.dim() != 4:
        raise ValueError("batch_norm_act takes NCHW x, got %d dimensions" % x.dim())
    n, c, h, w = x.shape
    if any(t.dim() != 1 or t.shape[0] != c for t in ts[1:]):
        raise ValueError("batch_norm_act: parameters %s do not fit x with %d channels"
                         % ([tuple(t.shape) for t in ts[1:]], c))
    if not (running_mean.is_contiguous() and running_var.is_contiguous()):
        raise ValueError("batch_norm_act: the running statistics are updated in place and must be contiguous")
    if n * h * w <= 1:
        raise ValueError("batch_norm_act: expected more than 1 value per channel when training, got input size %s"
                         % (tuple(x.shape),))
    if momentum is None:
        raise ValueError("batch_norm_act: momentum None (a cumulative moving average) is not supported")
    if act not in (ACT_NONE, ACT_RELU, ACT_RELU6):
        raise ValueError("batch_norm_act: act %r (ACT_NONE, ACT_RELU or ACT_RELU6)" % (act,))


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


class _BatchNormAct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, momentum, eps, act):
        lib = _lib.load()
        n, c, h, w = x.shape
        y = torch.empty_like(x, memory_format=torch.contiguous_format)
        saved = torch.empty(4, c, dtype=torch.float32, device=x.device)
        nb = lib.lp_bn_nchw_workspace_bytes(n, c, h, w)
        ws = torch.empty(max(nb, 8), dtype=torch.uint8, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check(lib.lp_bn_nchw_fwd(x.data_ptr(), weight.data_ptr(), bias.data_ptr(), running_mean.data_ptr(),
                                          running_var.data_ptr(), float(momentum), float(eps), y.data_ptr(),
                                          saved.data_ptr(), n, c, h, w, act, _DTYPES[x.dtype], ws.data_ptr(), nb,
                                          _stream(x.device)), "lp_bn_nchw_fwd")
        # the kernel wrote the running statistics: move their version counters as an in-place op would, so that
        # caches keyed on them (the eval engine's) see the change
        torch.autograd.graph.increment_version(running_mean)
        torch.autograd.graph.increment_version(running_var)
        ctx.save_for_backward(x, weight, saved)
        ctx.act = act
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, weight, saved = ctx.saved_tensors
        need_x, need_w, need_b = ctx.needs_input_grad[:3]
        dx = dw = db = None
        if need_x or need_w or need_b:
            lib = _lib.load()
            n, c, h, w = x.shape
            dy = dy.to(x.dtype).contiguous()
            dx = torch.empty_like(x, memory_format=torch.contiguous_format) if need_x else None
            dw = torch.empty(c, dtype=torch.float32, device=x.device) if need_w else None
            db = torch.empty(c, dtype=torch.float32, device=x.device) if need_b else None
            nb = lib.lp_bn_nchw_workspace_bytes(n, c, h, w)
            ws = torch.empty(max(nb, 8), dtype=torch.uint8, device=x.device)
            with torch.cuda.device(x.device):
                _lib.check(lib.lp_bn_nchw_bwd(x.data_ptr(), dy.data_ptr(), weight.data_ptr(), saved.data_ptr(),
                                              _lib.ptr(dx), _lib.ptr(dw), _lib.ptr(db), n, c, h, w, ctx.act,
                                              _DTYPES[x.dtype], ws.data_ptr(), nb, _stream(x.device)),
                           "lp_bn_nchw_bwd")
        return dx, dw, db, None, None, None, None, None


def batch_norm_act(x, weight, bias, running_mean, running_var, momentum=0.1, eps=1e-5, act=ACT_NONE):
    """act(F.batch_norm(x, running_mean, running_var, weight, bias, True, momentum, eps)) for an NCHW CUDA x, on the
    sm_90a kernels, with autograd (once differentiable: double backward raises); act is ACT_NONE, ACT_RELU or
    ACT_RELU6.

    Train mode: normalises with the batch statistics (biased variance) and updates running_mean / running_var in place
    to (1 - momentum) * running + momentum * batch statistic (unbiased variance).  Runs on x's device and its current
    stream and never synchronises the host.  x is fp32 or fp16 (network_to_half, autocast), weight, bias and the
    running statistics fp32; the output has x's dtype and is NCHW-contiguous.  Backward computes only the gradients
    that are needed: dx in x's dtype, dweight / dbias in fp32.  NaN and inf propagate as under F.batch_norm +
    F.relu / F.relu6.  Raises ValueError for CPU tensors, bf16 / fp64 x, parameters that are not fp32, one value per
    channel (N*H*W == 1) and momentum None."""
    _check(x, weight, bias, running_mean, running_var, momentum, act)
    return _BatchNormAct.apply(x.contiguous(), weight.contiguous(), bias.contiguous(), running_mean, running_var,
                               momentum, eps, act)


def _fused(bn, x, weight, bias, running_mean, running_var):
    y = batch_norm_act(x, weight, bias, running_mean, running_var, bn.momentum, bn.eps, bn.lp_act)
    if bn.lp_act != ACT_NONE:
        y._lp_act = (bn.lp_act, y._version)
    return y


def _applied(x):
    """the activation a converted BatchNorm applied to x, if x is still that output unchanged"""
    tag = getattr(x, "_lp_act", None)
    return tag[0] if tag is not None and tag[1] == x._version else ACT_NONE


class BatchNormAct2d(nn.BatchNorm2d):
    """An ``nn.BatchNorm2d`` whose train-mode forward on CUDA tensors runs the sm_90a kernels, with the activation
    ``lp_act`` (set by ``convert_batchnorm``) fused; eval mode and CPU tensors take ``nn.BatchNorm2d.forward``."""
    lp_act = ACT_NONE
    lp_base = nn.BatchNorm2d

    def forward(self, x):
        if not (x.is_cuda and self.training):
            return super().forward(x)
        self._check_input_dim(x)
        if self.momentum is None:
            raise ValueError("BatchNormAct2d: momentum None (a cumulative moving average) is not supported")
        if self.num_batches_tracked is not None:     # as _BatchNorm.forward counts it
            self.num_batches_tracked.add_(1)
        return _fused(self, x, self.weight, self.bias, self.running_mean, self.running_var)


class SuperBatchNormAct2d(SuperBatchNorm2d):
    """A ``SuperBatchNorm2d`` (the leading [:c] channels of its parameters and statistics) whose train-mode forward on
    CUDA tensors runs the sm_90a kernels with ``lp_act`` fused.  num_batches_tracked is not counted, as
    ``SuperBatchNorm2d``'s ``F.batch_norm`` call does not count it."""
    lp_act = ACT_NONE
    lp_base = SuperBatchNorm2d

    def forward(self, x):
        if not (x.is_cuda and self.training):
            return super().forward(x)
        if self.momentum is None:
            raise ValueError("SuperBatchNormAct2d: momentum None (a cumulative moving average) is not supported")
        c = x.shape[1]
        return _fused(self, x, self.weight[:c], self.bias[:c], self.running_mean[:c], self.running_var[:c])


class FusedReLU(nn.ReLU):
    """nn.ReLU after a converted BatchNorm: returns that BatchNorm's fused output (ReLU or ReLU6 applied) unchanged."""

    def forward(self, x):
        if _applied(x) in (ACT_RELU, ACT_RELU6):
            return x
        return super().forward(x)


class FusedReLU6(nn.ReLU6):
    """nn.ReLU6 after a converted BatchNorm: returns that BatchNorm's fused output (ReLU6 applied) unchanged."""

    def forward(self, x):
        if _applied(x) == ACT_RELU6:
            return x
        return super().forward(x)


_CONVERTED = {nn.BatchNorm2d: BatchNormAct2d, SuperBatchNorm2d: SuperBatchNormAct2d}
_FUSED_ACT = {nn.ReLU: FusedReLU, nn.ReLU6: FusedReLU6}


def is_eligible(m):
    """A plain nn.BatchNorm2d or SuperBatchNorm2d the kernels compute exactly as it is configured."""
    return type(m) in _CONVERTED and m.affine and m.track_running_stats and m.momentum is not None


def convert_batchnorm(module):
    """Every eligible BatchNorm in ``module`` (``module`` itself included) becomes a BatchNormAct2d /
    SuperBatchNormAct2d, in place, fused with the ReLU / ReLU6 that directly follows it in an nn.Sequential; returns
    ``module``.  Call it before wrapping the model in DistributedDataParallel / DataParallel."""
    for seq in module.modules():
        if isinstance(seq, nn.Sequential):
            kids = list(seq.children())
            for bn, act in zip(kids, kids[1:]):
                if is_eligible(bn) and type(act) in _ACTS:
                    bn.lp_act = _ACTS[type(act)]
                    act.__class__ = _FUSED_ACT[type(act)]
    for m in module.modules():
        if is_eligible(m):
            m.__class__ = _CONVERTED[type(m)]
    return module
