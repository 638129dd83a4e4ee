"""Training LitePose with its depthwise convolutions on the sm_90a kernels (csrc/dw_train.cu).

    model = convert_depthwise(model)          # before the DDP / DataParallel wrap, as with convert_sync_batchnorm

``convert_depthwise(module)`` turns every eligible depthwise ``nn.Conv2d`` of ``module`` (groups == in == out
channels, kernel 3, 5 or 7, stride 1 or 2, padding k // 2, dilation 1, zero padding, no bias) into a
``DepthwiseConv2d`` in place and returns ``module``.  The converted module keeps its ``Parameter`` objects, its state
dict and its ``isinstance(m, nn.Conv2d)``; only ``forward`` changes: a CUDA tensor goes through ``depthwise_conv2d``,
a CPU tensor through ``nn.Conv2d.forward`` as before.  The super-network's functional depthwise calls
(``SuperSepConv2d``, ``SuperInvBottleneck``) follow their converted module the same way.  Eval-mode CUDA inference of
the LitePose modules does not run the module tree at all (it runs the engine) and is unchanged.

``depthwise_conv2d(x, weight, stride)`` is the autograd function: forward, input gradient and weight gradient on the
kernels, on x's device and that device's current stream.  What stays on PyTorch: the 1x1 convolutions, BatchNorm,
the deconvolutions, the loss and the optimizer."""
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.autograd.function import once_differentiable

from litepose_b200 import _lib

_DTYPES = {torch.float32: _lib.LP_DT_F32, torch.float16: _lib.LP_DT_F16}
KERNELS = (3, 5, 7)
STRIDES = (1, 2)


def _out(h, s):
    return (h - 1) // s + 1


def _check(x, weight, stride):
    if not (torch.is_tensor(x) and torch.is_tensor(weight)):
        raise ValueError("depthwise_conv2d takes tensors x and weight")
    if not (x.is_cuda and weight.is_cuda and x.device == weight.device):
        raise ValueError("depthwise_conv2d runs on the sm_90a kernels: x and weight must be CUDA tensors on one device "
                         "(got %s and %s)" % (x.device, weight.device))
    if x.dtype != weight.dtype:
        raise ValueError("depthwise_conv2d: x is %s but weight is %s; the kernels take one dtype for both (use "
                         "torch.autocast or convert the model)" % (x.dtype, weight.dtype))
    if x.dtype not in _DTYPES:
        raise ValueError("depthwise_conv2d: %s is not supported; the kernels are fp32 and fp16 (bf16 and fp64 are not "
                         "implemented)" % x.dtype)
    if x.dim() != 4:
        raise ValueError("depthwise_conv2d takes NCHW x, got %d dimensions" % x.dim())
    c = x.shape[1]
    if weight.dim() != 4 or weight.shape[0] != c or weight.shape[1] != 1 or weight.shape[2] != weight.shape[3] or \
            weight.shape[2] not in KERNELS:
        raise ValueError("depthwise_conv2d: weight %s does not fit x with %d channels (weight [C, 1, k, k], k in "
                         "3, 5, 7)" % (tuple(weight.shape), c))
    if stride not in STRIDES:
        raise ValueError("depthwise_conv2d: stride %r (1 or 2)" % (stride,))
    if x.shape[2] < 1 or x.shape[3] < 1:
        raise ValueError("depthwise_conv2d: empty plane %s" % (tuple(x.shape),))


class _DepthwiseConv(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, stride):
        lib = _lib.load()
        n, c, h, w = x.shape
        k = weight.shape[-1]
        y = torch.empty((n, c, _out(h, stride), _out(w, stride)), dtype=x.dtype, device=x.device)
        with torch.cuda.device(x.device):
            st = torch.cuda.current_stream(x.device).cuda_stream
            _lib.check(lib.lp_dw_nchw_fwd(x.data_ptr(), weight.data_ptr(), y.data_ptr(), n, c, h, w, k, stride,
                                          _DTYPES[x.dtype], st), "lp_dw_nchw_fwd")
        ctx.save_for_backward(x, weight)
        ctx.stride = stride
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        lib = _lib.load()
        n, c, h, w = x.shape
        k, s, dt = weight.shape[-1], ctx.stride, _DTYPES[x.dtype]
        dy = dy.to(x.dtype).contiguous()
        dx = dw = None
        with torch.cuda.device(x.device):
            st = torch.cuda.current_stream(x.device).cuda_stream
            if ctx.needs_input_grad[0]:
                dx = torch.empty_like(x, memory_format=torch.contiguous_format)
                _lib.check(lib.lp_dw_nchw_dgrad(dy.data_ptr(), weight.data_ptr(), dx.data_ptr(), n, c, h, w, k, s, dt,
                                                st), "lp_dw_nchw_dgrad")
            if ctx.needs_input_grad[1]:
                dw = torch.empty_like(weight, memory_format=torch.contiguous_format)
                nb = lib.lp_dw_nchw_wgrad_workspace_bytes(n, c, h, w, k, s)
                ws = torch.empty(max(nb, 4), dtype=torch.uint8, device=x.device)
                _lib.check(lib.lp_dw_nchw_wgrad(x.data_ptr(), dy.data_ptr(), dw.data_ptr(), n, c, h, w, k, s, dt,
                                                ws.data_ptr(), nb, st), "lp_dw_nchw_wgrad")
        return dx, dw, None


def depthwise_conv2d(x, weight, stride=1):
    """F.conv2d(x, weight, None, stride, k // 2, 1, C) for an NCHW CUDA x [N, C, H, W] and weight [C, 1, k, k], on the
    sm_90a kernels, with autograd (once differentiable: double backward raises).

    Runs on x's device and its current stream.  x, weight and the incoming gradient are made contiguous when they are
    not (a sliced super-network weight is not; autograd routes its gradient back through the slice).  The output is
    NCHW-contiguous whatever x's memory format: a channels_last x gives a contiguous_format output.  Under
    ``torch.autocast("cuda", torch.float16)`` x and weight are cast to fp16 as F.conv2d casts them and the fp16
    kernels run.  Raises ValueError for CPU tensors, bf16 / fp64, x and weight of different dtypes outside autocast,
    bf16 autocast, and shapes the kernels do not take (k not 3, 5 or 7, stride not 1 or 2)."""
    if torch.is_tensor(x) and x.is_cuda and torch.is_autocast_enabled("cuda"):
        if torch.get_autocast_dtype("cuda") != torch.float16:
            raise ValueError("depthwise_conv2d: autocast to %s is not supported (the kernels are fp32 and fp16)"
                             % torch.get_autocast_dtype("cuda"))
        # autocast's rule for conv2d: every floating-point operand but fp64 runs in the autocast dtype
        x = x.to(torch.float16) if x.is_floating_point() and x.dtype != torch.float64 else x
        weight = weight.to(torch.float16) if weight.is_floating_point() and weight.dtype != torch.float64 else weight
    _check(x, weight, stride)
    return _DepthwiseConv.apply(x.contiguous(), weight.contiguous(), stride)


class DepthwiseConv2d(nn.Conv2d):
    """An ``nn.Conv2d`` (depthwise, as ``convert_depthwise`` admits it) whose forward on CUDA tensors runs the sm_90a
    kernels; CPU tensors take ``nn.Conv2d.forward``."""

    def forward(self, x):
        if x.is_cuda:
            return depthwise_conv2d(x, self.weight, self.stride[0])
        return super().forward(x)

    def forward_weight(self, x, weight):
        """This conv's depthwise convolution of x with another weight [C', 1, k', k'] (C' = x's channels, padding
        k' // 2): the super-network's sliced / transformed weights.  CPU tensors take F.conv2d."""
        if x.is_cuda:
            return depthwise_conv2d(x, weight, self.stride[0])
        return F.conv2d(x, weight, None, self.stride, weight.shape[-1] // 2, self.dilation, x.shape[1])


def is_eligible(m):
    """A plain nn.Conv2d the kernels compute exactly as it is configured."""
    if type(m) is not nn.Conv2d:
        return False
    k = m.kernel_size
    return (m.groups == m.in_channels == m.out_channels and k[0] == k[1] and k[0] in KERNELS and
            m.stride in ((1, 1), (2, 2)) and m.padding == (k[0] // 2, k[0] // 2) and m.dilation == (1, 1) and
            m.padding_mode == "zeros" and m.bias is None)


def convert_depthwise(module):
    """Every eligible depthwise nn.Conv2d in ``module`` (``module`` itself included) becomes a DepthwiseConv2d, in
    place; returns ``module``.  Call it before wrapping the model in DistributedDataParallel / DataParallel."""
    for m in module.modules():
        if is_eligible(m):
            m.__class__ = DepthwiseConv2d
    return module
