"""Error-budget emulation of the packed-fp16 depthwise arithmetic (test infrastructure, CPU only; not collected by pytest):

    python tests/emulate_dw_precision.py [ARCH SIZE ...]        # default: XS 128, S 128, S 256

Runs the BN-folded network (oracle.model_ref.fold_bn) with fp16 storage of every activation and every depthwise
convolution computed by the bit-exact emulator of the kernels (tests/dw_emul.py, mirrored lanes included):
  None  fp32 depthwise (F.conv2d)
  0/1/2 the 7x7 and stem 3x3 depthwise at lp_set_dw_precision 0 / 1 / 2, the 5x5 heads at precision 0 -- mode 2 is the
        shipped arithmetic (dwconv.cu default, dwpw.cu / dwblock.cu / stem_fused.cu packed chains)
and prints max|out - fp32 oracle| / (2e-3 * max|ref| + 1e-4) for the two network outputs.  Measured (random BN-folded
weights, synth.make_frames input):
            None           0              1              2 (shipped)
  XS 128    0.302 0.286    0.315 0.285    0.331 0.289    0.336 0.283
  S 128     0.272 0.254    0.282 0.258    0.332 0.328    0.270 0.314
  S 256     0.291 0.266    0.285 0.282    0.330 0.293    0.318 0.287
  M 512     0.616 0.382    0.663 0.425    0.682 0.393    0.671 0.415
The shipped arithmetic moves the ratios by at most 0.06 from an fp32 depthwise: the budget is dominated by the fp16
activation storage, which the reference's own fp16 path shares."""
import os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch.nn.functional as F
import dw_emul
from litepose_b200 import synth
from litepose_b200.config import get_arch, get_cfg
from litepose_b200.lib.models.pose_mobilenet import get_pose_net
from oracle import model_ref

ACTS = {None: dw_emul.ACT_NONE, "relu": dw_emul.ACT_RELU, "relu6": dw_emul.ACT_RELU6}

def h(t): return t.half().float()

def dw_emul_nchw(x, w, b, stride, act, prec):
    """x [N,C,H,W] fp32 holding fp16 values, w [C,1,k,k], b [C] -> the kernel's fp16 output (activation applied), NCHW"""
    C, k = w.shape[0], w.shape[-1]
    xn = x.permute(0, 2, 3, 1).contiguous().numpy().astype(np.float16)
    wt = w.reshape(C, k * k).t().contiguous().numpy().astype(np.float16)
    y = dw_emul.dwconv(xn, wt, b.numpy().astype(np.float32), k, stride, ACTS[act], prec)
    return torch.from_numpy(y.astype(np.float32)).permute(0, 3, 1, 2).contiguous()

def forward(fp, arch, x, mode):
    q = h
    def conv(name, x, stride=1, groups=1, act=None):
        w, b = fp[name]
        if mode is not None and groups > 1:
            return dw_emul_nchw(x, q(w), b, stride, act, 0 if w.shape[-1] == 5 else mode)
        y = F.conv2d(x, q(w), b, stride, w.shape[-1] // 2, 1, groups)
        if act == "relu6": y = F.relu6(y)
        elif act == "relu": y = F.relu(y)
        return y
    x = q(x.float())
    x = q(conv("first.0", x, 2, 1, "relu6")); x = q(conv("first.1", x, 1, x.shape[1], "relu6")); x = q(conv("first.2", x))
    x_list = [x]
    for si, st in enumerate(arch["backbone_setting"]):
        for bi in range(st["num_blocks"]):
            p = "stage.%d.%d." % (si, bi); stride = st["stride"] if bi == 0 else 1
            inp = x
            y = q(conv(p + "inv", x, 1, 1, "relu6"))
            y = q(conv(p + "depth_conv", y, stride, y.shape[1], "relu6"))
            y = conv(p + "point_conv", y)
            if stride == 1 and inp.shape[1] == y.shape[1]: y = y + inp
            x = q(y)
        x_list.append(x)
    outs = []
    refined, raw = x_list[-1], x_list[-2]
    for i in range(3):
        wr, b = fp["deconv_refined.%d" % i]; ww, _ = fp["deconv_raw.%d" % i]
        y = F.conv_transpose2d(refined, q(wr), None, 2, 1) + F.conv_transpose2d(raw, q(ww), None, 2, 1)
        refined = q(F.relu(y + b.view(1, -1, 1, 1))); raw = x_list[-i - 3]
        if i > 0:
            o = 0
            for nm, src in (("final_refined", refined), ("final_raw", raw)):
                p = "%s.%d.conv." % (nm, i - 1)
                t = q(conv(p + "dw", src, 1, src.shape[1], "relu"))
                o = o + F.conv2d(t, q(fp[p + "pw"][0]))
            outs.append(o)
    return outs

torch.set_num_threads(8)
args = sys.argv[1:]
cases = [(args[i], int(args[i + 1])) for i in range(0, len(args) - 1, 2)] or [("XS", 128), ("S", 128), ("S", 256)]
for name, size in cases:
    cfg = get_cfg(input_size=size); arch = get_arch(name)
    torch.manual_seed(0)
    model = synth.randomize_bn_(get_pose_net(cfg, False, arch), 1).eval()
    sd = model.state_dict()
    x = synth.make_frames(1, size, seed=11)
    with torch.no_grad():
        ref = model_ref.forward(sd, arch, x)
        fp = model_ref.fold_bn(sd, arch)
        for mode in (None, 0, 1, 2):
            o = forward(fp, arch, x, mode)
            r = [float((a - b).abs().max() / (2e-3 * b.abs().max() + 1e-4)) for a, b in zip(o, ref)]
            print(name, size, mode, ["%.3f" % v for v in r], flush=True)
