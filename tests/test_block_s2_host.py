"""CPU: host side of the fused stride-2 block kernel - the shape gate of lp_block_s2_supported, argument checks that
reject a launch before it reaches the device, and the engine's plan (which blocks run fused, scratch sizing)."""
import torch

from litepose_b200 import _lib, engine, synth
from litepose_b200.config import get_arch, get_cfg
from litepose_b200.lib.models.pose_mobilenet import get_pose_net


def test_block_s2_supported_gate():
    lib = _lib.load()
    ok = [(16, 96, 16), (16, 96, 32), (16, 96, 24), (8, 48, 16), (16, 32, 8), (16, 160, 16), (16, 96, 64)]
    assert [lib.lp_block_s2_supported(*c) for c in ok] == [1] * len(ok)
    assert lib.lp_block_s2_supported(32, 192, 48) == 0      # Cin > 16: one K = 16 expansion slice only
    assert lib.lp_block_s2_supported(24, 144, 32) == 0
    assert lib.lp_block_s2_supported(16, 96, 72) == 0       # Co > 64
    assert lib.lp_block_s2_supported(12, 96, 16) == 0       # multiples of 8
    assert lib.lp_block_s2_supported(16, 100, 16) == 0
    assert lib.lp_block_s2_supported(16, 96, 20) == 0
    assert lib.lp_block_s2_supported(16, 1024, 16) == 0     # shared-memory budget


def test_block_s2_rejects_bad_args_on_host():
    lib = _lib.load()
    p = 1 << 20                                              # never dereferenced: the checks come first
    for (h, w, cin, ce, co) in ((255, 256, 16, 96, 16), (256, 257, 16, 96, 16), (256, 256, 32, 192, 48),
                                (256, 256, 16, 96, 72)):
        rc = lib.lp_block_s2_f16(p, p, None, p, None, p, None, p, 1, h, w, cin, ce, co, None)
        assert rc == 1, (h, w, cin, ce, co)
        assert b"lp_block_s2_f16" in lib.lp_last_error()
    assert lib.lp_block_s2_f16(None, p, None, p, None, p, None, p, 1, 256, 256, 16, 96, 16, None) == 1


def _plan(arch_name, size):
    arch = get_arch(arch_name)
    torch.manual_seed(0)
    model = synth.randomize_bn_(get_pose_net(get_cfg(input_size=size), False, arch), 1).eval()
    eng = engine.LitePoseEngine(model.state_dict(), arch, "cpu")
    return eng._build_plan(2, size, size, torch.float16, True, alloc=engine._Bump())


def test_litepose_s_plan_fuses_the_narrow_stride2_blocks():
    plan = _plan("S", 512)
    s2 = [tuple(op.args[8:14]) for op in plan["ops"] if op.name == "block_s2"]
    assert s2 == [(2, 256, 256, 16, 96, 16), (2, 128, 128, 16, 96, 32)]
    dw7_s2 = [tuple(op.args[4:10]) for op in plan["ops"] if op.name == "dw7" and tuple(op.args[8:10]) == (7, 2)]
    assert len(dw7_s2) == 1 and dw7_s2[0][0] == 2 and dw7_s2[0][2:] == (64, 64, 7, 2)    # stage 2, block 0 (Cin 32)
    # the expansion scratch serves only the blocks that still run unfused: stage 2 block 0 (64 x 64 x 192) is the largest
    e_buf = [k for k in plan["keep"] if len(k.shape) == 1][0]
    assert e_buf.shape[0] == 2 * 64 * 64 * 192


def test_litepose_xs_plan_fuses_the_narrow_stride2_blocks():
    plan = _plan("XS", 256)
    assert [op.name for op in plan["ops"]].count("block_s2") == 2
