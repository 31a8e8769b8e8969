"""GPU parity of the fused FPN pyramid pieces (SURVEY §8 f.1): conv1x1 + bias + add as one wgmma GEMM and the two-pass
GroupNorm, against the stock PyTorch modules in true fp32 (forward and all gradients).  The end-to-end check is
tests/test_gpu_shells.py, whose Segtran3d / Segtran2d fixtures (produced by the real reference) run through these stages."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _true_fp32():
    torch.manual_seed(0)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.mark.parametrize("shape,cout", [((2, 24, 6, 8, 10), 40), ((3, 16, 12, 20), 72), ((1, 192, 8, 8, 8), 480)])
def test_conv1x1_add_matches_torch(shape, cout):
    from segtran_b200 import ops
    nd = len(shape) - 2
    conv = (torch.nn.Conv3d if nd == 3 else torch.nn.Conv2d)(shape[1], cout, 1).cuda()
    x = torch.randn(*shape, device="cuda", requires_grad=True)
    add = torch.randn(shape[0], cout, *shape[2:], device="cuda", requires_grad=True)
    G = torch.randn(shape[0], cout, *shape[2:], device="cuda")
    ref = conv(x) + add
    (ref * G).sum().backward()
    want = [x.grad.clone(), add.grad.clone(), conv.weight.grad.clone(), conv.bias.grad.clone()]
    x.grad = add.grad = conv.weight.grad = conv.bias.grad = None
    assert ops.conv1x1_ok(x, conv)
    y = ops.conv1x1_add(x, conv.weight, conv.bias, addend=add)
    (y * G).sum().backward()
    assert _rel(y, ref) < 1e-3                              # TF32 operands, fp32 accumulation
    for got, w in zip([x.grad, add.grad, conv.weight.grad, conv.bias.grad], want):
        assert _rel(got, w) < 2e-3
    ops.set_precision("tf32x3")                             # 3-pass validation mode: fp32-level
    try:
        y3 = ops.conv1x1_add(x, conv.weight, conv.bias, addend=add)
        assert _rel(y3, ref) < 2e-6
    finally:
        ops.set_precision("tf32")


@pytest.mark.parametrize("shape,groups", [((2, 24, 6, 8, 10), 8), ((3, 16, 13, 7), 8), ((2, 832, 4, 6, 6), 8)])
def test_group_norm_matches_torch(shape, groups):
    from segtran_b200 import ops
    gn = torch.nn.GroupNorm(groups, shape[1]).cuda()
    with torch.no_grad():
        gn.weight.uniform_(0.5, 1.5)
        gn.bias.uniform_(-0.5, 0.5)
    x = (torch.randn(*shape, device="cuda") * 2 + 0.7).requires_grad_(True)
    G = torch.randn(*shape, device="cuda")
    ref = gn(x)
    (ref * G).sum().backward()
    want = [x.grad.clone(), gn.weight.grad.clone(), gn.bias.grad.clone()]
    x.grad = gn.weight.grad = gn.bias.grad = None
    y = ops.group_norm(x, gn.weight, gn.bias, groups, gn.eps)
    (y * G).sum().backward()
    assert _rel(y, ref) < 1e-5
    for got, w in zip([x.grad, gn.weight.grad, gn.bias.grad], want):
        assert _rel(got, w) < 5e-5


@pytest.mark.parametrize("scheme", ["AN", "NA"])
def test_fpn_stage_matches_stock_modules(scheme):
    from segtran_b200 import ops
    conv = torch.nn.Conv3d(16, 32, 1).cuda()
    gn = torch.nn.GroupNorm(8, 32).cuda()
    with torch.no_grad():
        gn.weight.uniform_(0.5, 1.5)
        gn.bias.uniform_(-0.5, 0.5)
    Gw = torch.randn(2, 32, 8, 12, 12, device="cuda")     # (sum y^2 would be invariant to the GroupNorm input: zero gradient)
    cur = torch.randn(2, 16, 8, 12, 12, device="cuda", requires_grad=True)
    hi = torch.randn(2, 32, 4, 6, 6, device="cuda", requires_grad=True)
    up = conv(cur)
    h = F.interpolate(hi, size=up.shape[2:], mode="trilinear", align_corners=False)
    ref = gn(up + h) if scheme == "AN" else gn(up) + h
    (ref * Gw).sum().backward()
    want = [cur.grad.clone(), hi.grad.clone(), conv.weight.grad.clone(), gn.weight.grad.clone()]
    cur.grad = hi.grad = conv.weight.grad = conv.bias.grad = gn.weight.grad = gn.bias.grad = None
    y = ops.fpn_stage(cur, hi, conv, gn, scheme)
    (y * Gw).sum().backward()
    errs = [_rel(got, w) for got, w in zip([cur.grad, hi.grad, conv.weight.grad, gn.weight.grad], want)]
    print(scheme, "tf32 fwd %.2e grads" % _rel(y, ref), ["%.2e" % e for e in errs])
    assert _rel(y, ref) < 1e-3
    assert max(errs) < 3e-3
    # 3-pass validation mode: the same stage agrees with the stock modules to fp32 round-off
    cur.grad = hi.grad = conv.weight.grad = conv.bias.grad = gn.weight.grad = gn.bias.grad = None
    ops.set_precision("tf32x3")
    try:
        y3 = ops.fpn_stage(cur, hi, conv, gn, scheme)
        (y3 * Gw).sum().backward()
    finally:
        ops.set_precision("tf32")
    errs3 = [_rel(got, w) for got, w in zip([cur.grad, hi.grad, conv.weight.grad, gn.weight.grad], want)]
    print(scheme, "tf32x3 fwd %.2e grads" % _rel(y3, ref), ["%.2e" % e for e in errs3])
    assert _rel(y3, ref) < 1e-5 and max(errs3) < 1e-4
