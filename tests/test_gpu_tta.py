"""Mirror test-time augmentation of the sliding-window drop-ins (``mirror_axes`` of segtran_b200.inference: csrc/
sx_infer.cu sx_sw_gather and the mirrored sx_sw_accumulate / sx_sw2d_accumulate) on the GPU: against the fixtures made
from the reference's functions (tests/golden/tta_*.pt), against the stock torch.flip restatement at a BraTS-size volume
and a REFUGE-size batch, on a mirror-equivariant net, run to run, and in peak memory."""
import pytest
import torch

from oracle import tta_oracle as IO
from tests.test_tta_cpu import TTA, run_oracle, sure_mask
from tests.helpers import load_golden

pytestmark = pytest.mark.gpu


def run_lib(fx, net, image, mirror_axes=None):
    from segtran_b200.inference import test_single_batch, test_single_case
    axes = fx["mirror_axes"] if mirror_axes is None else mirror_axes
    if fx["kind"] == "tta3d":
        return test_single_case(net, image, fx["orig_patch"], fx["input_patch"], fx["batch_size"], fx["stride_xy"],
                                fx["stride_z"], fx["task"], "segtran", fx["K"], mirror_axes=axes)
    return test_single_batch(net, image, fx["orig"], fx["patch"], fx["stride"], "fundus", fx["K"], "segtran",
                             mirror_axes=axes)


def check(hard, soft, ref_hard, ref_soft, kind, tol=1e-5):
    hard, soft, ref_hard, ref_soft = hard.cpu(), soft.cpu(), ref_hard.cpu(), ref_soft.cpu()
    assert soft.shape == ref_soft.shape and hard.shape == ref_hard.shape and hard.dtype == ref_hard.dtype
    err = float((soft - ref_soft).abs().max())
    assert err < tol, err
    sure = sure_mask(ref_soft, ref_hard, kind)
    assert float(sure.float().mean()) > 0.99
    assert torch.equal(hard[sure], ref_hard[sure])


@pytest.mark.parametrize("name", TTA)
def test_tta_matches_reference_fixtures(name):
    fx = load_golden(name)
    hard, soft = run_lib(fx, IO.AsymNet(**fx["net"]), fx["image"].cuda())
    check(hard, soft, fx["hard"], fx["soft"], fx["kind"])


@pytest.mark.parametrize("name", TTA)
def test_tta_is_deterministic(name):
    fx = load_golden(name)
    net, image = IO.AsymNet(**fx["net"]), fx["image"].cuda()
    h1, s1 = run_lib(fx, net, image)
    h2, s2 = run_lib(fx, net, image)
    assert torch.equal(s1, s2) and torch.equal(h1, h2)


BRATS = dict(kind="tta3d", task="brats", K=4, orig_patch=(112, 112, 96), input_patch=(96, 96, 80), batch_size=3,
             stride_xy=56, stride_z=40, mirror_axes=(0, 1, 2))
REFUGE = dict(kind="tta2d", K=3, orig=(576, 576), patch=(288, 288), stride=(288, 288), mirror_axes=(0, 1))


def _image(kind):
    g = torch.Generator(device="cuda").manual_seed(5)
    shape = (4, 150, 170, 120) if kind == "tta3d" else (4, 3, 576, 576)
    return torch.randn(shape, device="cuda", generator=g) * 2.0


@pytest.mark.parametrize("fx", [BRATS, dict(BRATS, task="other", K=3, mirror_axes=(2, 1)), REFUGE,
                                dict(REFUGE, patch=(576, 576), mirror_axes=(1,))], ids=["brats", "brats_argmax",
                                                                                        "refuge", "refuge_same_size"])
def test_tta_matches_torch_flip_restatement_at_full_size(fx):
    image = _image(fx["kind"])
    net = IO.AsymNet(**IO.AsymNet.params(fx["K"], image.shape[0 if fx["kind"] == "tta3d" else 1], seed=9))
    hard, soft = run_lib(fx, net, image)
    ref_hard, ref_soft = run_oracle(fx, net, image)
    # 3-D with resizes: the library mirrors the windows before the input resize and reads the scores mirrored after the
    # output resize, torch.flip does it after / before.  The two agree up to the fp32 rounding of the source coordinate
    # ((j + 0.5) * ratio - 0.5 is ~95 at the far edge, one ulp 7.6e-6) times the step between neighbouring cells, which
    # on this white-noise image is a few units.
    resized = fx["kind"] == "tta3d" and fx["input_patch"] != fx["orig_patch"]
    check(hard, soft, ref_hard, ref_soft, fx["kind"], tol=5e-5 if resized else 1e-5)


class Pointwise(torch.nn.Module):
    """a 1x1(x1) convolution: mirror-equivariant, so TTA must return the plain output"""

    def __init__(self, C, K, dims):
        super().__init__()
        conv = torch.nn.Conv3d if dims == 3 else torch.nn.Conv2d
        torch.manual_seed(4)
        self.conv = conv(C, K, 1)

    def forward(self, x):
        return self.conv(x)


@pytest.mark.parametrize("fx", [BRATS, REFUGE], ids=["brats", "refuge"])
def test_mirror_equivariant_net_gives_the_plain_output(fx):
    image = _image(fx["kind"])
    C = image.shape[0 if fx["kind"] == "tta3d" else 1]
    net = Pointwise(C, fx["K"], 3 if fx["kind"] == "tta3d" else 2).cuda().eval()
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False        # the mirrored input differs from the plain one in rounding only
    try:
        plain_hard, plain_soft = run_lib(fx, net, image, mirror_axes=())
        hard, soft = run_lib(fx, net, image)
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    check(hard, soft, plain_hard, plain_soft, fx["kind"])


@pytest.mark.parametrize("fx", [BRATS, REFUGE, dict(REFUGE, patch=(576, 576))], ids=["brats", "refuge", "refuge_same"])
def test_tta_peak_memory_is_the_plain_peak_plus_one_window_batch(fx):
    image = _image(fx["kind"])
    net = IO.AsymNet(**IO.AsymNet.params(fx["K"], image.shape[0 if fx["kind"] == "tta3d" else 1], seed=9))

    def peak(axes):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = run_lib(fx, net, image, mirror_axes=axes)
        torch.cuda.synchronize()
        p = torch.cuda.max_memory_allocated() - base
        del out
        return p

    peak(())                                                   # warm-up
    plain, tta = peak(()), peak(fx["mirror_axes"])
    if fx["kind"] == "tta3d":
        gathered = fx["batch_size"] * image.shape[0] * 112 * 112 * 96 * 4
    else:
        gathered = image.shape[0] * image.shape[1] * 576 * 576 * 4
    print("peak plain %.1f MB, TTA %.1f MB, window batch %.1f MB" % (plain / 2**20, tta / 2**20, gathered / 2**20))
    assert tta <= plain + gathered
