"""Gaussian window blending of the sliding-window drop-ins (``gaussian_sigma_scale`` of segtran_b200.inference: the
weighted instantiations of sx_sw_accumulate / sx_sw2d_accumulate, given an sx_sw_weights descriptor) on the GPU: against
the stock-PyTorch oracle (oracle/gauss_oracle.py) on the inference and TTA fixture inputs and at a BraTS-size volume and
a REFUGE-size batch, with every mirror_axes combination, on nets whose scores are constant or depend on the position,
run to run, weighted and unweighted calls at the C ABI, and peak memory."""
import ctypes
import itertools

import pytest
import torch

from oracle import gauss_oracle as GO
from oracle import tta_oracle as TO
from segtran_b200 import _lib as L
from tests.helpers import AffinePickNet, load_golden
from tests.test_gpu_tta import BRATS, REFUGE, _image, check
from tests.test_tta_cpu import TTA

pytestmark = pytest.mark.gpu

S = 0.125
REFUGE_OVERLAP = dict(REFUGE, orig=(384, 384), stride=(96, 96))       # 576^2 images, 3 x 3 overlapping windows


def win(fx):
    return tuple(fx["orig_patch"] if fx["kind"] == "tta3d" else fx["orig"])


def run_lib(fx, net, image, mirror_axes=None, **kw):
    from segtran_b200.inference import test_single_batch, test_single_case
    axes = fx["mirror_axes"] if mirror_axes is None else mirror_axes
    if fx["kind"] == "tta3d":
        return test_single_case(net, image, fx["orig_patch"], fx["input_patch"], fx["batch_size"], fx["stride_xy"],
                                fx["stride_z"], fx["task"], "segtran", fx["K"], mirror_axes=axes, **kw)
    return test_single_batch(net, image, fx["orig"], fx["patch"], fx["stride"], "fundus", fx["K"], "segtran",
                             mirror_axes=axes, **kw)


def run_oracle(fx, net, image, s, mirror_axes=None):
    axes = fx["mirror_axes"] if mirror_axes is None else mirror_axes
    w = GO.gaussian_weight(win(fx), s) if s is not None else torch.ones(win(fx))
    if fx["kind"] == "tta3d":
        return GO.test_single_case_gauss(net, image, fx["orig_patch"], fx["input_patch"], fx["batch_size"],
                                         fx["stride_xy"], fx["stride_z"], fx["task"], "segtran", fx["K"], axes, w)
    return GO.test_single_batch_gauss(net, image, fx["orig"], fx["patch"], fx["stride"], "fundus", fx["K"], "segtran",
                                      axes, w)


def tol(fx, axes):
    """5e-5 for mirror variants with a resized net input whose ratio is not exact in binary (as in test_gpu_tta.py: the
    library mirrors the window before the input resize, the oracle after it, which differs by the rounding of the fp32
    source coordinate times the step between neighbouring cells of a white-noise image), 1e-5 otherwise"""
    if not axes:
        return 1e-5
    win_, net_in = (fx["orig_patch"], fx["input_patch"]) if fx["kind"] == "tta3d" else (fx["orig"], fx["patch"])
    return 1e-5 if all(a == b or a == 2 * b for a, b in zip(win_, net_in)) else 5e-5


def infer_cases():
    """the fixtures of the plain 3-D and 2-D drop-ins, as (fx, net, image) with no mirror axes"""
    out = []
    for key, c in load_golden("infer_sw")["cases"].items():
        fx = dict(kind="tta3d", task=c["task"], K=c["K"], orig_patch=tuple(c["orig_patch"]),
                  input_patch=tuple(c["input_patch"]), batch_size=c["batch_size"], stride_xy=c["stride_xy"],
                  stride_z=c["stride_z"], mirror_axes=())
        out.append(("infer_sw/" + key, fx, AffinePickNet(c["a"], c["b"], c["ch"]), c["image"]))
    for key, c in load_golden("eval2d")["sw"].items():
        fx = dict(kind="tta2d", K=c["K"], orig=tuple(c["orig"]), patch=tuple(c["patch"]), stride=tuple(c["stride"]),
                  mirror_axes=())
        out.append(("eval2d/" + key, fx, AffinePickNet(c["a"], c["b"], c["ch"]), c["image"]))
    for name in TTA:
        fx = load_golden(name)
        out.append((name, fx, TO.AsymNet(**fx["net"]), fx["image"]))
    return out


CASES = infer_cases()
IDS = [c[0] for c in CASES]


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_none_gives_the_bits_of_a_call_without_the_keyword(case):
    _, fx, net, image = case
    image = image.cuda()
    h0, s0 = run_lib(fx, net, image)
    h1, s1 = run_lib(fx, net, image, gaussian_sigma_scale=None)
    assert torch.equal(s0, s1) and torch.equal(h0, h1)


@pytest.mark.parametrize("s", [S, 0.3])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_weighted_output_matches_the_oracle_on_the_fixture_inputs(case, s):
    _, fx, net, image = case
    hard, soft = run_lib(fx, net, image.cuda(), gaussian_sigma_scale=s)
    ref_hard, ref_soft = run_oracle(fx, net, image, s)
    check(hard, soft, ref_hard, ref_soft, fx["kind"], tol=tol(fx, fx["mirror_axes"]))


@pytest.mark.parametrize("fx", [BRATS, dict(BRATS, task="other", K=3, mirror_axes=(2, 1)), dict(BRATS, mirror_axes=()),
                                REFUGE, dict(REFUGE, patch=(576, 576), mirror_axes=(1,)), dict(REFUGE, mirror_axes=()),
                                REFUGE_OVERLAP, dict(REFUGE_OVERLAP, mirror_axes=())],
                         ids=["brats", "brats_argmax", "brats_plain", "refuge", "refuge_same_size", "refuge_plain",
                              "refuge_overlap", "refuge_overlap_plain"])
def test_weighted_output_matches_the_oracle_at_full_size(fx):
    image = _image(fx["kind"])
    net = TO.AsymNet(**TO.AsymNet.params(fx["K"], image.shape[0 if fx["kind"] == "tta3d" else 1], seed=9))
    hard, soft = run_lib(fx, net, image, gaussian_sigma_scale=S)
    ref_hard, ref_soft = run_oracle(fx, net, image, S)
    check(hard, soft, ref_hard, ref_soft, fx["kind"], tol=tol(fx, fx["mirror_axes"]))


SMALL3 = dict(kind="tta3d", task="brats", K=4, orig_patch=(24, 24, 16), input_patch=(16, 20, 12), batch_size=2,
              stride_xy=12, stride_z=8, mirror_axes=())
SMALL2 = dict(kind="tta2d", K=3, orig=(32, 40), patch=(24, 24), stride=(16, 12), mirror_axes=())
AXES3 = [c for r in range(4) for c in itertools.permutations(range(3), r)]
AXES2 = [c for r in range(3) for c in itertools.permutations(range(2), r)]


@pytest.mark.parametrize("fx,axes", [(SMALL3, a) for a in AXES3] + [(SMALL2, a) for a in AXES2],
                         ids=["3d%s" % (a,) for a in AXES3] + ["2d%s" % (a,) for a in AXES2])
def test_every_mirror_axes_combination_is_weighted(fx, axes):
    g = torch.Generator().manual_seed(11)
    image = torch.randn((4, 20, 30, 12) if fx["kind"] == "tta3d" else (2, 3, 30, 44), generator=g) * 2
    net = TO.AsymNet(**TO.AsymNet.params(fx["K"], image.shape[0 if fx["kind"] == "tta3d" else 1], seed=3))
    hard, soft = run_lib(fx, net, image.cuda(), mirror_axes=axes, gaussian_sigma_scale=S)
    ref_hard, ref_soft = run_oracle(fx, net, image, S, mirror_axes=axes)
    check(hard, soft, ref_hard, ref_soft, fx["kind"], tol=tol(fx, axes))


class ConstNet(torch.nn.Module):
    """scores that do not depend on the input or the position: class k scores c[k] everywhere"""

    def __init__(self, c):
        super().__init__()
        self.c = c

    def forward(self, x):
        shape = (x.shape[0], len(self.c)) + tuple(x.shape[2:])
        return torch.tensor(self.c, device=x.device).view((1, -1) + (1,) * (x.dim() - 2)).expand(shape).contiguous()


@pytest.mark.parametrize("fx", [BRATS, dict(BRATS, task="other", K=3), REFUGE_OVERLAP],
                         ids=["brats", "brats_argmax", "refuge_overlap"])
def test_constant_scores_give_the_plain_output(fx):
    """every window adds w * p and w, so the weights cancel in the average, up to the fp32 rounding of the weighted
    sums (up to 8 windows x 8 variants per voxel at the BraTS size)"""
    image = _image(fx["kind"])
    net = ConstNet([-2.0, 1.5, -0.7, 0.4][:fx["K"]])
    plain_hard, plain_soft = run_lib(fx, net, image)
    hard, soft = run_lib(fx, net, image, gaussian_sigma_scale=S)
    assert float((soft - plain_soft).abs().max()) < 1e-5
    assert torch.equal(hard, plain_hard)


@pytest.mark.parametrize("fx", [BRATS, REFUGE_OVERLAP], ids=["brats", "refuge_overlap"])
def test_position_dependent_scores_change_the_output(fx):
    image = _image(fx["kind"])
    net = TO.AsymNet(**TO.AsymNet.params(fx["K"], image.shape[0 if fx["kind"] == "tta3d" else 1], seed=9))
    _, plain = run_lib(fx, net, image, mirror_axes=())
    _, weighted = run_lib(fx, net, image, mirror_axes=(), gaussian_sigma_scale=S)
    assert float((weighted - plain).abs().max()) > 1e-2


@pytest.mark.parametrize("fx", [BRATS, REFUGE], ids=["brats", "refuge"])
def test_weighted_runs_give_the_same_bits(fx):
    image = _image(fx["kind"])
    net = TO.AsymNet(**TO.AsymNet.params(fx["K"], image.shape[0 if fx["kind"] == "tta3d" else 1], seed=9))
    h1, s1 = run_lib(fx, net, image, gaussian_sigma_scale=S)
    h2, s2 = run_lib(fx, net, image, gaussian_sigma_scale=S)
    assert torch.equal(s1, s2) and torch.equal(h1, h2)


def _st():
    return torch.cuda.current_stream().cuda_stream


def test_an_accumulate_without_weights_is_unweighted():
    """An accumulate given tables adds w * sigmoid and w; one given none adds sigmoid and 1, also right after a refused
    weighted call."""
    dev = "cuda"
    K, d = 2, (3, 4, 5)
    scores = torch.zeros((K,) + d, device=dev)                              # sigmoid(0) = 1/2
    tab = torch.cat([torch.full((n,), v, device=dev) for n, v in zip(d, (0.5, 0.25, 0.5))])
    px = tab.data_ptr()
    wts = ctypes.byref(L.sx_sw_weights(px, px + 4 * d[0], px + 4 * (d[0] + d[1]), *d))
    preds = torch.zeros((K,) + d, device=dev)
    cnt = torch.zeros(d, device=dev)
    acc3 = (scores.data_ptr(), K, *d, preds.data_ptr(), cnt.data_ptr(), *d, 0, 0, 0)
    L.call("sx_sw_accumulate", *acc3, 0, wts, _st())
    assert torch.equal(cnt, torch.full(d, 0.0625, device=dev)) and torch.equal(preds, torch.full_like(preds, 0.03125))
    L.call("sx_sw_accumulate", *acc3, 0, None, _st())
    assert torch.equal(cnt, torch.full(d, 1.0625, device=dev)) and torch.equal(preds, torch.full_like(preds, 0.53125))
    with pytest.raises(L.SxError, match="mirror mask 8"):
        L.call("sx_sw_accumulate", *acc3, 8, wts, _st())
    L.call("sx_sw_accumulate", *acc3, 0, None, _st())
    assert torch.equal(cnt, torch.full(d, 2.0625, device=dev))

    # 2-D: the weight sits on the upsampled window
    B, h, w, dx, dy = 2, 3, 5, 6, 10
    s2 = torch.zeros(B, K, h, w, device=dev)
    tab2 = torch.cat([torch.full((dx,), 0.5, device=dev), torch.full((dy,), 0.5, device=dev)])
    wts2 = ctypes.byref(L.sx_sw_weights(tab2.data_ptr(), tab2.data_ptr() + 4 * dx, None, dx, dy, 1))
    p2 = torch.zeros(B, K, dx, dy, device=dev)
    c2 = torch.zeros(dx, dy, device=dev)
    acc2 = (s2.data_ptr(), B, K, h, w, dx, dy, p2.data_ptr(), c2.data_ptr(), dx, dy, 0, 0, 0)
    L.call("sx_sw2d_accumulate", *acc2, wts2, _st())
    L.call("sx_sw2d_accumulate", *acc2, None, _st())
    assert torch.equal(c2, torch.full((dx, dy), 1.25, device=dev)) and torch.equal(p2, torch.full_like(p2, 0.625))


def test_weights_are_floored_at_the_window_corners():
    """a tiny sigma: the corners of a lone window weigh 1e-3, so the count stays positive and the average is defined"""
    fx = dict(SMALL3, orig_patch=(24, 24, 16), input_patch=(24, 24, 16))
    image = torch.randn(4, 24, 24, 16, generator=torch.Generator().manual_seed(2)).cuda()
    net = TO.AsymNet(**TO.AsymNet.params(4, 4, seed=1))
    hard, soft = run_lib(fx, net, image, gaussian_sigma_scale=0.01)
    assert bool(torch.isfinite(soft).all())
    ref_hard, ref_soft = run_oracle(fx, net, image.cpu(), 0.01)
    check(hard, soft, ref_hard, ref_soft, fx["kind"])


@pytest.mark.parametrize("fx", [BRATS, REFUGE, dict(REFUGE, patch=(576, 576))], ids=["brats", "refuge", "refuge_same"])
def test_weighted_peak_memory_is_the_plain_peak_plus_the_tables(fx):
    image = _image(fx["kind"])
    net = TO.AsymNet(**TO.AsymNet.params(fx["K"], image.shape[0 if fx["kind"] == "tta3d" else 1], seed=9))

    def peak(**kw):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = run_lib(fx, net, image, **kw)
        torch.cuda.synchronize()
        p = torch.cuda.max_memory_allocated() - base
        del out
        return p

    peak()                                                     # warm-up
    for axes in ((), fx["mirror_axes"]):
        plain, weighted = peak(mirror_axes=axes), peak(mirror_axes=axes, gaussian_sigma_scale=S)
        tables = -(-4 * sum(win(fx)) // 512) * 512               # one fp32 tensor, in the allocator's 512-byte blocks
        print("axes %s: peak plain %.3f MB, weighted %.3f MB, tables %d B" % (axes, plain / 2**20, weighted / 2**20,
                                                                              tables))
        assert weighted <= plain + tables
