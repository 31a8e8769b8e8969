"""GPU checks of the 3-D batch preparation (segtran_b200/datasets3d.py, csrc/sx_prep3d.cu): brats_map_label and
RandomResizedCrop against the fixtures of the reference's own functions (oracle/gen_prep3d_golden.py), the full BraTS
shape against the stock F.interpolate / F.pad / slice formulation on the same GPU, memory, the device draws, run-to-run
identity, and a captured training step that prepares its batch inside the graph."""
import glob
import os
from argparse import Namespace

import pytest
import torch

from tests.helpers import GOLDEN, load_golden

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

from oracle import prep3d_oracle as PO  # noqa: E402
from segtran_b200 import ops  # noqa: E402
from segtran_b200.datasets3d import RandomResizedCrop, brats_map_label, draw_resized_crop  # noqa: E402

DEV = "cuda"
CROPS = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(GOLDEN, "prep3d_crop_*.pt")))
LABEL_DTYPES = [torch.uint8, torch.int16, torch.int32, torch.int64, torch.float32]
BRATS = (4, 112, 112, 96)


def _permuted(mask):
    """The reference's n-hot layout: a [B,K,...] view of a [K,B,...] tensor."""
    return mask.permute(1, 0, 2, 3, 4).contiguous().permute(1, 0, 2, 3, 4)


@pytest.mark.parametrize("dtype", LABEL_DTYPES)
@pytest.mark.parametrize("key", ["batched", "unbatched"])
def test_label_maps_are_bit_exact(dtype, key):
    c = load_golden("prep3d_labels")["cases"][key]
    lab = c["labels"].to(dtype).to(DEV)
    for binarize, ref in ((False, c["map4"]), (True, c["map2"])):
        out = brats_map_label(lab, binarize)
        assert out.is_contiguous() and out.dtype == torch.float32 and out.device == lab.device
        assert torch.equal(out.cpu(), ref), (dtype, key, binarize)


def test_label_map_values_outside_the_classes():
    """Negative and fractional labels, as the reference compares them in the label's type."""
    lab = torch.tensor([-3, -1, 0, 1, 2, 3, 4, 7, 255, 1000], device=DEV).view(1, 10, 1, 1)
    for dtype in (torch.int16, torch.int32, torch.int64, torch.float32):
        for binarize in (False, True):
            got = brats_map_label(lab.to(dtype), binarize)
            assert torch.equal(got, PO.brats_map_label(lab.to(dtype), binarize).contiguous())
    f = torch.tensor([0.5, -0.0, 3.0, float("nan")], device=DEV).view(4, 1, 1)
    for binarize in (False, True):
        assert torch.equal(brats_map_label(f, binarize), PO.brats_map_label(f, binarize))


@pytest.mark.parametrize("name", CROPS)
@pytest.mark.parametrize("layout", ["contiguous", "permuted"])
def test_resized_crop_matches_the_reference_fixtures(name, layout):
    fx = load_golden(name)
    volume, mask = fx["volume"].to(DEV), fx["mask"].to(DEV)
    if layout == "permuted":
        mask = _permuted(mask)
        draws = fx["draws"].to(DEV)                          # a device record
    else:
        draws = fx["draws"]                                  # a host record
    v3, m3 = RandomResizedCrop(volume, mask, fx["out_size"], fx["crop_percents"], fx["isotropic"], draws=draws)
    assert v3.shape == fx["volume3"].shape and m3.shape == fx["mask3"].shape
    assert float((v3.cpu() - fx["volume3"]).abs().max()) <= 1e-6
    assert float((m3.cpu() - fx["mask3"]).abs().max()) <= 1e-6


def _brats_batch(seed):
    g = torch.Generator().manual_seed(seed)
    volume = torch.randn((4,) + BRATS, generator=g).to(DEV)
    labels = torch.randint(0, 4, (4,) + BRATS[1:], generator=g, dtype=torch.uint8).to(DEV)
    return volume, brats_map_label(labels, False)


@pytest.mark.parametrize("scale", [0.9, 1.1])
def test_full_brats_shape_matches_the_stock_formulation(scale):
    volume, mask = _brats_batch(5)
    out = BRATS[1:]
    s = float(torch.tensor(scale, dtype=torch.float32))
    padded = [max(int(torch.tensor(float(L)) * s), O) for L, O in zip(out, out)]
    rec = torch.tensor([s, s, s] + [(p - O) // 3 for p, O in zip(padded, out)], dtype=torch.float32)
    v3, m3 = RandomResizedCrop(volume, mask, out, (-0.1, 0.1), draws=rec)
    rv, rm = PO.resized_crop(volume, mask, out, rec)
    assert float((v3 - rv).abs().max()) <= 1e-5
    assert float((m3 - rm).abs().max()) <= 1e-5
    # the reference's permuted n-hot view gives the same result
    v3p, m3p = RandomResizedCrop(volume, _permuted(mask), out, (-0.1, 0.1), draws=rec.to(DEV))
    assert torch.equal(v3p, v3) and torch.equal(m3p, m3)


def test_no_intermediate_is_allocated():
    volume, mask = _brats_batch(6)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    v3, m3 = RandomResizedCrop(volume, mask, BRATS[1:], (-0.1, 0.1))         # device draws: seed + record
    torch.cuda.synchronize()
    # the caching allocator hands each large output its whole 2 MiB-rounded segment when the rest is too small to split
    outputs = sum(-(-t.numel() * 4 // (2 << 20)) * (2 << 20) for t in (v3, m3))
    assert torch.cuda.max_memory_allocated() - base <= outputs + 64 * 1024
    del v3, m3


def _geometry_ok(rec, in_size, out_size):
    """rec [N,6]: every start is an integer in [0, max(int(L * s), out) - out]."""
    s = rec[:, :3]
    for a, (L, O) in enumerate(zip(in_size, out_size)):
        padded = torch.clamp((torch.tensor(float(L)) * s[:, a]).long(), min=O)
        st = rec[:, 3 + a]
        assert torch.equal(st, st.round()) and bool((st >= 0).all()) and bool((st.long() <= padded - O).all())


@pytest.mark.parametrize("isotropic", [True, False])
def test_device_draws_stay_in_range(isotropic):
    in_size, out_size, cp = (20, 16, 12), (18, 16, 10), (-0.2, 0.2)
    recs = torch.stack([draw_resized_crop(in_size, out_size, cp, isotropic, seed=s) for s in range(3000)]).cpu()
    lo, hi = float(torch.tensor(0.8, dtype=torch.float32)), float(torch.tensor(1.2, dtype=torch.float32))
    s = recs[:, :3]
    assert bool((s >= lo).all()) and bool((s < hi).all())
    if isotropic:
        assert torch.equal(s[:, 0], s[:, 1]) and torch.equal(s[:, 0], s[:, 2])
    else:
        assert bool((s[:, 0] != s[:, 1]).any()) and bool((s[:, 1] != s[:, 2]).any())
    # U[0.8, 1.2): mean 1, quartiles 0.9 and 1.1 (3000 draws: the standard error of the mean is 0.002)
    assert abs(float(s.mean()) - 1.0) < 0.01
    q = torch.quantile(s[:, 0].double(), torch.tensor([0.25, 0.75], dtype=torch.float64))
    assert abs(float(q[0]) - 0.9) < 0.02 and abs(float(q[1]) - 1.1) < 0.02
    _geometry_ok(recs, in_size, out_size)


def test_every_start_of_a_small_range_occurs():
    recs = torch.stack([draw_resized_crop((16, 16, 16), (12, 12, 12), (0.0, 0.0), seed=s) for s in range(2000)]).cpu()
    assert bool((recs[:, :3] == 1.0).all())
    for a in range(3):
        assert sorted(recs[:, 3 + a].unique().tolist()) == [0.0, 1.0, 2.0, 3.0, 4.0]


def test_seeds_fix_the_record():
    args = ((112, 112, 96), (112, 112, 96), (-0.1, 0.1), False)
    a = draw_resized_crop(*args, seed=1234)
    b = draw_resized_crop(*args, seed=1234)
    c = draw_resized_crop(*args, seed=torch.tensor([1234], device=DEV))
    d = draw_resized_crop(*args, seed=1235)
    assert torch.equal(a, b) and torch.equal(a, c)
    assert not torch.equal(a, d)
    # per-call device seeds: two calls draw different records
    e, f = draw_resized_crop(*args), draw_resized_crop(*args)
    assert not torch.equal(e, f)


def test_out_of_range_records_read_nothing_outside():
    g = torch.Generator().manual_seed(3)
    volume = torch.rand(2, 3, 9, 8, 7, generator=g).to(DEV)
    mask = torch.rand(2, 2, 9, 8, 7, generator=g).to(DEV)
    out = (6, 6, 6)
    for rec in ([1.0, 1.0, 1.0, 6.0, -2.0, 4.0], [0.5, 1.3, 0.8, -100.0, 1e9, 2.0], [1.0, 1.0, 1.0, 1e30, 0.0, -1e30]):
        v3, m3 = RandomResizedCrop(volume, mask, out, (-0.6, 0.4), draws=rec)
        resized, pads, starts = PO.crop_geometry(volume.shape[2:], out, rec)
        for x, y in ((volume, v3), (mask, m3)):
            full = PO.resized_crop(x, x, [r + p[0] + p[1] for r, p in zip(resized, pads)], [*rec[:3], 0, 0, 0])[0]
            ref = torch.zeros_like(y)
            idx = [torch.arange(out[a], device=DEV) + max(min(starts[a], 1 << 30), -(1 << 30)) for a in range(3)]
            ok = [(i >= 0) & (i < full.shape[2 + a]) for a, i in enumerate(idx)]
            sel = [i.clamp(0, full.shape[2 + a] - 1) for a, i in enumerate(idx)]
            g_ = full[:, :, sel[0]][:, :, :, sel[1]][:, :, :, :, sel[2]]
            m_ = ok[0].view(-1, 1, 1) & ok[1].view(1, -1, 1) & ok[2].view(1, 1, -1)
            ref = torch.where(m_, g_, ref)
            assert float((y - ref).abs().max()) <= 1e-6, rec


def test_two_runs_are_bit_identical():
    volume, mask = _brats_batch(7)
    rec = draw_resized_crop(BRATS[1:], BRATS[1:], (-0.1, 0.1), seed=99)
    a = RandomResizedCrop(volume, mask, BRATS[1:], (-0.1, 0.1), draws=rec)
    b = RandomResizedCrop(volume, mask, BRATS[1:], (-0.1, 0.1), draws=rec)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    lab = torch.randint(0, 5, (2, 30, 20, 10), device=DEV)
    assert torch.equal(brats_map_label(lab, False), brats_map_label(lab, False))


class FixedFeat3d(torch.nn.Module):
    def __init__(self, feats):
        super().__init__()
        self.feats = feats

    def extract_features(self, x):
        keys = ["MaxPool3d_2a_3x3", "Conv3d_2c_3x3", "Mixed_3c", "Mixed_4f", "Mixed_5c"]
        return dict(zip(keys, self.feats))


def test_captured_step_with_batch_preparation():
    """labels, volume -> brats_map_label -> draw_resized_crop + RandomResizedCrop -> Segtran3d -> seg_loss -> backward ->
    FlatBertAdam, captured as one CUDA graph: each replay after ops.advance_seed takes a new crop, and its loss and
    parameters equal those of an eager step given that replay's record."""
    import segtran_b200.networks.segtran3d as M
    import segtran_b200.networks.segtran_shared as S
    from segtran_b200.graph import CapturedStep
    from segtran_b200.train import FlatBertAdam, seg_loss
    fx = load_golden("seg3d_tiny")
    args = Namespace(**fx["args"])
    args.device = DEV
    S.bb2feat_dims[args.backbone_type] = fx["bb_feat_dims"]
    cfg = M.Segtran3dConfig()
    cfg.update_config(args)
    net = M.Segtran3d(cfg, backbone=FixedFeat3d([f.to(DEV) for f in fx["feats"]]))
    net.load_state_dict(fx["state_dict"], strict=False)
    net = net.to(DEV).train()                                       # dropout 0 in the fixture
    params = [p for p in net.parameters() if p.requires_grad]
    opt = FlatBertAdam([{"params": params, "lr": 1e-3, "weight_decay": 1e-4}], grad_clip=0.1)
    g = torch.Generator().manual_seed(8)
    volume = fx["batch"].to(DEV)
    labels = torch.randint(0, 4, (2, 32, 32, 32), generator=g, dtype=torch.uint8).to(DEV)
    out, cp = (32, 32, 32), (-0.1, 0.1)

    def step(draws=None):
        opt.zero_grad()
        mask = brats_map_label(labels, False)
        rec = draw_resized_crop(out, out, cp) if draws is None else draws
        v3, m3 = RandomResizedCrop(volume, mask, out, cp, draws=rec)
        loss, _, _ = seg_loss(net(v3), m3)
        loss.backward()
        opt.step()
        return loss, rec

    cudnn_det = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True                      # the stock in-bridge Conv3d's weight gradient
    try:
        _replays_match_eager(step, opt, volume.device, CapturedStep)
    finally:
        torch.backends.cudnn.deterministic = cudnn_det


def _replays_match_eager(step, opt, device, CapturedStep):
    graph = CapturedStep(step, warmup=2)
    state = [opt.flat_p, opt.flat_r, opt.flat_m, opt.flat_v, opt.step_count]
    recs = []
    for _ in range(3):
        ops.advance_seed(device)
        before = [t.clone() for t in state]
        loss, rec = graph()
        torch.cuda.synchronize()
        loss, rec = loss.clone(), rec.clone()
        after = [t.clone() for t in state]
        recs.append(rec.cpu())
        for t, b in zip(state, before):                            # the same step, eagerly, from the same state
            t.copy_(b)
        eloss, _ = step(draws=rec)
        torch.cuda.synchronize()
        assert torch.equal(eloss, loss)
        for t, a in zip(state, after):
            assert torch.equal(t, a)
    assert not torch.equal(recs[0], recs[1]) and not torch.equal(recs[1], recs[2])
    assert graph.kernel_launches > 20
