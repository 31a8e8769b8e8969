"""Generate tests/golden/prep3d_*.pt from the REAL reference functions (build container only: reads the reference).

TEST INFRASTRUCTURE ONLY.  Run:  python -m oracle.gen_prep3d_golden
code/dataloaders/datasets3d.py is imported with an empty `h5py` module in sys.modules (h5py is not installed here; the
functions used never call it).  Its `torch` name is replaced by a proxy that
  * records every torch.rand / torch.randint result, which gives the reference's own draws of RandomResizedCrop as the
    record (s_h, s_w, s_d, h_start, w_start, d_start), and
  * sends brats_map_label's hard-coded device='cuda' (datasets3d.py:23) to the CPU.  That literal sits in torch.zeros,
    which oracle/ref_import.cuda_literal_to_cpu (a torch.tensor redirect) does not cover.
Files:
  prep3d_labels.pt     labels with the values 0-4 and 255, batched [2,6,5,7] and unbatched [6,5,7], int64, and the
                       reference's 4-class and binarized maps of each (contiguous copies of its permuted views);
  prep3d_crop_<c>.pt   volume, the reference's permuted n-hot mask made contiguous, the call's arguments, the recorded
                       draws and the two outputs, for the cases of CASES.
"""
from __future__ import annotations

import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_import as R                      # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")

# name: (B, volume channels, in size, out size, crop_percents, isotropic, binarize, seed, geometry the draws must give)
#   up:    every axis scaled > 1 and cropped            down: every axis scaled < 1 and padded (F.pad branch)
#   aniso: three scales, H padded, W and D cropped      odd:  odd sizes, B = 3
CASES = {
    "up": (2, 1, (16, 14, 12), (16, 14, 12), (0.1, 0.3), True, False, 1, "ccc"),
    "down": (1, 4, (12, 10, 8), (12, 10, 8), (-0.3, -0.1), True, False, 2, "ppp"),
    "aniso": (2, 2, (14, 12, 10), (14, 12, 10), (-0.25, 0.25), False, True, 3, "pcc"),
    "odd": (3, 1, (13, 10, 7), (12, 9, 6), (-0.1, 0.1), True, False, 4, None),
}


class _TorchProxy(types.ModuleType):
    def __init__(self, real):
        super().__init__("torch")
        self._real = real
        self.log = []

    def __getattr__(self, name):
        return getattr(self._real, name)

    def rand(self, *a, **k):
        v = self._real.rand(*a, **k)
        self.log.append(v.clone())
        return v

    def randint(self, *a, **k):
        v = self._real.randint(*a, **k)
        self.log.append(v.clone())
        return v

    def zeros(self, *a, **k):
        if k.get("device") == "cuda":
            k["device"] = "cpu"
        return self._real.zeros(*a, **k)


def _reference():
    if not R.available():
        raise RuntimeError("reference not present at %s" % R.REF_ROOT)
    if R.REF_CODE not in sys.path:
        sys.path.insert(0, R.REF_CODE)
    sys.modules.setdefault("h5py", types.ModuleType("h5py"))
    import dataloaders.datasets3d as D3
    proxy = _TorchProxy(torch)
    D3.torch = proxy
    return D3, proxy


def _labels(gen, shape):
    vals = torch.tensor([0, 1, 2, 3, 4, 255])
    return vals[torch.randint(0, len(vals), shape, generator=gen)]


def _geometry(rec, in_size, out_size):
    """'p' for a padded axis, 'c' for a cropped one (int(L * s) in float32, as the reference)."""
    return "".join("p" if int(L * rec[a:a + 1]) < O else "c" for a, (L, O) in enumerate(zip(in_size, out_size)))


def gen_labels(D3):
    gen = torch.Generator().manual_seed(11)
    out = {}
    for key, shape in (("batched", (2, 6, 5, 7)), ("unbatched", (6, 5, 7))):
        lab = _labels(gen, shape)
        lab.view(-1)[:6] = torch.tensor([0, 1, 2, 3, 4, 255])                    # every value occurs
        out[key] = dict(labels=lab, map4=D3.brats_map_label(lab, False).contiguous(),
                        map2=D3.brats_map_label(lab, True).contiguous())
        print("labels", key, tuple(out[key]["map4"].shape), tuple(out[key]["map2"].shape))
    torch.save(dict(kind="prep3d_labels", cases=out), os.path.join(OUT, "prep3d_labels.pt"))


def gen_crop(D3, proxy, name):
    B, Cv, in_size, out_size, cp, iso, binarize, seed, want = CASES[name]
    gen = torch.Generator().manual_seed(100 + seed)
    volume = torch.rand((B, Cv) + in_size, generator=gen)         # unit range: 1e-6 is ~16 float32 ulps
    mask = D3.brats_map_label(_labels(gen, (B,) + in_size), binarize)             # the reference's permuted view
    for s in range(seed, seed + 10000):
        torch.manual_seed(s)
        proxy.log.clear()
        v3, m3 = D3.RandomResizedCrop(volume, mask, out_size, cp, isotropic=iso)
        draws = proxy.log
        # the scale from its torch.rand draw, by the reference's own expression (datasets3d.py:618-623)
        u = [draws[0]] * 3 if iso else draws[:3]
        scales = [t * ((1 + cp[1]) - (1 + cp[0])) + (1 + cp[0]) for t in u]
        starts = draws[-3:]
        rec = torch.cat([t.float().reshape(1) for t in scales + starts])
        if want is None or _geometry(rec, in_size, out_size) == want:
            break
    else:
        raise RuntimeError("no seed gives geometry %s for case %s" % (want, name))
    fx = dict(kind="prep3d_crop", name=name, volume=volume, mask=mask.contiguous(), out_size=out_size,
              crop_percents=cp, isotropic=iso, binarize=binarize, torch_seed=s, draws=rec, volume3=v3, mask3=m3)
    print("crop", name, "seed", s, "draws", rec.tolist(), "geometry", _geometry(rec, in_size, out_size),
          tuple(v3.shape), tuple(m3.shape))
    torch.save(fx, os.path.join(OUT, "prep3d_crop_%s.pt" % name))


if __name__ == "__main__":
    D3, proxy = _reference()
    gen_labels(D3)
    for n in CASES:
        gen_crop(D3, proxy, n)
