"""Float64 restatement of the class head without the out-FPN (out_fpn_layers == in_fpn_layers; CPU, checker only).

Reference: segtran2d.py:198-209 (ConvTranspose2d(C, K, 2, 2)) and :421-437 (bilinear to the input size);
segtran3d.py:234-245 (ConvTranspose3d(C, K, (2,2,1), (2,2,1))) and :478-498 (tokens permuted to (H2,W2,D2), trilinear to
the input size (H,W,D)).  Kept next to head_oracle.py, which restates the out-FPN heads.
"""
from __future__ import annotations

import torch.nn.functional as F


def direct_head(vfeat, Wt, bt, out_size):
    """2-D: vfeat [B,C,H2,W2], Wt [C,K,2,2] -> logits [B,K,H,W].  3-D: vfeat [B,C,D2,H2,W2] (the token order),
    Wt [C,K,2,2,1] -> logits [B,K,H,W,D].  Float64 throughout; bt may be None."""
    x, W = vfeat.double(), Wt.double()
    b = None if bt is None else bt.double()
    if x.dim() == 5:
        s = F.conv_transpose3d(x.permute(0, 1, 3, 4, 2), W, b, stride=(2, 2, 1))
        return F.interpolate(s, size=tuple(out_size), mode='trilinear', align_corners=False)
    s = F.conv_transpose2d(x, W, b, stride=2)
    return F.interpolate(s, size=tuple(out_size), mode='bilinear', align_corners=False)
