"""A1: TPVQueryLifter (reference model/lifter/tpv_query_lifter.py:6-36) and BEVQueryLifter (bev_query_lifter.py) -- same
names, ctor kwargs, parameter names (``tpv_hw``, ``tpv_zh``, ``tpv_wz`` / ``bev``) and output dicts."""
import torch
import torch.nn as nn
from .registry import MODELS


@MODELS.register_module()
class TPVQueryLifter(nn.Module):
    def __init__(self, tpv_h, tpv_w, tpv_z, dim, init_cfg=None, **kwargs):
        super().__init__()
        self.tpv_h, self.tpv_w, self.tpv_z, self.dim = tpv_h, tpv_w, tpv_z, dim
        self.tpv_hw = nn.Parameter(torch.randn(1, tpv_h * tpv_w, dim))
        self.tpv_zh = nn.Parameter(torch.randn(1, tpv_z * tpv_h, dim))
        self.tpv_wz = nn.Parameter(torch.randn(1, tpv_w * tpv_z, dim))

    def forward(self, ms_img_feats, *args, **kwargs):
        bs = ms_img_feats[0].shape[0]
        if bs == 1:  # the planes are read-only downstream: no 30 MB copy per frame
            return {'representation': [self.tpv_hw, self.tpv_zh, self.tpv_wz]}
        return {'representation': [p.repeat(bs, 1, 1) for p in (self.tpv_hw, self.tpv_zh, self.tpv_wz)]}


@MODELS.register_module()
class BEVQueryLifter(nn.Module):
    """bev_query_lifter.py:6-26: one learned BEV plane, parameter ``bev`` [1, H*W, C]; the representation is a tensor."""

    def __init__(self, bev_h, bev_w, dim, init_cfg=None, **kwargs):
        super().__init__()
        self.bev_h, self.bev_w, self.dim = bev_h, bev_w, dim
        self.bev = nn.Parameter(torch.randn(1, bev_h * bev_w, dim))

    def forward(self, ms_img_feats, *args, **kwargs):
        bs = ms_img_feats[0].shape[0]
        bev = self.bev.to(ms_img_feats[0].dtype)
        return {'representation': bev if bs == 1 else bev.repeat(bs, 1, 1)}
