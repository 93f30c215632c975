"""Sparse-convolution encoder / U-Net of NKSRNetwork -- SURVEY 8(f) row 2.

The reference's network lives in the closed wheel; what the open tree shows is its call contract
(models/nksr_net.py:73-78: `encoder(xyz, feat, svh, 0)`, `unet(feat, enc_svh, adaptive_depth=, gt_decoder_svh=)`),
its size (configs/default/train.yaml:9-25: kernel_dim 4, tree_depth 4, unet.f_maps 32) and what its outputs feed
(:93-94 basis features, :101 normal features, models/loss.py:152 structure logits, :117-118 udf features).  The layer
list below is therefore OURS (a point encoder with per-voxel pooling, a residual sparse-conv U-Net over the hierarchy,
linear heads per level), sized by those hparams; `state_dict()` keys are ours as well.  Weights are seeded random: the
pretrained checkpoint is a network download (models/nksr_net.py:36-38).

Where the time goes is the 3x3x3 sparse convolution, and that is a hand-written kernel (csrc/sparse_conv.cu,
`nksr_gather_gemm`): a gather-GEMM over the index tables the hierarchy already holds (nbr27 for the 3^3 stencil,
child8 for the stride-2 convolution, a parent-by-octant table for the up-projection), fp32 FFMA, TF32 mma.sync, or TF32
wgmma.mma_async on the Hopper tensor cores (`precision='tc'`).  The skip concatenation is never materialised (the decoder
convolution runs over its two inputs in turn).  Point-wise MLPs and the heads are dense library GEMMs (torch), as
BASELINE.json's north_star keeps the network on PyTorch.

Every module has `impl='torch'`: the same arithmetic in plain torch (dense gathers) -- the fp32 reference the GPU
tests compare the kernel with (tests/test_gpu_network.py).
"""
from __future__ import annotations

import math
import weakref
from types import SimpleNamespace

import torch
from torch import nn

from ._lib import call, stream_ptr


def round_tf32(w: torch.Tensor) -> torch.Tensor:
    """fp32 -> nearest TF32 value (10-bit mantissa, ties away from zero: what cvt.rna.tf32.f32 does), kept as fp32"""
    return ((w.contiguous().view(torch.int32) + 0x1000) & -0x2000).view(torch.float32)


def gather_gemm(x, idx, weight, bias=None, res=None, relu=False, tf32=False, impl="cuda"):
    """y[i] = act(bias + res[i] + sum_k x[idx[i, k]] @ weight[k]) over the valid (>= 0) entries of idx (n_out, K).
    tf32: False / 0 = fp32 FFMA kernel; True / 1 = TF32 mma.sync kernel; 2 = the same, `weight` already TF32-rounded;
    3 = the wgmma kernel (register accumulator), `weight` already TF32-rounded and transposed to (K, c_out, c_in)."""
    n_out, K = idx.shape
    if int(tf32) == 3 and impl == "cuda":
        c_out, c_in = weight.shape[1], weight.shape[2]
    else:
        c_in, c_out = weight.shape[1], weight.shape[2]
    assert weight.shape[0] == K and x.shape[1] == c_in
    if impl == "torch":
        y = torch.zeros((n_out, c_out), dtype=torch.float32, device=x.device)
        if bias is not None:
            y += bias
        if res is not None:
            y += res
        xp = torch.cat([x, x.new_zeros((1, c_in))])                 # row -1 -> zeros
        step = max(1, (1 << 24) // max(c_in, 1))
        for k in range(K):
            for s in range(0, n_out, step):
                y[s:s + step] += xp[idx[s:s + step, k].long()] @ weight[k]
        return torch.relu(y) if relu else y
    x = x.contiguous()
    idx = idx.contiguous()
    w = weight.contiguous()
    y = torch.empty((n_out, c_out), dtype=torch.float32, device=x.device)
    call("nksr_gather_gemm", x, idx, n_out, K, w, bias.contiguous() if bias is not None else None,
         res.contiguous() if res is not None else None, y, c_in, c_out, int(bool(relu)), int(tf32),
         stream_ptr(x.device))
    return y


def kernel_weights(weight, mode, splits=None):
    """`weight` (K, c_in, c_out) in the form the kernel of `mode` takes, cut along c_in into `splits` parts (the inputs of
    a convolution over a channel concatenation): mode 0 as is; 1 / 2 rounded to TF32; 3 rounded and transposed to
    (K, c_out, c_in).  Rebuilt on every call: no key can tell that the parameter was written in place through `.data`
    (EMA updates, weight surgery), which bumps no version counter, and the weights are at most a few MB."""
    w = weight.detach()
    if mode:
        w = round_tf32(w)
    parts = [w] if splits is None else list(torch.split(w, list(splits), dim=1))
    return [(q.transpose(1, 2) if int(mode) == 3 else q).contiguous() for q in parts]


_KERNEL_FLAG = {0: 0, 1: 2, 2: 2, 3: 3}          # the weights are always rounded on the host (flag 2), never per fragment


def conv_parts(parts, idx, weights, bias, res, relu, mode):
    """y = act(bias + res + sum_p conv(parts[p], weights[p])): the convolution of the channel concatenation of `parts`
    without materialising it -- one kernel call per part, each adding to the previous one's output"""
    y = res
    for i, (x, w) in enumerate(zip(parts, weights)):
        last = i == len(parts) - 1
        y = gather_gemm(x, idx, w, bias if last else None, y, relu and last, _KERNEL_FLAG[int(mode)])
    return y


class SparseConv(nn.Module):
    """K-tap sparse convolution: weight (K, c_in, c_out) + bias; the taps' sources come from an index table.  `x` may be
    a tuple of tensors: the convolution then runs over their channel concatenation (the U-Net's skip connections)."""

    def __init__(self, taps, c_in, c_out):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(taps, c_in, c_out))
        self.bias = nn.Parameter(torch.zeros(c_out))
        bound = math.sqrt(6.0 / (taps * c_in))                       # He-uniform over the full stencil
        nn.init.uniform_(self.weight, -bound, bound)

    def forward(self, x, idx, res=None, relu=True, tf32=False, impl="cuda"):
        parts = tuple(x) if isinstance(x, (tuple, list)) else (x,)
        if impl != "cuda":
            xc = parts[0] if len(parts) == 1 else torch.cat(parts, dim=1)
            return gather_gemm(xc, idx, self.weight, self.bias, res, relu, False, impl)
        mode = int(tf32)
        splits = tuple(int(q.shape[1]) for q in parts) if len(parts) > 1 else None
        ws = kernel_weights(self.weight, mode, splits)
        return conv_parts(parts, idx, ws, self.bias, res, relu, mode)


class PointEncoder(nn.Module):
    """points -> finest voxels: local coordinates (+ the per-point feature) through a small residual MLP whose blocks
    see the per-voxel maximum (the local-pooling PointNet of the convolutional occupancy family), then the mean over
    the points of a voxel.  Voxels that only exist through the 8-voxel splat get zeros (the U-Net's first convolutions
    spread the signal)."""

    def __init__(self, feat_dim, hidden, out_dim, n_blocks=2):
        super().__init__()
        self.fc_in = nn.Linear(3 + feat_dim, hidden)
        self.blocks = nn.ModuleList([nn.Sequential(nn.Linear(2 * hidden, hidden), nn.ReLU(), nn.Linear(hidden, hidden))
                                     for _ in range(n_blocks)])
        self.fc_out = nn.Linear(hidden, out_dim)

    def forward(self, xyz, feat, svh):
        n0 = svh.num_voxels(0)
        base0 = svh.locate(xyz)[0].long()
        ok = base0 >= 0
        if not bool(ok.all()):
            xyz, base0 = xyz[ok], base0[ok]
            feat = feat[ok] if feat is not None else None
        u = xyz / svh.voxel_size
        local = u - torch.floor(u) - 0.5
        h = torch.relu(self.fc_in(torch.cat([local, feat.to(torch.float32)], dim=1) if feat is not None else local))
        for blk in self.blocks:
            pooled = torch.zeros((n0, h.shape[1]), device=h.device).index_reduce_(0, base0, h, "amax",
                                                                                    include_self=False)
            h = h + blk(torch.cat([h, pooled[base0]], dim=1))
        out = torch.zeros((n0, self.fc_out.out_features), device=h.device).index_add_(0, base0, self.fc_out(h))
        cnt = torch.zeros(n0, device=h.device).index_add_(0, base0, torch.ones_like(base0, dtype=torch.float32))
        return out / cnt.clamp(min=1.0)[:, None]


def octant_of_children(child8, n_children):
    """octant (0..7, the column of child8) of every child voxel; -1 for a voxel without a parent"""
    c = child8.reshape(-1).long()
    valid = c >= 0
    octant = torch.full((n_children,), -1, dtype=torch.long, device=child8.device)
    octant[c[valid]] = (torch.arange(c.numel(), device=c.device) % 8)[valid]
    return octant


def up_table(svh, l):
    """(n_l, 8) int32 gather table of the up-projection l+1 -> l: row i holds its parent's index in the column of its
    octant and -1 elsewhere.  Built once per hierarchy level (cached on the hierarchy object, keyed by the tables it was
    derived from)."""
    child8, parent = svh.child8[l + 1], svh.parent[l]
    cache = svh.__dict__.setdefault("_unet_up_tables", {})
    hit = cache.get(l)
    # valid while the very tensor objects it was derived from are the hierarchy's tables (a rebuilt or moved hierarchy
    # holds new ones; weak references, so a recycled address or id cannot pass for the old table)
    if hit is None or hit[0][0]() is not child8 or hit[0][1]() is not parent:
        key = (weakref.ref(child8), weakref.ref(parent))
        n_l = svh.num_voxels(l)
        octant = octant_of_children(child8, n_l)
        rows = torch.nonzero((octant >= 0) & (parent >= 0)).squeeze(1)
        idx = torch.full((n_l, 8), -1, dtype=torch.int32, device=parent.device)
        idx[rows, octant[rows]] = parent[rows].to(torch.int32)
        cache[l] = (key, idx)
    return cache[l][1]


class SparseUNet(nn.Module):
    """Residual sparse-conv U-Net over the levels of a SparseFeatureHierarchy (level 0 = finest):
       down path  l = 0..D-1:  x_l = ResBlock_l(x_l)  (two 3^3 convs);  x_{l+1} = relu(stride-2 conv of x_l)
       up path    l = D-2..0:  y_l = relu(conv3([x_l ; up_l(y_{l+1})]))  with a per-octant linear up-projection
       heads      per level:   structure (3) | normal (3) | basis (kernel_dim) | udf (kernel_dim)"""

    def __init__(self, depth, f_maps, kernel_dim, max_channels=256):
        super().__init__()
        self.depth = depth
        self.kernel_dim = kernel_dim
        ch = [min(f_maps * 2 ** l, max_channels) for l in range(depth)]
        self.channels = ch
        self.enc_a = nn.ModuleList([SparseConv(27, ch[l], ch[l]) for l in range(depth)])
        self.enc_b = nn.ModuleList([SparseConv(27, ch[l], ch[l]) for l in range(depth)])
        self.down = nn.ModuleList([SparseConv(8, ch[l], ch[l + 1]) for l in range(depth - 1)])
        self.up = nn.ParameterList([nn.Parameter(torch.empty(8, ch[l + 1], ch[l])) for l in range(depth - 1)])
        for p in self.up:
            nn.init.uniform_(p, -math.sqrt(6.0 / p.shape[1]), math.sqrt(6.0 / p.shape[1]))
        self.dec = nn.ModuleList([SparseConv(27, 2 * ch[l], ch[l]) for l in range(depth - 1)])
        self.heads = nn.ModuleList([nn.Linear(ch[l], 6 + 2 * kernel_dim) for l in range(depth)])

    def up_project(self, y_coarse, svh, l, tf32=False, impl="cuda"):
        """level l+1 -> level l: every child takes its parent's features through the weight of its octant.  On the GPU
        this is the gather-GEMM kernel again, 8 taps with one valid source per row (`up_table`); impl='torch' is the
        plain per-octant loop the tests compare it with."""
        if impl == "cuda":
            ws = kernel_weights(self.up[l], int(tf32))
            return conv_parts((y_coarse,), up_table(svh, l), ws, None, None, False, int(tf32))
        n_l = svh.num_voxels(l)
        out = torch.zeros((n_l, self.channels[l]), device=y_coarse.device)
        octant = octant_of_children(svh.child8[l + 1], n_l)
        parent = svh.parent[l].long()
        for o in range(8):
            rows = torch.nonzero((octant == o) & (parent >= 0)).squeeze(1)
            if rows.numel():
                out[rows] = y_coarse[parent[rows]] @ self.up[l][o]
        return out

    def forward(self, x0, svh, tf32=False, impl="cuda"):
        D = min(self.depth, svh.depth)
        kw = dict(tf32=tf32, impl=impl)
        xs, x = [], x0
        for l in range(D):
            nbr = svh.nbr27[l]
            h = self.enc_a[l](x, nbr, relu=True, **kw)
            x = self.enc_b[l](h, nbr, res=x, relu=True, **kw)
            xs.append(x)
            if l + 1 < D:
                x = self.down[l](x, svh.child8[l + 1], relu=True, **kw)
        ys = [None] * D
        y = xs[D - 1]
        ys[D - 1] = y
        for l in range(D - 2, -1, -1):
            u = self.up_project(y, svh, l, **kw)
            y = self.dec[l]((xs[l], u), svh.nbr27[l], relu=True, **kw)         # conv over [skip ; up], not concatenated
            ys[l] = y
        C = self.kernel_dim
        out = SimpleNamespace(structure={}, normal={}, basis={}, udf={}, decoder={})
        for l in range(D):
            o = self.heads[l](ys[l])
            out.structure[l], out.normal[l] = o[:, :3], o[:, 3:6]
            out.basis[l], out.udf[l] = o[:, 6:6 + C], o[:, 6 + C:6 + 2 * C]
            out.decoder[l] = ys[l]
        return out


def restrict_to(feat_by_level, src_svh, dst_svh):
    """features living on src_svh's voxels -> dst_svh's voxels (matched by key; voxels src lacks get zeros): the
    decoder hierarchy may be a pruned / ground-truth one (models/nksr_net.py:74-78, gt_decoder_svh)"""
    if dst_svh is src_svh:
        return feat_by_level
    out = {}
    for l, f in feat_by_level.items():
        sk, dk = src_svh.keys[l], dst_svh.keys[l]
        if dk.numel() == 0 or sk.numel() == 0:
            out[l] = f.new_zeros((dk.numel(), f.shape[1]))
            continue
        pos = torch.searchsorted(sk, dk).clamp(max=sk.numel() - 1)
        hit = sk[pos] == dk
        out[l] = torch.where(hit[:, None], f[pos], torch.zeros((), device=f.device))
    return out
