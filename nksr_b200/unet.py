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

from ._lib import NksrError, _ws, call, stream_ptr


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
        y = torch.zeros((n_out, c_out), dtype=x.dtype, device=x.device)
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


def kernel_weights(weight, mode, splits=None, transposed=False):
    """`weight` (K, c_in, c_out) in the form the kernel of `mode` takes, cut along c_in into `splits` parts (the inputs of
    a convolution over a channel concatenation): mode 0 as is; 1 / 2 rounded to TF32; 3 rounded and transposed to
    (K, c_out, c_in).  transposed=True gives the per-tap transposes W_k^T the input gradient runs the same kernel with:
    (K, c_out, c_in) for modes 0-2, rounded (K, c_in, c_out) for mode 3.  Rebuilt on every call: no key can tell that the
    parameter was written in place through `.data` (EMA updates, weight surgery), which bumps no version counter, and
    the weights are at most a few MB."""
    w = weight.detach()
    if mode:
        w = round_tf32(w)
    parts = [w] if splits is None else list(torch.split(w, list(splits), dim=1))
    flip = (int(mode) == 3) != bool(transposed)
    return [(q.transpose(1, 2) if flip else q).contiguous() for q in parts]


def gather_gemm_wgrad(x, idx, g, tf32=False, bias=True, impl="cuda"):
    """weight and bias gradient of `gather_gemm` for the output gradient g (n_out, c_out) (already through the
    activation's derivative): dW[k] = sum_i [idx[i, k] >= 0] x[idx[i, k]]^T g[i]  (K, c_in, c_out), db = sum_i g[i]
    (None unless `bias`).  tf32: 0 = fp32 FFMA, 1..3 = TF32 mma.sync (x and g rounded); deterministic
    (csrc/sparse_conv_bwd.cu).  impl='torch' is the definition."""
    n_out, K = idx.shape
    c_in, c_out = x.shape[1], g.shape[1]
    if impl == "torch":
        xp = torch.cat([x, x.new_zeros((1, c_in))])                 # row -1 -> zeros
        dw = torch.stack([xp[idx[:, k].long()].transpose(0, 1) @ g for k in range(K)]) if n_out else \
            x.new_zeros((K, c_in, c_out))
        return dw, (g.sum(dim=0) if bias else None)
    x, idx, g = x.contiguous(), idx.contiguous(), g.contiguous()
    dw = torch.empty((K, c_in, c_out), dtype=torch.float32, device=x.device)
    db = torch.empty(c_out, dtype=torch.float32, device=x.device) if bias else None
    nb = call("nksr_gather_gemm_wgrad_workspace_bytes", n_out, K, c_in, c_out, int(tf32))
    ws = _ws(nb, x.device)
    call("nksr_gather_gemm_wgrad", x, idx, n_out, K, g, c_in, c_out, dw, db, ws, nb, int(tf32), stream_ptr(x.device))
    return dw, db


def transpose_taps(idx, n_src, impl="cuda"):
    """(n_src, K) int32 transpose of a gather table that is injective per tap: idx_t[j, k] = i iff idx[i, k] = j, -1
    elsewhere.  The input gradient of a convolution over idx is the convolution over idx_t with W_k^T.  A table with a
    repeated (source, tap) or a source >= n_src raises NksrError."""
    n_out, K = idx.shape
    if impl == "torch":
        ok = idx >= 0
        rows = torch.arange(n_out, device=idx.device)[:, None].expand(n_out, K)[ok]
        key = idx.long()[ok] * K + torch.arange(K, device=idx.device)[None, :].expand(n_out, K)[ok]
        if key.numel() and (int(key.max()) >= n_src * K or key.unique().numel() != key.numel()):
            raise NksrError("transpose_taps: the table is not injective per tap or a source is out of range")
        idx_t = torch.full((n_src * K,), -1, dtype=torch.int32, device=idx.device)
        idx_t[key] = rows.to(torch.int32)
        return idx_t.view(n_src, K)
    idx = idx.contiguous()
    idx_t = torch.empty((n_src, K), dtype=torch.int32, device=idx.device)
    status = torch.zeros(1, dtype=torch.int32, device=idx.device)
    call("nksr_transpose_taps", idx, n_out, K, n_src, idx_t, status, stream_ptr(idx.device))
    st = int(status.item())
    if st:
        raise NksrError(f"nksr_transpose_taps: " + ("a (source, tap) pair occurs twice; " if st & 1 else "") +
                        ("a source index is >= n_src" if st & 2 else "").rstrip("; "))
    return idx_t


def transposed_table(svh, idx, n_src):
    """`transpose_taps(idx, n_src)`, cached on the hierarchy object while `idx` is alive (the rule of `up_table`: a weak
    reference to the very tensor it was derived from, so a rebuilt table or a recycled id cannot pass for the old one)"""
    cache = svh.__dict__.setdefault("_unet_transposes", {})
    key = (id(idx), int(n_src))
    hit = cache.get(key)
    if hit is None or hit[0]() is not idx:
        for stale in [k for k, v in cache.items() if v[0]() is None]:
            del cache[stale]
        cache[key] = (weakref.ref(idx), transpose_taps(idx, n_src))
    return cache[key][1]


_KERNEL_FLAG = {0: 0, 1: 2, 2: 2, 3: 3}          # the weights are always rounded on the host (flag 2), never per fragment


def _per_part(idx, n_parts):
    """one gather table per part: `idx` itself when it is a tuple / list of them, else the one table for every part"""
    if isinstance(idx, (tuple, list)):
        if len(idx) != n_parts:
            raise ValueError(f"{len(idx)} index tables for {n_parts} parts")
        return tuple(idx)
    return (idx,) * n_parts


def conv_parts(parts, idx, weights, bias, res, relu, mode):
    """y = act(bias + res + sum_p conv(parts[p], weights[p])): the convolution of the channel concatenation of `parts`
    without materialising it -- one kernel call per part, each adding to the previous one's output.  `idx`: one table
    for all parts, or one per part (the decoder's skip input comes from another hierarchy through its own table)."""
    y = res
    idxs = _per_part(idx, len(parts))
    for i, (x, w) in enumerate(zip(parts, weights)):
        last = i == len(parts) - 1
        y = gather_gemm(x, idxs[i], w, bias if last else None, y, relu and last, _KERNEL_FLAG[int(mode)])
    return y


class GatherConv(torch.autograd.Function):
    """Autograd of `conv_parts` with the weight in parameter layout (K, sum_p c_p, c_out).  The forward is `conv_parts`
    itself (the same kernels and bits as without grad).  Backward, with g = dY * [y > 0] under ReLU (relu'(0) = 0):
      d_res = g,  d_bias = sum_i g[i],  dW = the weight-gradient kernel per part, concatenated along c_in,
      d_part_p = the forward kernel over the transposed table with part p's slice of W_k^T.
    idx_t: the transposed table, a function returning it (called once, in backward), or None (computed in backward).
    With one table per part (`idx` a tuple), every part's weight and input gradient run over its own table, and idx_t
    is a tuple of one such entry per part (or None)."""

    @staticmethod
    def forward(ctx, idx, idx_t, mode, relu, weight, bias, res, *parts):
        splits = tuple(int(q.shape[1]) for q in parts) if len(parts) > 1 else None
        y = conv_parts(parts, idx, kernel_weights(weight, mode, splits), bias, res, relu, mode)
        ctx.idx, ctx.idx_t, ctx.mode, ctx.relu, ctx.splits = idx, idx_t, int(mode), bool(relu), splits
        ctx.save_for_backward(weight, y if relu else None, *parts)
        return y

    @staticmethod
    def backward(ctx, dy):
        weight, y, *parts = ctx.saved_tensors
        need = ctx.needs_input_grad
        g = dy.contiguous()
        if ctx.relu:
            g = g * (y > 0)
        d_w = d_b = d_res = None
        if need[6]:
            d_res = g
        idxs = _per_part(ctx.idx, len(parts))
        if need[4] or need[5]:
            dws = []
            for p, x in enumerate(parts):
                dw, db = gather_gemm_wgrad(x, idxs[p], g, ctx.mode, bias=p == 0 and need[5])
                dws.append(dw)
                d_b = db if p == 0 else d_b
            d_w = dws[0] if len(dws) == 1 else torch.cat(dws, dim=1)
        d_parts = [None] * len(parts)
        if any(need[7:]):
            if isinstance(ctx.idx, (tuple, list)):
                idx_ts = ctx.idx_t if isinstance(ctx.idx_t, (tuple, list)) else (None,) * len(parts)
            else:
                idx_t = ctx.idx_t() if callable(ctx.idx_t) else ctx.idx_t
                if idx_t is None:
                    idx_t = transpose_taps(ctx.idx, parts[0].shape[0])
                idx_ts = (idx_t,) * len(parts)
            wts = kernel_weights(weight, ctx.mode, ctx.splits, transposed=True)
            for p in range(len(parts)):
                if need[7 + p]:
                    t = idx_ts[p]() if callable(idx_ts[p]) else idx_ts[p]
                    if t is None:
                        t = transpose_taps(idxs[p], parts[p].shape[0])
                    d_parts[p] = gather_gemm(g, t, wts[p], None, None, False, _KERNEL_FLAG[ctx.mode])
        return (None, None, None, None, d_w, d_b, d_res, *d_parts)


def _wants_grad(*tensors):
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors)


class SparseConv(nn.Module):
    """K-tap sparse convolution: weight (K, c_in, c_out) + bias; the taps' sources come from an index table.  `x` may be
    a tuple of tensors: the convolution then runs over their channel concatenation (the U-Net's skip connections);
    `idx` is then one table for all of them or a tuple of one table per part (and `idx_t` one entry per part).
    With grad enabled and an input or parameter that requires grad, the CUDA path runs through `GatherConv`; `idx_t`
    (the transposed table or a function returning it) saves its computation in backward."""

    def __init__(self, taps, c_in, c_out):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(taps, c_in, c_out))
        self.bias = nn.Parameter(torch.zeros(c_out))
        bound = math.sqrt(6.0 / (taps * c_in))                       # He-uniform over the full stencil
        nn.init.uniform_(self.weight, -bound, bound)

    def forward(self, x, idx, res=None, relu=True, tf32=False, impl="cuda", idx_t=None):
        parts = tuple(x) if isinstance(x, (tuple, list)) else (x,)
        if impl != "cuda":
            if isinstance(idx, (tuple, list)):          # one table per part: the sum of the per-part convolutions
                ws = torch.split(self.weight, [int(q.shape[1]) for q in parts], dim=1)
                y = sum(gather_gemm(q, t, w, None, None, False, False, impl)
                        for q, t, w in zip(parts, _per_part(idx, len(parts)), ws))
                y = y + self.bias
                if res is not None:
                    y = y + res
                return torch.relu(y) if relu else y
            xc = parts[0] if len(parts) == 1 else torch.cat(parts, dim=1)
            return gather_gemm(xc, idx, self.weight, self.bias, res, relu, False, impl)
        mode = int(tf32)
        if _wants_grad(self.weight, self.bias, res, *parts):
            return GatherConv.apply(idx, idx_t, mode, relu, self.weight, self.bias, res, *parts)
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
            idx = up_table(svh, l)
            if _wants_grad(self.up[l], y_coarse):
                n_src = svh.num_voxels(l + 1)
                return GatherConv.apply(idx, lambda: transposed_table(svh, idx, n_src), int(tf32), False, self.up[l],
                                        None, None, y_coarse)
            ws = kernel_weights(self.up[l], int(tf32))
            return conv_parts((y_coarse,), idx, ws, None, None, False, int(tf32))
        n_l = svh.num_voxels(l)
        out = torch.zeros((n_l, self.channels[l]), dtype=y_coarse.dtype, device=y_coarse.device)
        octant = octant_of_children(svh.child8[l + 1], n_l)
        parent = svh.parent[l].long()
        for o in range(8):
            rows = torch.nonzero((octant == o) & (parent >= 0)).squeeze(1)
            if rows.numel():
                out[rows] = y_coarse[parent[rows]] @ self.up[l][o]
        return out

    def _encode(self, x0, svh, D, kw, tt):
        """the down path: the encoder output x_l of every level"""
        xs, x = [], x0
        for l in range(D):
            nbr = svh.nbr27[l]
            h = self.enc_a[l](x, nbr, relu=True, idx_t=tt(nbr, l), **kw)
            x = self.enc_b[l](h, nbr, res=x, relu=True, idx_t=tt(nbr, l), **kw)
            xs.append(x)
            if l + 1 < D:
                x = self.down[l](x, svh.child8[l + 1], relu=True, idx_t=tt(svh.child8[l + 1], l), **kw)
        return xs

    def _heads(self, out, l, y):
        C = self.kernel_dim
        o = self.heads[l](y)
        out.structure[l], out.normal[l] = o[:, :3], o[:, 3:6]
        out.basis[l], out.udf[l] = o[:, 6:6 + C], o[:, 6 + C:6 + 2 * C]
        out.decoder[l] = y

    def forward(self, x0, svh, tf32=False, impl="cuda", grow=None):
        """the U-Net on the encoder hierarchy `svh`; with `grow` (a dict of `forward_grown`'s keyword arguments) the
        decoder runs on the hierarchy grown from the structure logits instead"""
        if grow is not None:
            return self.forward_grown(x0, svh, tf32=tf32, impl=impl, **grow)
        D = min(self.depth, svh.depth)
        kw = dict(tf32=tf32, impl=impl)
        # transposed tables for the input gradients, built on first use in backward and cached on the hierarchy
        tt = lambda idx, l: (lambda: transposed_table(svh, idx, svh.num_voxels(l))) if impl == "cuda" else None
        xs = self._encode(x0, svh, D, kw, tt)
        ys = [None] * D
        y = xs[D - 1]
        ys[D - 1] = y
        for l in range(D - 2, -1, -1):
            u = self.up_project(y, svh, l, **kw)
            y = self.dec[l]((xs[l], u), svh.nbr27[l], relu=True, idx_t=tt(svh.nbr27[l], l), **kw)   # [skip ; up], not cat
            ys[l] = y
        C = self.kernel_dim
        out = SimpleNamespace(structure={}, normal={}, basis={}, udf={}, decoder={})
        for l in range(D):
            o = self.heads[l](ys[l])
            out.structure[l], out.normal[l] = o[:, :3], o[:, 3:6]
            out.basis[l], out.udf[l] = o[:, 6:6 + C], o[:, 6 + C:6 + 2 * C]
            out.decoder[l] = ys[l]
        return out

    def forward_grown(self, x0, svh, adaptive_depth, forced=None, max_ratio=None, tf32=False, impl="cuda"):
        """The decoder on the hierarchy T grown from its own structure logits (DESIGN.md SPEC S16).  The down path is
        `forward`'s.  Going up, level l of T is decoded as y_l = relu(dec_l([skip ; u])) over T.nbr27[l], u the
        up-projection of y_{l+1} through T's parent-by-octant table and the skip input E's encoder output x_l gathered
        through skip27 = join_l o T.nbr27[l]; the heads run on y_l at once, and the structure logits of level l (or
        `forced(T, l)`, the classes of teacher forcing) decide T_{l-1}.
        Returns the heads and decoder outputs per level on T (structure / normal / basis / udf / decoder), plus
        `udf_svh` (T), `dec_svh` (the kept voxels), `kept[l]` (indices into T_l of dec_svh's voxels), `classes[l]`
        and `growth` (the StructureGrowth, with its join and skip tables).  impl='torch' grows with the torch
        restatement and convolves with the dense-gather torch path."""
        from .structure import DEFAULT_MAX_RATIO, StructureGrowth
        D = min(self.depth, svh.depth)
        kw = dict(tf32=tf32, impl=impl)
        tt = lambda idx, l: (lambda: transposed_table(svh, idx, svh.num_voxels(l))) if impl == "cuda" else None
        xs = self._encode(x0, svh, D, kw, tt)
        g = StructureGrowth(svh, D, adaptive_depth, DEFAULT_MAX_RATIO if max_ratio is None else max_ratio, impl)
        T = g.T
        out = SimpleNamespace(structure={}, normal={}, basis={}, udf={}, decoder={})
        y = xs[D - 1]
        for l in range(D - 1, -1, -1):
            if l < D - 1:
                u = self.up_project(y, T, l, **kw)
                skip, nbr = g.skip27(l), T.nbr27[l]
                n_e, n_t = svh.num_voxels(l), T.num_voxels(l)
                idx_t = ((lambda s=skip, n=n_e: transposed_table(T, s, n)),
                         (lambda b=nbr, n=n_t: transposed_table(T, b, n))) if impl == "cuda" else None
                y = self.dec[l]((xs[l], u), (skip, nbr), relu=True, idx_t=idx_t, **kw)
            self._heads(out, l, y)
            c = forced(T, l) if forced is not None else None
            g.step(l, logits=None if c is not None else out.structure[l].detach(), forced=c)
        out.dec_svh = g.finish()
        out.udf_svh, out.kept, out.classes, out.growth = T, g.kept, g.classes, g
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
