"""NKSRNetwork stand-in (PyTorch).

The reference's sparse-conv encoder / U-Net lives in the closed wheel and its pretrained
weights are a network download (models/nksr_net.py:35-38, README.md:108-110).  BASELINE.json's
north_star keeps the network on PyTorch and outside the hot path, so this module is a small,
seeded, deterministic replacement that produces the SAME OUTPUT CONTRACT the hot path consumes
(models/nksr_net.py:73-78, 93-94, 101, 117-118, 127-128):

    feat = network.encoder(xyz, point_feat, svh, 0)
    feat, dec_svh, udf_svh = network.unet(feat, svh, adaptive_depth=..., gt_decoder_svh=...)
    feat.basis_features[d]  (n_d, kernel_dim)   feat.normal_features[d]  (n_d, 3)
    feat.structure_features[d] (n_d, 3)         feat.udf_features[d]
    network.interpolators / .sdf_decoder / .udf_decoder

With backbone='unet', `structure` chooses the decoder hierarchy: 'encoder' (default) decodes on the encoder hierarchy and
returns it as dec_svh and udf_svh; 'predicted' grows it from the structure head level by level (DESIGN.md SPEC S16,
nksr_b200/structure.py) -- teacher-forced from gt_decoder_svh when one is given -- and returns the kept voxels as dec_svh
and the whole grown hierarchy (the reference's dec_tmp_svh) as udf_svh.

For backbone='pool', normals are the pooled input normals (or view directions) -- i.e. the "prediction" is
geometric, not learned; kernel features are a seeded perturbation of a constant, which makes
the kernel close to the pure Bezier kernel (well conditioned).  Documented as synthetic in
bench.py (`"data": "synthetic"`).
"""
from __future__ import annotations

from types import SimpleNamespace

import torch
from torch import nn

from .svh import SparseFeatureHierarchy

_DEFAULTS = dict(kernel_dim=4, tree_depth=4, adaptive_depth=2, feature="normal",
                 interpolator=dict(n_hidden=2, hidden_dim=16), udf=dict(enabled=False), seed=0,
                 unet=dict(f_maps=32), backbone="pool", precision="fp32", trainable=False, structure="encoder",
                 structure_max_ratio=None, geometry="kernel")
# the UDF decoder of udf.enabled draws its initial weights from seed + this offset
UDF_DECODER_SEED_OFFSET = 0x5D17
# the SDF decoder of geometry='neural' draws its initial weights from seed + this offset
SDF_DECODER_SEED_OFFSET = 0x5DF0


def _get(hp, key, default):
    if hp is None:
        return default
    if isinstance(hp, dict):
        return hp.get(key, default)
    return getattr(hp, key, default)


class ResidualMLP(nn.Module):
    def __init__(self, dim, hidden, n_hidden, scale=0.1):
        super().__init__()
        layers, d = [], dim
        for _ in range(max(n_hidden, 0)):
            layers += [nn.Linear(d, hidden), nn.ReLU()]
            d = hidden
        layers.append(nn.Linear(d, dim))
        self.net = nn.Sequential(*layers)
        self.scale = scale

    def forward(self, x):
        return x + self.scale * torch.tanh(self.net(x))


class FeatureBundle(SimpleNamespace):
    pass


class NKSRNetwork(nn.Module):
    def __init__(self, hparams=None, **overrides):
        super().__init__()
        hp = {k: _get(hparams, k, v) for k, v in _DEFAULTS.items()}
        hp.update(overrides)
        self.kernel_dim = int(hp["kernel_dim"])
        self.tree_depth = int(hp["tree_depth"])
        self.adaptive_depth = int(hp["adaptive_depth"])
        self.feature = hp["feature"]
        self.compute_structure = False
        # backbone: 'pool' = the geometric stand-in below (sensible output without trained weights: what the benchmark and
        # the examples use); 'unet' = the sparse-conv encoder / U-Net (nksr_b200/unet.py, csrc/sparse_conv.cu), random init
        self.backbone = str(hp["backbone"])
        if self.backbone not in ("pool", "unet"):
            raise ValueError("backbone: 'pool' or 'unet'")
        # precision: 'fp32' (FFMA kernel), 'tf32' (mma.sync), 'tc' (wgmma tensor cores) -- csrc/sparse_conv.cu
        self.tf32 = {"tf32": True, "tc": 3}.get(str(hp["precision"]), False)
        # trainable: the U-Net backbone keeps requires_grad and encoder / unet follow the caller's grad mode (the sparse
        # convolution's backward: csrc/sparse_conv_bwd.cu); by default every parameter is frozen and both run without grad
        self.trainable = bool(hp["trainable"])
        if self.trainable and self.backbone != "unet":
            raise ValueError("trainable=True needs backbone='unet' (the 'pool' stand-in has nothing to train)")
        # structure: 'encoder' = the decoder runs on the encoder hierarchy; 'predicted' = it grows its own hierarchy
        # from the structure head, level by level (DESIGN.md SPEC S16, nksr_b200/structure.py) -- U-Net backbone only
        self.structure = str(hp["structure"])
        if self.structure not in ("encoder", "predicted"):
            raise ValueError("structure: 'encoder' or 'predicted'")
        if self.structure == "predicted" and self.backbone != "unet":
            raise ValueError("structure='predicted' needs backbone='unet' (the 'pool' stand-in has no structure head "
                             "to grow from)")
        # children a grown level may hold, as a multiple of the encoder voxels of that level (None: the default of
        # nksr_b200/structure.py, DEFAULT_MAX_RATIO)
        self.structure_max_ratio = hp["structure_max_ratio"]
        # udf.enabled: the mask of a reconstruction is the UDF NeuralField on the decoder hierarchy (DESIGN.md SPEC S17,
        # models/nksr_net.py:124-130) and training adds its UDF loss over every level -- U-Net backbone only
        self.udf_enabled = bool(_get(hp["udf"], "enabled", False))
        if self.udf_enabled and self.backbone != "unet":
            raise ValueError("udf.enabled needs backbone='unet' (the 'pool' stand-in has no UDF head)")
        # geometry: the output field of a reconstruction (models/nksr_net.py:89-122).  'kernel' = the KernelField solved
        # from the basis features; 'neural' = the NeuralField sdf_decoder(u(x)) over the basis features of every decoder
        # level (no solve) -- U-Net backbone only
        self.geometry = str(hp["geometry"])
        if self.geometry not in ("kernel", "neural"):
            raise ValueError(f"geometry: 'kernel' or 'neural', not {self.geometry!r}")
        if self.geometry == "neural" and self.backbone != "unet":
            raise ValueError("geometry='neural' needs backbone='unet' (the 'pool' stand-in has no decoder to train)")
        interp = hp["interpolator"]
        gen = torch.Generator().manual_seed(int(hp["seed"]))
        state = torch.random.get_rng_state()
        torch.manual_seed(int(hp["seed"]))
        try:
            C = self.kernel_dim
            self.basis_heads = nn.ModuleList([nn.Linear(4, C) for _ in range(self.tree_depth)])
            self.interpolators = nn.ModuleList([
                ResidualMLP(C, int(_get(interp, "hidden_dim", 16)), int(_get(interp, "n_hidden", 2)))
                for _ in range(self.tree_depth)])
            self.structure_heads = nn.ModuleList([nn.Linear(4, 3) for _ in range(self.tree_depth)])
            self.sdf_decoder = nn.Sequential(nn.Linear(C, 16), nn.ReLU(), nn.Linear(16, 1))
            self.udf_decoder = nn.Sequential(nn.Linear(C, 16), nn.ReLU(), nn.Linear(16, 1))
            if self.backbone == "unet":
                from .unet import PointEncoder, SparseUNet
                f_maps = int(_get(hp["unet"], "f_maps", 32))
                if f_maps % 32:
                    raise ValueError("unet.f_maps must be a multiple of 32 (csrc/sparse_conv.cu stages 32-channel chunks)")
                self.point_encoder = PointEncoder(0 if self.feature in (None, "none") else 3, f_maps, f_maps)
                self.backbone_net = SparseUNet(self.tree_depth, f_maps, C)
            if self.udf_enabled:
                # the decoder of u(x), C columns per level; built last from its own seed, so that every other parameter
                # is bitwise what it is with udf disabled (the Linear(C, 16) above only keeps the draws in step)
                torch.manual_seed(int(hp["seed"]) + UDF_DECODER_SEED_OFFSET)
                self.udf_decoder = nn.Sequential(nn.Linear(C * self.tree_depth, 32), nn.ReLU(), nn.Linear(32, 32),
                                                 nn.ReLU(), nn.Linear(32, 1))
            if self.geometry == "neural":
                # the decoder of the neural output field, C columns per level; built after every other module from its
                # own seed, like the UDF decoder, so that every other parameter is bitwise that of geometry='kernel'
                torch.manual_seed(int(hp["seed"]) + SDF_DECODER_SEED_OFFSET)
                self.sdf_decoder = nn.Sequential(nn.Linear(C * self.tree_depth, 32), nn.ReLU(), nn.Linear(32, 32),
                                                 nn.ReLU(), nn.Linear(32, 1))
        finally:
            torch.random.set_rng_state(state)
        del gen
        if not self.trainable:
            for p in self.parameters():
                p.requires_grad_(False)

    def _grad_mode(self):
        """the caller's grad mode for a trainable network, no grad otherwise"""
        return torch.set_grad_enabled(self.trainable and torch.is_grad_enabled())

    # ---- encoder: pool point features into the voxels of every level ---------------------
    def encoder(self, xyz: torch.Tensor, feat, svh: SparseFeatureHierarchy, depth: int = 0):
        with self._grad_mode():
            return self._encoder(xyz, feat, svh, depth)

    def _encoder(self, xyz, feat, svh, depth):
        from ._lib import call, stream_ptr
        if self.backbone == "unet":
            if feat is None and self.point_encoder.fc_in.in_features > 3:
                feat = torch.zeros_like(xyz)
            return SimpleNamespace(svh=svh, x0=self.point_encoder(xyz.to(torch.float32), feat, svh))
        base0 = svh.locate(xyz)[0].long()                               # finest containing voxel
        ones = torch.ones((xyz.shape[0], 1), device=xyz.device)
        src = torch.cat([feat.to(torch.float32) if feat is not None else torch.zeros_like(xyz), ones], dim=1)
        pooled, acc = [], None
        for l in range(svh.depth):
            n = svh.num_voxels(l)
            if l == 0:
                acc = torch.zeros((n, 4), device=xyz.device)
                ok = base0 >= 0
                acc.index_add_(0, base0[ok], src[ok])
            else:                                                       # sum of the (<= 8) children
                up = torch.empty((n, 4), device=xyz.device)
                call("nksr_pool_children", svh.child8[l], acc, n, 4, up, stream_ptr(xyz.device))
                acc = up
            # smooth over the 27-neighbourhood so that splat-only voxels receive a value
            out = torch.empty_like(acc)
            call("nksr_pool27", svh.nbr27[l], acc, n, 4, out, stream_ptr(xyz.device))
            pooled.append(out)
        return SimpleNamespace(svh=svh, pooled=pooled)

    # ---- "U-Net": heads on the pooled statistics; hierarchy passes through -----------------
    def unet(self, feat, svh: SparseFeatureHierarchy, adaptive_depth: int = None, gt_decoder_svh=None):
        with self._grad_mode():
            return self._unet(feat, svh, adaptive_depth, gt_decoder_svh)

    def _unet(self, feat, svh, adaptive_depth, gt_decoder_svh):
        if self.structure == "predicted":
            return self._unet_grown(feat, svh, adaptive_depth, gt_decoder_svh)
        dec_svh = gt_decoder_svh if gt_decoder_svh is not None else svh
        C = self.kernel_dim
        if self.backbone == "unet":
            # structure='encoder': the decoder runs on the encoder hierarchy; a given decoder hierarchy (ground truth at
            # training time, models/nksr_net.py:77) receives the features of the voxels it shares with it.
            # structure='predicted' grows the decoder hierarchy from the structure logits instead (_unet_grown).
            from .unet import restrict_to
            o = self.backbone_net(feat.x0, svh, tf32=self.tf32)
            return (FeatureBundle(basis_features=restrict_to(o.basis, svh, dec_svh),
                                  normal_features=restrict_to(o.normal, svh, dec_svh),
                                  structure_features=restrict_to(o.structure, svh, dec_svh),
                                  udf_features=restrict_to(o.udf, svh, dec_svh)), dec_svh, dec_svh)
        basis, normal, structure, udf = {}, {}, {}, {}
        up = None
        for l in range(svh.depth - 1, -1, -1):
            s = feat.pooled[l]
            cnt = s[:, 3:4]
            mean = s[:, :3] / cnt.clamp(min=1.0)
            nrm = mean / (mean.norm(dim=1, keepdim=True) + 1e-6)
            if up is not None and svh.parent[l] is not None:           # fill empties from the parent
                nrm = torch.where(cnt > 0, nrm, up[svh.parent[l].long()])
            up = nrm
            x = torch.cat([nrm, torch.log1p(cnt)], dim=1)
            basis[l] = (1.0 + 0.1 * torch.tanh(self.basis_heads[l](x))) / (C ** 0.5)
            normal[l] = nrm
            if self.compute_structure:          # only the training losses read it (models/loss.py:152)
                structure[l] = self.structure_heads[l](x)
            udf[l] = basis[l]
        out = FeatureBundle(basis_features=basis, normal_features=normal, structure_features=structure,
                            udf_features=udf)
        return out, dec_svh, dec_svh

    def _unet_grown(self, feat, svh, adaptive_depth, gt_decoder_svh, impl="cuda"):
        """structure='predicted' (DESIGN.md SPEC S16): the decoder grows its hierarchy T from its structure logits, or
        from gt_decoder_svh's voxel status when one is given (teacher forcing, models/nksr_net.py:74-86).  Returns
        (features, dec_svh, udf_svh): udf_svh = T, where the structure and UDF features live; dec_svh = T's kept voxels,
        where the basis and normal features live."""
        from .structure import teacher_classes
        ad = self.adaptive_depth if adaptive_depth is None else int(adaptive_depth)
        forced = teacher_classes(gt_decoder_svh) if gt_decoder_svh is not None else None
        o = self.backbone_net(feat.x0, svh, tf32=self.tf32, impl=impl,
                              grow=dict(adaptive_depth=ad, forced=forced, max_ratio=self.structure_max_ratio))
        kept = o.kept
        bundle = FeatureBundle(basis_features={l: f[kept[l]] for l, f in o.basis.items()},
                               normal_features={l: f[kept[l]] for l, f in o.normal.items()},
                               structure_features=o.structure, udf_features=o.udf, classes=o.classes)
        return bundle, o.dec_svh, o.udf_svh


def load_checkpoint_from_url(url: str):
    """nksr.configs.load_checkpoint_from_url (models/nksr_net.py:17,37-38).  There is no network
    in this environment: only local paths are honoured; URLs raise."""
    import os
    if os.path.exists(url):
        return torch.load(url, map_location="cpu")
    raise RuntimeError(f"cannot fetch checkpoint '{url}': no network access; this build uses the seeded "
                       "stand-in network (nksr_b200/network.py)")
