"""Training losses of the U-Net backbone: the structure loss and the UDF loss of the reference (models/loss.py:143-160
and :106-140), with the samplers and ground-truth transform of configs/default/train.yaml
(supervision.structure_weight, supervision.udf, supervision.spatial.gt_band / gt_soft), and -- opt-in,
`train_step(..., kernel=True)` -- the kernel-field losses, which backpropagate through the kernel solve
(supervision.gt_surface and supervision.spatial, models/loss.py:163-260; fields._KernelSolve), or with
geometry='neural' the same losses on the NeuralField output field, whose normal loss backpropagates through its position
gradient (fields._NeuralJacobian).

    feat, dec_svh, _ = net.unet(net.encoder(xyz, normal, svh, 0), svh)
    l_struct, per_level = structure_loss(feat.structure_features, dec_svh, gt_svh)
    l_udf = udf_loss(net.udf_decoder, feat.udf_features, dec_svh, ref_xyz, ref_normal, voxel_size)
    (with udf.enabled: udf_field_loss, the same loss on the NeuralField over every level)

Both are plain torch on top of the hierarchy's CUDA tables; the gradients flow into the network through the sparse
convolution's backward kernels (nksr_b200/unet.py, csrc/sparse_conv_bwd.cu).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .fields import KernelField, NeuralField
from .sdfgen import sdf_from_points
from .svh import SparseFeatureHierarchy

# configs/default/train.yaml: supervision.structure_weight, supervision.udf (weight, samplers), spatial.gt_band
STRUCTURE_WEIGHT = 20.0
UDF_WEIGHT = 150.0
UDF_SAMPLERS = (dict(type="uniform", n_samples=80000, expand=1, expand_top=5),
                dict(type="band", n_samples=20000, eps=0.5))
GT_BAND = 1.0
# supervision.gt_surface (value / normal weights, subsample) and supervision.spatial (weight, samplers); solver weights
GT_SURFACE_VALUE_WEIGHT = 200.0
GT_SURFACE_NORMAL_WEIGHT = 100.0
GT_SURFACE_SUBSAMPLE = 50000
SPATIAL_WEIGHT = 300.0
SPATIAL_SAMPLERS = (dict(type="uniform", n_samples=50000, expand=1, expand_top=3),
                    dict(type="band", n_samples=50000, eps=0.5))
POS_WEIGHT = 1.0e4
NORMAL_WEIGHT = 1.0e4


def structure_loss(structure_features, dec_svh: SparseFeatureHierarchy, gt_svh: SparseFeatureHierarchy):
    """sum over the levels of the cross-entropy of the structure logits (n_l, 3) of the decoder hierarchy's voxels
    against gt_svh.evaluate_voxel_status (0 absent, 1 leaf, 2 with children; models/loss.py:150-156).  Returns
    (total, {level: loss}); levels without voxels are skipped."""
    grids = dec_svh.grids
    per_level = {}
    for d, logits in structure_features.items():
        if logits.shape[0] == 0:
            continue
        gt = gt_svh.evaluate_voxel_status(grids[d], d)
        per_level[d] = F.cross_entropy(logits, gt)
    total = sum(per_level.values()) if per_level else torch.zeros((), device=dec_svh.device)
    return total, per_level


def svh_samples(svh: SparseFeatureHierarchy, n: int, expand: int = 0, expand_top: int = 0, generator=None):
    """n points uniform over the voxels of every level (models/loss.py:22-52): a voxel drawn uniformly from all levels'
    voxels, then a point uniform inside it; a level's voxels are first dilated by `expand` (`expand_top` on the
    coarsest level) when that is >= 3"""
    dev = svh.device
    coords, scales = [], []
    grids = svh.grids
    for d in range(svh.depth):
        if grids[d] is None:
            continue
        ijk = grids[d].active_grid_coords().long()
        e = expand if d != svh.depth - 1 else expand_top
        if e >= 3:
            o = torch.arange(-e // 2 + 1, e // 2 + 1, device=dev)
            o = torch.stack(torch.meshgrid(o, o, o, indexing="ij"), dim=3).view(-1, 3)
            ijk = torch.unique((ijk[:, None, :] + o[None]).view(-1, 3), dim=0)
        coords.append(grids[d].grid_to_world(ijk))
        scales.append(torch.full((ijk.shape[0],), grids[d].voxel_size, device=dev))
    coords, scales = torch.cat(coords), torch.cat(scales)
    pick = (torch.rand((n,), device=dev, generator=generator) * coords.shape[0]).long()
    local = (torch.rand((n, 3), device=dev, generator=generator) - 0.5) * scales[pick, None]
    return coords[pick] + local


def band_samples(ref_xyz, ref_normal, n: int, eps: float, generator=None):
    """n points displaced from random reference points along their normals by N(0, eps) (models/loss.py:60-66)"""
    dev = ref_xyz.device
    pick = (torch.rand((n,), device=dev, generator=generator) * ref_xyz.shape[0]).long()
    return ref_xyz[pick] + ref_normal[pick] * torch.randn((n, 1), device=dev, generator=generator) * eps


def transform_field(f, voxel_size, gt_band=GT_BAND):
    """soft truncation tanh(f / T) T, T = gt_band * voxel_size (models/loss.py:68-80, gt_soft: true)"""
    t = gt_band * voxel_size
    return torch.tanh(f / t) * t


def udf_samples(svh, ref_xyz, ref_normal, voxel_size, samplers=UDF_SAMPLERS, generator=None):
    out = []
    for s in samplers:
        if s["type"] == "uniform":
            out.append(svh_samples(svh, s["n_samples"], s["expand"], s["expand_top"], generator))
        else:
            out.append(band_samples(ref_xyz, ref_normal, s["n_samples"], s["eps"] * voxel_size, generator))
    return torch.cat(out, 0)


def udf_gt(q, ref_xyz, ref_normal, voxel_size, gt_band=GT_BAND, gt=None):
    """|transform(-sdf_from_points(q, ref, 8, 0.02))|, or with ground truth geometry (a PointTSDFVolume or a
    MeshGroundTruth) |transform(gt.query_sdf(q))| (models/loss.py:84-86, 111-118)"""
    if gt is not None:
        return transform_field(gt.query_sdf(q), voxel_size, gt_band).abs()
    sdf = -sdf_from_points(q, ref_xyz, ref_normal, 8, 0.02, False)[0]
    return transform_field(sdf, voxel_size, gt_band).abs()


def udf_loss(udf_decoder, udf_features, svh: SparseFeatureHierarchy, ref_xyz, ref_normal, voxel_size,
             samplers=UDF_SAMPLERS, gt_band=GT_BAND, generator=None, q=None, gt=None):
    """mean |transform(pd) - gt| / voxel_size over the UDF samples (models/loss.py:120-140).  pd is the UDF NeuralField
    evaluated differentiably as udf_decoder(NeuralField._interp(q)) on the finest level's UDF features (the decoder
    takes kernel_dim inputs); `q` overrides the samplers; `gt` (ground truth geometry) gives the ground truth (udf_gt).
    Zero when the finest level is empty (a hierarchy grown from a prediction that kept nothing there): there is no
    field to evaluate."""
    if svh.num_voxels(0) == 0:
        return torch.zeros((), device=svh.device)
    if q is None:
        q = udf_samples(svh, ref_xyz, ref_normal, voxel_size, samplers, generator)
    gt = udf_gt(q, ref_xyz, ref_normal, voxel_size, gt_band, gt)
    field = NeuralField(svh, udf_decoder, {0: udf_features[0]})
    pd = udf_decoder(field._interp(q.to(torch.float32).contiguous())).reshape(-1)
    return torch.mean((transform_field(pd, voxel_size, gt_band) - gt).abs()) / voxel_size


def udf_field_loss(udf_decoder, udf_features, svh: SparseFeatureHierarchy, ref_xyz, ref_normal, voxel_size,
                   samplers=UDF_SAMPLERS, gt_band=GT_BAND, generator=None, q=None, gt=None):
    """the UDF loss of udf.enabled (models/loss.py:120-140): the same samples, ground truth and L1 as `udf_loss`, but pd
    is the UDF NeuralField over every level of `svh` (the decoder takes kernel_dim columns per level), evaluated and
    backpropagated through the interpolation kernels (csrc/neural_field.cu)"""
    if q is None:
        q = udf_samples(svh, ref_xyz, ref_normal, voxel_size, samplers, generator)
    gt = udf_gt(q, ref_xyz, ref_normal, voxel_size, gt_band, gt)
    field = NeuralField(svh, udf_decoder, udf_features)
    pd = field.evaluate_f(q.to(torch.float32).contiguous()).value
    return torch.mean((transform_field(pd, voxel_size, gt_band) - gt).abs()) / voxel_size


class TrainingScene:
    """one oriented cloud with its encoder hierarchy (point splatting) and ground-truth hierarchy (adaptive, from the
    normals, models/nksr_net.py:175-179).  The decoder runs on the encoder hierarchy: the predicted-structure regime,
    where all three structure classes occur.  `gt`: ground truth geometry on the same device, any object with
    torch_attr() -> (xyz, normal, ...), query_sdf(q) and query_classification(q) (0 near, 1 empty, 2 unknown):
    gt_geometry.PointTSDFVolume (volume ground truth) or gt_geometry.MeshGroundTruth (a mesh).  Every loss then takes
    its reference from it, as models/nksr_net.py and models/loss.py do with DS.GT_GEOMETRY: the ground-truth hierarchy and
    the surface samples from torch_attr(), the SDF from gt.query_sdf and the spatial loss's empty-space term from
    gt.query_classification."""

    def __init__(self, xyz, normal, voxel_size, depth, adaptive_depth=2, gt=None):
        dev = xyz.device
        self.xyz, self.normal, self.voxel_size = xyz.contiguous(), normal.contiguous(), float(voxel_size)
        self.gt = gt
        self.ref_xyz, self.ref_normal = (self.xyz, self.normal) if gt is None else gt.torch_attr()[:2]
        self.enc_svh = SparseFeatureHierarchy(voxel_size, depth, dev).build_point_splatting(self.xyz)
        self.gt_svh = SparseFeatureHierarchy(voxel_size, depth, dev).build_adaptive_normal_variation(
            self.ref_xyz, self.ref_normal, adaptive_depth=adaptive_depth)
        self.adaptive_depth = adaptive_depth


def kernel_field(net, feat, dec_svh: SparseFeatureHierarchy, scene: TrainingScene, timer=None, operator=None):
    """the KernelField of models/nksr_net.py:91-112: basis features through the interpolators, position constraints at
    the input points, normal constraints (value -normal_features) at the voxel centres of the `adaptive_depth` finest
    levels, solved with the solver weights of train.yaml.  Differentiable when grad is enabled (fields._KernelSolve).
    `operator` ('assembled' or 'matrix_free'), if given, sets field.solver_config['operator']: the matrix-free operator
    runs the forward and the adjoint PCG without assembling the Gram matrix."""
    field = KernelField(dec_svh, net.interpolators, feat.basis_features)
    if operator is not None:
        field.solver_config["operator"] = operator
    if timer is not None:
        field._timer = timer
        timer.mark("solve_start")
    ad = min(scene.adaptive_depth, dec_svh.depth)
    normal_xyz = torch.cat([dec_svh.get_voxel_centers(d) for d in range(ad)])
    normal_value = torch.cat([feat.normal_features[d] for d in range(ad)])
    normal_weight = NORMAL_WEIGHT / normal_xyz.shape[0] * (scene.voxel_size ** 2)
    field.solve(scene.xyz, normal_xyz, -normal_value, POS_WEIGHT / scene.xyz.shape[0], normal_weight, 1.0)
    return field


def gt_surface_loss(field, ref_xyz, ref_normal, subsample=GT_SURFACE_SUBSAMPLE, generator=None):
    """(value, normal) losses at a subsample of the reference points (models/loss.py:163-198): mean |f| and
    1 - mean <-grad f / |grad f|, n>"""
    if 0 < subsample < ref_xyz.shape[0]:
        idx = (torch.rand((subsample,), device=ref_xyz.device, generator=generator) * ref_xyz.shape[0]).long()
    else:
        idx = torch.arange(ref_xyz.shape[0], device=ref_xyz.device)
    ev = field.evaluate_f(ref_xyz[idx], grad=True)
    g = -ev.gradient / (torch.linalg.norm(ev.gradient, dim=-1, keepdim=True) + 1.0e-6)
    return ev.value.abs().mean(), 1.0 - torch.sum(g * ref_normal[idx], dim=-1).mean()


def spatial_loss(field, ref_xyz, ref_normal, voxel_size, samplers=SPATIAL_SAMPLERS, gt_band=GT_BAND, generator=None,
                 gt=None):
    """near-surface L1 of the transformed field against the transformed point-cloud SDF, / voxel_size, over the uniform +
    band samples (models/loss.py:201-260).  Without GT geometry every sample counts as near-surface; with `gt` (a
    PointTSDFVolume or a MeshGroundTruth, see TrainingScene) the loss is spatial_volume_terms' near + empty sums over
    the number of samples."""
    if gt is not None:
        near, empty, n = spatial_volume_terms(field, ref_xyz, ref_normal, voxel_size, gt, samplers, gt_band, generator)
        return (near + empty) / n
    q = udf_samples(field.svh, ref_xyz, ref_normal, voxel_size, samplers, generator)
    gt = transform_field(-sdf_from_points(q, ref_xyz, ref_normal, 8, 0.02, False)[0], voxel_size, gt_band)
    pd = transform_field(field.evaluate_f(q).value, voxel_size, gt_band)
    return torch.sum(torch.abs((pd - gt) / voxel_size)) / q.shape[0]


EMPTY_SPACE_WEIGHT = 0.1     # models/loss.py:244-245: 0.1 exp(pd / (2 voxel_size)) on empty-space samples


def spatial_volume_terms(field, ref_xyz, ref_normal, voxel_size, gt, samplers=SPATIAL_SAMPLERS, gt_band=GT_BAND,
                         generator=None):
    """the spatial loss's two sums with ground truth geometry (models/loss.py:227-248) and the number of samples:
    near = sum over the near-surface samples (class 0 of gt.query_classification) of |transform(pd) -
    transform(gt.query_sdf(q))| / voxel_size; empty = sum over the empty-space samples (class 1) of
    0.1 exp(pd / (2 voxel_size)) of the raw prediction, which pushes the field down in observed free space.  Unknown
    samples (class 2) get neither term."""
    q = udf_samples(field.svh, ref_xyz, ref_normal, voxel_size, samplers, generator)
    pd = field.evaluate_f(q).value
    gt_tsdf = transform_field(gt.query_sdf(q), voxel_size, gt_band)
    cls = gt.query_classification(q)
    near, empty = cls == 0, cls == 1
    pd_tsdf = transform_field(pd, voxel_size, gt_band)
    l_near = torch.sum(torch.abs((pd_tsdf[near] - gt_tsdf[near]) / voxel_size))
    l_empty = torch.sum(EMPTY_SPACE_WEIGHT * torch.exp(pd[empty] / (2.0 * voxel_size)))
    return l_near, l_empty, q.shape[0]


def neural_field(net, feat, dec_svh: SparseFeatureHierarchy):
    """the output field of geometry='neural' (models/nksr_net.py:114-119): the SDF decoder over the basis features of
    every level, with its position gradient; differentiable in both when grad is enabled.  The interpolators and the
    normal features are not used."""
    return NeuralField(dec_svh, net.sdf_decoder, feat.basis_features, position_gradient=True)


def kernel_losses(net, scene: TrainingScene, generator=None, feat=None, dec_svh=None, timer=None, operator=None):
    """the field losses of a trainable NKSRNetwork on the scene: dict(total, gt_value, gt_normal, spatial, field), on
    the KernelField (kernel_field), or with geometry='neural' on the NeuralField (neural_field, no solve).  `feat`,
    `dec_svh`: an existing forward of the network (else one is run).  With ground truth geometry (scene.gt) the dict
    also holds spatial_empty, the empty-space term's share of spatial.  `operator`: the kernel solve's (kernel_field)."""
    if feat is None:
        enc = net.encoder(scene.xyz, scene.normal, scene.enc_svh, 0)
        feat, dec_svh, _ = net.unet(enc, scene.enc_svh, adaptive_depth=scene.adaptive_depth)
    if getattr(net, "geometry", "kernel") == "neural":
        field = neural_field(net, feat, dec_svh)
    else:
        field = kernel_field(net, feat, dec_svh, scene, timer, operator)
    l_val, l_nrm = gt_surface_loss(field, scene.ref_xyz, scene.ref_normal, generator=generator)
    extra = {}
    if scene.gt is None:
        l_sp = spatial_loss(field, scene.xyz, scene.normal, scene.voxel_size, generator=generator)
    else:
        near, empty, n = spatial_volume_terms(field, scene.ref_xyz, scene.ref_normal, scene.voxel_size, scene.gt,
                                              generator=generator)
        l_sp = (near + empty) / n
        extra["spatial_empty"] = empty / n
    total = GT_SURFACE_VALUE_WEIGHT * l_val + GT_SURFACE_NORMAL_WEIGHT * l_nrm + SPATIAL_WEIGHT * l_sp
    return dict(total=total, gt_value=l_val, gt_normal=l_nrm, spatial=l_sp, **extra, field=field)


def use_predicted_structure(pd_structure_prob, generator=None):
    """whether this step grows the decoder from the network's own structure prediction instead of teacher forcing
    (the reference's should_use_pd_structure, models/nksr_net.py:218-226): never for a probability <= 0, always for
    >= 1, else a draw from `generator` (only then is one consumed, so that the default keeps every random stream as
    it was)"""
    p = float(pd_structure_prob)
    if p <= 0.0:
        return False
    if p >= 1.0:
        return True
    dev = generator.device if generator is not None else "cpu"
    return bool(torch.rand((1,), generator=generator, device=dev).item() < p)


def losses(net, scene: TrainingScene, generator=None, kernel=False, timer=None, pd_structure_prob=0.0, operator=None):
    """forward of a trainable NKSRNetwork on the scene and its weighted losses: (total, structure, udf), and with
    `kernel` the kernel_losses dict as a fourth element (its total is included in the first).  The structure and UDF
    losses live on the third hierarchy unet() returns: the encoder hierarchy for structure='encoder', the grown one for
    structure='predicted' -- teacher-forced from the scene's ground truth, or grown from the prediction with
    probability `pd_structure_prob`.  `operator`: the kernel solve's (kernel_field)."""
    enc = net.encoder(scene.xyz, scene.normal, scene.enc_svh, 0)
    if getattr(net, "structure", "encoder") == "predicted":
        gt_dec = None if use_predicted_structure(pd_structure_prob, generator) else scene.gt_svh
        feat, dec_svh, udf_svh = net.unet(enc, scene.enc_svh, adaptive_depth=scene.adaptive_depth,
                                          gt_decoder_svh=gt_dec)
    else:
        feat, dec_svh, udf_svh = net.unet(enc, scene.enc_svh, adaptive_depth=scene.adaptive_depth)
    l_struct, _ = structure_loss(feat.structure_features, udf_svh, scene.gt_svh)
    loss_fn = udf_field_loss if getattr(net, "udf_enabled", False) else udf_loss
    l_udf = loss_fn(net.udf_decoder, feat.udf_features, udf_svh, scene.ref_xyz, scene.ref_normal, scene.voxel_size,
                    generator=generator, gt=scene.gt)
    total = STRUCTURE_WEIGHT * l_struct + UDF_WEIGHT * l_udf
    if not kernel:
        return total, l_struct, l_udf
    k = kernel_losses(net, scene, generator, feat, dec_svh, timer, operator)
    return total + k["total"], l_struct, l_udf, k


GRAD_CLIP = 0.5         # configs/default/train.yaml: grad_clip
LEARNING_RATE = 1e-4    # configs/default/train.yaml: learning_rate.init


def make_optimizer(net):
    return torch.optim.Adam([p for p in net.parameters() if p.requires_grad], lr=LEARNING_RATE)


def train_step(net, opt, scene: TrainingScene, generator=None, marks=None, kernel=False, timer=None,
               pd_structure_prob=0.0, operator=None):
    """one Adam step (gradient norm clipped to GRAD_CLIP); returns the (structure, udf) losses as tensors, and with
    `kernel` (the kernel-field losses added, trained through the kernel solve) a third element: the dict of the
    detached kernel losses.  `marks`, if given, is called with 'forward' / 'backward' / 'step' after each phase has
    been enqueued; `timer` (a StageTimer) receives the kernel solve's stage marks.  `pd_structure_prob`: see
    `losses` (structure='predicted' only).  `operator` ('assembled' or 'matrix_free'): the kernel solve's operator
    (kernel_field); None keeps the field's own choice, which assembles for a grad-recording solve."""
    opt.zero_grad(set_to_none=True)
    out = losses(net, scene, generator, kernel, timer, pd_structure_prob, operator)
    total, l_struct, l_udf = out[:3]
    if marks:
        marks("forward")
    total.backward()
    if marks:
        marks("backward")
    torch.nn.utils.clip_grad_norm_([p for p in net.parameters() if p.requires_grad], GRAD_CLIP)
    opt.step()
    if marks:
        marks("step")
    if kernel:
        k = {key: v.detach() for key, v in out[3].items() if key != "field"}
        return l_struct.detach(), l_udf.detach(), k
    return l_struct.detach(), l_udf.detach()
