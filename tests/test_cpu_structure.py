"""The torch restatement of DESIGN.md SPEC S16 (the structure-grown decoder hierarchy, nksr_b200/structure.py,
impl='torch') on CPU tensors: the class rule (torch.argmax semantics), the growth invariants and teacher forcing on a
hierarchy built in torch.  The CUDA kernels are held to this restatement bit for bit in tests/test_gpu_structure.py."""
import math

import pytest
import torch

from nksr_b200 import structure as S


class _Hierarchy:
    """a parent-closed hierarchy in plain torch (the tables StructureGrowth reads from an encoder hierarchy)"""

    def __init__(self, fine_keys, depth):
        self.depth, self.voxel_size = depth, 0.1
        keys = [torch.unique(fine_keys >> (3 * l)) for l in range(depth)]
        self.keys = keys
        self.top_keys = torch.unique(keys[-1] >> 3)
        allk = keys + [self.top_keys]
        self.parent = [None] * (depth + 1)
        self.child8 = [None] * (depth + 1)
        self.nbr27 = [S.nbr27_torch(k) for k in allk]
        for l in range(depth):
            self.parent[l] = S._lookup(allk[l + 1], allk[l] >> 3)
            c8 = torch.full((allk[l + 1].numel(), 8), -1, dtype=torch.int32)
            c8[self.parent[l].long(), (allk[l] & 7)] = torch.arange(allk[l].numel(), dtype=torch.int32)
            self.child8[l + 1] = c8
        self.nbr125_top = None

    def num_voxels(self, l):
        return int(self.keys[l].numel())


def _cloud_keys(n=400, seed=0, extent=40):
    g = torch.Generator().manual_seed(seed)
    ijk = torch.randint(0, extent, (n, 3), generator=g) + (1 << 19)
    return torch.unique(S.morton_encode(ijk[:, 0], ijk[:, 1], ijk[:, 2]))


def test_morton_round_trip():
    g = torch.Generator().manual_seed(3)
    x, y, z = (torch.randint(0, 1 << 21, (1000,), generator=g) for _ in range(3))
    k = S.morton_encode(x, y, z)
    dx, dy, dz = S.morton_decode(k)
    assert torch.equal(dx, x) and torch.equal(dy, y) and torch.equal(dz, z)
    assert int(S.morton_encode(torch.tensor([1]), torch.tensor([0]), torch.tensor([0]))) == 4


def test_class_rule_follows_torch_argmax():
    nan = math.nan
    logits = torch.tensor([[0.0, 1.0, 1.0],      # tie between leaf and subdivide: the first wins
                           [2.0, 2.0, 2.0],      # three-way tie: empty
                           [nan, 5.0, 9.0],      # NaN counts as the largest value
                           [0.0, nan, nan],      # the first NaN
                           [0.0, 0.0, 3.0],
                           [-1.0, 0.5, 0.0]])
    want = torch.argmax(logits, dim=1)
    for level, a in [(0, 2), (1, 2), (2, 2), (3, 1)]:
        c, keep, sub = S.classify_torch(logits, level, a)
        assert torch.equal(c.long(), want)
        assert torch.equal(keep, want >= 1)
        exp_sub = ((want == 2) | ((want == 1) & (level >= a))) & (level >= 1)
        assert torch.equal(sub, exp_sub), (level, a)


def _grow(E, D, a, logits_for):
    g = S.StructureGrowth(E, D, a, max_ratio=None, impl="torch")
    for l in range(D - 1, -1, -1):
        g.step(l, logits=logits_for(l, g.T.num_voxels(l)))
    return g


@pytest.mark.parametrize("D,a", [(3, 1), (4, 2), (4, 3)])
def test_growth_invariants(D, a):
    E = _Hierarchy(_cloud_keys(), D)
    gen = torch.Generator().manual_seed(D * 10 + a)
    g = _grow(E, D, a, lambda l, n: torch.randn((n, 3), generator=gen) + torch.tensor([0.0, 0.3, 0.6]))
    T = g.T
    assert torch.equal(T.keys[D - 1], E.keys[D - 1])
    for l in range(D):
        k = T.keys[l]
        assert bool((k[1:] > k[:-1]).all())                                       # sorted and unique
        assert torch.equal(T.nbr27[l], S.nbr27_torch(k))
        assert torch.equal(g.join[l], S._lookup(E.keys[l], k))
        assert torch.equal(g.skip27(l).long(), torch.where(T.nbr27[l] >= 0, g.join[l].long()[T.nbr27[l].long().clamp(min=0)],
                                                           torch.full_like(T.nbr27[l].long(), -1)))
        assert torch.equal(g.kept[l], torch.nonzero(g.classes[l] >= 1).squeeze(1))
        if l < D - 1:
            assert torch.equal(k >> 3, T.keys[l + 1][T.parent[l].long()])        # parent-closed
            c8 = T.child8[l + 1]
            full = (c8 >= 0).all(dim=1)
            assert bool(((c8 >= 0).any(dim=1) == full).all())                      # rows are full or empty
            sub = (g.classes[l + 1] == 2) | ((g.classes[l + 1] == 1) & (l + 1 >= a))
            assert torch.equal(full, sub)
            assert k.numel() == 8 * int(sub.sum())
    # the kept voxels of every level hang under kept voxels
    for l in range(D - 1):
        kept_keys, up = T.keys[l][g.kept[l]], T.keys[l + 1][g.kept[l + 1]]
        assert bool(torch.isin(kept_keys >> 3, up).all())


def test_teacher_forcing_with_the_encoder_itself_gives_it_back():
    D, a = 4, 2
    E = _Hierarchy(_cloud_keys(seed=5), D)

    def status(T, l):                   # evaluate_voxel_status of E on T_l
        k = T.keys[l]
        pos = S._lookup(E.keys[l], k).long()
        st = (pos >= 0).long()
        if l > 0:
            has = (E.child8[l] >= 0).any(dim=1)
            st = torch.where((pos >= 0) & has[pos.clamp(min=0)], torch.full_like(st, 2), st)
        return st

    g = S.StructureGrowth(E, D, a, max_ratio=None, impl="torch")
    for l in range(D - 1, -1, -1):
        g.step(l, forced=status(g.T, l))
    for l in range(D):
        assert torch.equal(g.T.keys[l][g.kept[l]], E.keys[l])


def test_empty_level_empties_the_finer_ones():
    D = 3
    E = _Hierarchy(_cloud_keys(seed=2), D)
    g = _grow(E, D, 1, lambda l, n: torch.tensor([[1.0, 0.0, 0.0]]).expand(n, 3))
    for l in range(D - 1):
        assert g.T.num_voxels(l) == 0 and g.T.child8[l + 1].shape == (g.T.num_voxels(l + 1), 8)
        assert bool((g.T.child8[l + 1] < 0).all())
    assert all(g.kept[l].numel() == 0 for l in range(D))


def test_size_guard_names_the_level():
    D = 3
    E = _Hierarchy(_cloud_keys(seed=4), D)
    g = S.StructureGrowth(E, D, 1, max_ratio=1.0, impl="torch")
    from nksr_b200._lib import NksrError
    with pytest.raises(NksrError, match="level 1"):
        g.step(D - 1, logits=torch.tensor([[0.0, 0.0, 1.0]]).expand(E.num_voxels(D - 1), 3))


def test_predicted_structure_needs_the_unet_backbone():
    from nksr_b200.network import NKSRNetwork
    with pytest.raises(ValueError, match="backbone='unet'"):
        NKSRNetwork(dict(backbone="pool", structure="predicted"))
    with pytest.raises(ValueError):
        NKSRNetwork(dict(backbone="unet", structure="grown"))
    assert NKSRNetwork(dict(backbone="pool")).structure == "encoder"
