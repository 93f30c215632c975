"""Generates tests/golden/sdfgen/reference_outputs.npz: outputs of the reference's own GT-SDF generator
(ext.sdfgen.sdf_from_points of nv-tlabs/NKSR, built unmodified into oracle/_ref/ by oracle/Makefile.ref) on the inputs of tests/test_gpu_sdfgen.py.

Needs a GPU and oracle/_ref/nksr_sdfgen_ref.so (`NKSR_REFERENCE=<checkout> python -c "import __graft_entry__ as g;
g.build()"`).  Run from the repository root:  python tests/golden/make_sdfgen_golden.py [OUT.npz]

For every (case, argument set) a fixed, seeded sample of SAMPLE queries is kept: their indices, the query points
themselves (so that the test can tell its inputs are still the ones the reference saw), the signed distance and the
gradient.  Regenerate only when the test's inputs change on purpose.
"""
import importlib.util
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests.test_gpu_sdfgen import ARG_IDS, ARGS, CASES, _case  # noqa: E402

SAMPLE = 2500


def sample_indices(n_queries):
    return np.sort(np.random.default_rng(11).choice(n_queries, SAMPLE, replace=False)).astype(np.int32)


def main(out):
    import torch
    so = os.path.join(ROOT, "oracle", "_ref", "nksr_sdfgen_ref.so")
    spec = importlib.util.spec_from_file_location("nksr_sdfgen_ref", so)
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    data = {}
    for case in CASES:
        xyz, nrm, q = _case(case)
        idx = sample_indices(q.shape[0])
        for aid, kw in zip(ARG_IDS, ARGS):
            r = ref.sdf_from_points(t(q), t(xyz), t(nrm), kw["nb_points"], kw["stdv"], True, kw["imls"],
                                    kw["adaptive_knn"])
            key = f"{case}_{aid}"
            data[key + "_idx"] = idx
            data[key + "_q"] = q[idx]
            data[key + "_sdf"] = r[0].cpu().numpy()[idx].astype(np.float32)
            data[key + "_grad"] = r[1].cpu().numpy()[idx].astype(np.float32)
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    np.savez_compressed(out, **data)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    here = os.path.dirname(os.path.abspath(__file__))
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(here, "sdfgen", "reference_outputs.npz"))
