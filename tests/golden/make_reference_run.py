"""Records what the unmodified reference computes for the checks of tests/test_reference_live.py: PathIndex, edge_to_affinity,
propagate_to_edge and AffinityDisplacementLoss.to_affinity on small seeded inputs -> tests/golden/reference_run.npz.

    IRN_REFERENCE=<reference checkout> python tests/golden/make_reference_run.py
"""
import hashlib
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import make_golden as mg  # noqa: E402
from irn_b200 import synth  # noqa: E402
from oracle import refshim  # noqa: E402


def main():
    refshim.install()
    os.chdir(refshim.REF)
    from misc import indexing as ref_indexing
    from net import resnet50_irn as ref_irn
    out = {}
    out["path_sha"] = mg.sha_path_index(ref_indexing.PathIndex(5, (21, 26)))
    h, w, r = 12, 17, 5
    edge = synth.edge_map(h, w, "uniform", 7)
    pi = ref_indexing.PathIndex(r, (h + r, w + 2 * r))
    ep = torch.nn.functional.pad(torch.from_numpy(edge), (r, r, 0, r), value=1.0)
    out["aff_sha"] = hashlib.sha256(np.ascontiguousarray(ref_indexing.edge_to_affinity(ep[None], pi.path_indices).numpy()).tobytes()).hexdigest()
    name, hh, ww, C, et, kind, seed = mg.RW_CASES[1]
    with torch.no_grad():
        rw = ref_indexing.propagate_to_edge(torch.from_numpy(synth.seeds(C, hh, ww, seed)), torch.from_numpy(synth.edge_map(hh, ww, kind, seed)),
                                            radius=5, beta=10, exp_times=et).numpy().astype(np.float32)
    out["rw_name"] = name
    out["rw"] = rw
    # AffinityDisplacementLoss.to_affinity, forward and autograd gradient, case "r5" of make_golden.gen_to_affinity
    r, h, w, B, kind, seed = 5, 24, 31, 3, "uniform", 5
    pi = ref_indexing.PathIndex(r, (h, w))
    stub = types.SimpleNamespace(n_path_lengths=len(pi.path_indices),
                                 _buffers={ref_irn.AffinityDisplacementLoss.path_indices_prefix + str(i): torch.from_numpy(p) for i, p in enumerate(pi.path_indices)})
    e = torch.from_numpy(np.stack([synth.edge_map(h, w, kind, seed + b) for b in range(B)])).requires_grad_(True)
    aff = ref_irn.AffinityDisplacementLoss.to_affinity(stub, e)
    aff.backward(torch.from_numpy(np.random.RandomState(seed).standard_normal(tuple(aff.shape)).astype(np.float32)))
    out["toaff_sha"] = hashlib.sha256(np.ascontiguousarray(aff.detach().numpy()).tobytes()).hexdigest()
    out["toaff_grad"] = e.grad.numpy()
    np.savez_compressed(os.path.join(HERE, "reference_run.npz"), **{k: np.asarray(v) for k, v in out.items()})


if __name__ == "__main__":
    main()
