"""Host-side checks that need no GPU: the C-ABI library loads, exports every symbol the header
declares, and its host-only entry points (PathIndex) are integer bit-exact."""
import hashlib
import json
import os
import re

import numpy as np
import pytest

from conftest import ROOT, golden_path


def test_header_symbols_exported(built_lib):
    from irn_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "irn_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(irn_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    assert declared == set(_lib.SIGNATURES), "ctypes table and header drifted: %s" % (declared ^ set(_lib.SIGNATURES))
    for name in declared:
        assert hasattr(built_lib, name)
    assert built_lib.irn_version() >= 100


PI = json.load(open(golden_path("path_index.json")))


@pytest.mark.parametrize("key", sorted(PI))
def test_path_index_abi_bit_exact(built_lib, key):
    from irn_b200.indexing import PathIndex
    g = PI[key]
    pi = PathIndex(g["radius"], tuple(g["size"]))
    assert pi.radius == g["radius"] and pi.radius_floor == g["radius"] - 1
    assert [list(p.shape) for p in pi.path_indices] == g["group_shapes"]
    assert pi.search_dst.tolist() == g["search_dst"]
    assert pi.src_indices[:5].tolist() == g["src_head"]
    h = hashlib.sha256()
    for p in pi.path_indices:
        assert p.dtype == np.int64
        h.update(np.ascontiguousarray(p).tobytes())
    h.update(pi.src_indices.tobytes())
    h.update(np.ascontiguousarray(pi.dst_indices).tobytes())
    h.update(np.ascontiguousarray(pi.search_dst).tobytes())
    assert h.hexdigest() == g["sha256"]


def test_path_index_matches_oracle_paths(built_lib):
    from irn_b200.indexing import PathIndex
    from oracle import indexing as oi
    for r in (2, 3, 5, 7):
        a, b = PathIndex(r, (3 * r + 2, 4 * r + 3)), oi.PathIndex(r, (3 * r + 2, 4 * r + 3))
        assert len(a.search_paths) == len(b.search_paths)
        for p, q in zip(a.search_paths, b.search_paths):
            assert np.array_equal(p, q)
        for p, q in zip(a.path_indices, b.path_indices):
            assert np.array_equal(p, q)


def test_errors_are_reported(built_lib):
    from irn_b200 import _lib
    rc = built_lib.irn_path_index_fill(5, 3, 3, None, None, None, None, None)   # grid too small
    assert rc == -1
    assert b"too small" in built_lib.irn_last_error()
    assert built_lib.irn_rw_workspace_bytes(0, 8, 8, 1, 5) == 0
    with pytest.raises(_lib.IrnError):
        _lib.check(rc, "irn_path_index_fill")


def test_walk_variant_refused_before_any_launch(built_lib):
    """irn_random_walk_variant checks the kernel choice on the host, before any CUDA call: an unknown variant is kBadArg (-1)
    and variant 2 (per-step TMA kernel, radius 5 only) at another radius is kUnsupported (-4).  The device pointers are
    dummies that are never dereferenced, so this runs without a GPU."""
    import ctypes
    offs = np.array([0, 2], dtype=np.int32)
    dummy = ctypes.c_void_p(0x100000)
    call = lambda variant, radius: built_lib.irn_random_walk_variant(dummy, dummy, dummy, 1, offs.ctypes.data, 16, 16, radius,
                                                                     10.0, 4, dummy, 1 << 20, variant, None)
    for variant in (3, 5, 7, -1):
        assert call(variant, 5) == -1
        assert built_lib.irn_rw_last_launch_count() == 0
        assert b"variant %d" % variant in built_lib.irn_last_error()
    assert call(2, 3) == -4
    assert built_lib.irn_rw_last_launch_count() == 0
    assert b"variant 2" in built_lib.irn_last_error() and b"radius 5" in built_lib.irn_last_error()


def test_device_entry_points_refuse_cpu_tensors(built_lib):
    import torch
    from irn_b200 import indexing, _lib
    with pytest.raises(_lib.IrnError):
        indexing.propagate_to_edge(torch.zeros(1, 8, 8), torch.zeros(1, 8, 8))


def test_to_affinity_refuses_cpu_tensors_and_bad_arguments(built_lib):
    """N4's differentiable op has no CPU path either; argument errors are raised before anything is launched."""
    import torch
    from irn_b200 import indexing, _lib
    with pytest.raises(_lib.IrnError):
        indexing.to_affinity(torch.zeros(1, 1, 12, 24), radius=5)
    with pytest.raises(_lib.IrnError):
        indexing.to_affinity(torch.zeros(1, 12, 24), indexing.PathIndex(5, (12, 24)))
