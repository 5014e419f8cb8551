"""Host side of the ragged CRF (no device needed): workspace queries, chunking by per-image workspace, unpacking."""
import ctypes

import numpy as np
import torch

from irn_b200 import _lib, crf


def _ragged_bytes(sizes, groups, labels):
    hw = np.ascontiguousarray(np.asarray(sizes, np.int32).reshape(-1, 2))
    return _lib.lib().irn_crf_ragged_workspace_bytes(len(sizes), hw.ctypes.data_as(ctypes.c_void_p), groups, labels)


def test_ragged_workspace_of_equal_sizes_is_the_one_size_workspace():
    L = _lib.lib()
    for n, H, W, g, m in ((1, 1, 1, 1, 2), (3, 375, 500, 2, 4), (8, 640, 640, 2, 81)):
        assert _ragged_bytes([(H, W)] * n, g, m) == L.irn_crf_workspace_bytes(n, H, W, g, m) > 0
    # mixed sizes: at least the sum of the pixels' share, at most the per-image workspaces added up
    mixed = [(375, 500), (1, 1), (640, 427)]
    assert max(_ragged_bytes([s], 2, 7) for s in mixed) < _ragged_bytes(mixed, 2, 7) <= sum(_ragged_bytes([s], 2, 7) for s in mixed)


def test_workspace_query_is_zero_for_calls_that_are_refused():
    L = _lib.lib()
    assert _ragged_bytes([(10, 10), (0, 5)], 2, 3) == 0
    assert _ragged_bytes([(10, 10)], 3, 3) == 0
    assert _ragged_bytes([(10, 10)], 2, crf.max_labels() + 1) == 0
    assert L.irn_crf_ragged_workspace_bytes(1, None, 2, 3) == 0
    # 6 pairs per pixel past 2^31: the compute call refuses the batch, so the query gives no (partial) size
    assert L.irn_crf_workspace_bytes(1, 20000, 20000, 1, 2) == 0
    assert _ragged_bytes([(100, 100), (20000, 20000)], 1, 2) == 0
    assert L.irn_crf_workspace_bytes(1, 10000, 10000, 1, 2) > 0


def test_ragged_chunks_follow_the_workspace_bound_in_list_order():
    assert crf._ragged_chunks([5, 5, 5, 20, 1], 10) == [(0, 2), (2, 3), (3, 4), (4, 5)]
    assert crf._ragged_chunks([5, 5, 5], 100) == [(0, 3)]
    assert crf._ragged_chunks([50], 10) == [(0, 1)]


def test_unpack_splits_packed_results():
    sizes = [(2, 3), (1, 1), (4, 2)]
    flat = torch.arange(6 + 1 + 8)
    maps = crf.unpack(flat, sizes)
    assert [tuple(m.shape) for m in maps] == sizes and maps[2][3, 1].item() == 14
    q = torch.arange(2 * 15)
    qs = crf.unpack(q, sizes, 2)
    assert [tuple(m.shape) for m in qs] == [(2, 2, 3), (2, 1, 1), (2, 4, 2)] and qs[1].flatten().tolist() == [12, 13]
