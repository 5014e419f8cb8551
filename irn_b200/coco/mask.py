"""COCO masks on the device (irn_b200/csrc/coco_mask.cu) and the RLE helpers of make_cocoann.

A batch's masks are bit planes (`plane_words(H, W)` uint32 words each; the layout is coco_mask.cu's) back to back in one device
tensor.  `rasterize` turns ground-truth segmentations (polygons or uncompressed RLE) into planes, `pack_masks` turns the steps' bool
prediction masks into planes, `overlaps` counts every prediction/ground-truth intersection and every mask's area of each image.  The
counts are exact integers, equal to oracle/coco_mask.py's."""
import ctypes

import numpy as np
import torch

from .. import _lib


def plane_words(h, w):
    n = int(_lib.lib().irn_coco_plane_words(int(h), int(w)))
    if n < 0:
        raise _lib.IrnError("bad mask size %sx%s" % (h, w))
    return n


def _host(a, dtype):
    a = np.ascontiguousarray(a, dtype)
    return a, a.ctypes.data_as(ctypes.c_void_p)


def segmentation_parts(segm, h, w, ann_id):
    """One annotation's segmentation -> list of parts: ("poly", float64 [k,2]) per polygon, or one ("rle", int64 toggle positions)."""
    if isinstance(segm, list):
        parts = []
        for p in segm:
            xy = np.asarray(p, np.float64).reshape(-1)
            parts.append(("poly", xy[:len(xy) // 2 * 2].reshape(-1, 2)))
        return parts
    if isinstance(segm, dict) and isinstance(segm.get("counts"), list) and "size" in segm:
        if [int(s) for s in segm["size"]] != [int(h), int(w)]:
            raise ValueError("annotation %s: RLE size %s, image %dx%d" % (ann_id, segm["size"], h, w))
        counts = np.asarray(segm["counts"], np.int64)
        if (counts < 0).any() or counts.sum() != h * w:
            raise ValueError("annotation %s: RLE counts add up to %d, image %dx%d" % (ann_id, counts.sum(), h, w))
        return [("rle", np.cumsum(counts)[:-1])]
    raise ValueError("annotation %s: unsupported segmentation %s (polygons or uncompressed RLE only)" %
                     (ann_id, type(segm.get("counts") if isinstance(segm, dict) else segm).__name__))


def rasterize(anns, device):
    """anns: [(h, w, segmentation, annotation id)] -> (planes uint32 [sum plane_words] on device, word offset of each plane int64 [n+1])."""
    L = _lib.lib()
    n = len(anns)
    hw = np.array([(int(a[0]), int(a[1])) for a in anns], np.int32).reshape(-1, 2)
    offs = np.concatenate([[0], np.cumsum([plane_words(h, w) for h, w in hw])]).astype(np.int64)
    part_ann, edges, verts, toggles = [], [], [], []
    nv = 0
    for i, (h, w, segm, ann_id) in enumerate(anns):
        for kind, data in segmentation_parts(segm, int(h), int(w), ann_id):
            p = len(part_ann)
            part_ann.append(i)
            if kind == "poly":
                k = len(data)
                if k:
                    edges.append(np.stack([np.full(k, p), np.full(k, nv), np.full(k, k), np.arange(k)], 1))
                    verts.append(data)
                    nv += k
            else:
                toggles.append(np.stack([np.full(len(data), p), data], 1))
    part_ann, pa_p = _host(part_ann, np.int32)
    part_hw = np.ascontiguousarray(hw[part_ann]) if len(part_ann) else np.zeros((0, 2), np.int32)
    edges, e_p = _host(np.concatenate(edges) if edges else np.zeros((0, 4)), np.int32)
    verts, v_p = _host(np.concatenate(verts) if verts else np.zeros((0, 2)), np.float64)
    toggles, t_p = _host(np.concatenate(toggles) if toggles else np.zeros((0, 2)), np.int32)
    hw_c, hw_p = _host(hw, np.int32)
    planes = torch.empty(int(offs[-1]), dtype=torch.int32, device=device)
    nb = L.irn_coco_raster_workspace_bytes(len(part_ann), part_hw.ctypes.data_as(ctypes.c_void_p), len(edges), len(verts), len(toggles))
    if nb == 0:
        raise _lib.IrnError("irn_coco_raster_workspace_bytes refused the batch")
    ws = torch.empty(nb, dtype=torch.uint8, device=device)
    with torch.cuda.device(device):
        _lib.check(L.irn_coco_rasterize(n, hw_p, len(part_ann), pa_p, len(edges), e_p, len(verts), v_p, len(toggles), t_p,
                                        _lib.ptr(planes), int(offs[-1]), _lib.ptr(ws), nb, _lib.stream_ptr()), "irn_coco_rasterize")
    return planes, offs


def pack_masks(masks_u8, hwm):
    """masks_u8: uint8 [sum M_i*H_i*W_i] on the device (image i's bool [M_i,H_i,W_i] back to back), hwm [(H_i, W_i, M_i)] -> planes
    uint32 [sum M_i * plane_words(H_i, W_i)] (stored as int32)."""
    _lib.require_cuda(masks_u8)
    L = _lib.lib()
    hwm, hwm_p = _host(np.asarray(hwm).reshape(-1, 3), np.int32)
    words = int(sum(int(m) * plane_words(h, w) for h, w, m in hwm))
    planes = torch.empty(words, dtype=torch.int32, device=masks_u8.device)
    nb = L.irn_coco_pack_workspace_bytes(len(hwm))
    ws = torch.empty(nb, dtype=torch.uint8, device=masks_u8.device)
    with torch.cuda.device(masks_u8.device):
        _lib.check(L.irn_coco_pack_masks(_lib.ptr(masks_u8), masks_u8.numel(), len(hwm), hwm_p, _lib.ptr(planes), words, _lib.ptr(ws), nb,
                                         _lib.stream_ptr()), "irn_coco_pack_masks")
    return planes


def overlaps(pred_planes, gt_planes, hwmg):
    """hwmg [(H_i, W_i, M_i, G_i)] -> per image (inter int32 [M_i,G_i], area_pred int32 [M_i], area_gt int32 [G_i]) on the host."""
    L = _lib.lib()
    dev = pred_planes.device
    hwmg, hp = _host(np.asarray(hwmg).reshape(-1, 4), np.int32)
    M, G = hwmg[:, 2].astype(np.int64), hwmg[:, 3].astype(np.int64)
    inter = torch.empty(int((M * G).sum()), dtype=torch.int32, device=dev)
    ap = torch.empty(int(M.sum()), dtype=torch.int32, device=dev)
    ag = torch.empty(int(G.sum()), dtype=torch.int32, device=dev)
    nb = L.irn_coco_overlap_workspace_bytes(len(hwmg), hp)
    if nb == 0:
        raise _lib.IrnError("irn_coco_overlap_workspace_bytes refused the batch %s" % hwmg.tolist())
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(L.irn_coco_overlaps(_lib.ptr(pred_planes), pred_planes.numel(), _lib.ptr(gt_planes), gt_planes.numel(), len(hwmg), hp,
                                       _lib.ptr(inter), _lib.ptr(ap), _lib.ptr(ag), _lib.ptr(ws), nb, _lib.stream_ptr()), "irn_coco_overlaps")
    inter, ap, ag = inter.cpu().numpy(), ap.cpu().numpy(), ag.cpu().numpy()
    out, io, po, go = [], 0, 0, 0
    for m, g in zip(M, G):
        out.append((inter[io:io + m * g].reshape(m, g), ap[po:po + m], ag[go:go + g]))
        io, po, go = io + m * g, po + m, go + g
    return out


# ---------------------------------------------------------------------------------------------------------------- RLE on the host
def rle_encode(mask):
    """bool [h,w] -> uncompressed RLE {"counts": [...], "size": [h, w]}: column-major runs, the first one of zeros (possibly 0 long)."""
    mask = np.asarray(mask, bool)
    flat = mask.ravel(order="F")
    change = np.flatnonzero(flat[1:] != flat[:-1]) + 1
    bounds = np.concatenate([[0], change, [flat.size]])
    counts = np.diff(bounds).tolist()
    if flat.size and flat[0]:
        counts = [0] + counts
    return {"counts": [int(c) for c in counts], "size": [int(mask.shape[0]), int(mask.shape[1])]}


def rle_area(rle):
    """pycocotools' area: the sum of the runs of ones."""
    return int(sum(rle["counts"][1::2]))


def rle_bbox(rle):
    """pycocotools' toBbox [x, y, w, h] (floats): the extent of the runs of ones, except that a run which continues into the next
    column makes the box span every row; [0, 0, 0, 0] for an empty mask."""
    h = int(rle["size"][0])
    c = np.asarray(rle["counts"], np.int64)
    m = len(c) // 2 * 2
    if m == 0:
        return [0.0, 0.0, 0.0, 0.0]
    cs = np.cumsum(c[:m])
    start, last = cs[0::2], cs[1::2] - 1
    xs_, xe_ = start // h, last // h
    ys, ye = int(min(start.min() % h, last.min() % h)), int(max(start.max() % h, last.max() % h))
    if (xs_ < xe_).any():
        ys, ye = 0, h - 1
    x0, x1 = int(min(xs_.min(), xe_.min())), int(max(xs_.max(), xe_.max()))
    return [float(x0), float(ys), float(x1 - x0 + 1), float(ye - ys + 1)]
