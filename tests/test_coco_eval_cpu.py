"""COCO instance evaluation without a GPU: the cocoeval protocol on hand-computable cases, the oracle rasteriser on cases that follow
from its stated rule, make_cocoann's file, and the driver flags."""
import json
import os
import types

import numpy as np
import pytest

from irn_b200.coco import cocoeval as ce
from irn_b200.coco import mask as cmask
from oracle import coco_mask as ocm


def _im(image_id, gts, dts, inter):
    """gts [(cat, json area, crowd, pixel count)], dts [(cat, score, pixel count)]."""
    g = list(zip(*gts)) if gts else [[], [], [], []]
    d = list(zip(*dts)) if dts else [[], [], []]
    return ce.ImageEval(image_id, g[0], g[1], g[2], g[3], d[0], d[1], d[2], np.asarray(inter, np.int64).reshape(len(dts), len(gts)))


def _stats(images, n_cat=1):
    return dict(zip(ce.STAT_NAMES, ce.evaluate(images, n_cat)["stats"]))


def _close(a, b):
    return abs(a - b) < 1e-12


def test_thresholds():
    assert ce.IOU_THRS[8] == 0.8999999999999999 and ce.IOU_THRS[2] == 0.6 and len(ce.REC_THRS) == 101


def test_perfect_match_is_one_everywhere_it_is_defined():
    s = _stats([_im(1, [(0, 2000.0, False, 2000)], [(0, 0.9, 2000)], [[2000]])])
    for k in ("AP", "AP50", "AP75", "APm", "AR1", "AR10", "AR100", "ARm"):
        assert _close(s[k], 1.0), k
    for k in ("APs", "APl", "ARs", "ARl"):      # no ground truth of that size
        assert s[k] == -1, k


@pytest.mark.parametrize("inter,area_d,area_g,n_met", [(6, 8, 8, 3), (3, 4, 4, 3), (9, 9, 10, 9)])
def test_iou_exactly_at_a_threshold_meets_it(inter, area_d, area_g, n_met):
    """6/10 and 3/5 meet 0.6 (the third threshold); 9/10 meets linspace's 0.8999999999999999 (the ninth)."""
    s = _stats([_im(1, [(0, 5000.0, False, area_g)], [(0, 0.9, area_d)], [[inter]])])
    assert _close(s["AP50"], 1.0)
    assert _close(s["AP"], n_met / 10)


def test_iou_06_gives_ap50_1_ap75_0_ap_03():
    s = _stats([_im(1, [(0, 5000.0, False, 8)], [(0, 0.9, 8)], [[6]])])
    assert _close(s["AP50"], 1.0) and s["AP75"] == 0.0 and _close(s["AP"], 0.3)


def test_detection_on_a_crowd_region_is_neither_tp_nor_fp():
    # det 0 (the higher score) lies inside the crowd region: IoU = inter / area_d = 1, matched to an ignored ground truth
    im = _im(1, [(0, 2000.0, False, 2000), (0, 10000.0, True, 10000)], [(0, 0.95, 100), (0, 0.9, 2000)], [[0, 100], [2000, 0]])
    s = _stats([im])
    assert _close(s["AP"], 1.0) and _close(s["AR100"], 1.0)
    # the same region without the crowd flag: IoU 0.01, so the first detection is a false positive and the region a miss
    im = _im(1, [(0, 2000.0, False, 2000), (0, 10000.0, False, 10000)], [(0, 0.95, 100), (0, 0.9, 2000)], [[0, 100], [2000, 0]])
    s = _stats([im])
    assert _close(s["AR100"], 0.5) and s["AP"] < 0.5


def test_area_ranges_ignore_ground_truth_and_detections():
    # a small ground truth matched by the lower score; the higher score is an unmatched medium-sized detection
    im = _im(1, [(0, 500.0, False, 500)], [(0, 0.95, 5000), (0, 0.9, 500)], [[0], [500]])
    s = _stats([im])
    assert _close(s["AP"], 0.5)             # all: the false positive ranks first
    assert _close(s["APs"], 1.0)            # small: the medium detection is unmatched and outside the range, so ignored
    assert s["APm"] == -1 and s["APl"] == -1    # no ground truth of those sizes
    # the ground truth's JSON area chooses its range, not its pixel count
    s = _stats([_im(1, [(0, 5000.0, False, 500)], [(0, 0.9, 500)], [[500]])])
    assert _close(s["APm"], 1.0) and s["APs"] == -1


def test_max_dets_truncation():
    im = _im(1, [(0, 2000.0, False, 2000), (0, 3000.0, False, 3000)], [(0, 0.9, 2000), (0, 0.8, 3000)], [[2000, 0], [0, 3000]])
    s = _stats([im])
    assert _close(s["AR1"], 0.5) and _close(s["AR10"], 1.0) and _close(s["AR100"], 1.0)
    # 100 false positives above the only match: the match is cut at 100 detections
    dts = [(0, 0.99 - 1e-4 * i, 50) for i in range(100)] + [(0, 0.1, 2000)]
    inter = [[0]] * 100 + [[2000]]
    s = _stats([_im(1, [(0, 2000.0, False, 2000)], dts, inter)])
    assert s["AR100"] == 0.0 and s["AP"] == 0.0


def test_two_images_with_interleaved_scores_follow_the_precision_envelope():
    a = _im(1, [(0, 2000.0, False, 2000)], [(0, 0.9, 2000), (0, 0.6, 2000)], [[2000], [0]])
    b = _im(2, [(0, 2000.0, False, 2000)], [(0, 0.8, 2000), (0, 0.7, 2000)], [[0], [2000]])
    # ranked TP FP TP FP: recall .5 .5 1 1, precision 1 .5 2/3 .5 -> envelope 1 2/3 2/3 .5; recall thresholds <= .5 sample index 0
    r = ce.REC_THRS
    want = (np.sum(r <= 0.5) * 1.0 + np.sum(r > 0.5) * (2 / 3)) / len(r)
    for order in ([a, b], [b, a]):      # images are taken in ascending image id whatever the input order
        s = _stats(order)
        assert abs(s["AP50"] - want) < 1e-12
        assert _close(s["AR100"], 1.0)


def test_category_without_ground_truth_is_minus_one_and_left_out():
    im = _im(1, [(0, 2000.0, False, 2000)], [(0, 0.9, 2000), (1, 0.8, 500)], [[2000], [0]])
    res = ce.evaluate([im], 2)
    assert (res["precision"][:, :, 1] == -1).all() and (res["recall"][:, 1] == -1).all()
    assert _close(res["stats"][0], 1.0)


def test_equal_iou_later_ground_truth_wins():
    im = _im(1, [(0, 2000.0, False, 100), (0, 2000.0, False, 100)], [(0, 0.9, 100), (0, 0.8, 100)], [[80, 80], [80, 80]])
    e = ce.evaluate_img(im, 0, ce.AREA_RNG[0])
    # IoU 80/120 = 2/3 with both: the first detection takes the later ground truth, the second the earlier one
    assert e["dt_matched"][0].all() and e["dt_matched"][1].all()


# ---------------------------------------------------------------------------------------------------------------- oracle rasteriser
def test_rle_decode_inverts_make_cocoann_encode():
    rng = np.random.RandomState(0)
    for h, w in ((1, 1), (1, 7), (9, 1), (13, 17), (40, 33)):
        for p in (0.0, 0.1, 0.5, 1.0):
            m = rng.rand(h, w) < p
            rle = cmask.rle_encode(m)
            assert rle["size"] == [h, w] and sum(rle["counts"]) == h * w
            assert np.array_equal(ocm.rle_decode(rle), m)
            assert cmask.rle_area(rle) == int(m.sum())


def _rect(x0, y0, x1, y1):
    return [x0, y0, x1, y0, x1, y1, x0, y1]


def test_polygon_integral_rectangle_is_half_open():
    m = ocm.ann_mask([_rect(2, 3, 6, 8)], 10, 12)
    want = np.zeros((10, 12), bool)
    want[3:8, 2:6] = True
    assert np.array_equal(m, want)


def test_polygon_half_integral_rectangle_rounds_up():
    m = ocm.ann_mask([_rect(2.5, 3.5, 6.5, 8.5)], 10, 12)
    want = np.zeros((10, 12), bool)
    want[4:9, 3:7] = True
    assert np.array_equal(m, want)


def test_polygon_triangle_lies_in_its_box():
    m = ocm.ann_mask([[0, 0, 8, 0, 0, 8]], 10, 10)
    box = np.zeros((10, 10), bool)
    box[0:8, 0:8] = True
    assert not (m & ~box).any() and 24 <= m.sum() <= 40
    assert m[0, 0] and m[0, 6] and m[6, 0] and not m[7, 7]


def test_polygon_vertices_outside_and_slightly_negative():
    m = ocm.ann_mask([_rect(-3, -0.2, 20, 4)], 10, 12)
    want = np.zeros((10, 12), bool)
    want[0:4, :] = True
    assert np.array_equal(m, want)


@pytest.mark.parametrize("poly", [[], [3, 3], [1, 1, 5, 5], [1, 1, 5, 5, 7]])
def test_polygon_of_fewer_than_three_points_is_empty(poly):
    assert not ocm.ann_mask([poly], 10, 12).any()


def test_several_polygons_are_a_union():
    m = ocm.ann_mask([_rect(1, 1, 6, 6), _rect(4, 4, 9, 8)], 10, 12)
    want = np.zeros((10, 12), bool)
    want[1:6, 1:6] = True
    want[4:8, 4:9] = True
    assert np.array_equal(m, want)


@pytest.mark.parametrize("segm", [{"counts": "PPYo0", "size": [10, 12]}, {"size": [10, 12]}, 7])
def test_unsupported_segmentation_raises_naming_the_annotation(segm):
    with pytest.raises(ValueError, match="annotation 4242"):
        ocm.ann_mask(segm, 10, 12, 4242)
    with pytest.raises(ValueError, match="annotation 4242"):
        cmask.segmentation_parts(segm, 10, 12, 4242)


def test_pack_layout():
    m = np.zeros((33, 2), bool)
    m[0, 0] = m[31, 0] = m[32, 0] = m[5, 1] = True
    assert ocm.pack(m).tolist() == [1 | (1 << 31), 1, 1 << 5, 0]


# ---------------------------------------------------------------------------------------------------------------- make_cocoann
def test_rle_bbox_and_area_follow_to_bbox():
    m = np.zeros((6, 8), bool)
    m[2:5, 3:6] = True
    r = cmask.rle_encode(m)
    assert cmask.rle_bbox(r) == [3.0, 2.0, 3.0, 3.0] and cmask.rle_area(r) == 9
    m = np.zeros((6, 8), bool)
    m[5, 2] = m[0, 3] = True        # one run that continues into the next column: the box spans every row
    assert cmask.rle_bbox(cmask.rle_encode(m)) == [2.0, 0.0, 2.0, 6.0]
    assert cmask.rle_bbox(cmask.rle_encode(np.zeros((6, 8), bool))) == [0.0, 0.0, 0.0, 0.0]


def _coco_instances(tmp_path):
    inst = {"images": [{"id": 11, "file_name": "COCO_a_000000000011.jpg", "height": 6, "width": 8},
                       {"id": 5, "file_name": "COCO_a_000000000005.jpg", "height": 4, "width": 5}],
            "annotations": [], "categories": [{"id": 7, "name": "c"}, {"id": 1, "name": "a"}, {"id": 3, "name": "b"}]}
    p = tmp_path / "instances_a.json"
    p.write_text(json.dumps(inst))
    (tmp_path / "list.txt").write_text("a/COCO_a_000000000011\na/COCO_a_000000000005\n")
    return p


def test_make_cocoann_coco_file(tmp_path):
    from irn_b200.step import make_cocoann
    inst = _coco_instances(tmp_path)
    os.makedirs(tmp_path / "ins")
    m0 = np.zeros((3, 6, 8), bool)
    m0[0, 1:3, 1:4] = True
    m0[1, 4, :] = True
    m0[2, 0, 0] = True
    np.save(tmp_path / "ins" / "COCO_a_000000000011.npy", {"score": np.array([0.9, 1e-6, 0.5]), "mask": m0, "class": np.array([2, 0, 1])})
    m1 = np.ones((1, 4, 5), bool)
    np.save(tmp_path / "ins" / "COCO_a_000000000005.npy", {"score": np.array([0.7]), "mask": m1, "class": np.array([0])})
    args = types.SimpleNamespace(dataset="coco", coco_instances=str(inst), infer_list=str(tmp_path / "list.txt"),
                                 ins_seg_out_dir=str(tmp_path / "ins"), cocoann_out=str(tmp_path / "out" / "ann.json"))
    make_cocoann.run(args)
    coco = json.loads((tmp_path / "out" / "ann.json").read_text())
    assert sorted(coco) == ["annotations", "categories", "images", "type"] and coco["type"] == "instances"
    assert [im["id"] for im in coco["images"]] == [11, 5]
    assert [(im["height"], im["width"]) for im in coco["images"]] == [(6, 8), (4, 5)]
    assert [c["id"] for c in coco["categories"]] == [1, 3, 7]
    anns = coco["annotations"]
    assert [a["id"] for a in anns] == [1, 2, 3]                 # unique over the file; the 1e-6 score is skipped
    assert [a["image_id"] for a in anns] == [11, 11, 5]
    assert [a["category_id"] for a in anns] == [7, 3, 1]        # class k -> the k-th category id
    assert all(a["iscrowd"] == 0 for a in anns)
    assert anns[0]["area"] == 6 and anns[0]["bbox"] == [1.0, 1.0, 3.0, 2.0]
    assert anns[2]["area"] == 20 and anns[2]["bbox"] == [0.0, 0.0, 5.0, 4.0]
    assert np.array_equal(ocm.rle_decode(anns[1]["segmentation"]), m0[2])


def test_make_cocoann_voc_categories_and_ids(tmp_path):
    from irn_b200.step import make_cocoann
    os.makedirs(tmp_path / "ins")
    m = np.zeros((2, 4, 5), bool)
    m[0, 1, 1] = m[1, 2, 2] = True
    np.save(tmp_path / "ins" / "2007_000032.npy", {"score": np.array([0.5, 0.4]), "mask": m, "class": np.array([0, 19])})
    cats = [{"supercategory": "none", "id": k + 1, "name": c} for k, c in enumerate(make_cocoann.VOC_CATEGORIES)]
    coco = make_cocoann.annotation_file([("2007_000032", 2007000032, "2007_000032.jpg", 4, 5)], cats, list(range(1, 21)),
                                        str(tmp_path / "ins"))
    assert len(coco["categories"]) == 20 and coco["categories"][0]["name"] == "aeroplane"
    assert [a["category_id"] for a in coco["annotations"]] == [1, 20]
    assert coco["images"][0]["id"] == 2007000032


# ---------------------------------------------------------------------------------------------------------------- flags
def test_run_sample_runs_coco_eval_ins_seg_only_with_coco_instances(tmp_path):
    import run_sample
    a = run_sample.parse(["--dataset", "coco", "--coco_gt_dir", str(tmp_path)])
    assert a.coco_instances == "" and a.make_cocoann_pass is False and a.cocoann_out == "voc2012_train_custom.json"
    assert not run_sample._has_ground_truth(a, "eval_ins_seg")
    assert run_sample._has_ground_truth(a, "eval_sem_seg")
    inst = _coco_instances(tmp_path)
    a = run_sample.parse(["--dataset", "coco", "--coco_instances", str(inst)])
    assert run_sample._has_ground_truth(a, "eval_ins_seg") and not run_sample._has_ground_truth(a, "eval_sem_seg")
    assert run_sample.parse(["--make_cocoann_pass", "True"]).make_cocoann_pass is True


def test_category_index_is_shared():
    from irn_b200.coco import make_cls_labels
    from irn_b200.step import eval_ins_seg
    inst = {"images": [{"id": 1, "file_name": "x.jpg", "height": 2, "width": 2}], "categories": [{"id": 9}, {"id": 2}],
            "annotations": [{"id": 1, "image_id": 1, "category_id": 9, "segmentation": [], "area": 0}]}
    assert make_cls_labels.category_index(inst) == ([2, 9], {2: 0, 9: 1})
    n_cat, gt = eval_ins_seg.coco_ground_truth(inst, ["x"])
    assert n_cat == 2 and gt[0][2].tolist() == [1]
    with pytest.raises(KeyError, match="y"):
        eval_ins_seg.coco_ground_truth(inst, ["y"])
