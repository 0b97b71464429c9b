"""prep_metrics_list's host side, without a GPU: APData.add's ground-truth checks and fp32 box scaling (_gt_image), and
the staging buffer every image's ground truth goes to the device in (_gt_layout / _fill_gt): the packed words of each
image's padded mask rows must be that image's YB_MASK_BITS block."""
import numpy as np
import pytest
import torch

from yolact_b200.metrics import _fill_gt, _gt_image, _gt_layout


def _image(r, g_all, h, w, num_crowd, dtype=np.float32):
    gt = np.zeros((g_all, 5), np.float32)
    gt[:, :4] = np.sort(r.rand(g_all, 4).astype(np.float32), 1)[:, [0, 1, 2, 3]]
    gt[:, 4] = r.randint(0, 80, g_all)
    masks = r.rand(g_all, h, w)
    masks[masks < 0.3] = 0.5   # exactly 0.5 is not set
    masks = masks.astype(dtype) if dtype != np.uint8 else (masks > 0.5).astype(np.uint8) * r.randint(1, 4)
    return gt, masks


def _rows_bits(masks, h, w):
    """Reference YB_MASK_BITS words of [g,h,w] masks (value > 0.5 after the fp32 conversion)."""
    m = np.asarray(masks).astype(np.float32) > 0.5
    wpr = (w + 31) // 32
    pad = np.zeros(m.shape[:2] + (32 * wpr,), bool)
    pad[:, :, :w] = m
    return np.packbits(pad.reshape(-1, 32), axis=1, bitorder="little").view(np.uint32).reshape(-1)


def test_layout_and_fill_pack_to_each_images_bit_block():
    r = np.random.RandomState(3)
    specs = [(3, 5, 31, 1), (0, 7, 9, 0), (2, 1, 1, 2), (4, 6, 33, 0), (1, 4, 32, 0), (2, 3, 70, 1)]
    images, raw = [], []
    for i, (g_all, h, w, nc) in enumerate(specs):
        gt, masks = _image(r, g_all, h, w, nc, (np.float32, np.float64, np.uint8)[i % 3])
        images.append(_gt_image(gt, masks, h, w, nc, 80, "t"))
        raw.append((gt, masks, h, w))
    lay = _gt_layout(images)
    assert lay.cls_at % 16 == 0 and lay.mask_at % 16 == 0
    buf = torch.full((lay.nbytes,), 0xAB, dtype=torch.uint8)
    assert _fill_gt(buf, images, lay) == []
    buf = buf.numpy()
    G = sum(s[0] for s in specs)
    boxes = buf[lay.box_at:lay.box_at + 16 * G].view(np.float32).reshape(G, 4)
    cls = buf[lay.cls_at:lay.cls_at + 4 * G].view(np.int32)
    masks_u8 = buf[lay.mask_at:]
    assert len(masks_u8) % 32 == 0
    words = np.packbits(masks_u8.reshape(-1, 32) != 0, axis=1, bitorder="little").view(np.uint32).reshape(-1)
    for j, (gt, masks, h, w) in enumerate(raw):
        g_all = gt.shape[0]
        rr, wd = lay.rows[j], lay.words[j]
        want = gt[:, :4].astype(np.float32) * np.array([w, h, w, h], np.float32)
        assert np.array_equal(boxes[rr:rr + g_all].view(np.uint32), want.view(np.uint32))
        assert np.array_equal(cls[rr:rr + g_all], gt[:, 4].astype(np.int32))
        n_words = g_all * h * ((w + 31) // 32)
        assert np.array_equal(words[wd:wd + n_words], _rows_bits(masks, h, w))
    assert lay.words[-1] + specs[-1][0] * specs[-1][1] * 3 == len(words)


def test_scaled_boxes_are_fp32_products():
    gt = np.array([[0.1, 0.2, 0.7, 0.9, 3], [1 / 3, 0.5, 2 / 3, 0.75, 4]], np.float64)
    im = _gt_image(gt, np.zeros((2, 17, 29), np.float32), 17, 29, 1, 80, "t")
    want = gt[:, :4].astype(np.float32)
    want[:, [0, 2]] *= np.float32(29)
    want[:, [1, 3]] *= np.float32(17)
    assert im.boxes.dtype == np.float32 and np.array_equal(im.boxes, want)
    assert im.cls.tolist() == [3, 4] and im.g_all == 2 and im.num_crowd == 1


def test_ground_truth_refusals():
    gm = np.zeros((2, 4, 4), np.float32)
    gt = np.array([[0, 0, 0.5, 0.5, 1], [0, 0, 1, 1, 2]], np.float32)
    for bad in (dict(num_crowd=3), dict(num_crowd=-1), dict(gt=np.array([[0, 0, 1, 1, 80], [0, 0, 1, 1, 1]], np.float32)),
                dict(gt=np.array([[0, 0, 1, 1, -1], [0, 0, 1, 1, 1]], np.float32)), dict(gm=np.zeros((2, 4, 5))),
                dict(gm=np.zeros((3, 4, 4)))):
        with pytest.raises(ValueError):
            _gt_image(bad.get("gt", gt), bad.get("gm", gm), 4, 4, bad.get("num_crowd", 0), 80, "t")
    # a crowd's class is not checked (APData.add checks the first g rows only); no ground truth at all is fine
    _gt_image(np.array([[0, 0, 1, 1, 1], [0, 0, 1, 1, 99]], np.float32), gm, 4, 4, 1, 80, "t")
    assert _gt_image(np.zeros((0, 5), np.float32), None, 4, 4, 0, 80, "t").g_all == 0
