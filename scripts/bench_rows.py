"""Device times (CUDA events, warm-up, L2-sized inputs where it matters) of the section-8f row kernels at the
BASELINE shapes: FastBaseTransform, traditional NMS vs Fast NMS, bit-packed mask IoU, COCO RLE, display blend.
Prints a markdown table with algorithmic bytes and the fraction of the measured HBM peak."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import yolact_b200
from yolact_b200.config import CONFIGS
from yolact_b200.augmentations import FastBaseTransform
from yolact_b200.detection import Detect
from yolact_b200.eval_utils import mask_iou, mask_run_lengths, display_blend
from yolact_b200.output_utils import assemble_masks, _ops_handle
from yolact_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
peak = 3350.0   # H100 SXM data-sheet HBM3 bandwidth (GB/s) unless MEASURED_PEAKS.json says otherwise
try:
    pk = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    peak = float(pk.get("hbm_gbs", peak))
except Exception:
    pass


def timeit(fn, iters=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


rows = []
r = np.random.RandomState(0)
cfg = CONFIGS["yolact_base_config"].copy()
yolact_b200.cfg.replace(cfg.copy())

# FastBaseTransform: 8 frames 720p uint8 -> 550x550
frames = torch.from_numpy(r.randint(0, 256, size=(8, 720, 1280, 3)).astype(np.uint8)).cuda()
xf = FastBaseTransform(cfg)
ms = timeit(lambda: xf(frames))
by = 8 * (550 * 550 * 4 * 3 + 550 * 550 * 3 * 4)   # <= 4 source pixels x 3 B per output pixel (upper bound) + fp32 NCHW write
rows.append(("fast_base_transform 8x720p u8 -> 550^2", ms, by))
ms = timeit(lambda: xf(frames.float()))
rows.append(("fast_base_transform 8x720p f32 -> 550^2", ms, 8 * (550 * 550 * 16 * 3 + 550 * 550 * 12)))

# Detect at P = 19248, B = 8: fast vs traditional
P, C = 19248, 81
pri = torch.from_numpy(np.concatenate([r.uniform(0.05, 0.95, (P, 2)), r.uniform(0.03, 0.4, (P, 2))], 1).astype(np.float32)).cuda()
loc = torch.from_numpy(r.standard_normal((8, P, 4)).astype(np.float32)).cuda()
logits = (r.standard_normal((8, P, C)) * 2.0).astype(np.float32)
logits[:, :, 0] += 3.0
hot = r.rand(8, P) < 0.1
cls = r.randint(1, C, size=(8, P))
for b in range(8):
    idx = np.nonzero(hot[b])[0]
    logits[b, idx, cls[b, idx]] += r.uniform(2.0, 9.0, size=idx.size).astype(np.float32)
conf = torch.softmax(torch.from_numpy(logits), -1).cuda()
coef = torch.from_numpy(np.tanh(r.standard_normal((8, P, 32))).astype(np.float32)).cuda()
for name, fast in (("detect fast_nms B=8 P=19248", True), ("detect traditional_nms B=8 P=19248", False)):
    d = Detect(C, 0, 200, 0.05, 0.5, cfg=cfg)
    d.use_fast_nms = fast
    ms = timeit(lambda: d.detect_padded(loc, conf, coef, pri))
    rows.append((name, ms, 8 * P * (C * 4 + 16 + 16)))

# masks: 100 detections at 550x550, bit-packed
proto = torch.from_numpy(np.maximum(r.standard_normal((138, 138, 32)), 0).astype(np.float32)).cuda()
cf = torch.from_numpy(np.tanh(r.standard_normal((100, 32))).astype(np.float32)).cuda()
c = r.uniform(0.2, 0.8, (100, 2)); wh = r.uniform(0.1, 0.5, (100, 2))
bx = torch.from_numpy(np.concatenate([c - wh / 2, c + wh / 2], 1).astype(np.float32)).cuda()
bits, _, _ = assemble_masks(proto, cf, bx, 550, 550, True, "bits")
gt = bits[:20].clone()
words = bits[0].numel()
ms = timeit(lambda: mask_iou(bits, gt, packed=True))
rows.append(("mask_iou 100x20 @550^2 (bits)", ms, 100 * 20 * 2 * words * 4))
ms = timeit(lambda: mask_run_lengths(bits, "bits", w=550), iters=5)
rows.append(("mask_rle 100 @550^2 (bits, incl. D2H of runs)", ms, 100 * words * 4 * 2))
lib = _lib.load()
counts = torch.empty(100, 4 * 550 + 64, dtype=torch.int32, device="cuda"); nr = torch.empty(100, dtype=torch.int32, device="cuda")
def rle_only():
    _lib.check(lib.yb_mask_rle(_ops_handle(bits.device), _lib.ptr(bits), _lib.YB_MASK_BITS, 100, 550, 550, _lib.ptr(counts),
                               counts.shape[1], _lib.ptr(nr), _lib.current_stream(bits.device)), "rle")
ms = timeit(rle_only)
rows.append(("mask_rle 100 @550^2 (kernel only)", ms, 100 * words * 4 * 2))
frame = torch.from_numpy(r.randint(0, 256, size=(550, 550, 3)).astype(np.float32)).cuda()
cols = r.uniform(0, 1, (15, 3)).astype(np.float32)
ms = timeit(lambda: display_blend(frame, bits[:15], cols, 0.45, w=550))
rows.append(("display_blend 15 masks @550^2 (bits)", ms, 550 * 550 * (12 + 3) + 15 * words * 4))

print("# section-8f row kernels, device time (CUDA events), %s; HBM peak used: %.0f GB/s\n" % (torch.cuda.get_device_name(), peak))
print("| kernel | ms | algorithmic MB | GB/s | frac of HBM peak |\n|---|---:|---:|---:|---:|")
for name, ms, by in rows:
    gbs = by / ms / 1e6
    print("| %s | %.4f | %.2f | %.0f | %.3f |" % (name, ms, by / 1e6, gbs, gbs / peak))
