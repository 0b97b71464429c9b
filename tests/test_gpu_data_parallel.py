"""Yolact under torch.nn.DataParallel, as eval.py's evalvideo runs it (CustomDataParallel(net), DataParallel(
FastBaseTransform()), eval.py:630-634,661-662,692-712): a replica runs on its root's handle for its device with the
root's weights, concurrent first calls create one handle, and detections from another GPU than the frame render as on
the frame's GPU.  The multi-GPU tests compare against the single-GPU run as tests/test_gpu_multi.py does (counts and
class ids exactly, floats to 1e-4: a shard and the whole batch may get different tile plans from the autotuner) and are
skipped with fewer than 2 GPUs; the host side is covered on CPU by tests/test_data_parallel_host.py."""
import threading
import types

import numpy as np
import pytest
import torch

import yolact_b200
from oracle.weights import deterministic_input, deterministic_state_dict
from yolact_b200 import _lib
from yolact_b200.augmentations import FastBaseTransform
from yolact_b200.config import CONFIGS
from yolact_b200.display import render_masks

pytestmark = pytest.mark.gpu


class CustomDataParallel(torch.nn.DataParallel):
    """ A Custom Data Parallel class that properly gathers lists of dictionaries. """   # eval.py:630-634
    def gather(self, outputs, output_device):
        # Note that I don't actually want to convert everything to the output_device
        return sum(outputs, [])


def fresh_net(config="yolact_resnet50_config", seed=0):
    """A net that has never run, on cuda:0 (eval.py:1099-1103)."""
    cfg = CONFIGS[config].copy()
    cfg.max_size = 256
    yolact_b200.cfg.replace(cfg.copy())
    net = yolact_b200.Yolact(cfg, precision="f16x3")
    net.detect.use_fast_nms = True
    net.load_state_dict(deterministic_state_dict(net.state_dict(), seed))
    return net.eval().cuda()


_nets = {}


def shared_net(config):
    if config not in _nets:
        _nets[config] = fresh_net(config)
    net = _nets[config]
    yolact_b200.cfg.replace(net.cfg.copy())
    return net


def gpus():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    return list(range(min(n, 4)))


def same(a, b):
    """Two eval-mode output lists, bit for bit."""
    assert len(a) == len(b)
    for p, q in zip(a, b):
        assert (p["detection"] is None) == (q["detection"] is None)
        if p["detection"] is not None:
            assert p["detection"].keys() == q["detection"].keys()
            for k in p["detection"]:
                assert torch.equal(p["detection"][k], q["detection"][k]), k


def close(got, want, tol=1e-4):
    """got and want per image: same counts and class ids, floats to tol (relative to the largest magnitude above 1:
    the prototypes are not bounded by 1 as boxes, scores and coefficients are)."""
    assert len(got) == len(want)
    for i, (p, q) in enumerate(zip(got, want)):
        assert (p["detection"] is None) == (q["detection"] is None), i
        if p["detection"] is None:
            continue
        for k, t in q["detection"].items():
            g, t = p["detection"][k].cpu(), t.cpu()
            assert g.shape == t.shape, (i, k)
            if k == "class":
                assert torch.equal(g, t), i
            elif g.numel():
                d = float((g - t).abs().max()) / max(1.0, float(t.abs().max()))
                assert d < tol, (i, k, d)


def shard_devices(B, ids):
    """The device DataParallel runs each of B images on: scatter chunks dim 0 into len(ids) parts."""
    return [ids[j] for j, c in enumerate(torch.arange(B).chunk(len(ids))) for _ in range(len(c))]


# ---- one GPU --------------------------------------------------------------------------------------------------------
def test_a_replica_runs_a_never_run_net_then_the_root_gives_the_same_bits():
    net = fresh_net()
    x = deterministic_input(2, 256, 256, 11).cuda()
    with torch.no_grad():
        replica = torch.nn.parallel.replicate(net, [0])[0]
        assert replica is not net and len(replica.state_dict()) < len(net.state_dict())
        got = replica(x)
        assert list(net._handles) == [0]
        want = net(x)
    assert list(net._handles) == [0]
    assert any(d["detection"] is not None for d in got)
    assert all(d["net"] is net for d in got)
    same(got, want)


def test_new_weights_reach_a_replica_made_before_the_load():
    net = fresh_net()
    x = deterministic_input(2, 256, 256, 12).cuda()
    with torch.no_grad():
        replica = torch.nn.parallel.replicate(net, [0])[0]
        before = replica(x)
        net.load_state_dict(deterministic_state_dict(net.state_dict(), 1))
        after = replica(x)
        want = net(x)
    same(after, want)    # had the replica kept the old weights, the root's call would have pushed the new ones
    scores = lambda out: torch.cat([d["detection"]["score"] for d in out if d["detection"] is not None])
    a, b = scores(before), scores(after)
    assert a.shape != b.shape or not torch.equal(a, b)


def test_four_threads_making_the_first_call_create_one_handle(monkeypatch):
    net = fresh_net()
    lib = _lib.load()
    real, created = lib.yb_create, []

    def counting(cfg, device, out):
        rc = real(cfg, device, out)
        if cfg._obj.backbone != _lib.YB_BACKBONE_NONE:
            created.append(device)
        return rc

    monkeypatch.setattr(lib, "yb_create", counting)
    x = deterministic_input(2, 256, 256, 13).cuda()
    barrier = threading.Barrier(4)
    outs, errors = [None] * 4, []

    def run(i):
        try:
            barrier.wait()
            with torch.no_grad():
                outs[i] = net(x)
            torch.cuda.current_stream(x.device).synchronize()
        except BaseException as e:   # noqa: B902 -- reported below
            errors.append(e)

    ts = [threading.Thread(target=run, args=(i,)) for i in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
    assert created == [0] and list(net._handles) == [0]
    assert any(d["detection"] is not None for d in outs[0])
    for o in outs[1:]:
        same(o, outs[0])


# ---- two or more GPUs -----------------------------------------------------------------------------------------------
def test_custom_data_parallel_equals_one_gpu():
    ids = gpus()
    net = shared_net("yolact_resnet50_config")
    x = deterministic_input(5, 256, 256, 77).cuda()
    with torch.no_grad():
        for n in range(2, len(ids) + 1):
            dp = CustomDataParallel(net, device_ids=ids[:n]).cuda()
            for B in (1, 2, 5):
                got = dp(x[:B])
                want = net(x[:B])
                assert any(d["detection"] is not None for d in want)
                close(got, want)
                for d, dev in zip(got, shard_devices(B, ids[:n])):
                    assert d["net"] is net
                    if d["detection"] is not None:
                        assert {t.device for t in d["detection"].values()} == {torch.device("cuda", dev)}


def test_custom_data_parallel_first_call_with_one_frame():
    """evalvideo's default --video_multiframe=1 on a box with several GPUs: one replica, on cuda:0, on a net that has
    never run (eval.py does not prime it before wrapping it)."""
    gpus()
    net = fresh_net()
    dp = CustomDataParallel(net).cuda()
    x = deterministic_input(1, 256, 256, 14).cuda()
    with torch.no_grad():
        got = dp(x)
        want = net(x)
    assert got[0]["net"] is net
    same(got, want)      # the replica ran on the root's cuda:0 handle


@pytest.mark.parametrize("dtype", [torch.float32, torch.uint8])
def test_data_parallel_fast_base_transform_is_bit_identical(dtype):
    ids = gpus()
    cfg = CONFIGS["yolact_resnet50_config"].copy()
    g = torch.Generator().manual_seed(5)
    frames = torch.randint(0, 256, (5, 120, 170, 3), generator=g, dtype=torch.uint8).cuda().to(dtype)
    plain = FastBaseTransform(cfg)
    dp = torch.nn.DataParallel(FastBaseTransform(cfg), device_ids=ids).cuda()
    with torch.no_grad():
        for B in (1, 2, 5):
            got = dp(frames[:B])
            assert got.device == frames.device
            assert torch.equal(got, plain(frames[:B]))


def fake_eval():
    """The parts of eval.py install_display reads: evalvideo's display flags at their defaults."""
    args = types.SimpleNamespace(top_k=5, score_threshold=0.0, crop=True, display_masks=True, display_fps=False,
                                 display_text=True, display_bboxes=True, display_scores=True, display_lincomb=False)

    def original(*a, **k):
        raise AssertionError("evalvideo's display must not reach the original prep_display")

    return types.SimpleNamespace(args=args, prep_display=original,
                                 cfg=types.SimpleNamespace(eval_mask_branch=True, rescore_bbox=False,
                                                           dataset=types.SimpleNamespace(
                                                               class_names=tuple("c%d" % i for i in range(80)))))


def moved(pred, dev):
    """pred (one {'detection', 'net'} entry) with its detection copied to dev."""
    det = pred["detection"]
    return dict(pred, detection=None if det is None else {k: v.to(dev) for k, v in det.items()})


@pytest.mark.parametrize("config", ["yolact_resnet50_config", "yolact_plus_resnet50_config"])
def test_detections_from_another_gpu_render_as_on_the_frame_gpu(config):
    ids = gpus()
    net = shared_net(config)
    g = torch.Generator().manual_seed(21)
    frames = [torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8).cuda() for h, w in
              [(120, 170), (97, 130), (256, 256)]]
    with torch.no_grad():
        replica = torch.nn.parallel.replicate(net, ids[:2])[1]   # the broadcast starts from the net's cuda:0
        x = torch.cat([FastBaseTransform(net.cfg)(f[None]) for f in frames]).to(ids[1])
        preds = replica(x)
    assert any(p["detection"] is not None for p in preds)
    assert all(p["detection"]["box"].device.index == ids[1] for p in preds if p["detection"] is not None)
    here = [moved(p, frames[0].device) for p in preds]
    for kw in ({}, {"top_k": 15, "class_color": True}, {"top_k": 15, "score_threshold": 0.15, "fps_box": (90, 14)}):
        images, drawn = render_masks(preds, frames, **kw)
        want_images, want_drawn = render_masks(here, frames, **kw)
        for a, b in zip(images, want_images):
            assert a.device == frames[0].device and torch.equal(a, b)
        for k in drawn:
            assert torch.equal(drawn[k], want_drawn[k]), k

    pytest.importorskip("cv2")
    from integration.use_b200 import install_display
    E = fake_eval()
    install_display(E)
    for p, q, f in zip(preds, here, frames):
        f = f.float()      # evalvideo: torch.from_numpy(frame).cuda().float()
        got = E.prep_display([p], f, None, None, undo_transform=False, class_color=True, fps_str="")
        want = E.prep_display([q], f, None, None, undo_transform=False, class_color=True, fps_str="")
        assert got.dtype == np.uint8 and np.array_equal(got, want)


def test_evalvideo_network_stage_and_display():
    """eval.py:692-712 restated: transform_frame (frames to cuda:0 as float, the DataParallel transform), eval_network
    (pad to --video_multiframe with copies of frame 0, CustomDataParallel(net), out[:-num_extra]) and prep_frame per
    frame through install_display's prep_display.  Runs on any number of GPUs; with several, a frame's detections come
    from the GPU of its shard while the frame stays on cuda:0."""
    pytest.importorskip("cv2")
    from integration.use_b200 import install_display
    n = torch.cuda.device_count()
    net = shared_net("yolact_resnet50_config")
    dp = CustomDataParallel(net).cuda()
    transform = torch.nn.DataParallel(FastBaseTransform(net.cfg)).cuda()
    E = fake_eval()
    install_display(E)
    g = np.random.RandomState(8)
    for multiframe in sorted({1, n, 2 * n}):
        for count in sorted({multiframe, max(1, multiframe - 1)}):    # a short last read pads with frame 0
            video = [g.randint(0, 256, (120, 170, 3)).astype(np.uint8) for _ in range(count)]
            with torch.no_grad():
                frames = [torch.from_numpy(frame).cuda().float() for frame in video]
                imgs = transform(torch.stack(frames, 0))
                num_extra = 0
                while imgs.size(0) < multiframe:
                    imgs = torch.cat([imgs, imgs[0].unsqueeze(0)], dim=0)
                    num_extra += 1
                out = dp(imgs)
                if num_extra > 0:
                    out = out[:-num_extra]
                assert len(out) == count
                for i, frame in enumerate(frames):
                    got = E.prep_display([out[i]], frame, None, None, undo_transform=False, class_color=True,
                                         fps_str="")
                    want = E.prep_display([moved(out[i], frame.device)], frame, None, None, undo_transform=False,
                                          class_color=True, fps_str="")
                    assert np.array_equal(got, want), (multiframe, count, i)
