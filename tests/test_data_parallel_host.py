"""Yolact under torch.nn.DataParallel, host side: a replica (what torch.nn.parallel.replicate makes on every DataParallel
call) pushes its root's weights to the root's handle for its device and names the root as 'net', and concurrent first
calls create one handle per device -- for the net's handles and for the postprocess ops-handle cache.  The library is
replaced by a stub that records the calls, so no GPU is needed."""
import gc
import threading
import time

import pytest
import torch

import yolact_b200
from yolact_b200 import _lib, output_utils
from yolact_b200.config import CONFIGS


class StubLib:
    """The entry points _handle_for, _push_weights, _ops_handle and Yolact.__del__ call, recording each call."""

    def __init__(self, create_delay=0.0):
        self.create_delay = create_delay
        self.lock = threading.Lock()
        self.created, self.loaded, self.finalized, self.destroyed = [], [], [], []

    def yb_create(self, cfg, device, out):
        time.sleep(self.create_delay)   # widens the window in which a second thread could also find no handle
        with self.lock:
            out._obj.value = 0x1000 + len(self.created)
            self.created.append((int(cfg._obj.backbone), device))
        return 0

    def yb_load_weight(self, h, name, data, shape, dim):
        self.loaded.append((h.value, name.decode(), data.value, tuple(shape[:dim])))
        return 0

    def yb_finalize_weights(self, h):
        self.finalized.append(h.value)
        return 0

    def yb_destroy(self, h):
        self.destroyed.append(h.value)
        return 0


def replicate_on_host(network):
    """torch.nn.parallel.replicate's module copy for one replica, without the CUDA broadcast: every module is copied
    with _replicate_for_data_parallel, children are re-linked to the copies, parameters become plain attributes
    (outside state_dict()) and buffers stay buffers."""
    modules = list(network.modules())
    index = {m: i for i, m in enumerate(modules)}
    copies = [m._replicate_for_data_parallel() for m in modules]
    for m, r in zip(modules, copies):
        for key, child in m._modules.items():
            if child is None:
                r._modules[key] = None
            else:
                setattr(r, key, copies[index[child]])
        for key, p in m._parameters.items():
            if p is None:
                r._parameters[key] = None
            else:
                setattr(r, key, p.detach().clone())
        for key, b in m._buffers.items():
            r._buffers[key] = None if b is None else b.clone()
    return copies[0]


@pytest.fixture
def stub(monkeypatch):
    lib = StubLib()
    monkeypatch.setattr(_lib, "load", lambda: lib)
    return lib


@pytest.fixture
def net(stub):
    net = yolact_b200.Yolact(CONFIGS["yolact_resnet50_config"].copy())
    yield net
    net._handles.clear()   # stub handles: nothing for the real library to destroy


def pushed_weights(net):
    """(name, data pointer, shape) of every tensor _push_weights sends for net's parameters."""
    return [(k, t.data_ptr(), tuple(t.shape)) for k, t in net.state_dict().items()
            if not k.endswith("num_batches_tracked") and not k.startswith("semantic_seg_conv")]


def test_a_replica_pushes_the_root_weights_to_the_root_handle(net, stub):
    replica = replicate_on_host(net)
    root_keys = list(net.state_dict())
    assert len(root_keys) == 354
    assert len(replica.state_dict()) == 159   # buffers only: what a replica's own state_dict() would push
    assert replica._root() is net

    h = replica._handle_for(torch.device("cuda", 1))
    assert stub.created == [(_lib.YB_BACKBONE_RESNET, 1)]
    assert net._handles == {1: h} and net._pushed == {1: net._version}
    # the root's own tensors, every one of them, into the one handle
    assert [(n, p, s) for _, n, p, s in stub.loaded] == pushed_weights(net)
    assert {hv for hv, _, _, _ in stub.loaded} == {h.value} and stub.finalized == [h.value]

    # the root on the same device takes the same handle without another push
    assert net._handle_for(torch.device("cuda", 1)) is h
    assert len(stub.finalized) == 1 and len(stub.created) == 1


def test_new_root_weights_reach_the_next_replica_call(net, stub):
    replica = replicate_on_host(net)
    replica._handle_for(torch.device("cuda", 0))
    sd = {k: v.clone() + 1 if v.is_floating_point() else v.clone() for k, v in net.state_dict().items()}
    net.load_state_dict(sd)
    n = len(stub.loaded)
    replica._handle_for(torch.device("cuda", 0))   # a replica made before the load
    assert len(stub.created) == 1 and len(stub.finalized) == 2
    assert [(name, p, s) for _, name, p, s in stub.loaded[n:]] == pushed_weights(net)
    assert net._pushed == {0: net._version}


def test_replica_detections_name_the_root_and_a_replica_destroys_nothing(net, stub):
    replica = replicate_on_host(net)
    B, M, k = 3, 4, net.cfg.mask_dim
    padded = (torch.rand(B, M, 4), torch.rand(B, M, k), torch.zeros(B, M, dtype=torch.int64), torch.rand(B, M),
              torch.tensor([2, 0, 4], dtype=torch.int32), torch.rand(B, 5, 5, k))
    out = replica._detection_list(padded)
    assert [d["net"] for d in out] == [net] * B
    assert out[1]["detection"] is None and out[2]["detection"]["box"].shape == (4, 4)

    replica._handle_for(torch.device("cuda", 0))
    del replica, out
    gc.collect()
    assert stub.destroyed == []      # the handle is the root's, and the root is alive
    assert len(net._handles) == 1


def race(fn, threads=8):
    """fn() from `threads` threads released together -> their results (re-raises the first exception)."""
    barrier = threading.Barrier(threads)
    results, errors = [None] * threads, []

    def run(i):
        try:
            barrier.wait()
            results[i] = fn(i)
        except BaseException as e:   # noqa: B902 -- reported below
            errors.append(e)

    ts = [threading.Thread(target=run, args=(i,)) for i in range(threads)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if errors:
        raise errors[0]
    return results


def test_concurrent_first_calls_create_one_handle_per_device(net, stub):
    stub.create_delay = 0.02
    replicas = [replicate_on_host(net) for _ in range(4)]
    mods = [net] + replicas
    got = race(lambda i: (i % 2, mods[i % len(mods)]._handle_for(torch.device("cuda", i % 2))))
    assert sorted(dev for _, dev in stub.created) == [0, 1]
    for dev, h in got:
        assert h is net._handles[dev]
    assert len(stub.finalized) == 2          # one push per handle
    assert net._pushed == {0: net._version, 1: net._version}


def test_concurrent_ops_handle_lookups_create_once(stub, monkeypatch):
    stub.create_delay = 0.02
    monkeypatch.setattr(output_utils, "_ops_handles", {})
    keys = [(i % 2, 32 if i < 6 else 4) for i in range(8)]   # three threads on each of (0, 32) and (1, 32)
    got = race(lambda i: output_utils._ops_handle(torch.device("cuda", keys[i][0]), keys[i][1]))
    assert sorted(stub.created) == [(_lib.YB_BACKBONE_NONE, 0)] * 2 + [(_lib.YB_BACKBONE_NONE, 1)] * 2
    assert set(output_utils._ops_handles) == set(keys)
    for key, h in zip(keys, got):
        assert h is output_utils._ops_handles[key]
