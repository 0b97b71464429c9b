"""Plan files on the H100: a handle that loads another's plan file runs the same kernels and reproduces its outputs bit
for bit, times nothing the file covers, obeys an edited entry, times only the shapes the file lacks, and refuses a
file that does not fit it without changing anything.

One writer handle (yolact_base, f16x3, 550^2, B = 2) tunes and saves; every other handle is fresh and runs the same
deterministic weights and input."""
import os
import subprocess
import sys

import pytest
import torch

import yolact_b200
from yolact_b200 import _lib
from oracle.weights import deterministic_state_dict, deterministic_input
from tests.conftest import ROOT
from tests.helpers import cfg_for, rel_err

pytestmark = pytest.mark.gpu

CFG = "yolact_base_config"
B, H, W = 2, 550, 550
HEAD = ("loc", "conf", "mask", "proto")
DET = ("box", "coef", "cls", "score", "count", "proto")


def _net(plans=None):
    cfg = cfg_for(CFG)
    yolact_b200.cfg.replace(cfg.copy())
    net = yolact_b200.Yolact(cfg, precision="f16x3")
    net.load_state_dict(deterministic_state_dict(net.state_dict(), 7))
    if plans:
        net.load_plans(plans)
    return net


def _run(net, b=B):
    """head tensors (train mode), detections and prototypes (infer_padded), op names with tilings and chains"""
    x = deterministic_input(b, H, W, seed=11).cuda()
    net.train()
    raw = net(x)
    out = {k: raw[k].clone() for k in HEAD}
    det = net.infer_padded(x)
    out.update({"det_" + k: v.clone() for k, v in zip(DET, det)})
    names = [n for n, _ in net.profile_conv_stack(x)]
    torch.cuda.synchronize()
    return out, names


def _assert_equal(a, b):
    for k in a:
        assert torch.equal(a[k], b[k]), (k, float((a[k].double() - b[k].double()).abs().max()))


def _entries(path):
    lines = open(path).read().splitlines()
    assert lines[-1] == "end"
    return lines[10:-1]


def _rewrite(src, dst, old, new):
    text = open(src).read()
    assert text.count(old) == 1, old
    open(dst, "w").write(text.replace(old, new))


@pytest.fixture(scope="module", autouse=True)
def _no_plan_file_from_the_environment():
    """every handle here starts with an empty table, whatever YB_PLANS names"""
    with pytest.MonkeyPatch.context() as mp:
        mp.delenv("YB_PLANS", raising=False)
        yield


@pytest.fixture(scope="module")
def writer(tmp_path_factory):
    d = tmp_path_factory.mktemp("plans")
    net = _net()
    out, names = _run(net)
    path = str(d / "b2.txt")
    net.save_plans(path)
    timed, loaded = net.plan_stats()
    assert timed > 0 and loaded == 0
    assert len(_entries(path)) == timed   # one entry per timed decision
    del net
    torch.cuda.empty_cache()
    return dict(path=path, out=out, names=names, dir=d)


@pytest.fixture(scope="module")
def reader(writer):
    """a handle that loaded the writer's file and ran the writer's input"""
    net = _net(writer["path"])
    out, names = _run(net)
    return dict(net=net, out=out, names=names)


def test_loaded_plans_reproduce_the_writers_outputs_bit_for_bit(writer, reader):
    _assert_equal(reader["out"], writer["out"])
    # the same tilings and chains, op by op
    assert reader["names"] == writer["names"]
    timed, loaded = reader["net"].plan_stats()
    assert timed == 0 and loaded > 0


def test_a_child_process_reproduces_the_writers_outputs(writer, tmp_path):
    code = (
        "import sys, torch\n"
        "sys.path.insert(0, %r)\n"
        "from tests import test_gpu_plan_file as T\n"
        "net = T._net(%r)\n"
        "out, names = T._run(net)\n"
        "torch.save({k: v.cpu() for k, v in out.items()}, %r)\n"
        "print('stats', *net.plan_stats())\n" % (ROOT, writer["path"], str(tmp_path / "out.pt")))
    env = dict(os.environ)
    env.pop("YB_PLANS", None)
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-3000:]
    stats = [l for l in r.stdout.splitlines() if l.startswith("stats")][-1].split()
    assert int(stats[1]) == 0 and int(stats[2]) > 0
    got = torch.load(str(tmp_path / "out.pt"))
    _assert_equal({k: v.cuda() for k, v in got.items()}, writer["out"])


def test_an_edited_entry_is_obeyed(writer, tmp_path):
    entries = _entries(writer["path"])
    # a prediction head (never chained, so its tiling shows in its op name): one pipeline stage fewer
    heads = [e for e in entries if e.startswith("tiling ") and e.split(" ")[1].split(",")[8].endswith("s3")
             and int(e.split("stages=")[1].split(" ")[0]) > 1]
    assert heads, entries
    old = heads[0]
    st = int(old.split("stages=")[1].split(" ")[0])
    new = old.replace("stages=%d" % st, "stages=%d" % (st - 1))
    key = old.split(" ")[1].split(",")
    hw = " %sx%s tc " % (key[1], key[2])
    # a chain decision flipped
    chains = [e for e in entries if e.startswith("chain ")]
    assert chains
    c_old = chains[0]
    was_chain = c_old.endswith(" chain")
    c_new = c_old[:c_old.rindex(" ")] + (" separate" if was_chain else " chain")
    first, last = c_old.split(" ")[1].split(":")[1].split("..")
    path = str(tmp_path / "edited.txt")
    text = open(writer["path"]).read().replace(old + "\n", new + "\n").replace(c_old + "\n", c_new + "\n")
    open(path, "w").write(text)

    net = _net(path)
    out, names = _run(net)
    assert net.plan_stats()[0] == 0

    def tiling(e):
        f = dict(kv.split("=") for kv in e.split(" ")[2:])
        s = "BN=%s st=%s g=%s" % (f["bn"], f["stages"], f["grid"])
        return s + "".join(n for v, n in ((f["pair"], " pair"), (f["mma_groups"] == "2" and "1" or "0", " epi2"),
                                          (f["pdl_friendly"], " pdlf"), (f["stream_k"], " sk")) if v == "1")

    def head_ops(ns):
        return [n for n in ns if "bbox+conf+mask" in n and hw in n]

    assert head_ops(writer["names"]) and all(n.endswith(" tc " + tiling(old)) for n in head_ops(writer["names"]))
    assert head_ops(names) and all(n.endswith(" tc " + tiling(new)) for n in head_ops(names))
    tag = "[%s .. %s]" % (first, last)
    assert any(tag in n for n in writer["names"]) == was_chain
    assert any(tag in n for n in names) == (not was_chain)
    for k in HEAD:   # stream-K adds partial tiles in another order: equal up to fp32 rounding
        assert rel_err(out[k].cpu().numpy(), writer["out"][k].cpu().numpy()) < 2e-4, k


def test_a_file_for_another_batch_times_only_the_missing_shapes(writer, reader, tmp_path):
    net = _net(writer["path"])
    _run(net, b=3)
    timed, loaded = net.plan_stats()
    superset = str(tmp_path / "b2b3.txt")
    net.save_plans(superset)
    old, new = set(_entries(writer["path"])), set(_entries(superset))
    assert old < new
    added = new - old
    assert timed == len(added) > 0 and loaded == 0
    for e in added:
        key = e.split(" ")[1]
        assert key.startswith("3,") if e.startswith("tiling ") else key.startswith("3x550x550:"), e
    # a save right after a load writes the loaded bytes
    for src in (writer["path"], superset):
        fresh = _net(src)
        again = str(tmp_path / "again.txt")
        fresh.save_plans(again)
        assert open(again, "rb").read() == open(src, "rb").read()
    # the reader has planned B = 2 from the file: the superset agrees with it and loads
    reader["net"].load_plans(superset)


def test_refused_files_leave_the_handle_untouched(writer, reader, tmp_path):
    src = writer["path"]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    bid = _lib.load().yb_build_id().decode()
    entries = _entries(src)
    tiling = [e for e in entries if e.startswith("tiling ")][0]
    st = int(tiling.split("stages=")[1].split(" ")[0])
    chain = [e for e in entries if e.startswith("chain ")][0]
    bad = {}
    for name, old, new, word in [
        ("precision", "precision f16x3\n", "precision f16tc\n", "precision"),
        ("sms", "sms %d\n" % sms, "sms %d\n" % (sms - 18), "sms"),
        ("build", "build %s\n" % bid, "build 0123456789abcdef\n", "build"),
        ("tiling", tiling + "\n", tiling.replace("stages=%d" % st, "stages=%d" % (st % 8 + 1)) + "\n", "tiling"),
        ("chain", chain + "\n", chain[:chain.rindex(" ")] + (" separate\n" if chain.endswith(" chain") else " chain\n"),
         "chain"),
    ]:
        p = str(tmp_path / (name + ".txt"))
        _rewrite(src, p, old, new)
        bad[name] = (p, word)
    text = open(src).read()
    p = str(tmp_path / "truncated.txt")
    open(p, "w").write(text[:len(text) // 2])
    bad["truncated"] = (p, "truncated")

    net = reader["net"]   # has planned every shape of the file (B = 2): the edited entries disagree with it
    before = net.plan_stats()
    for name, (p, word) in bad.items():
        with pytest.raises(_lib.YbError) as e:
            net.load_plans(p)
        assert "status -1" in str(e.value) and word in str(e.value), (name, str(e.value))
    out, names = _run(net)
    _assert_equal(out, writer["out"])
    assert names == writer["names"]
    assert net.plan_stats()[0] == before[0] == 0

    # a fresh handle refuses the header and truncation refusals too, and then plans by timing with nothing merged
    fresh = _net()
    fresh.num_priors_for(H, W)   # creates the handle
    for name in ("precision", "sms", "build", "truncated"):
        p, word = bad[name]
        with pytest.raises(_lib.YbError) as e:
            fresh.load_plans(p)
        assert word in str(e.value), (name, str(e.value))
    out, _ = _run(fresh)
    timed, loaded = fresh.plan_stats()
    assert timed == len(entries) and loaded == 0
    for k in HEAD:
        assert rel_err(out[k].cpu().numpy(), writer["out"][k].cpu().numpy()) < 2e-4, k
