"""Plan files on the CPU: the parser and writer behind yb_save_plans / yb_load_plans, through the host-only
yb_check_plans (parse, check format, version and build id, write back as yb_save_plans would).  Comparing the header
with a device and a handle, and obeying the entries, are GPU tests (test_gpu_plan_file.py)."""
import ctypes
import os

import pytest

from yolact_b200 import _lib
from yolact_b200 import build as _build
from tests import test_abi_and_host

PLAN_FUNCTIONS = ["yb_save_plans", "yb_load_plans", "yb_plan_stats", "yb_build_id", "yb_check_plans"]


def _build_id():
    return _lib.load().yb_build_id().decode()


def _text(build=None, version="1", header_extra="", entries=None, end="end\n"):
    if entries is None:
        entries = [
            "tiling 2,138,138,256,64,1,1,0,-hs0,128,2437632 bn=64 stages=4 grid=132 pair=0 mma_groups=1 "
            "pdl_friendly=0 stream_k=1 chain=0",
            "chain 2x550x550:backbone.layers.0.0.conv1..backbone.layers.0.2.conv3:2,138,138,64,64,1,1,0,-hs0,128,"
            "2437632;2,138,138,64,64,3,1,1,-hs0,128,2437632 separate",
            "tiling 1,69,69,512,128,1,1,0,-hs0,256,1218816 bn=128 stages=3 grid=132 pair=1 mma_groups=2 "
            "pdl_friendly=0 stream_k=0 chain=0",
        ]
    return ("yolact_b200 plans %s\n" % version + "build %s\n" % (build or _build_id()) +
            "device NVIDIA H100 80GB HBM3\ncompute_capability 9.0\nsms 132\nprecision f16x3\nsk_candidates 1\n"
            "chain_mode 1\npdl 0\n" + header_extra + "entries %d\n" % len(entries) +
            "".join(e + "\n" for e in entries) + end)


def _check(tmp_path, text, out=False):
    p = tmp_path / "plans.txt"
    p.write_bytes(text.encode())
    o = tmp_path / "out.txt"
    lib = _lib.load()
    st = lib.yb_check_plans(str(p).encode(), str(o).encode() if out else None)
    return st, lib.yb_last_error().decode(), (o.read_bytes().decode() if out and st == 0 else None)


def _refused(tmp_path, text, *words):
    st, err, _ = _check(tmp_path, text)
    assert st == -1, "accepted: %r" % text[-200:]   # YB_ERR_INVALID
    for w in words:
        assert w in err, (w, err)
    return err


def test_library_exports_the_plan_functions():
    test_abi_and_host.test_library_exports_every_declared_symbol()
    syms = test_abi_and_host._header_symbols()
    for name in PLAN_FUNCTIONS:
        assert name in syms and name in _lib.SIGNATURES
    assert ctypes.CDLL(_lib.LIB_PATH).yb_save_plans   # exported by the library itself


def test_build_id_is_the_hash_build_py_passes():
    bid = _build_id()
    assert len(bid) == 16 and all(c in "0123456789abcdef" for c in bid)
    assert bid == _build.build_id(), "the library was built from other sources: python -m yolact_b200.build"


def test_round_trip_is_canonical_and_stable(tmp_path):
    st, err, out = _check(tmp_path, _text(), out=True)
    assert st == 0, err
    lines = out.splitlines()
    # header unchanged, entries sorted (tilings by key, then chains), count and end line written
    assert lines[:10] == _text().splitlines()[:10]
    body = lines[10:-1]
    assert lines[-1] == "end" and len(body) == 3
    assert [l.split(" ")[0] for l in body] == ["tiling", "tiling", "chain"]
    assert body[0].startswith("tiling 1,69,69") and body[1].startswith("tiling 2,138,138")
    assert sorted(body) == sorted(_text().splitlines()[10:-1])
    # the canonical text reads back to itself byte for byte
    st, err, again = _check(tmp_path, out, out=True)
    assert st == 0 and again == out


def test_empty_file_round_trips(tmp_path):
    st, err, out = _check(tmp_path, _text(entries=[]), out=True)
    assert st == 0, err
    assert out == _text(entries=[])


def test_truncated_files_are_refused(tmp_path):
    full = _text()
    # every cut: at each line boundary and in the middle of each line
    cuts = set()
    pos = 0
    for line in full.splitlines(keepends=True):
        cuts.add(pos)
        cuts.add(pos + len(line) // 2)
        pos += len(line)
    cuts.discard(len(full))
    for n in sorted(cuts):
        _refused(tmp_path, full[:n])
    assert "truncated" in _refused(tmp_path, full[:full.index("entries")])
    assert "truncated" in _refused(tmp_path, full[:full.index("\nend") + 1])
    # a missing end line behind a complete entry list is truncation too, and text after it is refused
    _refused(tmp_path, _text(end=""), "truncated")
    _refused(tmp_path, _text(end="end\nmore\n"), "after the end line")


def test_wrong_version_or_build_id_is_refused(tmp_path):
    _refused(tmp_path, _text(version="2"), "version")
    _refused(tmp_path, _text(version="1 "), "version")
    _refused(tmp_path, "some other file\n", "not a yolact_b200 plan file")
    _refused(tmp_path, _text(build="0123456789abcdef"), "build", _build_id())


def test_duplicate_keys_are_refused(tmp_path):
    e = _text().splitlines()[10:-1]
    _refused(tmp_path, _text(entries=e + [e[0]]), "duplicate tiling key")
    _refused(tmp_path, _text(entries=e + [e[1].replace("separate", "chain")]), "duplicate chain key")
    # one key may name a tiling and a chain: they are different tables
    st, err, _ = _check(tmp_path, _text(entries=e[:1] + ["chain " + e[0].split(" ")[1] + " chain"]))
    assert st == 0, err


def test_unknown_or_malformed_fields_are_refused(tmp_path):
    t = _text()
    _refused(tmp_path, _text(header_extra="clock 1980\n"), "'clock'")
    _refused(tmp_path, t.replace("sms 132\nprecision f16x3\n", "precision f16x3\nsms 132\n"), "'precision'", "'sms'")
    _refused(tmp_path, t.replace("sms 132", "sms 13x"), "'sms'")
    _refused(tmp_path, t.replace("sms 132", "sms"), "'sms'")
    e = t.splitlines()[10:-1]
    tiling = e[0]
    for bad, word in [
        (tiling.replace(" chain=0", " chain=0 colour=1"), "fields, not 8"),
        (tiling.replace(" chain=0", ""), "fields, not 8"),
        (tiling.replace("stages=", "depth="), "'depth'"),
        (tiling.replace("bn=64 stages=4", "stages=4 bn=64"), "'stages' where 'bn'"),
        (tiling.replace("bn=64", "bn=48"), "'bn'"),
        (tiling.replace("bn=64", "bn=6.4"), "'bn'"),
        (tiling.replace("stages=4", "stages=0"), "'stages'"),
        (tiling.replace("stages=4", "stages=9"), "'stages'"),
        (tiling.replace("grid=132", "grid=-1"), "'grid'"),
        (tiling.replace("pair=0", "pair=2"), "'pair'"),
        (tiling.replace("mma_groups=1", "mma_groups=3"), "'mma_groups'"),
        (tiling.replace("stream_k=1", "stream_k=yes"), "'stream_k'"),
        (tiling.replace("chain=0", "chain=1"), "'chain'"),
        (tiling.replace("tiling ", "tilling "), "unknown entry kind 'tilling'"),
        (e[1].replace(" separate", " maybe"), "'chain' or 'separate'"),
        (e[1].replace(" separate", ""), "'chain' or 'separate'"),
        ("tiling", "a kind and a key"),
    ]:
        _refused(tmp_path, _text(entries=[bad] + e[1:]), word)
    # the entry count must match the entries
    _refused(tmp_path, t.replace("entries 3", "entries 2"), "expected 'end'")
    _refused(tmp_path, t.replace("entries 3", "entries -1"), "'entries'")


def test_unreadable_path_is_refused(tmp_path):
    lib = _lib.load()
    assert lib.yb_check_plans(str(tmp_path / "missing.txt").encode(), None) == -1
    assert "cannot open" in lib.yb_last_error().decode()
    p = tmp_path / "plans.txt"
    p.write_text(_text())
    assert lib.yb_check_plans(str(p).encode(), str(tmp_path / "no" / "dir.txt").encode()) == -1
    assert "cannot" in lib.yb_last_error().decode()
    assert not os.path.exists(tmp_path / "no")


def test_tune_cli_parses_sizes():
    from yolact_b200 import tune
    assert tune._sizes("550") == [(550, 550)]
    assert tune._sizes("550,480x640") == [(550, 550), (480, 640)]
    with pytest.raises(SystemExit):
        tune.main(["--config", "no_such_config", "-o", os.devnull])
