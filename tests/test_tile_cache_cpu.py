"""CPU tests of the managed tile cache's interfaces: the Python mirror of sb_tile_cache_info has the header's layout, and
run_kitti --tile-cache-host reaches the engine, reports the counters and keeps resume working (an injected engine stands
in for the library; the CUDA path itself: tests/test_gpu_tile_cache.py)."""
import ctypes as C
import json
import os
import re

import pytest

from semantic_suma_b200 import api, run_kitti
from test_run_kitti_resume import FakeEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_tile_cache_info_layout_matches_header():
    src = open(os.path.join(ROOT, "include", "suma_b200.h")).read()
    body = re.search(r"typedef struct sb_tile_cache_info \{(.*?)\} sb_tile_cache_info;", src, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for typ, names in re.findall(r"(uint32_t|uint64_t)\s+([^;]+);", body):
        fields += [(n.strip(), typ) for n in names.split(",")]
    ctypes_of = {"uint32_t": C.c_uint32, "uint64_t": C.c_uint64}
    assert [(n, ctypes_of[t]) for n, t in fields] == list(api.TileCacheInfo._fields_)
    assert C.sizeof(api.TileCacheInfo) == 16 + 8 * (len(fields) - 4)


class CachedFakeEngine(FakeEngine):
    calls = []

    def setTileCache(self, pool, host):
        CachedFakeEngine.calls.append((pool, host))

    def tile_cache_info(self):
        return {"managed": 1, "evictions": 0}


@pytest.mark.parametrize("arg,host", [("inf", float("inf")), ("123456", 123456)])
def test_run_kitti_tile_cache_host_reaches_the_engine(tmp_path, capsys, arg, host):
    seq = str(tmp_path / "seq")
    run_kitti.make_synthetic_sequence(seq, 6, width=450)
    whole, resumed, state = (str(tmp_path / n) for n in ("whole.txt", "resumed.txt", "state.bin"))
    common = [seq, "--width", "450", "--tile-cache-host", arg]
    FakeEngine.fail_at = None
    CachedFakeEngine.calls = []
    assert run_kitti.main(common + ["--out", whole], make_engine=CachedFakeEngine) == 0
    report = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert report["tile_cache"]["managed"] == 1
    assert CachedFakeEngine.calls == [(run_kitti.TILE_POOL_SURFELS, host)]
    assert run_kitti.main(common + ["--max-scans", "3", "--save-state", state], make_engine=CachedFakeEngine) == 0
    assert run_kitti.main(common + ["--resume", state, "--out", resumed], make_engine=CachedFakeEngine) == 0
    assert open(resumed, "rb").read() == open(whole, "rb").read()


def test_run_kitti_default_cache_leaves_the_engine_alone(tmp_path, capsys):
    seq = str(tmp_path / "seq")
    run_kitti.make_synthetic_sequence(seq, 3, width=450)
    CachedFakeEngine.calls = []
    assert run_kitti.main([seq, "--width", "450", "--tile-cache-host", "0"], make_engine=CachedFakeEngine) == 0
    assert CachedFakeEngine.calls == []
    assert "tile_cache" not in json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    with pytest.raises(ValueError):
        run_kitti.parse_host_surfels("-1")
