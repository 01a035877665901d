"""The designed map-update cases of tests/update_cases.py against the reference's own shaders (oracle/_ref, pinned
built-ins): ref.Map and the oracle must agree bit for bit (index map, radius map, integrated flags, transform-feedback
counts, records and their order), and both must agree with tests/update_reference.py. With
tests/test_gpu_update_edges.py (CUDA = oracle = model) this closes reference shaders = oracle = CUDA = model at the
thresholds themselves."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import ref as R
import update_cases as U
import update_reference as M
from helpers import assert_bits_equal, surfel_fields_equal

pytestmark = pytest.mark.skipif(not R.available(), reason="oracle/_ref not built and /root/reference absent")


def _run(m, c):
    for t, T in c.poses.items():
        m.set_pose(t, T)
    m.upload(c.records(), U.TS)
    m.update(c.pose, c.frame())
    return m.update_debug() + (m.download(),)


@pytest.mark.parametrize("shape", U.SHAPES, ids=["%dx%d" % s for s in U.SHAPES])
@pytest.mark.parametrize("name", U.case_ids())
def test_update_case_equals_reference_shaders(name, shape):
    c = U.get(name, *shape)
    p = c.params(O)
    model = M.update(p, c.records(), c.frame(), c.pose, U.TS, c.poses)
    U.check_tags(c, model)
    rm = R.Map(p)
    d = rm.derived()
    for k, v in model["derived"].items():
        assert np.float32(d[k]) == v, "%s: derived %s: reference %r, model %r" % (name, k, d[k], v)
    r, o = _run(rm, c), _run(O.Map(p), c)
    assert np.array_equal(r[0], o[0]), name + ": index map"
    assert_bits_equal(r[1], o[1], name + ": radius map")
    assert np.array_equal(r[2], o[2]), name + ": integrated flags"
    assert r[3:5] == o[3:5], "%s: transform-feedback counts %s vs oracle %s" % (name, r[3:5], o[3:5])
    surfel_fields_equal(r[5], o[5], name + ": surfels")
    assert np.array_equal(r[0], model["index"]), name + ": index map vs model"
    assert_bits_equal(r[1], model["radius"], name + ": radius map vs model")
    assert np.array_equal(r[2], model["integrated"]), name + ": integrated flags vs model"
    assert r[3:5] == (model["n_updated"], model["n_new"]), name + ": counts vs model"
    M.compare(model, r[5], name + ": surfels vs model")


def test_parallel_normals_give_a_nan_normal_in_the_reference():
    """update_surfels.vert's slerp of exactly parallel normals: acos(1) = 0, 1 / sin(0) = inf, NaN weights -- the
    reference's surfel keeps a NaN normal, as the oracle's and the library's do"""
    c = U.get("slerp_parallel", *U.SHAPES[0])
    r = _run(R.Map(c.params(O)), c)[5]
    assert len(r) >= 1 and np.isnan(r[0]["nx"]) and np.isnan(r[0]["ny"]) and np.isnan(r[0]["nz"])
