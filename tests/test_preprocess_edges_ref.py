"""The designed preprocessing cases of tests/preprocess_cases.py against the reference's own shaders (oracle/_ref,
pinned built-ins): gen_vertexmap, gen_normalmap and floodfill must give the oracle's vertex, normal and semantic maps
bit for bit, and both must equal tests/preprocess_reference.py. With tests/test_gpu_preprocess_edges.py (CUDA = oracle =
model) this closes reference shaders = oracle = CUDA = model at the thresholds themselves."""
import pytest

from oracle import oracle as O
from oracle import ref as R
import preprocess_cases as U
import preprocess_reference as M
from helpers import assert_bits_equal

pytestmark = pytest.mark.skipif(not R.available(), reason="oracle/_ref not built and /root/reference absent")


@pytest.mark.parametrize("shape", U.SHAPES, ids=["%dx%d" % s for s in U.SHAPES])
@pytest.mark.parametrize("name", U.case_ids())
def test_preprocess_case_equals_reference_shaders(name, shape):
    c = U.get(name, *shape)
    p = c.params(O)
    pts, lab, prb = c.arrays()
    model = M.preprocess(p, pts, lab, prb, c.timestamp)
    U.check_tags(c, model)
    r = R.preprocess(p, pts, lab, prb, c.timestamp)
    o = O.preprocess(p, pts, lab, prb, c.timestamp)
    for a, b, nm in zip(r, o, ("vertex", "normal", "semantic")):
        assert_bits_equal(a, b, "%s: %s map, reference vs oracle" % (name, nm))
        assert_bits_equal(a, model[nm], "%s: %s map, reference vs model" % (name, nm))
