"""The map update's index map (K6a, gen_indexmap) written by the pipeline's post-ICP render instead of a pass of its own.
Without track-loss recovery the render sees the map at the pose and with the product table the index pass would see; on a
scan with recovery a gated index pass writes the keys at the recovered pose; with loop closure on the plain index pass
runs. Every case against the oracle, after every scan:
pose bits, the index map, every surfel record (the update's colour lane records every index-map win of its else-branch)."""
import numpy as np
import pytest

from oracle import oracle as O
from semantic_suma_b200 import api, synth
from helpers import assert_bits_equal, both_params, scans, sized, surfel_fields_equal

pytestmark = pytest.mark.gpu


def _step(osl, gsl, scan, what, compacted):
    """one scan on both. compacted: the map was downloaded (and so compacted) after the previous scan, so the physical
    slots the library's index map names are the surfels in order, as the oracle's are; otherwise (dead slots in front of
    live ones) only the pixels that have a winner are compared."""
    osl.process_scan(*scan)
    gsl.processScan(*scan)
    assert_bits_equal(gsl.getCurrentPose(), osl.pose(), what + " pose")
    oi = osl.map.update_debug()[0]
    gi = gsl.getMap().update_debug()[0]
    assert_bits_equal(gi != 0, oi != 0, what + " pixels with an index-map winner")
    if compacted:
        assert_bits_equal(gi, oi, what + " index map")
    assert gsl.getMap().size() == osl.map.size(), what + " surfel count"


def _lockstep(po, pp, sc, what, observe_every_scan=True, setup=None):
    """observe_every_scan: download and compare every surfel after every scan; else only after the last one (the
    in-place updates then leave dead slots for the next scans' renders to skip)"""
    osl, gsl = O.Slam(po), api.SurfelMapping(pp)
    try:
        if setup:
            setup(osl, gsl)
        compacted = True
        for t, scan in enumerate(sc):
            _step(osl, gsl, scan, "%s t=%d" % (what, t), compacted)
            if observe_every_scan or t == len(sc) - 1:
                surfel_fields_equal(gsl.getMap().getAllSurfels(), osl.map.download(), "%s t=%d surfels" % (what, t))
            compacted = observe_every_scan
        for g, o in zip(gsl.getLastModelFrame().maps(), osl.frame(1)):
            assert_bits_equal(g, o, what + " model frame")
        return osl.stats()
    finally:
        gsl.ctx.close()


def test_fused_index_map_64x2048():
    """the bench geometry: the fused render writes the keys on every scan after the first; three scans observed after
    each, then three on a map with dead slots"""
    po, pp = both_params(**sized(2048))
    sc, _ = scans(2048, n=6)
    _lockstep(po, pp, sc[:3], "2048 observed")
    _lockstep(po, pp, sc, "2048 dead slots", observe_every_scan=False)


def test_fused_index_map_through_track_loss_recovery():
    """the pose jump of test_track_loss_fallback_bit_exact: the recovery runs, the render writes no key and the gated
    index pass writes them all at the recovered pose"""
    po, pp = both_params(**sized(900))
    scene = synth.Scene(width=900, height=64)
    poses = synth.trajectory(8)
    J = synth.translate(0.8, 0.3, 0) @ synth.rot_z(np.deg2rad(8.0))
    sc = [scene.scan(f, poses[f] if f < 4 else poses[f] @ J) for f in range(7)]
    st = _lockstep(po, pp, sc, "fallback")
    assert st["track_loss"] >= 1, "the sequence must trigger the recovery"


@pytest.mark.parametrize("model", [
    dict(data_width=513, data_height=33, model_width=451, model_height=47),  # the render's projection serves the index
    dict(sized(900), model_fov_up=4.0, model_fov_down=-26.0),                # the index projects again with its own
], ids=["model_451x47_data_513x33", "model_fov_differs"])
def test_fused_index_map_model_differs_from_data(model):
    po, pp = both_params(**model)
    W, H = model["data_width"], model["data_height"]
    sc, _ = scans(W, H, n=5)
    _lockstep(po, pp, sc, "model != data")


def test_plain_index_pass_with_loop_closure():
    """checkLoopClosure runs between the pose update and the map update and renders: the plain index pass stays"""
    po, pp = both_params(**sized(900))
    sc, _ = scans(900, n=5)
    lp = dict(search_distance=3.0, min_trajectory_distance=15.0, min_verifications=2)

    def setup(osl, gsl):
        osl.enable_loop_closure(**lp)
        gsl.enableLoopClosure(True, **lp)

    _lockstep(po, pp, sc, "loop closure", setup=setup)

