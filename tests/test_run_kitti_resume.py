"""run_kitti --save-state / --save-every / --resume without a GPU: an injected engine with state that every scan depends
on stands in for the library, so that the plumbing (checkpoint and trajectory side file, where the resumed run starts,
the pose file) is checked on its own. The CUDA engine itself: tests/test_gpu_checkpoint.py."""
import numpy as np
import pytest

from semantic_suma_b200 import run_kitti


class FakeEngine:
    """pose chain driven by the scans and by a memory of all earlier scans; fails at scan `fail_at` (an interruption)"""
    fail_at = None

    def __init__(self, params):
        self.pose = np.eye(4)
        self.memory = np.zeros(3)
        self.t = 0

    def processScan(self, pts, labels, probs):
        if self.t == FakeEngine.fail_at:
            raise KeyboardInterrupt("interrupted at scan %d" % self.t)
        m = np.asarray(pts, np.float64)[:, :3].mean(axis=0)
        self.memory = 0.5 * self.memory + 1e-3 * m
        T = np.eye(4)
        T[:3, 3] = self.memory
        c, s = np.cos(self.memory[0]), np.sin(self.memory[0])
        T[:2, :2] = [[c, -s], [s, c]]
        self.pose = self.pose @ T
        self.t += 1

    def getCurrentPose(self):
        return self.pose

    def timestamp(self):
        return self.t

    def save_state(self):
        return np.concatenate([self.pose.reshape(-1), self.memory, [self.t]]).tobytes()

    def load_state(self, blob):
        a = np.frombuffer(blob, np.float64)
        self.pose, self.memory, self.t = a[:16].reshape(4, 4).copy(), a[16:19].copy(), int(a[19])


@pytest.fixture
def seq(tmp_path):
    d = str(tmp_path / "seq")
    run_kitti.make_synthetic_sequence(d, 12, width=450)
    return d


def _run(args):
    FakeEngine.fail_at = None
    assert run_kitti.main(args, make_engine=FakeEngine) == 0


def test_resume_after_an_interruption_writes_the_same_pose_file(seq, tmp_path):
    whole, resumed, state = str(tmp_path / "whole.txt"), str(tmp_path / "resumed.txt"), str(tmp_path / "state.bin")
    _run([seq, "--width", "450", "--out", whole])
    FakeEngine.fail_at = 8
    with pytest.raises(KeyboardInterrupt):
        run_kitti.main([seq, "--width", "450", "--save-state", state, "--save-every", "3"], make_engine=FakeEngine)
    assert len(np.load(run_kitti.trajectory_path(state))) == 6  # the last checkpoint before the interruption
    _run([seq, "--width", "450", "--resume", state, "--out", resumed])
    assert open(resumed, "rb").read() == open(whole, "rb").read()


def test_a_run_cut_short_and_resumed_writes_the_same_pose_file(seq, tmp_path):
    whole, resumed, state = str(tmp_path / "whole.txt"), str(tmp_path / "resumed.txt"), str(tmp_path / "state.bin")
    _run([seq, "--width", "450", "--out", whole])
    _run([seq, "--width", "450", "--max-scans", "5", "--save-state", state])
    assert len(np.load(run_kitti.trajectory_path(state))) == 5
    res = run_kitti.run_sequence(seq, None, make_engine=FakeEngine, resume=state)
    assert res["scans"] == 7 and len(res["poses"]) == 12
    _run([seq, "--width", "450", "--resume", state, "--out", resumed, "--save-state", state])
    assert open(resumed, "rb").read() == open(whole, "rb").read()
    assert len(np.load(run_kitti.trajectory_path(state))) == 12


def test_checkpoint_and_trajectory_must_agree(seq, tmp_path):
    state = str(tmp_path / "state.bin")
    _run([seq, "--width", "450", "--max-scans", "4", "--save-state", state])
    np.save(run_kitti.trajectory_path(state), np.zeros((3, 4, 4)))
    with pytest.raises(ValueError):
        run_kitti.run_sequence(seq, None, make_engine=FakeEngine, resume=state)
    with pytest.raises(SystemExit):
        run_kitti.main([seq, "--save-every", "2"], make_engine=FakeEngine)
