"""Row f15 on the CPU: the image shares of a multi-rank BOP run (`bop_run.shard_images`), the template-pose flags, and
the gloo steps of `bop_run.Ranks` with two CPU processes (tests/bop_run_shard_worker.py)."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

from gigapose_b200 import bop_run

WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "bop_run_shard_worker.py")


def _cases():
    rng = np.random.default_rng(3)
    yield [100] * 9 + [1] * 40, 8                              # HOPE-like: a few heavy images
    yield [5], 4                                               # fewer images than ranks
    yield [], 2
    yield [3, 3, 3, 3], 3                                      # ties
    for world in (1, 2, 3, 8):
        yield rng.integers(1, 120, int(rng.integers(1, 300))).tolist(), world


@pytest.mark.parametrize("counts,world", list(_cases()))
def test_shares_cover_every_image_once_and_are_balanced(counts, world):
    shares = bop_run.shard_images(counts, world)
    assert len(shares) == world
    assert sorted(i for s in shares for i in s) == list(range(len(counts)))
    assert all(s == sorted(s) for s in shares)
    assert shares == bop_run.shard_images(list(counts), world)
    if counts:
        loads = [sum(counts[i] for i in s) for s in shares]
        assert max(loads) <= sum(counts) / world + max(counts)


def test_shares_are_longest_first_with_ties_by_image_index():
    assert bop_run.shard_images([1, 5, 5, 2, 9], 2) == [[3, 4], [0, 1, 2]]      # 9 | 5 5 | 2 | 1
    assert bop_run.shard_images([4, 4, 4, 4], 2) == [[0, 2], [1, 3]]


BASE = ["--dataset-dir", "d", "--checkpoint", "c"]


def test_template_flags_default_to_the_reference_test_templates():
    a = bop_run.parser().parse_args(BASE)
    assert a.template_poses is None and a.template_level is None and a.pose_distribution is None
    a = bop_run.parser().parse_args(BASE + ["--template-level", "2", "--pose-distribution", "upper"])
    assert (a.template_level, a.pose_distribution) == (2, "upper")
    for bad in (["--template-level", "3"], ["--pose-distribution", "lower"]):
        with pytest.raises(SystemExit):
            bop_run.parser().parse_args(BASE + bad)


@pytest.mark.parametrize("extra", [["--template-level", "1"], ["--pose-distribution", "all"],
                                   ["--template-level", "0", "--pose-distribution", "upper"]])
def test_generated_template_flags_are_refused_with_template_poses(extra, capsys):
    with pytest.raises(SystemExit):
        bop_run.main(BASE + ["--template-poses", "p.npy"] + extra)
    assert "--template-poses" in capsys.readouterr().err


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _launch(out, fail_rank, fail_step, world=2):
    port = _free_port()
    procs = []
    for r in range(world):
        env = dict(os.environ, RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(port))
        procs.append(subprocess.Popen([sys.executable, WORKER, str(out), str(fail_rank), str(fail_step)], env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
    results = []
    try:
        for p in procs:
            _, err = p.communicate(timeout=120)
            results.append((p.returncode, err))
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()
    return results


def test_ranks_step_together(tmp_path):
    results = _launch(tmp_path, -1, -1)
    assert [rc for rc, _ in results] == [0, 0], results
    assert sorted(os.listdir(tmp_path)) == sorted(f"rank{r}_step{s}" for r in range(2) for s in range(3))


@pytest.mark.parametrize("fail_rank,fail_step", [(1, 1), (0, 0), (1, 2)])
def test_a_failing_rank_makes_every_rank_exit_naming_it(tmp_path, fail_rank, fail_step):
    results = _launch(tmp_path, fail_rank, fail_step)
    for r, (rc, err) in enumerate(results):
        assert rc != 0, (r, err)
        assert "RankFailed" in err and f"rank {fail_rank}: BopRunError: planted failure" in err, (r, err)
        with open(tmp_path / f"rank{r}_failed") as f:
            msg = f.read()
        assert msg.startswith(f"rank {fail_rank}: BopRunError: planted failure")
        assert "image 7 (scene 1, image 3)" in msg
        assert not (tmp_path / f"rank{r}_step{fail_step + 1}").exists()
    assert not (tmp_path / f"rank{fail_rank}_step{fail_step}").exists()
    assert (tmp_path / f"rank{1 - fail_rank}_step{fail_step}").exists()
