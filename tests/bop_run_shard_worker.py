"""One rank of tests/test_bop_run_shard_cpu.py: three `bop_run.Ranks` steps on a gloo group (RANK, WORLD_SIZE,
MASTER_ADDR and MASTER_PORT from the environment).  Each step writes <out>/rank{r}_step{s}; rank FAIL_RANK raises in
step FAIL_STEP (an error with the note `run_images` adds), after sleeping so that the other rank reaches the step's
end first; a rank that gets `RankFailed` writes its message to <out>/rank{r}_failed and exits with it.

    python tests/bop_run_shard_worker.py OUT FAIL_RANK FAIL_STEP
"""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gigapose_b200 import bop_run  # noqa: E402


def main(out, fail_rank, fail_step):
    ranks = bop_run.Ranks()
    try:
        for step in range(3):
            def fn():
                if ranks.rank == fail_rank and step == fail_step:
                    time.sleep(1.0)
                    e = bop_run.BopRunError("planted failure")
                    e.add_note("while running image 7 (scene 1, image 3)")
                    raise e
                open(os.path.join(out, f"rank{ranks.rank}_step{step}"), "w").close()
            ranks.step(fn)
    except bop_run.RankFailed as e:
        with open(os.path.join(out, f"rank{ranks.rank}_failed"), "w") as f:
            f.write(str(e))
        raise
    finally:
        ranks.close()


if __name__ == "__main__":
    main(sys.argv[1], int(sys.argv[2]), int(sys.argv[3]))
