"""N > 1 host path on CPU (not gpu): world_size-2 gloo run of the two-stage Q1 protocol."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_two_ranks_gloo_two_stage_q1():
    # --standalone: the rendezvous store takes a free port, so another job on the host that holds a fixed port (or joins it)
    # cannot stall or cross this run
    p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--nnodes=1", "--nproc-per-node", "2",
                        os.path.join(ROOT, "tests", "gloo_worker.py")],
                       capture_output=True, text=True, timeout=300, env=dict(os.environ, OMP_NUM_THREADS="1"))
    assert p.returncode == 0 and "GLOO PASS" in p.stdout, p.stdout[-2000:] + p.stderr[-3000:]
