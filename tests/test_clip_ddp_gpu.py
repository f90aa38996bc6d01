"""Gradient-norm clipping under data parallelism on 2 GPUs (NCCL): every rank takes the norm of the same averaged gradient, so
all ranks clip alike and skip alike. Needs >= 2 visible GPUs; skipped on a single-GPU machine."""
import json
import os
import signal
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_ranks_clip_and_skip_alike(tmp_path):
    out = tmp_path / "clip_ddp.json"
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ddp_clip_worker.py")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29543", worker, str(out)]
    # own process group: on a timeout the launcher and both ranks are ended together, nothing is left running
    proc = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, start_new_session=True)
    try:
        _, err = proc.communicate(timeout=600)
    except subprocess.TimeoutExpired:
        os.killpg(proc.pid, signal.SIGKILL)
        proc.communicate()
        pytest.fail("the 2-rank clipping worker did not finish within 600 s")
    assert proc.returncode == 0, err[-3000:]
    res = json.load(open(out))
    assert all(res["norm_equal"]) and all(res["params_equal"]), res
    assert all(n > 0.5 for n in res["norms"]), res            # the steps were really clipped
    assert res["skipped"] == 1 and res["skipped_on_every_rank"] == 1 and res["unchanged_after_skip"], res
    assert res["step_after_skip"] == 3 and res["params_equal_after"], res
