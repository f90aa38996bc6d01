"""Retrieval evaluation sharded over two ranks (evaluate_retrieval_both(group=...)) against the single-process evaluation, through
tests/_retrieval_ddp_worker.py: one GPU per rank over NCCL, and both ranks on one GPU with the collectives over gloo. Under
torch.use_deterministic_algorithms(True) the gathered scores, both directions' ranks and top-k lists, the metrics and R-sum are
bitwise the single-process ones, padded and packed, fine-tuned with task tokens and zero shot; without it the scores stay within
the packed / padded bound and ranks differ only at near ties. Both ranks return the same result, each rank scores its own block
only, and a weight one ulp off on one rank makes both raise ValueError."""
import json
import os
import signal
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_retrieval_ddp_worker.py")


def _launch(tmp_path, backend, port):
    out = tmp_path / f"retrieval_ddp_{backend}.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), WORKER, str(out), backend]
    # own process group: on a timeout the launcher and both ranks are ended together, nothing is left running
    proc = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, start_new_session=True)
    try:
        _, err = proc.communicate(timeout=600)
    except subprocess.TimeoutExpired:
        os.killpg(proc.pid, signal.SIGKILL)
        proc.communicate()
        pytest.fail(f"the 2-rank retrieval worker ({backend}) did not finish within 600 s")
    assert proc.returncode == 0, err[-3000:]
    return json.load(open(out))


def _check(ranks):
    r0, r1 = ranks
    cases = [k for k in r0 if not k.startswith("perturbed")]
    assert len(cases) == 16 and set(r0) == set(r1)
    for name in cases:
        C = int(name.rsplit("_C", 1)[1])
        for rank, res in enumerate(ranks):
            r = res[name]
            lo, hi = (0, C // 2) if rank == 0 else (C // 2, C)
            assert r["rows"] == [C] + ([hi - lo] if hi > lo else []), (name, rank, r["rows"])    # single call, then the block
            assert r["shape"] == [C, 12] and r["packed"] == ("packed" in name) and not r["fallbacks"], (name, r)
            if "_det_" in name:
                assert r["scores_equal"] and r["out_equal"], (name, rank, r["rel"])
            else:
                assert r["rel"] <= 1e-3, (name, rank, r["rel"])
                assert r["t2i_apart"] == [] and r["i2t_apart"] == [], (name, rank, r)
        # every rank returns the same gathered matrix and the same result
        assert r0[name]["scores_checksum"] == r1[name]["scores_checksum"] and r0[name]["out"] == r1[name]["out"], name
    for zero_shot in ("False", "True"):
        for res in ranks:
            assert "parameters" in res[f"perturbed_{zero_shot}"] and "caption ids" not in res[f"perturbed_{zero_shot}"], res


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_over_nccl_match_one_process(tmp_path):
    _check(_launch(tmp_path, "nccl", 29549))


def test_two_ranks_on_one_gpu_over_gloo_match_one_process(tmp_path):
    _check(_launch(tmp_path, "gloo", 29553))
