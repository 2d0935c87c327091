"""Lossless stream rounds across processes on hardware: one process per GPU under torch.distributed.run.  Rank 0 holds
the events; ranks >= 1 are told only the number of batches, and every rank runs ShardedBus.run_rounds (device rounds,
agreement through the publisher's memory) with consumers draining at random.  Every subscriber's drained records and
(count, digest) must equal the oracle's (mailbox_cap = ring_cap) at G = 1, 2, 4, 8.  G > device_count is skipped; the same
round kernels run at G >= 2 on one GPU in tests/test_gpu_stream_rounds.py."""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle_binding as ob
from multi_worker_lossless_rounds import make_case

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_SUBS, N_BATCHES, B, R = 256, 30, 64, 128


@pytest.mark.timeout(900)
@pytest.mark.parametrize("G", [1, 2, 4, 8])
def test_lossless_rounds_equal_oracle_at_every_shard_count(G, tmp_path):
    import torch
    if torch.cuda.device_count() < G:
        pytest.skip(f"needs {G} GPUs")
    out = tmp_path / f"rounds{G}"
    out.mkdir()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={G}", "--master-addr", "127.0.0.1",
           "--master-port", str(29850 + G), os.path.join(ROOT, "tests", "multi_worker_lossless_rounds.py"), "--out", str(out),
           "--subs", str(N_SUBS), "--batches", str(N_BATCHES), "--batch", str(B), "--ring", str(R)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    ranks = [np.load(out / f"rank{k}.npz") for k in range(G)]
    assert len({int(x["rounds"]) for x in ranks}) == 1 and len({int(x["publishes"]) for x in ranks}) == 1
    # every subscriber's whole delivered sequence, as the oracle delivers it (the drain points do not change it)
    case = make_case(N_SUBS, N_BATCHES, B)
    orc = ob.Oracle(N_SUBS, keep_window=0)
    for s in range(N_SUBS):
        orc.subscribe(int(case["masks"][s]))
    for j in range(N_BATCHES):
        assert orc.advance(case["now"][j]) == 0
        for c, s_ in zip(case["codes"][j], case["sources"][j]):
            assert orc.publish(int(c), int(s_)) == 0
    for x in ranks:
        recs = x["records"].view(ob.EVENT_DTYPE)
        ends = np.cumsum(x["lens"])
        for i, (lo, hi) in enumerate(zip(np.r_[0, ends[:-1]], ends)):
            s = int(x["first"]) + i
            assert int(x["count"][i]) == orc.count(s) and int(x["digest"][i]) == orc.digest(s), s
            assert recs[lo:hi].tobytes() == orc.mailbox(s).tobytes(), s
