"""The fleet-wide consumer backlog of a lossless ShardedBus across processes, on hardware: one process per GPU under
torch.distributed.run, device rounds queued until they stall, nobody consuming but the drains of exactly the blockers.
At every stall every rank's blockers() and lagging() must equal what a LocalShardedBus driven through the same steps on
one process returns.  G > device_count is skipped; the aggregation itself is checked on CPU in
tests/test_gloo_stream_blockers.py."""
import os
import subprocess
import sys

import numpy as np
import pytest

from multi_worker_stream_blockers import replay_on_one_process

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_SUBS, N_BATCHES, B, R = 64, 20, 32, 64


@pytest.mark.timeout(900)
@pytest.mark.parametrize("G", [1, 2, 4, 8])
def test_every_rank_answers_as_one_process_does(G, tmp_path):
    import torch
    if torch.cuda.device_count() < G:
        pytest.skip(f"needs {G} GPUs")
    out = tmp_path / f"blk{G}"
    out.mkdir()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={G}", "--master-addr", "127.0.0.1",
           "--master-port", str(29950 + G), os.path.join(ROOT, "tests", "multi_worker_stream_blockers.py"), "--out", str(out),
           "--subs", str(N_SUBS), "--batches", str(N_BATCHES), "--batch", str(B), "--ring", str(R)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    ranks = [np.load(out / f"rank{k}.npy", allow_pickle=True).tolist() for k in range(G)]
    want = replay_on_one_process(G, N_SUBS, N_BATCHES, B, R)
    assert len(want) >= 2 and all(a["blockers"] for a in want)
    for k, got in enumerate(ranks):
        assert got == want, k
