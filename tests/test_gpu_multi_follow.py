"""Stream followers across processes on hardware: one process per GPU under torch.distributed.run.  Rank 0 holds the
events; ranks >= 1 are told only the number of batches and follow the stream (ShardedBus.follow).  Every subscriber's
(count, digest) must equal the oracle's, and the global digest fold must be the same at G = 1, 2, 4, 8.  G > device_count
is skipped; the same follower kernels run at G >= 2 on one GPU in tests/test_gpu_stream_follow.py."""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle_binding as ob
from multi_worker_follow import make_case

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_SUBS, N_BATCHES, B = 512, 40, 64
_cache = {}


def _oracle():
    if "orc" not in _cache:
        case = make_case(N_SUBS, N_BATCHES, B)
        orc = ob.Oracle(N_SUBS, timers_per_sub=1, keep_window=0)
        for s in range(N_SUBS):
            orc.subscribe(int(case["masks"][s]))
            orc.timer_add(s, case["period"], case["timer_src0"] + s, False)
        for j in range(N_BATCHES):
            assert orc.advance(case["now"][j]) == 0
            for c, s_ in zip(case["codes"][j], case["sources"][j]):
                assert orc.publish(int(c), int(s_)) == 0
        _cache["orc"] = orc
    return _cache["orc"]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("G", [1, 2, 4, 8])
def test_followers_equal_oracle_at_every_shard_count(G, tmp_path):
    import torch
    if torch.cuda.device_count() < G:
        pytest.skip(f"needs {G} GPUs")
    orc = _oracle()
    out = tmp_path / f"follow{G}"
    out.mkdir()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={G}", "--master-addr", "127.0.0.1",
           "--master-port", str(29750 + G), os.path.join(ROOT, "tests", "multi_worker_follow.py"), "--out", str(out),
           "--subs", str(N_SUBS), "--batches", str(N_BATCHES), "--batch", str(B)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    ranks = [np.load(out / f"rank{k}.npz") for k in range(G)]
    count = np.concatenate([x["count"] for x in ranks]); digest = np.concatenate([x["digest"] for x in ranks])
    assert len(count) == N_SUBS
    want_c = np.array([orc.count(s) for s in range(N_SUBS)], dtype=np.uint64)
    want_d = np.array([orc.digest(s) for s in range(N_SUBS)], dtype=np.uint64)
    bad = np.nonzero((count != want_c) | (digest != want_d))[0]
    assert len(bad) == 0, f"{len(bad)} subscribers differ from the oracle, first {bad[:8]}"
    assert sum(int(x["deliveries"]) for x in ranks) == orc.total_deliveries()
    assert len({int(x["publishes"]) for x in ranks}) == 1         # every rank accounted every published record
    folds = {tuple(int(v) for v in x["fold"]) for x in ranks}
    assert len(folds) == 1
    _cache.setdefault("folds", {})[G] = folds.pop()
    assert len(set(_cache["folds"].values())) == 1
