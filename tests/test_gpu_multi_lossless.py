"""Lossless mode across processes on hardware: one process per GPU under torch.distributed.run (ShardedBus(lossless=True)),
small rings, a drain schedule after every stalled round, every rank retrying in lockstep.  Every subscriber's
(count, digest) must equal the oracle's with mailbox_cap = ring_cap (the Go bus blocking on a full channel), and the
global digest fold must be the same at G = 1, 2, 4, 8.  G > device_count is skipped; the same offer words and agree kernel
run at G >= 2 on one GPU in tests/test_gpu_stream_agree.py."""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle_binding as ob
from multi_worker_lossless import drain_schedule, make_case

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_SUBS, N_BATCHES, B, R = 256, 24, 32, 64
_cache = {}


def _oracle():
    """the same batches and the same drain schedule, event by event; returns (oracle, rounds, stalls)"""
    if "orc" not in _cache:
        case = make_case(N_SUBS, N_BATCHES, B)
        orc = ob.Oracle(N_SUBS, keep_window=0, mailbox_cap=R)
        for s in range(N_SUBS):
            orc.subscribe(int(case["masks"][s]))
        rounds = stalls = 0
        for j in range(N_BATCHES):
            assert orc.advance(case["now"][j]) == 0
            i = j * B
            while True:
                while i < (j + 1) * B and orc.publish(int(case["codes"][i]), int(case["sources"][i])) == 0:
                    i += 1
                rounds += 1
                if i == (j + 1) * B:
                    break
                stalls += 1
                for s, take in drain_schedule(rounds - 1, N_SUBS, R):
                    orc.consume(s, take)
        _cache["orc"] = (orc, rounds, stalls)
    return _cache["orc"]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("G", [1, 2, 4, 8])
def test_lossless_sharded_bus_equals_oracle_at_every_shard_count(G, tmp_path):
    import torch
    if torch.cuda.device_count() < G:
        pytest.skip(f"needs {G} GPUs")
    orc, rounds, stalls = _oracle()
    assert stalls > 0
    out = tmp_path / f"lossless{G}"
    out.mkdir()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={G}", "--master-addr", "127.0.0.1",
           "--master-port", str(29700 + G), os.path.join(ROOT, "tests", "multi_worker_lossless.py"), "--out", str(out),
           "--subs", str(N_SUBS), "--batches", str(N_BATCHES), "--batch", str(B), "--ring", str(R)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    ranks = [np.load(out / f"rank{k}.npz") for k in range(G)]
    assert all(int(x["rounds"]) == rounds and int(x["stalls"]) == stalls for x in ranks)   # lockstep, as the oracle
    count = np.concatenate([x["count"] for x in ranks]); digest = np.concatenate([x["digest"] for x in ranks])
    assert len(count) == N_SUBS
    want_c = np.array([orc.count(s) for s in range(N_SUBS)], dtype=np.uint64)
    want_d = np.array([orc.digest(s) for s in range(N_SUBS)], dtype=np.uint64)
    bad = np.nonzero((count != want_c) | (digest != want_d))[0]
    assert len(bad) == 0, f"{len(bad)} subscribers differ from the oracle, first {bad[:8]}"
    assert sum(int(x["deliveries"]) for x in ranks) == orc.total_deliveries()
    folds = {tuple(int(v) for v in x["fold"]) for x in ranks}
    assert len(folds) == 1
    _cache.setdefault("folds", {})[G] = folds.pop()
    assert len(set(_cache["folds"].values())) == 1                 # the fold does not depend on G
