"""The whole-fleet ring reference (`tests/ring_check.py`) against the C oracle, on the CPU: every mailbox of a small fleet
with code masks, exact {code, source} cases, unicast records (some for another shard), codes past the enum, two timer
slots (periodic and one-shot, equal due times across slots, records stamped exactly at a due time) and rings that wrap;
also as a shard whose mailboxes start at a non-zero global id."""
import numpy as np
import pytest

import oracle_binding as ob
import ring_check as rc


def _fleet(seed, n=160, R=64, E=900, B=128, base=0):
    rng = np.random.default_rng(seed)
    masks = rng.integers(0, 1 << 17, n).astype(np.uint32)
    masks[::7] = rc.MASK_ALL
    masks[3::11] = 0
    shapes = np.full((12, 16, 2), 0xFFFFFFFF, dtype=np.uint32)
    for s in range(1, 12):                                   # shape 0: no cases
        k = int(rng.integers(1, 17))
        shapes[s, :k, 0], shapes[s, :k, 1] = rng.integers(0, 17, k), rng.integers(0, 6, k)
    shape_of = rng.integers(0, 12, n)
    ts = np.sort(rng.integers(0, 40_000, E)).astype(np.uint64)
    ts[100:104] = 6_000                                      # stamped exactly at a due time (period 1_000 / 1_500 / 2_000)
    ts = np.sort(ts)
    rec = np.zeros(E, dtype=ob.EVENT_DTYPE)
    rec["seq"], rec["ts_ns"] = 10_000 + np.arange(E), ts
    rec["code"], rec["source_id"], rec["target"] = rng.integers(0, 17, E), rng.integers(0, 6, E), rc.TARGET_ALL
    rec["code"][::97] = 17 + rng.integers(0, 50, len(rec[::97]))              # past the enum: nobody takes it
    uni = rng.random(E) < 0.1
    rec["target"][uni] = base + rng.integers(-40 if base else 0, n + 40, int(uni.sum()))   # some for another shard
    rec["flags"][uni] = 0x2
    cuts = list(range(0, E, B)) + [E]
    # watermarks up to the next batch's first stamp (the last one past every record)
    batches = [(a, b, int(ts[b] if b < E else ts[-1] + 700) if i % 2 else int(ts[b - 1]))
               for i, (a, b) in enumerate(zip(cuts[:-1], cuts[1:]))]
    period = (1_000 + 500 * (np.arange(n) % 3)).astype(np.uint64)
    timers = [{"period": period, "source": (500 + np.arange(n)).astype(np.uint32), "oneshot": False},
              {"period": np.where(np.arange(n) % 4 == 0, period, 7_000 + 13 * np.arange(n)).astype(np.uint64),
               "source": (900 + np.arange(n)).astype(np.uint32), "oneshot": True}]
    return rc.FleetModel(n, R, rec, batches, masks, shapes, shape_of, timers, sub_id_base=base)


@pytest.mark.parametrize("seed", [1, 2])
def test_reference_equals_the_oracle_on_every_mailbox(seed):
    model = _fleet(seed)
    model.pin(range(model.n))
    count, _, written = model.expected(0, model.n, "cpu")
    assert (count > model.R).any() and (count < model.R).any()               # wrapped and partial rings both occur
    assert int(written.sum()) == int(np.minimum(count.numpy(), model.R).sum())


def test_reference_of_a_shard_at_a_nonzero_base_equals_the_oracle():
    """mailbox i is global id 70,000 + i: unicast records to the ids just below and past the shard reach nobody here, and
    tick records carry the global id as target (oracle at the same sub_id_base)"""
    base = 70_000
    model = _fleet(4, base=base)
    targets = model.records["target"][model.records["target"] != rc.TARGET_ALL].astype(np.int64)
    assert (targets < base).any() and (targets >= base + model.n).any() and ((targets >= base) & (targets < base + model.n)).any()
    model.pin(range(model.n))
    orc = ob.Oracle(model.n, timers_per_sub=2, keep_window=model.R, sub_id_base=base)
    for i in range(model.n):
        rows = model.pair_shapes[model.shape_of[i]]
        orc.subscribe(int(model.masks[i]), [(int(c), int(s)) for c, s in rows if c != 0xFFFFFFFF] or None)
        for tm in model.timers:
            orc.timer_add(base + i, int(tm["period"][i]), int(tm["source"][i]), bool(tm["oneshot"]))
    for a, b, w in model.batches:
        assert orc.publish_records(model.records[a:b], w) == 0
    count, _, _ = model.expected(0, model.n, "cpu")
    assert [int(c) for c in count] == [orc.count(base + i) for i in range(model.n)]
    for i in range(model.n):
        assert model.window(i).tobytes() == orc.mailbox(base + i).tobytes(), i
    ticks = model.window(model.n - 1)
    assert (ticks["target"][ticks["flags"] & 1 == 1] == base + model.n - 1).all()


def test_reference_chunks_agree_with_one_pass():
    model = _fleet(3)
    whole = model.expected(0, model.n, "cpu")
    for g0, g1 in ((0, 1), (1, 50), (50, 160)):
        part = model.expected(g0, g1, "cpu")
        R = model.R
        assert (part[0] == whole[0][g0:g1]).all()
        assert (part[1] == whole[1][g0 * R: g1 * R]).all() and (part[2] == whole[2][g0 * R: g1 * R]).all()
