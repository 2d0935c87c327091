"""The consumer half of the hot path on a fleet where few mailboxes receive records: what the `chan Event` pump costs per
batch with the dense drain (cpbus_drain_many over the whole id range) and with the sparse one (cpbus_drain_ready until
nothing is ready).

The fleet is the Job-shaped one of scripts/diag_pairs.py (exact {code, source} cases per subscriber).  512-event batches
from host buffers are published to twin buses; after every batch each bus is drained by one of the two paths, alternating
which goes first, with both C functions called directly on preallocated pinned buffers as a shim would.  Parity: the two
paths' records are identical per subscriber and equal a 1-subscriber oracle's for sampled subscribers.  Also the dense rate
of both paths on the `bridge` shape of bench.py (8,192 mailboxes x 512 records).  Prints one JSON line with the card's name
and power limit; exits 3 when a parity check fails.  Writes nothing.

  python scripts/bridge_sparse.py [--steps 200 --warmup 10 --subs 32768 1048576]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

import oracle_binding as ob
from containerpilot_b200 import _native as nat
from containerpilot_b200 import events as ev
from containerpilot_b200 import masks as mk
from containerpilot_b200.bus import Bus, EVENT_DTYPE, READY_DTYPE


def job_fleet(n: int, seed: int = 7):
    """The Job-shaped fleet of scripts/diag_pairs.py, built with numpy: subscriber j has the exact cases of a Job's switch
    (its own name, health check and timers, and, for j % 3 != 0, the ExitSuccess of a random other job as start event).
    Source ids: 0 "", 1 global, 2 closed, 3 SIGHUP, 4 SIGUSR2, then 5 per job.  Returns masks, pair rows (n x 16 x 2) and
    pair counts, as cpbus_subscribe_pairs_many takes them, and the number of source ids."""
    rng = np.random.default_rng(seed)
    dep = rng.integers(0, n, n).astype(np.int64)
    j = np.arange(n, dtype=np.int64)
    fixed = {"": 0, "global": 1, "closed": 2, "SIGHUP": 3, "SIGUSR2": 4}
    suffix = {"": 0, "heartbeat": 2, "run-every": 3, "wait-timeout": 4}

    def src_of(name):                        # templates use job0 (own) and job1 (the start event's job)
        if name in fixed:
            return lambda: np.full(n, fixed[name], dtype=np.int64)
        base, _, sfx = name.partition(".")
        if base == "check":
            who = j if sfx == "job0" else dep
            return lambda: 5 + 5 * who + 1
        who = j if base == "job0" else dep
        return lambda: 5 + 5 * who + suffix[sfx]
    masks = np.zeros(n, dtype=np.uint32)
    rows = np.full((n, 16, 2), 0xFFFFFFFF, dtype=np.uint32)
    cnt = np.zeros(n, dtype=np.uint32)
    for kind, start in ((0, ev.GlobalStartup), (1, ev.Event(ev.ExitSuccess, "job1"))):
        sel = (j % 3 != 0) if kind else (j % 3 == 0)
        m, cases = mk.JobSwitch("job0", start_event=start).cases()
        masks[sel] = m
        cnt[sel] = len(cases)
        for k, c in enumerate(cases):
            rows[sel, k, 0] = c.Code
            rows[sel, k, 1] = src_of(c.Source)()[sel]
    return masks, rows, cnt, 5 + 5 * n


def run(args):
    """Both drain paths per fleet size in args.subs, then the dense shape; returns the result record."""
    B, R = 512, 512                          # a 512-event batch goes out as two 256-event fan-outs (batch_cap <= ring/2)
    steps, warmup = args.steps, max(args.warmup, 3)
    lib = nat.load()

    def pinned(n_rec, dtype):
        t = torch.empty((n_rec * dtype.itemsize,), dtype=torch.uint8).pin_memory()
        return t, t.numpy().view(dtype)

    legs, ok = [], True
    for n_subs in args.subs:
        masks, rows, cnt, n_src = job_fleet(n_subs)
        rng = np.random.default_rng(0xB51D + n_subs)
        host = np.zeros((warmup + steps) * B, dtype=EVENT_DTYPE)
        host["code"] = rng.integers(1, 17, len(host)); host["source_id"] = rng.integers(0, n_src, len(host))
        buses = [Bus(n_subs, ring_cap=R, batch_cap=R // 2, digest=False, device=args.device) for _ in range(2)]
        for bus in buses:
            first = C.c_uint32()
            nat.check(lib.cpbus_subscribe_pairs_many(bus._h, masks.ctypes.data, rows.ctypes.data, cnt.ctypes.data, n_subs,
                                                     C.byref(first)), "cpbus_subscribe_pairs_many")
        cap = 1 << 16
        t_out_m, out_m = pinned(cap, EVENT_DTYPE); t_out_r, out_r = pinned(cap, EVENT_DTYPE)
        offs = np.zeros(n_subs, dtype=np.uint32); cnts = np.zeros(n_subs, dtype=np.uint32)
        ready_cap = 4096
        t_rdy, rdy = pinned(ready_cap, READY_DTYPE)
        total, n_ready, nxt = C.c_size_t(), C.c_size_t(), C.c_uint32()
        got = [{}, {}]
        t_many, t_ready, calls_ready = [], [], 0

        def pump_many(bus):                  # -> (runs, seconds spent in the C call)
            t0 = time.perf_counter()
            nat.check(lib.cpbus_drain_many(bus._h, 0, n_subs, out_m.ctypes.data, cap, offs.ctypes.data, cnts.ctypes.data,
                                           C.byref(total)), "cpbus_drain_many")
            dt = time.perf_counter() - t0
            return [(int(s), out_m[int(offs[s]):int(offs[s]) + int(cnts[s])].copy()) for s in np.nonzero(cnts)[0]], dt, 1

        def pump_ready(bus):                 # -> (runs, seconds spent in the C calls, calls)
            runs, start, n_calls, dt = [], 0, 0, 0.0
            while True:
                t0 = time.perf_counter()
                nat.check(lib.cpbus_drain_ready(bus._h, 0, n_subs, start, out_r.ctypes.data, cap, rdy.ctypes.data, ready_cap,
                                                C.byref(n_ready), C.byref(total), C.byref(nxt)), "cpbus_drain_ready")
                dt += time.perf_counter() - t0
                n_calls += 1
                for e in rdy[:n_ready.value]:
                    runs.append((int(e["sub_id"]), out_r[int(e["offset"]):int(e["offset"]) + int(e["count"])].copy()))
                if not n_ready.value or nxt.value == start:   # next_sub == start_sub: everything ready was taken
                    return runs, dt, n_calls
                start = nxt.value

        for i in range(warmup + steps):
            for bus in buses:
                nat.check(bus.publish_many(host[i * B:(i + 1) * B]), "cpbus_publish"); nat.check(bus.flush(), "cpbus_flush")
                bus.sync()
            for leg in ((0, 1) if i % 2 == 0 else (1, 0)):   # alternate which path goes first
                runs, dt, n_calls = (pump_many(buses[0]) if leg == 0 else pump_ready(buses[1]))
                if i >= warmup and leg == 1:
                    calls_ready += n_calls
                if i >= warmup:
                    (t_many if leg == 0 else t_ready).append(dt)
                for s, r in runs:
                    got[leg].setdefault(s, []).append(r)
        same = got[0].keys() == got[1].keys() and all(np.concatenate(got[0][s]).tobytes() == np.concatenate(got[1][s]).tobytes()
                                                      for s in got[0])
        sample = sorted(got[1])[:4] + [int(x) for x in rng.integers(0, n_subs, 2)]
        oracle_ok = True
        for s in sample:
            o = ob.Oracle(1, keep_window=0, sub_id_base=s)
            o.subscribe(int(masks[s]), [(int(c), int(x)) for c, x in rows[s, :cnt[s]]])
            o.publish_many(host["code"], host["source_id"])
            want = o.mailbox(s).tobytes()
            oracle_ok = oracle_ok and np.concatenate(got[1].get(s, [np.zeros(0, dtype=EVENT_DTYPE)])).tobytes() == want
        delivered = sum(len(r) for parts in got[1].values() for r in parts)
        ok = ok and same and oracle_ok
        legs.append({"subscribers": n_subs, "us_per_batch_drain_many": float(np.median(t_many)) * 1e6,
                     "us_per_batch_drain_ready": float(np.median(t_ready)) * 1e6,
                     "drain_ready_calls_per_batch": calls_ready / steps, "records_per_batch": delivered / (warmup + steps),
                     "mailboxes_with_records": len(got[1]), "identical_per_subscriber": same, "oracle_sampled": sample,
                     "oracle_ok": oracle_ok})
        for bus in buses:
            bus.close()
    # dense: the `bridge` shape, both paths on one bus in alternation
    n_drain, R2 = 8192, 1024
    bus = Bus(n_drain, ring_cap=R2, batch_cap=512, digest=False, device=args.device)
    bus.subscribe_many(np.full(n_drain, nat.MASK_ALL, dtype=np.uint32))
    cap = n_drain * 512
    t_out, out = pinned(cap, EVENT_DTYPE)
    offs = np.zeros(n_drain, dtype=np.uint32); cnts = np.zeros(n_drain, dtype=np.uint32)
    t_rdy, rdy = pinned(n_drain, READY_DTYPE)
    total, n_ready, nxt = C.c_size_t(), C.c_size_t(), C.c_uint32()
    host = np.zeros(512, dtype=EVENT_DTYPE)
    host["code"] = np.arange(512) % 16 + 1
    times = [[], []]
    for rep in range(10):
        for leg in ((0, 1) if rep % 2 == 0 else (1, 0)):
            nat.check(bus.publish_many(host), "cpbus_publish"); nat.check(bus.flush(), "cpbus_flush"); bus.sync()
            t0 = time.perf_counter()
            if leg == 0:
                nat.check(lib.cpbus_drain_many(bus._h, 0, n_drain, out.ctypes.data, cap, offs.ctypes.data, cnts.ctypes.data,
                                               C.byref(total)), "cpbus_drain_many")
            else:
                nat.check(lib.cpbus_drain_ready(bus._h, 0, n_drain, 0, out.ctypes.data, cap, rdy.ctypes.data, n_drain,
                                                C.byref(n_ready), C.byref(total), C.byref(nxt)), "cpbus_drain_ready")
                ok = ok and n_ready.value == n_drain
            dt = time.perf_counter() - t0
            ok = ok and total.value == n_drain * 512
            if rep >= 2:                                           # the first calls allocate the device staging
                times[leg].append(dt)
    bus.close()
    del t_out, t_rdy
    recs = n_drain * 512
    dense = {"workload": f"{n_drain} mailboxes x 512 records -> pinned host memory",
             "drain_many_records_per_s": recs / float(np.median(times[0])),
             "drain_ready_records_per_s": recs / float(np.median(times[1]))}
    return {"name": "bridge-sparse",
            "workload": "Job-shaped fleet (exact cases per subscriber, scripts/diag_pairs.py), 512-event batches from host buffers; "
                        "after every batch the pump drains everything that arrived: cpbus_drain_many over the whole range vs "
                        "cpbus_drain_ready until nothing is ready (twin buses, alternating)",
            "unit": "us/batch (median host time of the pump step, ends in a stream sync)", "steps": steps,
            "legs": legs, "dense": dense, "parity_checked": bool(ok)}


def card(device: int):
    """Name and power limit of the card, read in the same process as the measurement."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(device), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": limit}
    except Exception:
        return {"name": torch.cuda.get_device_name(device), "power_limit": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200, help="timed batches per fleet size")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--subs", type=int, nargs="+", default=[32_768, 1_048_576])
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bridge_sparse.py: no CUDA device; cpbus has no CPU fallback")
    torch.cuda.set_device(args.device)
    res = run(args)
    res["gpu"] = card(args.device)
    print(json.dumps(res), flush=True)
    if not res["parity_checked"]:
        sys.exit(3)


if __name__ == "__main__":
    main()
