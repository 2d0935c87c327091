"""Host µs per pump step of the acknowledged drain (cpbus_take_ready until nothing is ready, then one cpbus_ack_many of
everything taken) against the plain one (cpbus_drain_ready until nothing is ready), alternated in one run.

The fleet is the Job-shaped one of scripts/bridge_sparse.py (exact {code, source} cases per subscriber), on twin lossless
buses (512-record rings).  Each step publishes one 512-event batch from a host buffer to both buses and flushes, then pumps
each bus with its path, alternating which goes first; the C functions are called directly on preallocated pinned buffers,
as a shim would.  Parity: both paths return byte-identical records and ready lists at every step.  Rows give, per fleet
size, the median over the steps of each round, then the median and min..max of those over the rounds; the take + ack path
is also split into its take and ack parts.  With --profile, a separate run under torch.profiler gives the device time of
each kernel and copy of both paths.  Prints one JSON line naming the card and its power limit; exits 3 when a
parity check fails.  A run without a GPU stops.

  python scripts/diag_take_ack.py [--steps 200 --warmup 10 --rounds 3 --subs 32768 1048576] [--profile 50] [--out FILE]
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import numpy as np
import torch

from bridge_sparse import job_fleet
from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus, EVENT_DTYPE, READY_DTYPE

B, R = 512, 512


def _card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return out[0] if out else "unknown card"


def _pinned(n, dtype):
    t = torch.empty((n * dtype.itemsize,), dtype=torch.uint8).pin_memory()
    return t, t.numpy().view(dtype)


def run_fleet(n_subs, steps, warmup, rounds, device, profile):
    lib = nat.load()
    masks, rows, cnt, n_src = job_fleet(n_subs)
    buses = [Bus(n_subs, ring_cap=R, batch_cap=R // 2, digest=False, lossless=True, device=device) for _ in range(2)]
    for bus in buses:
        first = C.c_uint32()
        nat.check(lib.cpbus_subscribe_pairs_many(bus._h, masks.ctypes.data, rows.ctypes.data, cnt.ctypes.data, n_subs,
                                                 C.byref(first)), "cpbus_subscribe_pairs_many")
    cap, ready_cap = 1 << 16, 4096
    keep = []
    outs, rdys = [], []
    for _ in range(2):
        t, o = _pinned(cap, EVENT_DTYPE); keep.append(t); outs.append(o)
        t, r = _pinned(ready_cap, READY_DTYPE); keep.append(t); rdys.append(r)
    n_ready, total, nxt = C.c_size_t(), C.c_size_t(), C.c_uint32()
    ack_ids, ack_cnt = np.zeros(n_subs, dtype=np.uint32), np.zeros(n_subs, dtype=np.uint32)
    applied = C.c_uint32()

    def pump(k):   # k = 0: drain_ready; 1: take_ready + ack_many.  -> (runs, seconds, take seconds, ack seconds)
        bus, out, rdy = buses[k], outs[k], rdys[k]
        fn = lib.cpbus_take_ready if k else lib.cpbus_drain_ready
        runs, start, n_ack, t_take = [], 0, 0, 0.0
        while True:
            t0 = time.perf_counter()
            nat.check(fn(bus._h, 0, n_subs, start, out.ctypes.data, cap, rdy.ctypes.data, ready_cap, C.byref(n_ready),
                         C.byref(total), C.byref(nxt)), "take/drain_ready")
            t_take += time.perf_counter() - t0
            got = rdy[:n_ready.value]
            runs.append((got.tobytes(), out[:total.value].tobytes()))
            if k:
                ack_ids[n_ack:n_ack + len(got)] = got["sub_id"]; ack_cnt[n_ack:n_ack + len(got)] = got["count"]
                n_ack += len(got)
            if not n_ready.value or nxt.value == start:
                break
            start = nxt.value
        t_ack = 0.0
        if k and n_ack:
            t0 = time.perf_counter()
            nat.check(lib.cpbus_ack_many(bus._h, ack_ids.ctypes.data, ack_cnt.ctypes.data, n_ack, None, C.byref(applied)),
                      "cpbus_ack_many")
            t_ack = time.perf_counter() - t0
            if applied.value != n_ack:
                raise SystemExit(3)
        return runs, t_take + t_ack, t_take, t_ack

    rng = np.random.default_rng(0xAC4 + n_subs)
    per_round, ok, records = [], True, 0
    for rnd in range(rounds):
        host = np.zeros((warmup + steps) * B, dtype=EVENT_DTYPE)
        host["code"] = rng.integers(1, 17, len(host)); host["source_id"] = rng.integers(0, n_src, len(host))
        t = {"drain_ready": [], "take_ack": [], "take": [], "ack": []}
        for i in range(warmup + steps):
            batch = host[i * B:(i + 1) * B]
            for bus in buses:
                nat.check(bus.publish_many(batch), "publish"); nat.check(bus.flush(), "flush")
            res = [None, None]
            for k in ((0, 1) if (i + rnd) % 2 == 0 else (1, 0)):
                res[k] = pump(k)
            ok &= res[0][0] == res[1][0]
            if i >= warmup:
                records += sum(len(r[1]) // 32 for r in res[0][0])
                t["drain_ready"].append(res[0][1]); t["take_ack"].append(res[1][1])
                t["take"].append(res[1][2]); t["ack"].append(res[1][3])
        per_round.append({k: float(np.median(v)) * 1e6 for k, v in t.items()})
    kernels = {}
    if profile:   # device time of each kernel and copy of both paths, in a run of its own after the timed rounds
        from torch.profiler import ProfilerActivity, profile as prof_ctx
        host = np.zeros(profile * B, dtype=EVENT_DTYPE)
        host["code"] = rng.integers(1, 17, len(host)); host["source_id"] = rng.integers(0, n_src, len(host))
        with prof_ctx(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(profile):
                for k, bus in enumerate(buses):
                    nat.check(bus.publish_many(host[i * B:(i + 1) * B]), "publish"); nat.check(bus.flush(), "flush")
                    pump(k)
        for e in prof.key_averages():
            name = e.key
            if any(s in name for s in ("ready_scan", "gather", "ack_kernel", "Memcpy", "Memset")):
                kernels[name[:60]] = {"count": e.count, "avg_us": round(e.device_time_total / max(e.count, 1), 2)}
    for bus in buses:
        bus.close()
    summary = {}
    for k in per_round[0]:
        v = [r[k] for r in per_round]
        summary[k] = {"median_us": round(float(np.median(v)), 1), "min_us": round(min(v), 1), "max_us": round(max(v), 1)}
    summary["ratio"] = round(summary["take_ack"]["median_us"] / summary["drain_ready"]["median_us"], 3)
    return {"subs": n_subs, "records_per_step": round(records / (rounds * steps), 1), "parity": bool(ok),
            "rounds": per_round, "summary": summary, "device": kernels}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--subs", type=int, nargs="+", default=[32768, 1048576])
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--profile", type=int, default=0, metavar="STEPS",
                    help="also run STEPS pump steps of both paths under torch.profiler and report device time per kernel and copy")
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: this script measures on the device")
    legs = [run_fleet(n, args.steps, max(args.warmup, 3), args.rounds, args.device, args.profile) for n in args.subs]
    rec = {"card": _card(), "batch": B, "ring_cap": R, "steps": args.steps, "legs": legs}
    line = json.dumps(rec)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    if not all(leg["parity"] for leg in legs):
        raise SystemExit(3)


if __name__ == "__main__":
    main()
