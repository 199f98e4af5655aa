"""The gather step's cost (DESIGN.md §9a): cook_state_user_stats, cook_state_instance_stats, cook_state_history_stats and
cook_state_list_completed over several pools as handles, with every handle on device 0 (the one-device path), with
COOK_STAGE_HANDLES=1 (every handle after the first compacts on its own stream and its rows are copied to the first
handle's range with cudaMemcpyPeerAsync), and, when two devices are visible, with the handles on two devices.

  python tools/measure_multidevice.py --config c3              # config #3's four pools as four handles
  python tools/measure_multidevice.py --config c5 --scale 0.2  # config #5's sixteen pools, placed by sharding.py

For config #5 the handles are ordered by sharding.assign_pools_lpt's placement on two GPUs, the first GPU's pools
first; the first handle is the leader.  Per call and arm it prints the median over --reps calls (after 3 warm-up
calls) of the device time (the call's own CUDA events on the leader's stream: upload + device + download) and the
wall time of the binding call, the launches, and whether the answer equals the one-device answer bit for bit.  The
card line carries the GPU's name and power limit; the numbers are only meaningful beside it.
"""
import argparse
import json
import os
import struct
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cook_b200 import abi, engine, sharding, traces  # noqa: E402
from cook_b200.engine import GpuEngine  # noqa: E402

STAGE = "COOK_STAGE_HANDLES"
DAY_MS = 86_400_000


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                                       "--format=csv,noheader"], text=True)
        return out.strip().splitlines()
    except Exception as e:   # noqa: BLE001
        return [f"unknown ({e})"]


def device_count():
    import torch
    return torch.cuda.device_count()


def canon(x):
    if isinstance(x, dict):
        return {k: canon(v) for k, v in sorted(x.items()) if k != "stats"}
    if isinstance(x, np.ndarray):
        return (str(x.dtype), x.shape, x.tobytes())
    if isinstance(x, (list, tuple)):
        return [canon(v) for v in x]
    if isinstance(x, float):
        return struct.unpack("<q", struct.pack("<d", x))[0]
    return x


def load(ts, devices, rng):
    """One handle per trace pool on devices[p]: its running and pending rows, reason and unknown facts, a history of
    as many finished rows as it runs tasks over 31 days, and a completed-job log of as many records as it has jobs."""
    es = []
    t_end = 1_700_000_000_000
    for p, (t, d) in enumerate(zip(ts, devices)):
        run = {k: np.asarray(v).copy() for k, v in t["cols"]["running"].items()}
        pc = t["cols"]["pending"]
        n, J = len(run["task_id"]), t["jobs"].n
        e = GpuEngine(pool_name=f"md-{p}", device=d)
        e.state_apply(abi.make_delta(reset=True, running=abi.make_tasks(**run), pending=t["jobs"],
                                     pending_priority=pc["priority"], pending_job_id=pc["job_id"]))
        e.state_task_reason(run["task_id"], np.where(rng.random(n) < 0.1, rng.choice([1001, 2003], n), -1))
        e.state_task_facts(run["task_id"], unknown=(rng.random(n) < 0.05).astype(np.uint8))
        k = rng.integers(0, n, n)
        start = np.sort(rng.integers(t_end - 31 * DAY_MS, t_end, n))
        e.state_history_seed(t_end - 31 * DAY_MS, task_id=np.arange(n, dtype=np.int64) + 10 ** 12 + 10 ** 9 * p,
                             user=run["user"][k], start_ms=start, end_ms=start + rng.integers(0, 7_200_000, n),
                             cpus=np.asarray(run["cpus"], np.float64)[k], mem=np.asarray(run["mem"], np.float64)[k],
                             success=(rng.random(n) < 0.7).astype(np.uint8),
                             reason_code=np.where(rng.random(n) < 0.3, 3001, -1))
        users = np.asarray(pc["user"], np.int32)
        e.state_completed_seed(t_end - 32 * DAY_MS, np.asarray(pc["job_id"], np.int64) + 10 ** 10 * p,
                               np.arange(J, dtype=np.int64), users,
                               np.sort(rng.integers(t_end - 32 * DAY_MS, t_end, J)), np.full(J, p, np.int32),
                               np.zeros(J, np.int32), np.where(rng.random(J) < 0.7, 1, 2).astype(np.uint8))
        es.append(e)
    return es, t_end


def calls(es, ts, t_end):
    U = max(t["users"].n_users for t in ts)
    users = abi.make_users(U)
    heavy = int(np.bincount(np.concatenate([np.asarray(t["cols"]["pending"]["user"]) for t in ts])).argmax())
    return {
        "user_stats": lambda: engine.state_user_stats(es, users),
        "instance_stats": lambda: engine.state_instance_stats(es, t_end + 10 ** 9, abi.IS_RUNNING, 0, t_end + 10 ** 9),
        "history_stats": lambda: engine.state_history_stats(es, abi.IS_SUCCESS, t_end - 31 * DAY_MS, t_end),
        "history_stats_day": lambda: engine.state_history_stats(es, abi.IS_SUCCESS, t_end - DAY_MS, t_end),
        "list_completed": lambda: engine.state_list_completed(es, heavy, abi.LC_COMPLETED, t_end - 7 * DAY_MS, t_end,
                                                              cap=1 << 20),
    }


def timed(fn, reps):
    for _ in range(3):
        got = fn()
    dev, wall = [], []
    for _ in range(reps):
        w0 = time.perf_counter()
        got = fn()
        wall.append(time.perf_counter() - w0)
        s = got["stats"]
        dev.append(s["ms_h2d"] + s["ms_device"] + s["ms_d2h"])
    return got, float(np.median(dev)), 1e3 * float(np.median(wall))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", choices=["c3", "c5"], default="c3")
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--seed", type=int, default=7)
    a = ap.parse_args()
    n_pools = 4 if a.config == "c3" else 16
    ts = [traces.gen_config_pool(a.config, p, scale=a.scale) for p in range(n_pools)]
    if a.config == "c5":   # LPT on two GPUs, the first GPU's pools first
        gpu_of = sharding.assign_pools_lpt([sharding.pool_cycle_cost(t["jobs"].n, t["offers"].n) for t in ts], 2)
        order = sorted(range(n_pools), key=lambda p: (gpu_of[p], p))
    else:
        gpu_of, order = [p % 2 for p in range(n_pools)], list(range(n_pools))
    ts = [ts[p] for p in order]
    place = [gpu_of[p] for p in order]
    two = device_count() >= 2
    print(json.dumps({"card": card(), "config": a.config, "scale": a.scale, "handles": n_pools,
                      "running": sum(len(t["cols"]["running"]["task_id"]) for t in ts),
                      "pending": sum(t["jobs"].n for t in ts), "placement": place, "devices_visible": device_count()}),
          flush=True)
    arms = [("one_device", [0] * n_pools, None), ("staged", [0] * n_pools, "1")]
    if two:
        arms.append(("two_devices", place, None))
    base = {}
    for arm, devices, env in arms:
        os.environ.pop(STAGE, None)
        if env:
            os.environ[STAGE] = env
        es, t_end = load(ts, devices, np.random.default_rng(a.seed))
        for name, fn in calls(es, ts, t_end).items():
            got, dev, wall = timed(fn, a.reps)
            same = base.setdefault(name, canon(got)) == canon(got)
            print(json.dumps({"arm": arm, "call": name, "device_ms": round(dev, 4), "wall_ms": round(wall, 4),
                              "n_launches": got["stats"]["n_launches"], "identical_to_one_device": same}), flush=True)
        for e in es:
            e.close()
    os.environ.pop(STAGE, None)
    if not two:
        print(json.dumps({"two_devices": "not measured: one device visible"}), flush=True)


if __name__ == "__main__":
    main()
