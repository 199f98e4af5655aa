"""Per-turn timeline of the matcher's commit chain on C2 and on its non-saturating variant (GPU box).

Runs the PROF instantiation (COOK_PROF=1) with COOK_PROF_TRACE set, so the kernel stamps every queue
entry's turn with clock64 on the resolver SM, and splits each turn's wall time
T_done(g) - T_done(g-1) into:
  (a) owner late      T_ready > T_done(g-1): the owner's top-3 was not built yet
                      (a_land: the result itself landed after T_done(g-1); a_look: it landed in time)
  (b) hand-off        T_seen - max(T_done(g-1), T_ready): from turn g-1's chain word and mbarrier arrive
                      to the next owner's turn; split on the turns whose owner was ready in time into
                        detect   T_hand - T_done(g-1): until the owner learned that turn g-1 had ended
                        rest     T_seen - T_hand: from there to the start of the turn body
                      with how often the owner waited for a turn to end before T_hand and whether it
                      learned of the turn right after folding an older entry (mid-fold)
  (c) turn body       T_done - T_seen
  (d) END turns       the whole wall time of end-of-block entries
  (e) block boundary  the part of (a) before the driver saw every row of the turn's block scored
The terms add up to the chain's wall time exactly.  Prints the card, power limit and SM clock read in
the same run.  COOK_GPU_LIB selects an A/B build of the library.

usage: python tools/prof_turn.py [--out DIR] [--only c2|nonsat]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cook_b200 import traces  # noqa: E402
from cook_b200.engine import GpuEngine  # noqa: E402

TT_FREE, TT_LAND, TT_READY, TT_SEEN, TT_DONE, TT_FENCE, TT_INFO, TT_K, TT_EVAL, TT_DEC, TT_HAND, TT_POLL = range(12)
PATHS = ["exact", "take_z", "fallback", "group"]
TERMS = ["a_land", "a_look", "b_handoff", "c_body", "d_end", "e_block"]


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError):
        out = []
    return out[0] if out else "unknown"


def read_trace(path):
    raw = np.fromfile(path, dtype=np.uint64)
    assert raw[0] == 0x314e5254, "not a turn trace"
    n_turn, n_blk, words = int(raw[1]), int(raw[2]), int(raw[3])
    hdr = {"res_total": int(raw[4]), "n_cons": int(raw[5]), "matched": int(raw[6])}
    turns = raw[8:8 + n_turn * words].reshape(n_turn, words).astype(np.int64)
    blk = raw[8 + n_turn * words:8 + n_turn * words + n_blk].astype(np.int64)
    return hdr, turns, blk


def split(hdr, T, blk):
    """Per-turn terms (cycles) for every turn g >= 1 whose predecessor was recorded."""
    n = int(np.nonzero(T[:, TT_DONE])[0].max()) + 1
    T = T[:n]
    assert (T[:, TT_DONE] != 0).all(), "a turn of the chain was not recorded"
    info = T[:, TT_INFO]
    is_end = (info & 0xF) == 1
    b = info >> 32
    prev = np.concatenate([[T[0, TT_FREE]], T[:-1, TT_DONE]])
    wall = T[:, TT_DONE] - prev
    ready, land, seen, done = T[:, TT_READY], T[:, TT_LAND], T[:, TT_SEEN], T[:, TT_DONE]
    late = np.maximum(ready - prev, 0)
    rows_at = blk[np.minimum(b, len(blk) - 1)]
    e = np.where(rows_at > 0, np.clip(rows_at - prev, 0, late), 0)
    a = late - e
    land_late = land > prev
    t = {
        "a_land": np.where(~is_end & land_late, a, 0),
        "a_look": np.where(~is_end & ~land_late, a, 0),
        "b_handoff": np.where(is_end, 0, seen - np.maximum(prev, ready)),
        "c_body": np.where(is_end, 0, done - seen),
        "d_end": np.where(is_end, wall, 0),
        "e_block": np.where(is_end, 0, e),
    }
    chk = sum(t.values())
    assert (chk == wall).all(), "the terms do not add up to the wall time"
    job = ~is_end
    # the first quarter of the queue: turns up to the last job with k < n_cons / 4
    k = T[:, TT_K]
    q1_end = int(np.nonzero(job & (k < hdr["n_cons"] // 4))[0].max()) + 1 if (job & (k < hdr["n_cons"] // 4)).any() else 0
    q1 = np.arange(n) < q1_end
    ev, dec = T[:, TT_EVAL], T[:, TT_DEC]
    fast = job & (ev > 0) & (dec > 0) & (((info >> 4) & 0xF) == 0) & (((info >> 8) & 0xF) == 0)
    extra = {
        # (c) split, exact-path turns without a relook: newest entry loaded and evaluated / decided / appended
        "body_eval": np.where(fast, ev - seen, 0),
        "body_decide": np.where(fast, dec - ev, 0),
        "body_append": np.where(fast, done - dec, 0),
        "first_look": np.where(job, ready - land, 0),      # off the chain: result landed -> top-3 built
        "wait_result": np.where(job, land - T[:, TT_FREE], 0),
        "end_fence": np.where(is_end, done - T[:, TT_FENCE], 0),
        "end_publish": np.where(is_end, T[:, TT_FENCE] - seen, 0),
        "end_handoff": np.where(is_end, seen - np.maximum(prev, ready), 0),
    }
    # (b) split: job turns whose owner was ready before turn g-1 ended and learned of its end afterwards
    # TT_HAND holds the low word of the clock: its distance from T_done(g-1) is taken modulo 2^32
    detect = (T[:, TT_HAND] - prev) & 0xFFFFFFFF
    in_time = job & (ready <= prev) & (((T[:, TT_HAND] >> 32) & 1) == 1) & (detect < 1 << 31)
    extra["hand_detect"] = np.where(in_time, detect, 0)
    extra["hand_rest"] = np.where(in_time, seen - prev - detect, 0)
    extra["hand_waits"] = np.where(in_time, T[:, TT_POLL] & 0xFFFFFFFF, 0)
    extra["hand_midfold"] = np.where(in_time, (T[:, TT_POLL] >> 32) & 1, 0)
    return dict(n=n, wall=wall, terms=t, extra=extra, job=job, is_end=is_end, q1=q1, info=info, fast=fast, in_time=in_time,
                placed=job & (((info >> 21) & 1) == 1), land_late=land_late)


def summarise(name, hdr, S, mhz):
    out = {"workload": name, "turns": int(S["n"]), "job_turns": int(S["job"].sum()), "end_turns": int(S["is_end"].sum()),
           "placements": int(S["placed"].sum()), "res_total_cycles": hdr["res_total"]}
    chain = int(S["wall"][1:].sum())
    out["chain_cycles"] = chain
    out["chain_share_of_resolver"] = chain / max(1, hdr["res_total"])
    out["cycles_per_placement"] = chain / max(1, out["placements"])
    out["us_per_placement_at_clock"] = out["cycles_per_placement"] / mhz if mhz else None

    def block(sel):
        sel = sel.copy()
        sel[0] = False
        tot = S["wall"][sel].sum()
        npl = max(1, int((S["placed"] & sel).sum()))
        r = {"placements": int((S["placed"] & sel).sum()), "cycles": int(tot), "cycles_per_placement": tot / npl, "terms": {},
             "in_time_turns": int((S["in_time"] & sel).sum())}
        for nm in TERMS:
            v = S["terms"][nm][sel]
            jv = S["terms"][nm][sel & (S["is_end"] if nm == "d_end" else S["job"])]
            r["terms"][nm] = {"per_placement": float(v.sum()) / npl, "share": float(v.sum()) / max(1, tot),
                              "p50": float(np.percentile(jv, 50)) if len(jv) else 0.0,
                              "p90": float(np.percentile(jv, 90)) if len(jv) else 0.0,
                              "p99": float(np.percentile(jv, 99)) if len(jv) else 0.0}
        for nm, v in S["extra"].items():
            kind = (S["is_end"] if nm.startswith("end") else S["fast"] if nm.startswith("body") else
                    S["in_time"] if nm.startswith("hand") else S["job"])
            sv = v[sel & kind]
            r.setdefault("diag", {})[nm] = {"mean": float(sv.mean()) if len(sv) else 0.0,
                                            "p50": float(np.percentile(sv, 50)) if len(sv) else 0.0}
        return r

    allsel = np.ones(S["n"], bool)
    out["all"] = block(allsel)
    out["q1"] = block(S["q1"])
    out["rest"] = block(~S["q1"])
    j = S["job"]
    info = S["info"]
    path = (info >> 4) & 0xF
    out["paths"] = {p: int((j & (path == i)).sum()) for i, p in enumerate(PATHS)}
    out["relooks"] = int(((info >> 8) & 0xF)[j].sum())
    out["slow_turns"] = int((j & (((info >> 20) & 1) == 1)).sum())
    fold = (info >> 12) & 0xFF
    out["folded_hist"] = {int(x): int(c) for x, c in zip(*np.unique(fold[j], return_counts=True))}
    out["result_landed_late"] = int((j & S["land_late"]).sum())
    return out


def show(r, mhz):
    print(f"== {r['workload']}: {r['turns']} turns ({r['job_turns']} job, {r['end_turns']} END), "
          f"{r['placements']} placements; chain {r['chain_cycles']} cycles = {100 * r['chain_share_of_resolver']:.1f} % "
          f"of the resolver's run; {r['cycles_per_placement']:.0f} cycles/placement"
          + (f" = {r['us_per_placement_at_clock']:.3f} us at {mhz} MHz" if mhz else ""))
    print(f"   paths {r['paths']}  relooks {r['relooks']}  slow turns {r['slow_turns']}  "
          f"results landed after the previous turn {r['result_landed_late']}")
    print(f"   entries folded one by one before the turn: {r['folded_hist']}")
    for part in ("all", "q1", "rest"):
        p = r[part]
        print(f"   [{part}] {p['placements']} placements, {p['cycles_per_placement']:.0f} cycles/placement")
        for nm in TERMS:
            x = p["terms"][nm]
            print(f"      {nm:10s} {x['per_placement']:8.1f} cyc/placement {100 * x['share']:5.1f} %   "
                  f"per turn p50 {x['p50']:7.0f} p90 {x['p90']:7.0f} p99 {x['p99']:8.0f}")
        print("      diag " + "  ".join(f"{k} mean {v['mean']:.0f} p50 {v['p50']:.0f}" for k, v in p["diag"].items()
                                   if not k.startswith("hand")))
        h = p["diag"]
        print(f"      (b) split over {p['in_time_turns']} turns with the owner ready in time: "
              f"detect mean {h['hand_detect']['mean']:.0f} p50 {h['hand_detect']['p50']:.0f}, "
              f"rest mean {h['hand_rest']['mean']:.0f} p50 {h['hand_rest']['p50']:.0f} cycles; "
              f"waits mean {h['hand_waits']['mean']:.1f} p50 {h['hand_waits']['p50']:.0f}; "
              f"mid-fold {100 * h['hand_midfold']['mean']:.1f} %")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="write the summaries as JSON into this directory")
    ap.add_argument("--only", choices=["c2", "nonsat"], default=None)
    args = ap.parse_args()
    cardinfo = card()
    print("card (name, power limit, SM clock, max SM clock):", cardinfo, flush=True)
    try:
        mhz = int(cardinfo.split(",")[2].strip().split()[0])
    except (IndexError, ValueError):
        mhz = None
    runs = [("c2", dict()), ("nonsat", dict(offer_scale=6))]
    results = []
    tmp = tempfile.mkdtemp(prefix="cook_turn_")
    for name, kw in runs:
        if args.only and args.only != name:
            continue
        t = traces.gen_c2(seed=2, **kw)
        eng = GpuEngine(pool_name="turns-" + name)
        ranked = eng.rank(t["running"], t["pending"], t["users"])["ranked"]
        prm = traces.match_params(t["jobs"].n)
        os.environ.pop("COOK_PROF", None)
        os.environ.pop("COOK_PROF_TRACE", None)
        ref = eng.match(ranked, t["jobs"], t["offers"], t["users"], prm)["assign"].copy()
        ms = [eng.match(ranked, t["jobs"], t["offers"], t["users"], prm)["stats"]["ms_match_kernel"] for _ in range(3)]
        os.environ["COOK_PROF"] = "1"
        path = os.path.join(tmp, name + ".bin")
        os.environ["COOK_PROF_TRACE"] = path
        eng.match(ranked, t["jobs"], t["offers"], t["users"], prm)   # module load of the PROF kernel
        m = eng.match(ranked, t["jobs"], t["offers"], t["users"], prm)
        os.environ.pop("COOK_PROF", None)
        os.environ.pop("COOK_PROF_TRACE", None)
        same = bool((m["assign"] == ref).all())
        hdr, T, blk = read_trace(path)
        r = summarise(name, hdr, split(hdr, T, blk), mhz)
        r["kernel_ms_plain"] = [round(x, 3) for x in ms]
        r["kernel_ms_traced"] = round(m["stats"]["ms_match_kernel"], 3)
        r["same_assign_as_plain"] = same
        r["card"] = cardinfo
        print(f"-- {name}: plain kernel ms {r['kernel_ms_plain']}, traced {r['kernel_ms_traced']}, "
              f"assignments {'identical' if same else 'DIFFERENT'}", flush=True)
        show(r, mhz)
        results.append(r)
        eng.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "prof_turn.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
