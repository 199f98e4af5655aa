"""Plain restatements of dru/sorted-merge (dru.clj:82-104) and builders of per-user score tables with
chosen runs of equal scores, for the tests of LessMerge (cook_b200/csrc/fold.cuh) and of cook_rank's merge
order.

A table is what cook_rank holds after its per-user fold: users in name order, each with its tasks in queue
order and a score per task (NaN for the tasks limit-over-quota-jobs cuts).  Position p is the p-th task of
that layout; segment k belongs to user perm[k], so segment order differs from user id."""
import heapq

import numpy as np

from cook_b200 import abi


def sorted_merge(colls, score):
    """dru.clj:89-94 literally: every step stable-sorts the remaining seqs by the score of their first item
    (`sort-by` is stable), yields the first item of the first seq and conses that seq's remainder to the
    FRONT of the others.  colls: lists of items, users in name order; score(item): a float, not NaN."""
    colls = [list(c) for c in colls if len(c)]
    out = []
    while colls:
        colls = sorted(colls, key=lambda c: score(c[0]))
        (y, *rest), others = colls[0], colls[1:]
        out.append(y)
        colls = ([rest] if rest else []) + others
    return out


def heap_merge(colls, score):
    """The same order from a heap keyed (score, newest arrival first, name): arrival is the step at which
    the user's previous item was emitted, 0 for its first."""
    heap = [(score(c[0]), 0, k, 0) for k, c in enumerate(colls) if len(c)]
    heapq.heapify(heap)
    out, step = [], 0
    while heap:
        _, _, k, i = heapq.heappop(heap)
        out.append(colls[k][i])
        step += 1
        if i + 1 < len(colls[k]):
            heapq.heappush(heap, (score(colls[k][i + 1]), -step, k, i + 1))
    return out


def _divs(div):
    """(cpus, mem) divisors of a user: one number stands for both."""
    return (div, div) if np.isscalar(div) else div


def left_fold_scores(mode, amounts, div, kept):
    """The scores of one user's tasks (dru.clj:50-80): running sums in queue order, one divide each; mode 0
    max(mem / div_mem, cpus / div_cpus) over (cpus, mem) pairs (clojure.core/max of a NaN from 0 / 0 and
    a number is the number), mode 1 gpus / div.  Tasks from `kept` on are NaN."""
    out = []
    acc = [np.float64(0.0), np.float64(0.0)]
    with np.errstate(divide="ignore", invalid="ignore"):
        for i, a in enumerate(amounts):
            if i >= kept:
                out.append(np.nan)
                continue
            if mode == 0:
                dc, dm = _divs(div)
                acc = [acc[0] + np.float64(a[0]), acc[1] + np.float64(a[1])]
                x, y = acc[1] / np.float64(dm), acc[0] / np.float64(dc)   # mem, cpus
                out.append(float(x if x > y else y))
            else:
                acc[0] = acc[0] + np.float64(a)
                out.append(float(acc[0] / np.float64(div)))
    return out


def table(users, mode=1, perm=None):
    """users: per user in name order, a dict with `amounts` (mode 1: gpus per task; mode 0: (cpus, mem) per
    task), `div` (the user's share of that resource; 0 gives +inf scores) and optionally `kept` (how many
    tasks survive limit-over-quota-jobs).  perm[k] is the user id of segment k (a permutation)."""
    U = len(users)
    perm = np.arange(U) if perm is None else np.asarray(perm)
    dru, user_at, lists = [], [], []
    seg_start = np.zeros(U, np.int32)
    seg_end = np.zeros(U, np.int32)
    name_rank = np.zeros(U, np.int32)
    for k, u in enumerate(users):
        uid = int(perm[k])
        kept = len(u["amounts"]) if u.get("kept") is None else u["kept"]
        s = len(dru)
        seg_start[uid], name_rank[uid] = s, k
        sc = left_fold_scores(mode, u["amounts"], u["div"], kept)
        lists.append(list(range(s, s + kept)))
        dru += sc
        user_at += [uid] * len(sc)
        seg_end[uid] = len(dru)
    dru = np.array(dru, np.float64)
    cut = [p for p in range(len(dru)) if dru[p] != dru[p]]
    return dict(users=users, mode=mode, perm=perm, dru=dru, user_at=np.array(user_at, np.int32),
                seg_start=seg_start, seg_end=seg_end, name_rank=name_rank, lists=lists,
                merge=sorted_merge(lists, lambda p: dru[p]), cut=cut)


def expected_positions(t):
    """LessMerge's order of every position: the merge, then the cut tasks in position order."""
    return np.array(t["merge"] + t["cut"], np.int32)


# ---- tables with chosen runs of equal scores
def hand_case():
    """Users A < B, two tasks each, all four scores equal: the merge emits a1 a2 b1 b2."""
    return table([dict(amounts=[0.0, 0.0], div=1.0), dict(amounts=[0.0, 0.0], div=1.0)])


def structured_gpu_table(perm_seed=None):
    """GPU mode, scores on a small integer grid so that runs meet runs of other users: a run at the start,
    in the middle and at the end of a list, a whole list as one run, a run right after the first task, a
    run just before an over-quota tail, single-task users."""
    users = [
        dict(amounts=[0, 0, 0, 1, 1], div=1.0),             # run at the start (score 0)
        dict(amounts=[1, 1, 0, 0, 1], div=1.0),             # run in the middle (2 2 2)
        dict(amounts=[1, 1, 1, 0, 0], div=1.0),             # run at the end (3 3 3)
        dict(amounts=[2, 0, 0, 0], div=1.0),                # whole list one run (2)
        dict(amounts=[1, 2, 0, 0], div=1.0),                # run right after the first task (1, 3 3 3)
        dict(amounts=[1, 1, 0, 4, 4], div=1.0, kept=3),     # run (2 2) just before a cut tail
        dict(amounts=[2], div=1.0),                         # single task
        dict(amounts=[0], div=1.0),                         # single task, score 0
        dict(amounts=[6, 0], div=2.0),                      # 3 3 through another share
        dict(amounts=[1, 0, 1, 0, 1, 0], div=1.0),          # runs of two: 1 1 2 2 3 3
        dict(amounts=[0, 0, 0, 0, 0, 0, 0], div=4.0),       # a long run of 0
        dict(amounts=[1, 0, 1, 0, 1], div=1.0, kept=2),     # 1 1, then cut
    ]
    perm = None if perm_seed is None else np.random.default_rng(perm_seed).permutation(len(users))
    return table(users, 1, perm)


def inf_default_table(perm_seed=None):
    """Default mode: users with a zero share score +inf on every task (one run), beside ordinary users and
    users with a zero mem share whose first tasks ask for no mem (finite scores, then a run of +inf that
    arrives late and so goes before the runs that start a list)."""
    users = [
        dict(amounts=[(1.0, 100.0), (1.0, 100.0)], div=0.0),
        dict(amounts=[(1.0, 0.0), (1.0, 8.0), (2.0, 1.0)], div=(1.0, 0.0)),   # 1 inf inf
        dict(amounts=[(1.0, 0.0), (1.0, 0.0), (1.0, 2.0)], div=(2.0, 0.0)),   # 0.5 1 inf
        dict(amounts=[(1.0, 0.0), (2.0, 5.0), (1.0, 1.0)], div=1.0),
        dict(amounts=[(2.0, 1.0)] * 4, div=0.0),
        dict(amounts=[(1.0, 1.0), (1.0, 1.0), (0.0, 0.0)], div=1.0),     # 1 2 2
        dict(amounts=[(0.5, 3.0)], div=0.0),
        dict(amounts=[(4.0, 1.0), (1.0, 1.0), (1.0, 1.0)], div=2.0, kept=2),
    ]
    perm = None if perm_seed is None else np.random.default_rng(perm_seed).permutation(len(users))
    return table(users, 0, perm)


def random_gpu_table(seed, n_users, max_len, frac_zero, frac_cut=0.2, divs=(1.0, 2.0, 4.0)):
    """GPU mode with random lists: gpus 0 with probability frac_zero, else 1, 2 or 4; some users cut."""
    rng = np.random.default_rng(seed)
    users = []
    for _ in range(n_users):
        n = int(rng.integers(1, max_len + 1))
        g = np.where(rng.random(n) < frac_zero, 0.0, rng.choice([1.0, 2.0, 4.0], n))
        kept = int(rng.integers(0, n + 1)) if rng.random() < frac_cut else None
        users.append(dict(amounts=[float(x) for x in g], div=float(rng.choice(divs)), kept=kept))
    return table(users, 1, rng.permutation(n_users))


def tie_tables():
    """Every hand-built tie table, by name."""
    out = {"hand": hand_case(), "structured": structured_gpu_table(), "structured_perm": structured_gpu_table(5),
           "inf_default": inf_default_table(), "inf_default_perm": inf_default_table(6)}
    for seed, (nu, ml, fz) in enumerate([(3, 5, 0.5), (17, 12, 0.3), (9, 25, 0.7), (2, 100, 0.5), (40, 6, 1.0),
                                         (25, 10, 0.0), (1, 60, 0.6), (60, 4, 0.5)]):
        out[f"random{seed}"] = random_gpu_table(100 + seed, nu, ml, fz)
    return out


def table_ranking(t, seed=0, off_grid=False):
    """The ABI inputs that make cook_rank hold table t: every task pending, queue order by job id, the
    columns in a shuffled input order.  Returns (pending, users, params, pos) where pos[i] is the position
    of input task i; a cut tail comes from quota_count = kept with max_over_quota_jobs = 0.  off_grid (GPU
    mode only): cpus of 1.1, which no score reads but which keep the sums off the exact grid."""
    assert not (off_grid and t["mode"] == 0)
    rng = np.random.default_rng(seed)
    n, U = len(t["dru"]), len(t["users"])
    cpus, mem, gpus = np.full(n, 1.1 if off_grid else 1.0), np.ones(n), np.zeros(n)
    qcount = np.full(U, np.finfo(np.float64).max)
    div_cpus, div_mem = np.zeros(U), np.zeros(U)
    for k, u in enumerate(t["users"]):
        uid, s = int(t["perm"][k]), int(t["seg_start"][int(t["perm"][k])])
        div_cpus[uid], div_mem[uid] = _divs(u["div"])
        for i, a in enumerate(u["amounts"]):
            if t["mode"] == 0:
                cpus[s + i], mem[s + i] = a
            else:
                gpus[s + i] = a
        if u.get("kept") is not None:
            qcount[uid] = u["kept"]
    inp = rng.permutation(n)                  # input task i sits at position inp[i]
    cols = dict(user=t["user_at"][inp], priority=np.full(n, 50, np.int32), start_time=np.full(n, abi.INT64_MAX),
                task_id=np.full(n, -1, np.int64), job_id=(1000 + inp).astype(np.int64) * 2,
                cpus=cpus[inp], mem=mem[inp], gpus=gpus[inp])
    pending = abi.make_tasks(**cols)
    users = abi.make_users(U, name_rank=t["name_rank"], div_mem=div_mem, div_cpus=div_cpus, div_gpus=div_cpus,
                           quota={"count": qcount})
    return pending, users, abi.RankParams(0, 0, 0.0, 0.0), inp.astype(np.int32)
