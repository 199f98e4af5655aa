"""Matcher inputs that reach the rare decisions of match_kernel in cook_b200/csrc/match.cu: equal-fitness ties,
fitnesses one ulp apart, exact fits, supply confined to one or two chunks, crowded commit turns, group conflicts
and the pipeline's size edges.  Test infrastructure only: no GPU code is imported here.

Every builder returns a dict:
  args    cook_match's arguments before params: (ranked, jobs, offers, users); the ranked list is the job order
  kw      its keyword arguments (groups, max_ports)
  nc      num_considerable (every job is considerable: one user without quota or rate limit)
  claims  what test_match_edges.py asserts of the oracle's answer; "want" pins a hand-computed assignment
  knobs   the settings to run it under: COOK_* environment variables, plus "max_ctas" (a match parameter)
  fails   considerable indices whose per-reason failure counts are compared (tie, exact-fit and group cases)

Offer name ranks are a fixed permutation of 0..O-1 ("perm") or its reverse ("rev"), never the identity (except
for a single offer), so the lowest hostname is neither the lowest input index nor the last.  The kernel sorts
the offers by name rank, so a VM's sorted index v (its chunk is v mod 32) equals its name rank here.  `constr`
adds a max-tasks-per-host column that no VM reaches: it selects the constraint kernel (match_kernel<true>)
without changing any answer.
"""
import numpy as np

from cook_b200 import abi

ORDERS = ("perm", "rev")
TOPK = 8            # candidates per (job, chunk) in a row (match.cu)
SL_MAX = 64         # live VMs per chunk in sparse mode (match.cu)

# Where the kernel's tables leave shared memory.  Sizes from the structs of match.cu, compiled for sm_90a:
# sizeof(EvalShared) = 49216, sizeof(SparseLive) = 8324, sizeof(ResolverShared) = 160224, NCW = 4 commit warps.
#  static VM table (evaluators): ev_base + 32 O + sizeof(SparseLive) <= 224 KiB, ev_base = 49216 rounded up to
#    128 = 49280: 32 O <= 229376 - 49280 - 8324 = 171772, so O <= 5367.
#  latest[] (resolver): res_base + 4 O <= 200 KiB, res_base = 160224 (a multiple of 16) plus, in the constraint
#    kernel, the four owners' verdict-bit rows NCW * ceil(O / 32) * 4 B (a multiple of 16).  Plain:
#    4 O <= 204800 - 160224 = 44576, O <= 11144.  Constraint: 4 O + 16 ceil(O / 32) <= 44576, O <= 9904
#    (9904: 39616 + 4960 = 44576; 9905: 39620 + 4960 = 44580).
#  SBW_MAX = 1024 verdict-bit words per row in sparse mode (constraint kernel): O <= 32768.
SMEM_STATIC_O = 5367
LATEST_O = {False: 11144, True: 9904}
SBW_O = 32 * 1024


def ranks(O, order):
    """Name ranks: a fixed permutation of 0..O-1 or its reverse, neither of them the identity (O > 1)."""
    p = np.random.default_rng(7919 + O).permutation(O)
    while O > 2 and ((p == np.arange(O)).all() or (p == np.arange(O)[::-1]).all()):
        p = np.roll(p, 1)
    return (p if order == "perm" else O - 1 - p).astype(np.int32)


def fitness(c, m, lc, lm, rc, rm, ac=0.0, am=0.0):
    """cpuMemBinPacker in the oracle's association (eval_pair): ((req + assigned) + running) / (lease + running)."""
    return (((c + ac) + rc) / (lc + rc) + ((m + am) + rm) / (lm + rm)) / 2.0


def step(x, n):
    """The double n ulps above (n < 0: below) a positive x."""
    return float((np.array([x], np.float64).view(np.int64) + n).view(np.float64)[0])


def make(c, m, lc, lm, rc, rm, order, constr, claims, knobs=None, fails=None, jports=None, vports=None,
         attr=None, groups=None, max_ports=0, rank=None):
    """The dict of one case.  vports: one (begin, end) port range per VM; groups: (per-job group lists,
    abi.Groups); attr: [n_cols][O] attribute values."""
    c, m = np.asarray(c, np.float64), np.asarray(m, np.float64)
    lc, lm, rc, rm = (np.asarray(x, np.float64) for x in (lc, lm, rc, rm))
    J, O = len(c), len(lc)
    rank = ranks(O, order) if rank is None else np.asarray(rank, np.int32)
    jk = {}
    if groups is not None:
        off, idx = abi.csr(groups[0])
        jk.update(group_off=off, group_idx=idx)
    jobs = abi.JobsSoA(n=J, user=np.zeros(J, np.int32), cpus=c, mem=m, gpus=np.zeros(J),
                       ports=np.zeros(J, np.int32) if jports is None else np.asarray(jports, np.int32),
                       allowed=np.ones(J, np.uint8), plugin_accept=np.ones(J, np.uint8), **jk)
    ok = {}
    if constr:
        ok.update(max_tasks=np.full(O, 1_000_000, np.int32), num_tasks=np.zeros(O, np.int32))
    if vports is not None:
        off, b = abi.csr([[p[0]] for p in vports])
        _, e = abi.csr([[p[1]] for p in vports])
        ok.update(port_off=off, port_begin=b, port_end=e)
    if attr is not None:
        attr = np.asarray(attr, np.int32)
        ok.update(n_attr_cols=attr.shape[0], attr=attr.reshape(-1))
    else:
        ok.update(n_attr_cols=0)
    offers = abi.OffersSoA(n=O, hostname_id=(7 * np.arange(O) + 3).astype(np.int32), name_rank=rank, cpus=lc,
                           mem=lm, run_cpus=rc, run_mem=rm, run_count=np.zeros(O, np.int32), **ok)
    users = abi.make_users(1, div_mem=1.0, div_cpus=1.0, div_gpus=1.0)
    return dict(args=(np.arange(J, dtype=np.int32), jobs, offers, users),
                kw=dict(groups=groups[1] if groups is not None else None, max_ports=max_ports),
                nc=J, claims=claims, knobs=knobs or [{}], fails=fails, constr=constr, rank=rank)


def by_rank(rank):
    """Input index of each name rank."""
    return np.argsort(rank, kind="stable")


def _full(O, lc, lm, rc, rm):
    return [np.full(O, x, np.float64) for x in (lc, lm, rc, rm)]


# ---- 1. ties ------------------------------------------------------------------------------------------------
TIE_O = (1, 31, 32, 33, 1023, 1024, 1025, 5121)
WIDE_KNOBS = [{}, {"COOK_NO_SPARSE": "1"}, {"COOK_NO_SMEM_STATIC": "1"}]


def ties(O, order, constr, per_vm=1, J=None, knobs=None):
    """O identical VMs; a job asks for 1 / per_vm of a VM, so every untouched VM ties for every job and a
    touched one is strictly better until it is full.  Job k goes to the VM of name rank k // per_vm; the jobs
    beyond the supply stay unplaced."""
    lc, lm, rc, rm = 4.0, 4096.0, 2.0, 1024.0
    cap = O * per_vm
    if J is None:
        J = cap + 3 if cap <= 64 else (400 if O == 4096 else min(cap, 200))
    rank = ranks(O, order)
    br = by_rank(rank)
    want = [int(br[k // per_vm]) if k < cap else -1 for k in range(J)]
    f0 = fitness(lc / per_vm, lm / per_vm, lc, lm, rc, rm)
    claims = dict(kind="ties", want=want, f0=f0, per_vm=per_vm)
    fails = sorted({0, min(J - 1, cap), J - 1})
    return make(np.full(J, lc / per_vm), np.full(J, lm / per_vm), *_full(O, lc, lm, rc, rm), order, constr,
                claims, knobs=knobs or (WIDE_KNOBS if O >= 1023 else None), fails=fails, rank=rank)


BOUND_TIE_KNOBS = [{}, {"COOK_KMIN": "1"}, {"COOK_KMIN": "1", "COOK_NSPEC": "1"},
                   {"COOK_KMIN": "1", "COOK_LOOKAHEAD": "8"}, {"COOK_NO_SMEM_STATIC": "1"}]
BT_T, BT_U = (16.0, 4096.0, 0.0, 0.0), (8.0, 2048.0, 0.0, 6144.0)      # VM (lease cpus, mem, running cpus, mem)
BT_X, BT_F, BT_Y = (6.0, 2560.0), (8.0, 64.0), (6.0, 1024.0)           # job (cpus, mem)


def bound_tie(side, order, constr, G=60):
    """A winner whose fitness equals the bound's.  G VMs T and 2 G + 4 VMs U; triples of jobs X, F, Y.  X fits
    only a T (mem) and takes the best-named untouched one; F fills the best-named untouched U.  For Y a T
    holding an X fits exactly as well as an untouched U (0.8125, bit for bit), and everything else fits worse
    or not at all.  A candidate set of Y computed before X and F were placed holds the U that F fills (with
    COOK_KMIN=1 that U alone) and the next untouched U as its bound; at Y's turn the T that X changed ties
    with that bound.  side "low": the T's rank below every U, so Y takes that T (the winner beats the bound on
    its name); "high": above, so Y takes the bound."""
    NU = 2 * G + 4
    O = G + NU
    rank = ranks(O, order)
    is_t = rank >= NU if side == "high" else rank < G
    vm = np.where(is_t[:, None], BT_T, BT_U)
    br = by_rank(rank)
    ts, us = [int(v) for v in br if is_t[v]], [int(v) for v in br if not is_t[v]]
    if side == "high":
        want = [x for i in range(G) for x in (ts[i], us[2 * i], us[2 * i + 1])]
    else:
        want = [x for i in range(G) for x in (ts[i], us[i], ts[i])]
    jobs = [BT_X, BT_F, BT_Y] * G
    f_t = fitness(*BT_Y, BT_T[0], BT_T[1], BT_T[2], BT_T[3], ac=BT_X[0], am=BT_X[1])
    f_u = fitness(*BT_Y, *BT_U)
    assert f_t == f_u == 0.8125
    claims = dict(kind="bound_tie", want=want, side=side, f_t=f_t, f_u=f_u, ts=ts, us=us)
    return make([j[0] for j in jobs], [j[1] for j in jobs], *vm.T, order, constr, claims, knobs=BOUND_TIE_KNOBS,
                fails=[0, 1, 2], rank=rank)


# ---- 2. one-ulp fitness -------------------------------------------------------------------------------------
ULP_JOB = (2.0, 400.0)          # cpus equal to every VM's lease: one job per VM, cpu fit exactly 1
ULP_VM = (2.0, 1000.3, 1.5, 300.7)


def ulp_partner(kind):
    """(lm, rm) of a VM whose fitness for ULP_JOB is one ulp above ULP_VM's ("ulp") or bit-equal to it from
    other inputs ("equal"): ULP_VM's mem lease and running mem moved by a few ulps."""
    lc, lm0, rc, rm0 = ULP_VM
    f0 = fitness(*ULP_JOB, lc, lm0, rc, rm0)
    want = float(np.nextafter(f0, np.inf)) if kind == "ulp" else f0
    for i in range(1, 41):
        for j in (0, 1, -1, 2, -2, 3, -3):
            lm, rm = step(lm0, j), step(rm0, i)
            if fitness(*ULP_JOB, lc, lm, rc, rm) == want:
                return lm, rm
    raise AssertionError("no partner within 40 ulps")


def ulp_pairs(kind, order, constr, P=40):
    """P VMs A (ULP_VM) and P VMs B (ulp_partner): "ulp": B fits one ulp better and every B ranks above every A,
    so the B's go first, in name order, then the A's; "equal": B ties A bit for bit, the roles alternate by
    name rank and the jobs take the VMs in name order.  One job per VM, plus one that finds no room."""
    O = 2 * P
    rank = ranks(O, order)
    isb = rank >= P if kind == "ulp" else rank % 2 == 1
    lc, lm0, rc, rm0 = ULP_VM
    lmb, rmb = ulp_partner(kind)
    lm, rm = np.where(isb, lmb, lm0), np.where(isb, rmb, rm0)
    br = by_rank(rank)
    if kind == "ulp":
        want = [int(v) for v in br[P:]] + [int(v) for v in br[:P]] + [-1]
    else:
        want = [int(v) for v in br] + [-1]
    fa, fb = fitness(*ULP_JOB, lc, lm0, rc, rm0), fitness(*ULP_JOB, lc, lmb, rc, rmb)
    assert (fb == np.nextafter(fa, np.inf)) if kind == "ulp" else (fb == fa and (lmb, rmb) != (lm0, rm0))
    claims = dict(kind="ulp_" + kind, want=want, fa=fa, fb=fb, b_vms=[int(v) for v in np.flatnonzero(isb)])
    J = O + 1
    return make(np.full(J, ULP_JOB[0]), np.full(J, ULP_JOB[1]), np.full(O, lc), lm, np.full(O, rc), rm,
                order, constr, claims, fails=[0, P, J - 1], rank=rank)


# ---- 3. exact fit -------------------------------------------------------------------------------------------
def exact_amounts(regime):
    """(lease, a, b, x): after requests a and b the running sum (0 + a) + b leaves exactly room x:
    (0 + a) + b + x <= lease < (0 + a) + b + nextafter(x).  Off the grid (tenths) the other association
    a + (b + x') of the one-ulp-larger request still fits, so a matcher that summed in another order would
    place it."""
    if regime == "grid":   # x in the binade of the lease: one ulp more is one ulp of the sum
        return 1.5, 0.125, 0.125, 1.25
    for L10 in range(5, 60):
        L = L10 / 10.0
        for a10 in range(1, L10):
            for b10 in range(1, L10 - a10):
                a, b = a10 / 10.0, b10 / 10.0
                acc = (0.0 + a) + b
                x = L - acc
                while acc + x > L:
                    x = float(np.nextafter(x, -np.inf))
                while acc + float(np.nextafter(x, np.inf)) <= L:
                    x = float(np.nextafter(x, np.inf))
                if a + (b + float(np.nextafter(x, np.inf))) <= L:
                    return L, a, b, x
    raise AssertionError("no association-sensitive exact fit")


def exact_fit(res, regime, edge, order, constr):
    """40 identical VMs.  Jobs a and b land on the best-named VM T (ties, then T is the touched one); job x asks
    for exactly T's room left in resource `res` (edge "exact": placed on T) or one ulp more (edge "ulp": it
    goes to the next-named VM).  Ports (constraint kernel only): T offers 10 ports, a and b take 3 each and x
    takes 4 (exact) or 5."""
    O = 40
    rank = ranks(O, order)
    br = by_rank(rank)
    T, D = int(br[0]), int(br[1])
    lc, lm = np.full(O, 16.0), np.full(O, 16384.0)
    c, m, jp, vp, mp = [1.0, 1.0, 1.0], [64.0, 64.0, 64.0], None, None, 0
    if res == "ports":
        assert constr
        jp = [3, 3, 4 if edge == "exact" else 5]
        vp = [(31000, 31009)] * O
        mp = 5
        claims_amounts = None
    else:
        L, a, b, x = exact_amounts(regime)
        if edge == "ulp":
            x = float(np.nextafter(x, np.inf))
        scale = 1.0 if res == "cpus" else 1024.0   # a power of two: the same roundings in mem
        amounts = [a * scale, b * scale, x * scale]
        if res == "cpus":
            lc, c = np.full(O, L), amounts
        else:
            lm, m = np.full(O, L * 1024.0), amounts
        claims_amounts = (L * scale, amounts)
    want = [T, T, T if edge == "exact" else D]
    ports = [[31000, 31001, 31002], [31003, 31004, 31005],
             [31006, 31007, 31008, 31009] if edge == "exact" else [31000 + i for i in range(5)]] if jp else None
    claims = dict(kind="exact_fit", want=want, res=res, regime=regime, edge=edge, amounts=claims_amounts,
                  ports=ports)
    return make(c, m, lc, lm, np.full(O, 1.0), np.full(O, 512.0), order, constr, claims, fails=[0, 1, 2],
                jports=jp, vports=vp, max_ports=mp, rank=rank)


# ---- 4. single-chunk supply ---------------------------------------------------------------------------------
def single_chunk(chunks, order, constr, tiles=48, per_chunk=24):
    """32 x tiles VMs; only those of the given chunks (name rank mod 32) can take a job, one job each, and they
    tie.  per_chunk jobs per chunk (more than TOPK): every job beyond a chunk's row needs a re-scan of the
    chunk behind the row's bound.  Job k goes to the k-th best-named VM of the chunks."""
    O = 32 * tiles
    rank = ranks(O, order)
    big = np.isin(rank % 32, chunks)
    lc, lm = np.where(big, 4.0, 1.0), np.where(big, 4096.0, 1024.0)
    J = per_chunk * len(chunks)
    br = by_rank(rank)
    want = [int(v) for v in br if big[v]][:J]
    claims = dict(kind="single_chunk", want=want, chunks=list(chunks))
    return make(np.full(J, 4.0), np.full(J, 4096.0), lc, lm, np.full(O, 1.0), np.full(O, 512.0), order,
                constr, claims, knobs=[{}, {"COOK_NO_SPARSE": "1"}, {"COOK_KMIN": "1"}], rank=rank)


def stale_rescan(order, constr):
    """Supply in one chunk (c = 5) across three blocks (B jobs per block: 64 plain, 128 constraint).  K tied VMs
    take one job Y each; VM W of the chunk also fits a Y job, but worst of all, and is the only VM a job X fits.
    Block 0 is B Y jobs, block 1 starts with X (the first log entry after block 0: W is full for Y from then on)
    and goes on with Y jobs, and block 2's Y jobs exhaust the K VMs.  The rows of block 2 were scored against
    the state after block 0, where W was free: a Y job that re-scans the chunk behind its row's bound must skip W
    as changed since that snapshot, and the Y jobs after the K VMs stay unplaced."""
    B = 128 if constr else 64
    K = B + (B - 1) + 10
    tiles = K + 3
    O = 32 * tiles
    rank = ranks(O, order)
    chunk = rank % 32 == 5
    w = int(np.flatnonzero(chunk & (rank == rank[chunk].max()))[0])
    tied = chunk & (rank // 32 < K)
    lc, lm = np.where(tied, 4.0, 1.0), np.where(tied, 4096.0, 1024.0)
    lc[w], lm[w] = 4.0, 16384.0
    y, x = (4.0, 4096.0), (1.0, 10000.0)
    jobs = [y] * B + [x] + [y] * (B - 1) + [y] * 20
    br = [int(v) for v in by_rank(rank) if tied[v]]
    ys = br[:K] + [-1] * 10
    want = ys[:B] + [w] + ys[B:]
    claims = dict(kind="stale_rescan", want=want, w=w, B=B)
    return make([j[0] for j in jobs], [j[1] for j in jobs], lc, lm, np.full(O, 1.0), np.full(O, 512.0), order,
                constr, claims, knobs=[{}, {"COOK_KMIN": "1"}, {"COOK_NO_SPARSE": "1"}], rank=rank)


# ---- 5. crowded turns ---------------------------------------------------------------------------------------
CROWD_KNOBS = [{}, {"COOK_KMIN": "1", "COOK_LOOKAHEAD": "2"}, {"COOK_KMIN": "2", "COOK_LOOKAHEAD": "8"},
               {"COOK_KMIN": "16", "COOK_LOOKAHEAD": "31"}, {"COOK_NSPEC": "1", "max_ctas": 3},
               {"COOK_NSPEC": "3", "max_ctas": 5}, {"COOK_KMIN": "1", "COOK_NSPEC": "1", "COOK_LOOKAHEAD": "31"},
               {"COOK_KMIN": "16", "COOK_NSPEC": "3", "COOK_LOOKAHEAD": "2", "max_ctas": 0},
               {"COOK_KMIN": "2", "COOK_LOOKAHEAD": "8", "COOK_NO_SMEM_STATIC": "1"}]


def crowded(per_vm, order, constr, O=600, J=500):
    """Every VM has a distinct fitness (distinct running mem) and room for per_vm identical jobs: the jobs fill
    the VMs best first, so each placement supersedes the best items every later owner holds (relooks, exact
    recomputations, the bound taken directly).  Job k goes to the (k // per_vm)-th best VM."""
    rank = ranks(O, order)
    q = np.random.default_rng(O + per_vm).permutation(O)
    rm = 1024.0 * (1 + q)
    lc, lm = 2.0 * per_vm, 4096.0 * per_vm
    best = np.argsort(-q, kind="stable")
    want = [int(best[k // per_vm]) if k < O * per_vm else -1 for k in range(J)]
    claims = dict(kind="crowded", want=want)
    return make(np.full(J, 2.0), np.full(J, 1024.0), np.full(O, lc), np.full(O, lm), np.full(O, 1.0), rm,
                order, constr, claims, knobs=CROWD_KNOBS, rank=rank)


SWAP_KNOBS = [{"COOK_KMIN": "1", "COOK_LOOKAHEAD": str(la), "COOK_NSPEC": ns} for la in (3, 4, 6, 31)
              for ns in ("1", "3")]


def swap_bound(order, constr, G=100):
    """Groups of three VMs X, Y, W (X and Y in one chunk) and triples of jobs Q, P, P'.  P-shaped jobs rank the
    VMs X1 > Y1 > W1 > X2 > ... (running mem); Q-shaped jobs prefer any Y (running cpus).  Q_i takes Y_i, P_i
    takes X_i, P'_i takes W_i.  A candidate set of P'_i computed before Q_i's placement holds X_i alone
    (COOK_KMIN=1) with Y_i as its bound: at P'_i's turn both are gone, and Y_i was changed by the very first
    placement after that version, so the bound may not be taken with the state the set recorded."""
    O = 64 * G
    rank = ranks(O, order)
    grp, pos = rank // 64, rank % 64
    role = np.select([pos == 5, pos == 37, pos == 9], [0, 1, 2], -1)   # X, Y (chunk 5), W (chunk 9)
    lc = np.where(role >= 0, 8.0, 0.5)
    rc = np.where(role == 1, 56.0, 0.0)
    rm = np.where(role >= 0, 4096.0 - 8.0 * (3 * grp + np.maximum(role, 0)), 0.0)
    p, q = (8.0, 1024.0), (5.0, 1024.0)   # either fills a VM for P; one Q fills a Y for Q
    jobs = [q, p, p] * G
    at = {(int(grp[v]), int(role[v])): int(v) for v in range(O) if role[v] >= 0}
    want = [at[(i, r)] for i in range(G) for r in (1, 0, 2)]
    claims = dict(kind="swap_bound", want=want)
    return make([j[0] for j in jobs], [j[1] for j in jobs], lc, np.full(O, 8192.0), rc, rm, order, constr, claims,
                knobs=SWAP_KNOBS, rank=rank)


# ---- 6. group conflicts -------------------------------------------------------------------------------------
def group_conflicts(order, O=96):
    """Identical VMs (four jobs each) with attribute column 0 = 1 + name rank mod 3.  Consecutive members of a
    unique group (6), a balanced group on column 0 (minimum 3, 9 members) and an attribute-equals group on
    column 0 (6), then 4 jobs without groups.  Each member's candidate set is stale once the member before it
    is placed: the resolver's exact full scan decides.  The unique members go to name ranks 0..5 (a touched VM
    is better, but its host is taken)."""
    rank = ranks(O, order)
    attr = (1 + rank % 3).astype(np.int32)[None, :]
    lists = [[0]] * 6 + [[1]] * 9 + [[2]] * 6 + [[]] * 4
    J = len(lists)
    groups = abi.Groups(n_groups=3, kind=np.array([abi.GROUP_UNIQUE, abi.GROUP_BALANCED, abi.GROUP_ATTR_EQUALS],
                                                  np.int32),
                        attr_col=np.zeros(3, np.int32), minimum=np.array([1, 3, 1], np.int32),
                        cot_off=np.zeros(4, np.int32), cot_hostname_id=np.zeros(1, np.int32),
                        cot_attr_val=np.zeros(1, np.int32))
    br = by_rank(rank)
    claims = dict(kind="groups", unique=[int(v) for v in br[:6]], members=[list(range(0, 6)), list(range(6, 15)),
                                                                            list(range(15, 21))], attr=attr[0])
    knobs = [{}, {"COOK_LOOKAHEAD": "2"}, {"COOK_KMIN": "1", "COOK_NSPEC": "1"}, {"max_ctas": 3}]
    return make(np.full(J, 1.0), np.full(J, 1024.0), *_full(O, 4.0, 4096.0, 2.0, 1024.0), order, True, claims,
                knobs=knobs, fails=[0, 6, 15, J - 1], attr=attr, groups=(lists, groups), rank=rank)


# ---- 7. pipeline and size edges -----------------------------------------------------------------------------
BLOCK_J = {False: (1, 63, 64, 65), True: (127, 128, 129)}


def hopeless(order, constr):
    """One job per VM and more jobs than VMs: the cluster fills in the middle of the second block (plain
    blocks of 64 jobs, constraint blocks of 128), the evaluators stop and the rest of the queue is marked
    unplaced without being scored."""
    O = 100 if not constr else 200
    return ties(O, order, constr, J=3 * O)


def sparse_edge(live, order, constr):
    """Chunk 5 holds B + `live` VMs that can take one job each (the best-named ones of the chunk, B = 64 plain,
    128 constraint jobs per block), every other VM is too small for any job, and there are 3 B + 10 jobs.
    Blocks 0 and 1 are scored against the initial state (dense).  Block 2 is scored against the state after
    block 0, which left `live` VMs: sparse mode iff live <= SL_MAX.  With 65 the scoring turns sparse at block
    3, once block 1 has filled all but one."""
    B = 128 if constr else 64
    N = B + live
    O = 32 * (N + 2)
    rank = ranks(O, order)
    big = (rank % 32 == 5) & (rank // 32 < N)
    J = 3 * B + 10
    br = by_rank(rank)
    want = ([int(v) for v in br if big[v]] + [-1] * J)[:J]
    claims = dict(kind="sparse", want=want, live=live, B=B)
    lc, lm = np.where(big, 4.0, 1.0), np.where(big, 4096.0, 1024.0)
    return make(np.full(J, 4.0), np.full(J, 4096.0), lc, lm, np.full(O, 1.0), np.full(O, 512.0), order, constr,
                claims, knobs=[{}, {"COOK_NO_SPARSE": "1"}], rank=rank)


SBW_TILES = (0, 511, 1022, 1023)


def sbw_edge(O, order):
    """The constraint kernel's verdict bits staged in shared memory in sparse mode (SBW_MAX words).  Only the
    VMs of tiles 0, 511, 1022 and 1023 (name rank // 32), and at O = 32769 the one VM of tile 1024, can take a
    job, one each: every chunk has at most 5 live VMs.  O = 32768: 1024 verdict words, the whole staging buffer
    with bits in its last word, and the live mask in use (O <= 64 x 32 x NW).  O = 32769: 1025 words and no
    live mask, so every row is scored dense."""
    rank = ranks(O, order)
    big = np.isin(rank // 32, SBW_TILES + (1024,))
    J = int(big.sum()) + 12
    br = by_rank(rank)
    want = ([int(v) for v in br if big[v]] + [-1] * J)[:J]
    claims = dict(kind="sbw", want=want)
    lc, lm = np.where(big, 4.0, 1.0), np.where(big, 4096.0, 1024.0)
    return make(np.full(J, 4.0), np.full(J, 4096.0), lc, lm, np.full(O, 1.0), np.full(O, 512.0), order, True,
                claims, knobs=[{}, {"COOK_NO_SPARSE": "1"}], rank=rank)


def threshold(O, order, constr, J=64):
    """Ties over O VMs on either side of a shared-memory limit (see the constants above), or of the bound of the
    evaluators' live mask and request pre-test (O <= 64 x 32 x NW = 32768)."""
    return ties(O, order, constr, J=J, knobs=[{}])


# ---- the catalogue ------------------------------------------------------------------------------------------
def catalogue():
    """{name: builder(order)} of every case, both kernels where the case applies to both."""
    out = {}
    for ck in (False, True):
        kn = "C" if ck else "P"
        for O in TIE_O:
            out[f"1-ties-{kn}-O{O}"] = lambda od, O=O, ck=ck: ties(O, od, ck)
        for O in (1, 32, 1024):
            out[f"1-ties4-{kn}-O{O}"] = lambda od, O=O, ck=ck: ties(O, od, ck, per_vm=4)
        out[f"1-ties-{kn}-O4096"] = lambda od, ck=ck: ties(4096, od, ck)
        for side in ("low", "high"):
            out[f"1-bound-{side}-{kn}"] = lambda od, side=side, ck=ck: bound_tie(side, od, ck)
        for kind in ("ulp", "equal"):
            for P in (3, 40):
                out[f"2-{kind}-{kn}-P{P}"] = lambda od, kind=kind, P=P, ck=ck: ulp_pairs(kind, od, ck, P)
        for res in ("cpus", "mem") + (("ports",) if ck else ()):
            for regime in (("grid", "off") if res != "ports" else ("grid",)):
                for edge in ("exact", "ulp"):
                    out[f"3-fit-{res}-{regime}-{edge}-{kn}"] = \
                        lambda od, res=res, regime=regime, edge=edge, ck=ck: exact_fit(res, regime, edge, od, ck)
        out[f"4-chunk-{kn}-1"] = lambda od, ck=ck: single_chunk([11], od, ck)
        out[f"4-chunk-{kn}-2"] = lambda od, ck=ck: single_chunk([3, 30], od, ck)
        out[f"4-stale-{kn}"] = lambda od, ck=ck: stale_rescan(od, ck)
        for per_vm in (1, 2):
            out[f"5-crowded-{kn}-{per_vm}"] = lambda od, per_vm=per_vm, ck=ck: crowded(per_vm, od, ck)
        out[f"5-swap-{kn}"] = lambda od, ck=ck: swap_bound(od, ck)
        for J in BLOCK_J[ck]:
            out[f"7-block-{kn}-J{J}"] = lambda od, J=J, ck=ck: ties(256, od, ck, J=J)
        out[f"7-hopeless-{kn}"] = lambda od, ck=ck: hopeless(od, ck)
        for live in (SL_MAX, SL_MAX + 1):
            out[f"7-sparse-{kn}-{live}"] = lambda od, live=live, ck=ck: sparse_edge(live, od, ck)
        for O in (SMEM_STATIC_O, SMEM_STATIC_O + 1, LATEST_O[ck], LATEST_O[ck] + 1):
            out[f"7-smem-{kn}-O{O}"] = lambda od, O=O, ck=ck: threshold(O, od, ck)
    out["6-groups"] = lambda od: group_conflicts(od)
    for O in (SBW_O, SBW_O + 1):
        out[f"7-sbw-C-O{O}"] = lambda od, O=O: sbw_edge(O, od)
        out[f"7-gate-P-O{O}"] = lambda od, O=O: threshold(O, od, False)
    return out


def greedy(case):
    """A plain restatement of the matcher without groups or hard constraints, for the CPU checks: jobs in
    order, every VM tried, the resource test `assigned + request > lease` (and ports), the fitness in the
    oracle's association, equal fitness to the lowest name rank.  Returns (assign, ports)."""
    _, jobs, offers, _ = case["args"]
    c, m, jp = jobs.col("cpus"), jobs.col("mem"), jobs.col("ports")
    lc, lm, rc, rm = (offers.col(k) for k in ("cpus", "mem", "run_cpus", "run_mem"))
    rank = offers.col("name_rank")
    O = len(lc)
    if offers.col("port_off") is not None:
        pb, pe = offers.col("port_begin"), offers.col("port_end")
        ptot = pe - pb + 1
    else:
        pb, ptot = np.zeros(O, np.int64), np.zeros(O, np.int64)
    ac, am, pu = np.zeros(O), np.zeros(O), np.zeros(O, np.int64)
    assign, ports = [], []
    for j in range(len(c)):
        no = (ac + c[j] > lc) | (am + m[j] > lm) | (jp[j] > ptot - pu)
        f = np.where(no, 0.0, (((c[j] + ac) + rc) / (lc + rc) + ((m[j] + am) + rm) / (lm + rm)) / 2.0)
        best = f.max() if O else 0.0
        if not best > 0.0:
            assign.append(-1)
            ports.append([])
            continue
        v = int(np.flatnonzero(f == best)[np.argmin(rank[f == best])])
        assign.append(v)
        ports.append([int(pb[v] + pu[v] + i) for i in range(jp[j])])
        ac[v] = ac[v] + c[j]
        am[v] = am[v] + m[j]
        pu[v] += jp[j]
    return np.array(assign, np.int32), ports
