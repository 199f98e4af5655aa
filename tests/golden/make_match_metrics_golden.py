"""Writes tests/golden/match_metrics_golden.json: the known answers of the match-cycle metrics.

"resource_maps" transcribes the reference's test-job->resource-maps (test/cook/test/scheduler/scheduler.clj:2461-2511):
each case's jobs as the reference builds them (COOK_GPU_MODEL, the resources with the disk map) and the resource maps
the reference asserts, string keys and all.

"rounds" are hand-computed edges.  Each case is a list of rounds over one pool; a round lists its considerable jobs in
take order ({job_id, user, cpus, mem, gpus, ports, facts (JF_* bits), gpu_model, disk_type, disk_request,
disk_limit}), the positions the match assigned, the positions the launch-rate filter dropped, and the expected answer
written out by hand:
  gpus_zero     a gpus resource of 0.0 is a key, gpus/unspecified-gpu-model = 0.0; a job with gpus 2.0 and no gpus
                resource has none
  disk_partial  disk without a limit (request 10 of type 1) and disk without a request (limit 20 of type 1)
  uris_0/1/2    no row, one row (position 1) and two rows with uris: two make jobs->stats the error string
  tie           cpus 4, 1, 4, 2: the last maximal row is position 2; sorted 1 2 4 4 gives p50 = 2, p95 = p100 = 4
  fold          cpus 0.1, 0.2, 0.3 in take order fold to (0.1 + 0.2) + 0.3 = 0.6000000000000001, not 0.6
  drops         three jobs, positions 0 and 2 assigned, 0 dropped: one matched, the head not matched, jobs 11 and 10
                at one cycle
  counters      job 1 unmatched, then out of the considerable set, then back: 1, absent, 1; job 2 unmatched twice: 2
  threshold     job 7 unmatched in 501 rounds with threshold 500: none too long at 500 cycles, one at 501
  empty         an empty round after an unmatched one forgets every count

Run from the repository root: python tests/golden/make_match_metrics_golden.py
"""
import json
import os

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "match_metrics_golden.json")
GPUS, DISK, REQ, LIM, URIS = 1, 2, 4, 8, 16


def job(jid, cpus, mem, facts=0, user=0, **kw):
    r = dict(job_id=jid, user=user, cpus=cpus, mem=mem, gpus=0.0, ports=0, facts=facts, gpu_model=-1, disk_type=-1,
             disk_request=0.0, disk_limit=0.0)
    r.update(kw)
    return r


RESOURCE_MAPS = [
    {"name": "adds up resources by type",
     "jobs": [{"gpu_model": "nvidia-tesla-k80",
               "resources": {"cpus": 1.2, "mem": 34, "gpus": 2, "disk": {"request": 10, "limit": 20, "type": "pd-ssd"}}},
              {"gpu_model": "nvidia-tesla-p100", "resources": {"cpus": 2.3, "mem": 45, "gpus": 4}}],
     "want": [{"cpus": 1.2, "mem": 34, "gpus/nvidia-tesla-k80": 2, "disk/pd-ssd/request": 10, "disk/pd-ssd/limit": 20},
              {"cpus": 2.3, "mem": 45, "gpus/nvidia-tesla-p100": 4}]},
    {"name": "gracefully handles unspecified gpu model",
     "jobs": [{"gpu_model": None, "resources": {"cpus": 1.2, "mem": 34, "gpus": 2}},
              {"gpu_model": None, "resources": {"cpus": 2.3, "mem": 45, "gpus": 4}}],
     "want": [{"cpus": 1.2, "mem": 34, "gpus/unspecified-gpu-model": 2},
              {"cpus": 2.3, "mem": 45, "gpus/unspecified-gpu-model": 4}]},
    {"name": "gracefully handles unspecified disk type",
     "jobs": [{"gpu_model": None, "resources": {"cpus": 1.2, "mem": 34, "disk": {"request": 10}}},
              {"gpu_model": None, "resources": {"cpus": 2.3, "mem": 45, "disk": {"request": 50, "limit": 100}}}],
     "want": [{"cpus": 1.2, "mem": 34, "disk/unspecified-disk-type/request": 10},
              {"cpus": 2.3, "mem": 45, "disk/unspecified-disk-type/request": 50,
               "disk/unspecified-disk-type/limit": 100}]},
]


def rnd(jobs, assigned=(), dropped=(), **want):
    return {"jobs": jobs, "assigned": list(assigned), "dropped": list(dropped), "want": want}


ROUNDS = {
    "gpus_zero": [rnd([job(1, 1.0, 10.0, GPUS, gpus=0.0), job(2, 1.0, 10.0, 0, gpus=2.0)],
                      keys=[[0, -1, 0.0]], total_cpus=2.0, total_mem=20.0)],
    "disk_partial": [rnd([job(1, 1.0, 1.0, DISK | REQ, disk_type=1, disk_request=10.0),
                          job(2, 1.0, 1.0, DISK | LIM, disk_type=1, disk_limit=20.0)],
                         keys=[[1, 1, 10.0], [2, 1, 20.0]])],
    "uris_0": [rnd([job(1, 1.0, 1.0), job(2, 1.0, 1.0)], uris=0, uris_position=-1, stats_error=False)],
    "uris_1": [rnd([job(1, 1.0, 1.0), job(2, 1.0, 1.0, URIS)], uris=1, uris_position=1, stats_error=False)],
    "uris_2": [rnd([job(1, 1.0, 1.0, URIS), job(2, 1.0, 1.0, URIS)], uris=2, uris_position=-1, stats_error=True)],
    "tie": [rnd([job(1, 4.0, 1.0), job(2, 1.0, 9.0), job(3, 4.0, 9.0), job(4, 2.0, 3.0)],
                largest_cpus=2, largest_mem=2, pct_cpus=[2.0, 4.0, 4.0], pct_mem=[3.0, 9.0, 9.0], total_cpus=11.0,
                total_mem=22.0)],
    "fold": [rnd([job(1, 0.1, 1.0), job(2, 0.2, 1.0), job(3, 0.3, 1.0)], total_cpus=0.6000000000000001,
                 total_mem=3.0)],
    "drops": [rnd([job(10, 1.0, 1.0, user=1), job(11, 1.0, 1.0), job(12, 1.0, 1.0)], assigned=[0, 2], dropped=[0],
                  matched=1, head_matched=0, user_considerable=[2, 1], user_matched=[1, 0],
                  cycles={"10": 1, "11": 1})],
    "counters": [rnd([job(1, 1.0, 1.0), job(2, 1.0, 1.0)], cycles={"1": 1, "2": 1}),
                 rnd([job(2, 1.0, 1.0)], cycles={"2": 2}),
                 rnd([job(1, 1.0, 1.0), job(2, 1.0, 1.0)], assigned=[1], cycles={"1": 1})],
    # 499 rounds without an expected answer ("repeat"), then the two at the boundary
    "threshold": [dict(rnd([job(7, 1.0, 1.0)]), repeat=499),
                  rnd([job(7, 1.0, 1.0)], cycles={"7": 500}, too_long=0),
                  rnd([job(7, 1.0, 1.0)], cycles={"7": 501}, too_long=1, first=[[7, 501]])],
    "empty": [rnd([job(1, 1.0, 1.0)], cycles={"1": 1}), rnd([], considerable=0, cycles={})],
}


if __name__ == "__main__":
    with open(OUT, "w") as f:
        json.dump({"threshold": 500, "n_users": 2, "resource_maps": RESOURCE_MAPS, "rounds": ROUNDS}, f, indent=0)
        f.write("\n")
    print("wrote", OUT)
