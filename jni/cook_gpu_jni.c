/*
 * cook_gpu_jni.c — JNI shim between Cook's JVM (namespace cook.scheduler.gpu, clj/cook/scheduler/gpu.clj)
 * and libcookgpu.so (include/cook_gpu.h).  One native method per C-ABI entry point; nothing here
 * computes: the methods unwrap direct ByteBuffers into the SoA structs and forward.
 *
 * Java side (package cook.gpu, class Native): every `long` is an opaque handle (cook_ctx*, cook_pool*,
 * ncclComm_t); every column is a java.nio.ByteBuffer allocated with allocateDirect and
 * ByteOrder.nativeOrder(), or null when the ABI allows NULL.  Columns travel as Object[] in the
 * FIELD ORDER of the struct in cook_gpu.h (the order cook_b200/abi.py mirrors as well), scalar
 * fields as int[] / double[] next to them.  Errors: the int32 code is returned unchanged; the Clojure
 * wrapper turns non-zero into ex-info with cook_last_error's text, which the existing catch blocks
 * (scheduler.clj:1521-1535) already handle.
 *
 * Build (where a JDK exists):  gcc -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux \
 *                                  -Iinclude jni/cook_gpu_jni.c -Lcook_b200 -lcookgpu -o libcookgpujni.so
 * This image has no JDK; the file is reviewed against cook_gpu.h, not compiled here.
 */
#include <jni.h>
#include <stdint.h>
#include <string.h>

#include "cook_gpu.h"

#define JFN(ret, name) JNIEXPORT ret JNICALL Java_cook_gpu_Native_##name

static void* buf(JNIEnv* env, jobjectArray cols, int i) {
  jobject b = (*env)->GetObjectArrayElement(env, cols, i);
  return b ? (*env)->GetDirectBufferAddress(env, b) : NULL;
}
static void* one(JNIEnv* env, jobject b) { return b ? (*env)->GetDirectBufferAddress(env, b) : NULL; }

/* ---- struct unpackers: Object[] columns in header field order ------------------------------ */
static void tasks_from(JNIEnv* env, jint n, jobjectArray c, cook_tasks_soa* t) {
  t->n = n; t->user = buf(env, c, 0); t->priority = buf(env, c, 1); t->start_time = buf(env, c, 2);
  t->task_id = buf(env, c, 3); t->job_id = buf(env, c, 4); t->cpus = buf(env, c, 5); t->mem = buf(env, c, 6);
  t->gpus = buf(env, c, 7);
}
static void users_from(JNIEnv* env, jint n, jobjectArray c, cook_user_table* u) {
  u->n_users = n; u->name_rank = buf(env, c, 0); u->div_mem = buf(env, c, 1); u->div_cpus = buf(env, c, 2);
  u->div_gpus = buf(env, c, 3); u->quota_count = buf(env, c, 4); u->quota_cpus = buf(env, c, 5);
  u->quota_mem = buf(env, c, 6); u->quota_gpus = buf(env, c, 7); u->usage_count = buf(env, c, 8);
  u->usage_cpus = buf(env, c, 9); u->usage_mem = buf(env, c, 10); u->usage_gpus = buf(env, c, 11);
  u->tokens = buf(env, c, 12);
}
static void quota_from(JNIEnv* env, jdoubleArray q, cook_pool_quota* out) {   /* null => (nil? quota) */
  memset(out, 0, sizeof(*out));
  if (!q) return;
  jdouble v[4];
  (*env)->GetDoubleArrayRegion(env, q, 0, 4, v);
  out->enabled = 1; out->count = v[0]; out->cpus = v[1]; out->mem = v[2]; out->gpus = v[3];
}
static void jobs_from(JNIEnv* env, jint n, jobjectArray c, cook_jobs_soa* j) {
  j->n = n; j->user = buf(env, c, 0); j->cpus = buf(env, c, 1); j->mem = buf(env, c, 2); j->gpus = buf(env, c, 3);
  j->ports = buf(env, c, 4); j->allowed = buf(env, c, 5); j->plugin_accept = buf(env, c, 6);
  j->novel_off = buf(env, c, 7); j->novel_host = buf(env, c, 8); j->gpu_model = buf(env, c, 9);
  j->disk_request = buf(env, c, 10); j->disk_type = buf(env, c, 11); j->attr_off = buf(env, c, 12);
  j->attr_col = buf(env, c, 13); j->attr_val = buf(env, c, 14); j->est_end_ms = buf(env, c, 15);
  j->ckpt_location = buf(env, c, 16); j->reserved_host = buf(env, c, 17); j->group_off = buf(env, c, 18);
  j->group_idx = buf(env, c, 19);
}
static void offers_from(JNIEnv* env, jint n, jint n_attr_cols, jobjectArray c, cook_offers_soa* o) {
  o->n = n; o->hostname_id = buf(env, c, 0); o->name_rank = buf(env, c, 1); o->cpus = buf(env, c, 2);
  o->mem = buf(env, c, 3); o->run_cpus = buf(env, c, 4); o->run_mem = buf(env, c, 5); o->run_count = buf(env, c, 6);
  o->port_off = buf(env, c, 7); o->port_begin = buf(env, c, 8); o->port_end = buf(env, c, 9);
  o->is_k8s = buf(env, c, 10); o->location = buf(env, c, 11); o->gpu_off = buf(env, c, 12);
  o->gpu_model = buf(env, c, 13); o->gpu_count = buf(env, c, 14); o->disk_off = buf(env, c, 15);
  o->disk_type = buf(env, c, 16); o->disk_space = buf(env, c, 17); o->max_tasks = buf(env, c, 18);
  o->num_tasks = buf(env, c, 19); o->host_start_time = buf(env, c, 20); o->n_attr_cols = n_attr_cols;
  o->attr = buf(env, c, 21); o->reserved = buf(env, c, 22);
}
static int groups_from(JNIEnv* env, jint n, jobjectArray c, cook_groups* g) {
  if (!c || n <= 0) return 0;
  g->n_groups = n; g->kind = buf(env, c, 0); g->attr_col = buf(env, c, 1); g->minimum = buf(env, c, 2);
  g->cot_off = buf(env, c, 3); g->cot_hostname_id = buf(env, c, 4); g->cot_attr_val = buf(env, c, 5);
  return 1;
}
static void hosts_from(JNIEnv* env, jint n, jint n_attr_cols, jobjectArray c, cook_host_table* h) {
  h->n = n; h->hostname_id = buf(env, c, 0); h->name_rank = buf(env, c, 1); h->has_spare = buf(env, c, 2);
  h->spare_cpus = buf(env, c, 3); h->spare_mem = buf(env, c, 4); h->spare_gpus = buf(env, c, 5);
  h->is_k8s = buf(env, c, 6); h->location = buf(env, c, 7); h->gpu_off = buf(env, c, 8); h->gpu_model = buf(env, c, 9);
  h->gpu_count = buf(env, c, 10); h->disk_off = buf(env, c, 11); h->disk_type = buf(env, c, 12);
  h->disk_space = buf(env, c, 13); h->host_start_time = buf(env, c, 14); h->n_attr_cols = n_attr_cols;
  h->attr = buf(env, c, 15);
}

/* ---- lifetime --------------------------------------------------------------------------------- */
JFN(jint, init)(JNIEnv* env, jclass k, jintArray devices, jlongArray out_ctx) {
  cook_gpu_config cfg; memset(&cfg, 0, sizeof(cfg));
  jint ids[64]; jsize n = devices ? (*env)->GetArrayLength(env, devices) : 0;
  if (n > 64) n = 64;
  if (n) { (*env)->GetIntArrayRegion(env, devices, 0, n, ids); cfg.n_devices = n; cfg.device_ids = (const int32_t*)ids; }
  cook_ctx* ctx = NULL;
  jint rc = cook_gpu_init(&cfg, &ctx);
  jlong h = (jlong)(intptr_t)ctx; (*env)->SetLongArrayRegion(env, out_ctx, 0, 1, &h);
  return rc;
}
JFN(jint, shutdown)(JNIEnv* env, jclass k, jlong ctx) { return cook_gpu_shutdown((cook_ctx*)(intptr_t)ctx); }
JFN(jint, poolOpen)(JNIEnv* env, jclass k, jlong ctx, jstring name, jint dru_mode, jint device, jlongArray out_pool) {
  const char* s = (*env)->GetStringUTFChars(env, name, NULL);
  cook_pool* p = NULL;
  jint rc = cook_pool_open((cook_ctx*)(intptr_t)ctx, s, dru_mode, device, &p);
  (*env)->ReleaseStringUTFChars(env, name, s);
  jlong h = (jlong)(intptr_t)p; (*env)->SetLongArrayRegion(env, out_pool, 0, 1, &h);
  return rc;
}
JFN(jint, poolClose)(JNIEnv* env, jclass k, jlong pool) { return cook_pool_close((cook_pool*)(intptr_t)pool); }
JFN(jstring, lastError)(JNIEnv* env, jclass k, jlong pool) {
  char b[512]; b[0] = 0; cook_last_error((cook_pool*)(intptr_t)pool, b, sizeof(b));
  return (*env)->NewStringUTF(env, b);
}
JFN(jstring, version)(JNIEnv* env, jclass k) { return (*env)->NewStringUTF(env, cook_gpu_version()); }

/* ---- R1-R7 ------------------------------------------------------------------------------------ */
JFN(jint, rank)(JNIEnv* env, jclass k, jlong pool, jint n_running, jobjectArray running, jint n_pending,
                jobjectArray pending, jint n_users, jobjectArray users, jdoubleArray pool_quota,
                jdoubleArray group_quota, jobject group_usage, jint max_over_quota_jobs, jint filter_offensive,
                jdouble off_mem_mb, jdouble off_cpus, jobject out_ranked, jintArray out_n, jobject out_dru,
                jobject out_order, jintArray out_order_n) {
  cook_tasks_soa r, p; cook_user_table u; cook_pool_quota pq, gq; cook_rank_params prm;
  memset(&r, 0, sizeof(r)); memset(&p, 0, sizeof(p)); memset(&u, 0, sizeof(u));
  tasks_from(env, n_running, running, &r); tasks_from(env, n_pending, pending, &p); users_from(env, n_users, users, &u);
  quota_from(env, pool_quota, &pq); quota_from(env, group_quota, &gq);
  prm.max_over_quota_jobs = max_over_quota_jobs; prm.filter_offensive = filter_offensive;
  prm.offensive_max_mem_mb = off_mem_mb; prm.offensive_max_cpus = off_cpus;
  int32_t n = 0, on = 0;
  jint rc = cook_rank((cook_pool*)(intptr_t)pool, &r, &p, &u, &pq, &gq, one(env, group_usage), &prm, one(env, out_ranked),
                      &n, one(env, out_dru), one(env, out_order), &on);
  (*env)->SetIntArrayRegion(env, out_n, 0, 1, (jint*)&n);
  if (out_order_n) (*env)->SetIntArrayRegion(env, out_order_n, 0, 1, (jint*)&on);
  return rc;
}

/* ---- M0-M6 ------------------------------------------------------------------------------------ */
JFN(jint, match)(JNIEnv* env, jclass k, jlong pool, jobject ranked_idx, jint n_ranked, jint n_jobs, jobjectArray jobs,
                 jint n_offers, jint n_attr_cols, jobjectArray offers, jint n_groups, jobjectArray groups, jint n_users,
                 jobjectArray users, jdoubleArray pool_quota, jintArray iparams /* num_considerable, enforce_rate_limit,
                 host_lifetime_mins, fitness_kind, reuse_resident, max_ctas */, jdouble good_enough_fitness,
                 jobject out_considerable, jobject out_assign, jobject out_ports, jint max_ports, jobject out_fail,
                 jobject out_stats /* sizeof(cook_match_stats) bytes */) {
  cook_jobs_soa j; cook_offers_soa o; cook_groups g; cook_user_table u; cook_pool_quota pq; cook_match_params prm;
  memset(&j, 0, sizeof(j)); memset(&o, 0, sizeof(o)); memset(&g, 0, sizeof(g)); memset(&u, 0, sizeof(u));
  jobs_from(env, n_jobs, jobs, &j); offers_from(env, n_offers, n_attr_cols, offers, &o);
  int have_g = groups_from(env, n_groups, groups, &g);
  users_from(env, n_users, users, &u); quota_from(env, pool_quota, &pq);
  jint ip[6]; (*env)->GetIntArrayRegion(env, iparams, 0, 6, ip);
  memset(&prm, 0, sizeof(prm));
  prm.num_considerable = ip[0]; prm.enforce_rate_limit = ip[1]; prm.host_lifetime_mins = ip[2]; prm.fitness_kind = ip[3];
  prm.good_enough_fitness = good_enough_fitness; prm.reuse_resident = ip[4]; prm.max_ctas = ip[5];
  return cook_match((cook_pool*)(intptr_t)pool, one(env, ranked_idx), n_ranked, &j, &o, have_g ? &g : NULL, &u, &pq, &prm,
                    one(env, out_considerable), one(env, out_assign), one(env, out_ports), max_ports, one(env, out_fail),
                    (cook_match_stats*)one(env, out_stats));
}
JFN(jint, matchFailures)(JNIEnv* env, jclass k, jlong pool, jobject k_idx, jint n, jobject out_counts) {
  return cook_match_failures((cook_pool*)(intptr_t)pool, one(env, k_idx), n, (cook_failure_counts*)one(env, out_counts));
}

/* ---- resident pool state (§8f-1) --------------------------------------------------------------- */
/* one batch from the tx-report tap: `pending` holds the jobs_from columns of the upserted rows */
JFN(jint, stateApply)(JNIEnv* env, jclass k, jlong pool, jint reset, jint n_pending, jobjectArray pending,
                      jobject pending_priority, jobject pending_job_id, jint n_pending_rm, jobject pending_rm_job_id,
                      jint n_running, jobjectArray running, jint n_running_rm, jobject running_rm_task_id,
                      jobject running_hostname_id, jobject running_group_off, jobject running_group_idx) {
  cook_state_delta d;
  memset(&d, 0, sizeof(d));
  d.reset = reset;
  if (pending) jobs_from(env, n_pending, pending, &d.pending);
  d.pending_priority = one(env, pending_priority); d.pending_job_id = one(env, pending_job_id);
  d.n_pending_rm = n_pending_rm; d.pending_rm_job_id = one(env, pending_rm_job_id);
  if (running) tasks_from(env, n_running, running, &d.running);
  d.n_running_rm = n_running_rm; d.running_rm_task_id = one(env, running_rm_task_id);
  d.running_hostname_id = one(env, running_hostname_id);
  d.running_group_off = one(env, running_group_off); d.running_group_idx = one(env, running_group_idx);
  return cook_state_apply((cook_pool*)(intptr_t)pool, &d);
}
/* launches by job id: the task columns the device already holds are not sent (hostname_id may be null) */
JFN(jint, stateLaunch)(JNIEnv* env, jclass k, jlong pool, jint n, jobject job_id, jobject task_id, jobject start_time,
                       jobject hostname_id) {
  return cook_state_launch((cook_pool*)(intptr_t)pool, n, one(env, job_id), one(env, task_id), one(env, start_time),
                           one(env, hostname_id));
}
/* match-time columns of pending jobs in place (a null column is unchanged); clear_reservations != 0 first
 * drops every reservation (reserve-hosts!) */
JFN(jint, statePatch)(JNIEnv* env, jclass k, jlong pool, jint n, jobject job_id, jobject allowed, jobject plugin_accept,
                      jobject reserved_host, jint clear_reservations) {
  return cook_state_patch((cook_pool*)(intptr_t)pool, n, one(env, job_id), one(env, allowed), one(env, plugin_accept),
                          one(env, reserved_host), clear_reservations);
}
/* the running usage of the live running rows: per user ([4][n_users] doubles), of the pool (4 doubles) and per
 * host of hostname_id (run_cpus, run_mem, run_count); every output may be null */
JFN(jint, stateUsage)(JNIEnv* env, jclass k, jlong pool, jint n_users, jobject out_user_usage, jobject out_pool_usage,
                      jint n_hosts, jobject hostname_id, jobject out_run_cpus, jobject out_run_mem,
                      jobject out_run_count) {
  return cook_state_usage((cook_pool*)(intptr_t)pool, n_users, one(env, out_user_usage), one(env, out_pool_usage),
                          n_hosts, one(env, hostname_id), one(env, out_run_cpus), one(env, out_run_mem),
                          one(env, out_run_count));
}
/* each group's running cotasks (the cot_* columns of `groups` for stateMatch / stateRebalance); `hosts` holds the
 * hosts_from columns (only hostname_id and attr are read) or is null; out_cot_hostname_id null: a size query */
JFN(jint, stateCotasks)(JNIEnv* env, jclass k, jlong pool, jint n_groups, jobject attr_col, jint n_hosts,
                        jint n_attr_cols, jobjectArray hosts, jint cap, jobject out_cot_off, jobject out_cot_hostname_id,
                        jobject out_cot_attr_val, jintArray out_n) {
  cook_host_table h;
  memset(&h, 0, sizeof(h));
  if (hosts) hosts_from(env, n_hosts, n_attr_cols, hosts, &h);
  int32_t n = 0;
  jint rc = cook_state_cotasks((cook_pool*)(intptr_t)pool, n_groups, one(env, attr_col), hosts ? &h : NULL, cap,
                               one(env, out_cot_off), one(env, out_cot_hostname_id), one(env, out_cot_attr_val), &n);
  if (rc == COOK_OK) (*env)->SetIntArrayRegion(env, out_n, 0, 1, (jint*)&n);
  return rc;
}
JFN(jint, stateRank)(JNIEnv* env, jclass k, jlong pool, jint n_users, jobjectArray users, jdoubleArray pool_quota,
                     jdoubleArray group_quota, jobject group_usage, jint max_over_quota_jobs, jint filter_offensive,
                     jdouble off_mem_mb, jdouble off_cpus, jobject out_ranked_job_id, jintArray out_n) {
  cook_user_table u; cook_pool_quota pq, gq; cook_rank_params prm;
  memset(&u, 0, sizeof(u));
  users_from(env, n_users, users, &u); quota_from(env, pool_quota, &pq); quota_from(env, group_quota, &gq);
  prm.max_over_quota_jobs = max_over_quota_jobs; prm.filter_offensive = filter_offensive;
  prm.offensive_max_mem_mb = off_mem_mb; prm.offensive_max_cpus = off_cpus;
  int32_t n = 0;
  jint rc = cook_state_rank((cook_pool*)(intptr_t)pool, &u, &pq, &gq, one(env, group_usage), &prm,
                            one(env, out_ranked_job_id), &n);
  (*env)->SetIntArrayRegion(env, out_n, 0, 1, (jint*)&n);
  return rc;
}
/* stateRank plus the jobs the rank dropped as offensive (filter-offensive-jobs), as job ids in out_offensive_job_id
 * (room for offensive_cap >= the live pending rows) and their number in out_n_offensive[0] */
JFN(jint, stateRankOffensive)(JNIEnv* env, jclass k, jlong pool, jint n_users, jobjectArray users,
                              jdoubleArray pool_quota, jdoubleArray group_quota, jobject group_usage,
                              jint max_over_quota_jobs, jint filter_offensive, jdouble off_mem_mb, jdouble off_cpus,
                              jobject out_ranked_job_id, jintArray out_n, jobject out_offensive_job_id,
                              jint offensive_cap, jintArray out_n_offensive) {
  cook_user_table u; cook_pool_quota pq, gq; cook_rank_params prm;
  memset(&u, 0, sizeof(u));
  users_from(env, n_users, users, &u); quota_from(env, pool_quota, &pq); quota_from(env, group_quota, &gq);
  prm.max_over_quota_jobs = max_over_quota_jobs; prm.filter_offensive = filter_offensive;
  prm.offensive_max_mem_mb = off_mem_mb; prm.offensive_max_cpus = off_cpus;
  int32_t n = 0, n_off = 0;
  jint rc = cook_state_rank_offensive((cook_pool*)(intptr_t)pool, &u, &pq, &gq, one(env, group_usage), &prm,
                                      one(env, out_ranked_job_id), &n, one(env, out_offensive_job_id), offensive_cap,
                                      &n_off);
  (*env)->SetIntArrayRegion(env, out_n, 0, 1, (jint*)&n);
  (*env)->SetIntArrayRegion(env, out_n_offensive, 0, 1, (jint*)&n_off);
  return rc;
}
/* M0 over the resident queue without a match; iparams = {num_considerable, enforce_rate_limit, quota_only,
 * usage_source, consume} (cook_considerable_params); the job ids go to out_job_id, their number to out_n[0] */
JFN(jint, stateConsiderable)(JNIEnv* env, jclass k, jlong pool, jint n_users, jobjectArray users,
                             jdoubleArray pool_quota, jintArray iparams, jobject out_job_id, jintArray out_n) {
  cook_user_table u; cook_pool_quota pq; cook_considerable_params prm;
  memset(&u, 0, sizeof(u));
  users_from(env, n_users, users, &u); quota_from(env, pool_quota, &pq);
  jint ip[5]; (*env)->GetIntArrayRegion(env, iparams, 0, 5, ip);
  prm.num_considerable = ip[0]; prm.enforce_rate_limit = ip[1]; prm.quota_only = ip[2]; prm.usage_source = ip[3];
  prm.consume = ip[4];
  int32_t n = 0;
  jint rc = cook_state_considerable((cook_pool*)(intptr_t)pool, &u, &pq, &prm, one(env, out_job_id), &n);
  (*env)->SetIntArrayRegion(env, out_n, 0, 1, (jint*)&n);
  return rc;
}
/* the monitor's user stats over the live rows of `pools` (a long[] of handles: one pool, or a quota group's pools);
 * out_jobs / out_cpus / out_mem hold [4][n_users] values, out_member n_users bytes, out_all_jobs / _cpus / _mem 4
 * values, out_users COOK_USERS_N longs, out_stats sizeof(cook_phase_stats) bytes; quota_rest_ok and out_stats may
 * be null.  More than 64 handles is COOK_E_BADARG: a quota group's stats over a subset of its pools would be wrong */
JFN(jint, stateUserStats)(JNIEnv* env, jclass k, jlongArray pools, jint n_users, jobjectArray users,
                          jobject quota_rest_ok, jobject out_jobs, jobject out_cpus, jobject out_mem, jobject out_member,
                          jobject out_all_jobs, jobject out_all_cpus, jobject out_all_mem, jobject out_users,
                          jobject out_stats) {
  cook_user_table u;
  memset(&u, 0, sizeof(u));
  users_from(env, n_users, users, &u);
  jsize n = (*env)->GetArrayLength(env, pools);
  if (n > 64) return COOK_E_BADARG;
  jlong* h = (*env)->GetLongArrayElements(env, pools, NULL);
  cook_pool* p[64];
  for (jsize i = 0; i < n; i++) p[i] = (cook_pool*)(intptr_t)h[i];
  (*env)->ReleaseLongArrayElements(env, pools, h, JNI_ABORT);
  return cook_state_user_stats(p, (int32_t)n, &u, one(env, quota_rest_ok), one(env, out_jobs), one(env, out_cpus),
                               one(env, out_mem), one(env, out_member), one(env, out_all_jobs), one(env, out_all_cpus),
                               one(env, out_all_mem), one(env, out_users), one(env, out_stats));
}
/* the killers' facts of live running tasks: task_id n longs, max_runtime_ms n longs, cancelled / unknown n bytes (each
 * but task_id may be null: unchanged) */
JFN(jint, stateTaskFacts)(JNIEnv* env, jclass k, jlong pool, jint n, jobject task_id, jobject max_runtime_ms,
                          jobject cancelled, jobject unknown) {
  return cook_state_task_facts((cook_pool*)(intptr_t)pool, n, one(env, task_id), one(env, max_runtime_ms),
                               one(env, cancelled), one(env, unknown));
}
/* the reason fact of running tasks: task_id n longs, reason_code n ints (-1: none) */
JFN(jint, stateTaskReason)(JNIEnv* env, jclass k, jlong pool, jint n, jobject task_id, jobject reason_code) {
  return cook_state_task_reason((cook_pool*)(intptr_t)pool, n, one(env, task_id), one(env, reason_code));
}
/* the stats keys of live pending jobs: job_id n longs, flags n bytes (COOK_JF_*), gpu_model n ints, disk_request and
 * disk_limit n doubles, disk_type n ints (each but job_id may be null: unchanged) */
JFN(jint, stateJobFacts)(JNIEnv* env, jclass k, jlong pool, jint n, jobject job_id, jobject flags, jobject gpu_model,
                         jobject disk_request, jobject disk_limit, jobject disk_type) {
  return cook_state_job_facts((cook_pool*)(intptr_t)pool, n, one(env, job_id), one(env, flags), one(env, gpu_model),
                              one(env, disk_request), one(env, disk_limit), one(env, disk_type));
}
/* the match-cycle metrics of the last resident match: dropped n_dropped ints (may be null when 0); outs = {counts
 * COOK_MMC_N longs, amounts COOK_MMA_N doubles, row ints 3 * COOK_MMR_NI longs, row amounts 3 * COOK_MMR_NF doubles,
 * first job ids 10 longs, first cycles 10 ints, user considerable n_users ints, user matched n_users ints, key kinds,
 * key codes key_cap ints each, key totals key_cap doubles}; out_stats a cook_phase_stats or null */
JFN(jint, stateMatchMetrics)(JNIEnv* env, jclass k, jlong pool, jint n_users, jint n_dropped, jobject dropped,
                             jint unmatched_warn_cycles, jint key_cap, jobjectArray outs, jobject out_stats) {
  return cook_state_match_metrics((cook_pool*)(intptr_t)pool, n_users, n_dropped, one(env, dropped),
                                  unmatched_warn_cycles, key_cap, buf(env, outs, 0), buf(env, outs, 1), buf(env, outs, 2),
                                  buf(env, outs, 3), buf(env, outs, 4), buf(env, outs, 5), buf(env, outs, 6),
                                  buf(env, outs, 7), buf(env, outs, 8), buf(env, outs, 9), buf(env, outs, 10),
                                  (cook_phase_stats*)one(env, out_stats));
}
/* finished tasks: task_id and end_time_ms n longs, success n bytes (null: none succeeded) */
JFN(jint, stateFinish)(JNIEnv* env, jclass k, jlong pool, jint n, jobject task_id, jobject end_time_ms,
                       jobject success) {
  return cook_state_finish((cook_pool*)(intptr_t)pool, n, one(env, task_id), one(env, end_time_ms), one(env, success));
}
/* records by hand: (group, runtime_s) n_add ints each, then forget_group n_forget ints */
JFN(jint, stateGroupRuntimes)(JNIEnv* env, jclass k, jlong pool, jint n_add, jobject group, jobject runtime_s,
                              jint n_forget, jobject forget_group) {
  return cook_state_group_runtimes((cook_pool*)(intptr_t)pool, n_add, one(env, group), one(env, runtime_s), n_forget,
                                   one(env, forget_group));
}
/* the three kill lists over `pools` (a long[] of handles on one device, at most 64); times = {now_ms,
 * default_timeout_ms, max_timeout_ms}; groups: the four group columns (kind, quantile, multiplier, n_jobs), n_groups
 * values each; lists: {linger task id, linger pool, cancel task id, cancel pool, straggler group, straggler task id,
 * straggler pool} (a null task id skips that sweep); caps = {row_cap, entry_cap}; out_n gets the three lengths */
JFN(jint, stateSweep)(JNIEnv* env, jclass k, jlongArray pools, jlongArray times, jint n_groups, jobjectArray groups,
                      jintArray caps, jobjectArray lists, jintArray out_n, jobject out_stats) {
  jsize n = (*env)->GetArrayLength(env, pools);
  if (n > 64) return COOK_E_BADARG;
  jlong* h = (*env)->GetLongArrayElements(env, pools, NULL);
  cook_pool* p[64];
  for (jsize i = 0; i < n; i++) p[i] = (cook_pool*)(intptr_t)h[i];
  (*env)->ReleaseLongArrayElements(env, pools, h, JNI_ABORT);
  jlong t[3]; (*env)->GetLongArrayRegion(env, times, 0, 3, t);
  jint c[2]; (*env)->GetIntArrayRegion(env, caps, 0, 2, c);
  int32_t nl = 0, nc = 0, ns = 0;
  jint rc = cook_state_sweep(p, (int32_t)n, t[0], t[1], t[2], n_groups, buf(env, groups, 0), buf(env, groups, 1),
                             buf(env, groups, 2), buf(env, groups, 3), c[0], buf(env, lists, 0), buf(env, lists, 1),
                             &nl, buf(env, lists, 2), buf(env, lists, 3), &nc, c[1], buf(env, lists, 4),
                             buf(env, lists, 5), buf(env, lists, 6), &ns, one(env, out_stats));
  jint got[3] = {nl, nc, ns};
  (*env)->SetIntArrayRegion(env, out_n, 0, 3, got);
  return rc;
}
/* users' running usage: user n_users ints (null: every user); caps [seg_cap, job_cap]; segs the direct buffers of
 * user, scope, group (ints), jobs (longs), cpus, mem, gpus (doubles), list_off (ints; null without by_group); job_id
 * job_cap longs (null without by_group); out_n gets [n_seg, n_job]; out_stats may be null */
JFN(jint, stateUserUsage)(JNIEnv* env, jclass k, jlongArray pools, jint n_users, jobject user, jint per_pool,
                          jint by_group, jintArray caps, jobjectArray segs, jobject job_id, jintArray out_n,
                          jobject out_stats) {
  jsize n = (*env)->GetArrayLength(env, pools);
  if (n > 64) return COOK_E_BADARG;
  jlong* h = (*env)->GetLongArrayElements(env, pools, NULL);
  cook_pool* p[64];
  for (jsize i = 0; i < n; i++) p[i] = (cook_pool*)(intptr_t)h[i];
  (*env)->ReleaseLongArrayElements(env, pools, h, JNI_ABORT);
  jint c[2]; (*env)->GetIntArrayRegion(env, caps, 0, 2, c);
  int32_t ns = 0, nj = 0;
  jint rc = cook_state_user_usage(p, (int32_t)n, one(env, user), n_users, per_pool, by_group, c[0], buf(env, segs, 0),
                                  buf(env, segs, 1), buf(env, segs, 2), buf(env, segs, 3), buf(env, segs, 4),
                                  buf(env, segs, 5), buf(env, segs, 6), buf(env, segs, 7), c[1], one(env, job_id), &ns,
                                  &nj, one(env, out_stats));
  jint got[2] = {ns, nj};
  (*env)->SetIntArrayRegion(env, out_n, 0, 2, got);
  return rc;
}
/* finished tasks with the history: as stateFinish, plus reason_code n ints (null: each row's reason fact) */
JFN(jint, stateFinishHistory)(JNIEnv* env, jclass k, jlong pool, jint n, jobject task_id, jobject end_time_ms,
                              jobject success, jobject reason_code) {
  return cook_state_finish_history((cook_pool*)(intptr_t)pool, n, one(env, task_id), one(env, end_time_ms),
                                   one(env, success), one(env, reason_code));
}
/* the reason dictionary: reason_code n_reasons ints, mea_culpa n_reasons bytes, failure_limit n_reasons ints */
JFN(jint, stateRetryConfig)(JNIEnv* env, jclass k, jlong pool, jint mea_culpa_limit, jint n_reasons, jobject reason_code,
                            jobject mea_culpa, jobject failure_limit) {
  return cook_state_retry_config((cook_pool*)(intptr_t)pool, mea_culpa_limit, n_reasons, one(env, reason_code),
                                 one(env, mea_culpa), one(env, failure_limit));
}
/* jobs' retry facts: job_id n longs, max_retries n ints, flags n bytes (COOK_RF_*), done_off n + 1 ints and
   done_reason ints (null: no done instance) */
JFN(jint, stateRetryFacts)(JNIEnv* env, jclass k, jlong pool, jint n, jobject job_id, jobject max_retries, jobject flags,
                           jobject done_off, jobject done_reason) {
  return cook_state_retry_facts((cook_pool*)(intptr_t)pool, n, one(env, job_id), one(env, max_retries), one(env, flags),
                                one(env, done_off), one(env, done_reason));
}
/* terminal statuses: as stateFinishHistory, plus preempted n bytes (null: none) and the outputs out_outcome and
   out_attempts, n ints each */
JFN(jint, stateStatus)(JNIEnv* env, jclass k, jlong pool, jint n, jobject task_id, jobject success, jobject end_time_ms,
                       jobject reason_code, jobject preempted, jobject out_outcome, jobject out_attempts) {
  return cook_state_status((cook_pool*)(intptr_t)pool, n, one(env, task_id), one(env, success), one(env, end_time_ms),
                           one(env, reason_code), one(env, preempted), one(env, out_outcome), one(env, out_attempts));
}
/* jobs' list facts: job_id n longs, submit_ms n longs, submit_pool n ints, custom_executor n ints (each null: kept) */
JFN(jint, stateListFacts)(JNIEnv* env, jclass k, jlong pool, jint n, jobject job_id, jobject submit_ms,
                          jobject submit_pool, jobject custom_executor) {
  return cook_state_list_facts((cook_pool*)(intptr_t)pool, n, one(env, job_id), one(env, submit_ms),
                               one(env, submit_pool), one(env, custom_executor));
}
/* the job listing: times [start_ms, end_ms, job_id_lo, job_id_hi]; args [user, states, pool_code,
 * include_custom_executor, limit, cap]; handle_pool n_pools ints (null with pool_code -1); outs the direct buffers of
 * state, job_id, submit_ms, pool (cap ints / longs); out_n gets [n, n_missing]; out_stats may be null */
JFN(jint, stateListJobs)(JNIEnv* env, jclass k, jlongArray pools, jlongArray times, jintArray args, jobject handle_pool,
                         jobjectArray outs, jintArray out_n, jobject out_stats) {
  jsize n = (*env)->GetArrayLength(env, pools);
  if (n > 64) return COOK_E_BADARG;
  jlong* h = (*env)->GetLongArrayElements(env, pools, NULL);
  cook_pool* p[64];
  for (jsize i = 0; i < n; i++) p[i] = (cook_pool*)(intptr_t)h[i];
  (*env)->ReleaseLongArrayElements(env, pools, h, JNI_ABORT);
  jlong t[4]; (*env)->GetLongArrayRegion(env, times, 0, 4, t);
  jint a[6]; (*env)->GetIntArrayRegion(env, args, 0, 6, a);
  int32_t got[2] = {0, 0};
  jint rc = cook_state_list_jobs(p, (int32_t)n, a[0], a[1], t[0], t[1], t[2], t[3], a[2], one(env, handle_pool), a[3],
                                 a[4], a[5], buf(env, outs, 0), buf(env, outs, 1), buf(env, outs, 2), buf(env, outs, 3),
                                 &got[0], &got[1], one(env, out_stats));
  jint g[2] = {got[0], got[1]};
  (*env)->SetIntArrayRegion(env, out_n, 0, 2, g);
  return rc;
}
/* the completed-job log: cols the direct buffers of job_id, stamp, user, submit_ms, submit_pool, custom_executor
 * (n ints: -1 nil, 0 false, 1 true), kind (n bytes) */
JFN(jint, stateCompletedSeed)(JNIEnv* env, jclass k, jlong pool, jlong since_ms, jint n, jobjectArray cols) {
  return cook_state_completed_seed((cook_pool*)(intptr_t)pool, since_ms, n, buf(env, cols, 0), buf(env, cols, 1),
                                   buf(env, cols, 2), buf(env, cols, 3), buf(env, cols, 4), buf(env, cols, 5),
                                   buf(env, cols, 6));
}
JFN(jint, stateCompletedRecord)(JNIEnv* env, jclass k, jlong pool, jint n, jobjectArray cols) {
  return cook_state_completed_record((cook_pool*)(intptr_t)pool, n, buf(env, cols, 0), buf(env, cols, 1),
                                     buf(env, cols, 2), buf(env, cols, 3), buf(env, cols, 4), buf(env, cols, 5),
                                     buf(env, cols, 6));
}
JFN(jint, stateCompletedAdvance)(JNIEnv* env, jclass k, jlong pool, jlong since_ms) {
  return cook_state_completed_advance((cook_pool*)(intptr_t)pool, since_ms);
}
/* the completed listing: times [start_ms, end_ms, job_id_lo, job_id_hi]; args [user, state, pool_code,
 * include_custom_executor, limit, cap]; handle_pool n_pools ints (null with pool_code -1); outs the direct buffers of
 * job_id, submit_ms, pool (cap longs / ints); out_n gets [n]; out_stats may be null */
JFN(jint, stateListCompleted)(JNIEnv* env, jclass k, jlongArray pools, jlongArray times, jintArray args,
                              jobject handle_pool, jobjectArray outs, jintArray out_n, jobject out_stats) {
  jsize n = (*env)->GetArrayLength(env, pools);
  if (n > 64) return COOK_E_BADARG;
  jlong* h = (*env)->GetLongArrayElements(env, pools, NULL);
  cook_pool* p[64];
  for (jsize i = 0; i < n; i++) p[i] = (cook_pool*)(intptr_t)h[i];
  (*env)->ReleaseLongArrayElements(env, pools, h, JNI_ABORT);
  jlong t[4]; (*env)->GetLongArrayRegion(env, times, 0, 4, t);
  jint a[6]; (*env)->GetIntArrayRegion(env, args, 0, 6, a);
  int32_t got = 0;
  jint rc = cook_state_list_completed(p, (int32_t)n, a[0], a[1], t[0], t[1], t[2], t[3], a[2], one(env, handle_pool),
                                      a[3], a[4], a[5], buf(env, outs, 0), buf(env, outs, 1), buf(env, outs, 2), &got,
                                      one(env, out_stats));
  jint g = got;
  (*env)->SetIntArrayRegion(env, out_n, 0, 1, &g);
  return rc;
}
/* the history's seed: cols the direct buffers of task_id, user, start_ms, end_ms, cpus, mem, success, reason_code */
JFN(jint, stateHistorySeed)(JNIEnv* env, jclass k, jlong pool, jlong since_ms, jint n, jobjectArray cols) {
  return cook_state_history_seed((cook_pool*)(intptr_t)pool, since_ms, n, buf(env, cols, 0), buf(env, cols, 1),
                                 buf(env, cols, 2), buf(env, cols, 3), buf(env, cols, 4), buf(env, cols, 5),
                                 buf(env, cols, 6), buf(env, cols, 7));
}
JFN(jint, stateHistoryAdvance)(JNIEnv* env, jclass k, jlong pool, jlong since_ms) {
  return cook_state_history_advance((cook_pool*)(intptr_t)pool, since_ms);
}
/* instance stats: times [now_ms, start_ms, end_ms, task_id_lo, task_id_hi]; segs the direct buffers of kind, user,
 * reason (seg_cap ints), count (seg_cap longs), total (3 * seg_cap doubles), pct (15 * seg_cap doubles); leaders the
 * direct buffers of user (2 * COOK_IS_LEADERS ints) and total (2 * COOK_IS_LEADERS doubles); out_n gets [n_seg,
 * n_leader]; out_stats may be null */
JFN(jint, stateInstanceStats)(JNIEnv* env, jclass k, jlongArray pools, jlongArray times, jint status, jint seg_cap,
                              jobjectArray segs, jobjectArray leaders, jintArray out_n, jobject out_stats) {
  jsize n = (*env)->GetArrayLength(env, pools);
  if (n > 64) return COOK_E_BADARG;
  jlong* h = (*env)->GetLongArrayElements(env, pools, NULL);
  cook_pool* p[64];
  for (jsize i = 0; i < n; i++) p[i] = (cook_pool*)(intptr_t)h[i];
  (*env)->ReleaseLongArrayElements(env, pools, h, JNI_ABORT);
  jlong t[5]; (*env)->GetLongArrayRegion(env, times, 0, 5, t);
  int32_t ns = 0, nl = 0;
  /* COOK_IS_SUCCESS and COOK_IS_FAILED read the histories (now_ms unused) */
  jint rc = status == COOK_IS_SUCCESS || status == COOK_IS_FAILED
                ? cook_state_history_stats(p, (int32_t)n, status, t[1], t[2], t[3], t[4], seg_cap, buf(env, segs, 0),
                                           buf(env, segs, 1), buf(env, segs, 2), buf(env, segs, 3), buf(env, segs, 4),
                                           buf(env, segs, 5), buf(env, leaders, 0), buf(env, leaders, 1), &ns, &nl,
                                           one(env, out_stats))
                : cook_state_instance_stats(p, (int32_t)n, t[0], status, t[1], t[2], t[3], t[4], seg_cap,
                                            buf(env, segs, 0), buf(env, segs, 1), buf(env, segs, 2), buf(env, segs, 3),
                                            buf(env, segs, 4), buf(env, segs, 5), buf(env, leaders, 0),
                                            buf(env, leaders, 1), &ns, &nl, one(env, out_stats));
  jint got[2] = {ns, nl};
  (*env)->SetIntArrayRegion(env, out_n, 0, 2, got);
  return rc;
}
/* why queried jobs are not scheduled: job_id n longs; outputs direct buffers of n bytes (status), 4n doubles (usage),
 * n ints (position, n_ahead), COOK_UNSCHED_AHEAD*n longs (ahead job ids), n bytes (plugin deferred); out_stats may be
 * null */
JFN(jint, stateUnscheduled)(JNIEnv* env, jclass k, jlong pool, jint n, jobject job_id, jobject out_status,
                            jobject out_usage, jobject out_position, jobject out_n_ahead, jobject out_ahead_job_id,
                            jobject out_plugin_deferred, jobject out_stats) {
  return cook_state_unscheduled((cook_pool*)(intptr_t)pool, n, one(env, job_id), one(env, out_status),
                                one(env, out_usage), one(env, out_position), one(env, out_n_ahead),
                                one(env, out_ahead_job_id), one(env, out_plugin_deferred), one(env, out_stats));
}
/* the fingerprints and the recount of the resident rows: out_digest is a direct buffer of sizeof(cook_state_digest_out),
 * out_pending_bucket / out_running_bucket direct buffers of n_buckets cook_fp each (null when n_buckets == 0) */
JFN(jint, stateDigest)(JNIEnv* env, jclass k, jlong pool, jint n_buckets, jobject out_digest, jobject out_pending_bucket,
                       jobject out_running_bucket) {
  return cook_state_digest((cook_pool*)(intptr_t)pool, n_buckets, (cook_state_digest_out*)one(env, out_digest),
                           (cook_fp*)one(env, out_pending_bucket), (cook_fp*)one(env, out_running_bucket));
}
/* the live rows (bucket_mask: those of the selected buckets) as a delta's arrays.  cols: 33 direct buffers in the field
 * order of cook_state_rows (the 20 of cook_jobs_rows, pending_priority, pending_job_id, the 8 of cook_tasks_rows,
 * running_hostname_id, running_group_off, running_group_idx), a null element skips the column; a null `cols` asks for
 * the sizes.  cap and out_n hold {pending, running, entries[4]} */
JFN(jint, stateExport)(JNIEnv* env, jclass k, jlong pool, jint n_buckets, jobject bucket_mask, jintArray cap,
                       jobjectArray cols, jintArray out_n) {
  cook_state_rows rows; cook_state_sizes c, n;
  void** field = (void**)&rows;   /* cook_state_rows holds nothing but pointers */
  memset(&rows, 0, sizeof(rows)); memset(&n, 0, sizeof(n));
  if (cols)
    for (int i = 0; i < (int)(sizeof(rows) / sizeof(void*)); i++)
      field[i] = one(env, (*env)->GetObjectArrayElement(env, cols, i));
  if (cap) (*env)->GetIntArrayRegion(env, cap, 0, 6, (jint*)&c);
  jint rc = cook_state_export((cook_pool*)(intptr_t)pool, n_buckets, (const uint8_t*)one(env, bucket_mask), cap ? &c : NULL,
                              cols ? &rows : NULL, &n);
  if (rc == COOK_OK) (*env)->SetIntArrayRegion(env, out_n, 0, 6, (jint*)&n);
  return rc;
}
/* the live queue as job ids (a null out_job_id asks for the length) */
JFN(jint, stateQueue)(JNIEnv* env, jclass k, jlong pool, jint cap, jobject out_job_id, jintArray out_n) {
  int32_t n = 0;
  jint rc = cook_state_queue((cook_pool*)(intptr_t)pool, cap, one(env, out_job_id), &n);
  if (rc == COOK_OK) (*env)->SetIntArrayRegion(env, out_n, 0, 1, (jint*)&n);
  return rc;
}
typedef int32_t (*state_match_fn)(cook_pool*, const cook_offers_soa*, const cook_groups*, const cook_user_table*,
                                  const cook_pool_quota*, const cook_match_params*, int64_t*, int32_t*, int32_t*, int32_t,
                                  uint8_t*, cook_match_stats*);
static jint state_match(state_match_fn fn, JNIEnv* env, jlong pool, jint n_offers, jint n_attr_cols, jobjectArray offers,
                        jint n_groups, jobjectArray groups, jint n_users, jobjectArray users, jdoubleArray pool_quota,
                        jintArray iparams, jdouble good_enough_fitness, jobject out_considerable_job_id,
                        jobject out_assign, jobject out_ports, jint max_ports, jobject out_fail, jobject out_stats) {
  cook_offers_soa o; cook_groups g; cook_user_table u; cook_pool_quota pq; cook_match_params prm;
  memset(&o, 0, sizeof(o)); memset(&g, 0, sizeof(g)); memset(&u, 0, sizeof(u));
  offers_from(env, n_offers, n_attr_cols, offers, &o);
  int have_g = groups_from(env, n_groups, groups, &g);
  users_from(env, n_users, users, &u); quota_from(env, pool_quota, &pq);
  jint ip[6]; (*env)->GetIntArrayRegion(env, iparams, 0, 6, ip);
  memset(&prm, 0, sizeof(prm));
  prm.num_considerable = ip[0]; prm.enforce_rate_limit = ip[1]; prm.host_lifetime_mins = ip[2]; prm.fitness_kind = ip[3];
  prm.good_enough_fitness = good_enough_fitness; prm.reuse_resident = ip[4]; prm.max_ctas = ip[5];
  return fn((cook_pool*)(intptr_t)pool, &o, have_g ? &g : NULL, &u, &pq, &prm, one(env, out_considerable_job_id),
            one(env, out_assign), one(env, out_ports), max_ports, one(env, out_fail), (cook_match_stats*)one(env, out_stats));
}
JFN(jint, stateMatch)(JNIEnv* env, jclass k, jlong pool, jint n_offers, jint n_attr_cols, jobjectArray offers,
                      jint n_groups, jobjectArray groups, jint n_users, jobjectArray users, jdoubleArray pool_quota,
                      jintArray iparams /* as match */, jdouble good_enough_fitness, jobject out_considerable_job_id,
                      jobject out_assign, jobject out_ports, jint max_ports, jobject out_fail, jobject out_stats) {
  return state_match(cook_state_match, env, pool, n_offers, n_attr_cols, offers, n_groups, groups, n_users, users,
                     pool_quota, iparams, good_enough_fitness, out_considerable_job_id, out_assign, out_ports, max_ports,
                     out_fail, out_stats);
}
/* stateMatch with the users' usage, the offers' run columns and the groups' cot lists derived on the device from
 * the resident running rows: those columns of `users`, `offers` and `groups` are not read and may be null */
JFN(jint, stateMatchDerived)(JNIEnv* env, jclass k, jlong pool, jint n_offers, jint n_attr_cols, jobjectArray offers,
                             jint n_groups, jobjectArray groups, jint n_users, jobjectArray users, jdoubleArray pool_quota,
                             jintArray iparams, jdouble good_enough_fitness, jobject out_considerable_job_id,
                             jobject out_assign, jobject out_ports, jint max_ports, jobject out_fail, jobject out_stats) {
  return state_match(cook_state_match_derived, env, pool, n_offers, n_attr_cols, offers, n_groups, groups, n_users,
                     users, pool_quota, iparams, good_enough_fitness, out_considerable_job_id, out_assign, out_ports,
                     max_ports, out_fail, out_stats);
}

/* the offers that arrived, one row each (offers in cook_offers_soa field order; name_rank, run_* and reserved are not
 * read), their ids, single-shot flags, "gpus" scalars and hostname bytes as a CSR (null hostname_off: all empty) */
JFN(jint, stateOffersAdd)(JNIEnv* env, jclass k, jlong pool, jint n_offers, jint n_attr_cols, jobjectArray offers,
                          jobject offer_id, jobject single_shot, jobject offer_gpus, jobject hostname,
                          jobject hostname_off, jlong now_ms) {
  cook_offers_soa o;
  memset(&o, 0, sizeof(o));
  offers_from(env, n_offers, n_attr_cols, offers, &o);
  return cook_state_offers_add((cook_pool*)(intptr_t)pool, &o, one(env, offer_id), one(env, single_shot),
                               one(env, offer_gpus), one(env, hostname), one(env, hostname_off), now_ms);
}
/* expiry, the merge of the live offers, the derived match, consumption; out_assign gets hostname codes and
 * out_gone_offer_id / out_gone_fate (gone_cap entries each) the offers that left, their count in out_n_gone[0] */
JFN(jint, stateMatchOffers)(JNIEnv* env, jclass k, jlong pool, jlong now_ms, jlong incubate_ms, jint n_groups,
                            jobjectArray groups, jint n_users, jobjectArray users, jdoubleArray pool_quota,
                            jintArray iparams, jdouble good_enough_fitness, jobject out_considerable_job_id,
                            jobject out_assign, jobject out_ports, jint max_ports, jobject out_fail,
                            jobject out_gone_offer_id, jobject out_gone_fate, jint gone_cap, jintArray out_n_gone,
                            jobject out_stats) {
  cook_groups g; cook_user_table u; cook_pool_quota pq; cook_match_params prm;
  memset(&g, 0, sizeof(g)); memset(&u, 0, sizeof(u));
  int have_g = groups_from(env, n_groups, groups, &g);
  users_from(env, n_users, users, &u); quota_from(env, pool_quota, &pq);
  jint ip[6]; (*env)->GetIntArrayRegion(env, iparams, 0, 6, ip);
  memset(&prm, 0, sizeof(prm));
  prm.num_considerable = ip[0]; prm.enforce_rate_limit = ip[1]; prm.host_lifetime_mins = ip[2]; prm.fitness_kind = ip[3];
  prm.good_enough_fitness = good_enough_fitness; prm.reuse_resident = ip[4]; prm.max_ctas = ip[5];
  int32_t n_gone = 0;
  jint rc = cook_state_match_offers((cook_pool*)(intptr_t)pool, now_ms, incubate_ms, have_g ? &g : NULL, &u, &pq, &prm,
                                    one(env, out_considerable_job_id), one(env, out_assign), one(env, out_ports),
                                    max_ports, one(env, out_fail), one(env, out_gone_offer_id), one(env, out_gone_fate),
                                    gone_cap, &n_gone, (cook_match_stats*)one(env, out_stats));
  (*env)->SetIntArrayRegion(env, out_n_gone, 0, 1, (jint*)&n_gone);
  return rc;
}

/* the rebalancer over the resident rows; out_victim_task_id holds victim_cap task ids */
typedef int32_t (*state_rebalance_fn)(cook_pool*, const cook_host_table*, const cook_groups*, const cook_user_table*,
                                      const cook_rebalance_params*, cook_decision*, int64_t*, int64_t*, int32_t, int32_t*);
static jint state_rebalance(state_rebalance_fn fn, JNIEnv* env, jlong pool, jint n_hosts, jint n_attr_cols,
                            jobjectArray hosts, jint n_groups, jobjectArray groups, jint n_users, jobjectArray users,
                            jint max_preemption, jdouble min_dru_diff, jdouble safe_dru_threshold, jint host_lifetime_mins,
                            jobject out_decisions, jobject out_decision_job_id, jobject out_victim_task_id,
                            jint victim_cap, jintArray out_n) {
  cook_host_table h; cook_groups g; cook_user_table u; cook_rebalance_params prm;
  memset(&h, 0, sizeof(h)); memset(&g, 0, sizeof(g)); memset(&u, 0, sizeof(u));
  hosts_from(env, n_hosts, n_attr_cols, hosts, &h);
  int have_g = groups_from(env, n_groups, groups, &g); users_from(env, n_users, users, &u);
  prm.max_preemption = max_preemption; prm.min_dru_diff = min_dru_diff; prm.safe_dru_threshold = safe_dru_threshold;
  prm.host_lifetime_mins = host_lifetime_mins;
  int32_t n = 0;
  jint rc = fn((cook_pool*)(intptr_t)pool, &h, have_g ? &g : NULL, &u, &prm, (cook_decision*)one(env, out_decisions),
               one(env, out_decision_job_id), one(env, out_victim_task_id), victim_cap, &n);
  (*env)->SetIntArrayRegion(env, out_n, 0, 1, (jint*)&n);
  return rc;
}
JFN(jint, stateRebalance)(JNIEnv* env, jclass k, jlong pool, jint n_hosts, jint n_attr_cols, jobjectArray hosts,
                          jint n_groups, jobjectArray groups, jint n_users, jobjectArray users, jint max_preemption,
                          jdouble min_dru_diff, jdouble safe_dru_threshold, jint host_lifetime_mins,
                          jobject out_decisions, jobject out_decision_job_id, jobject out_victim_task_id,
                          jint victim_cap, jintArray out_n) {
  return state_rebalance(cook_state_rebalance, env, pool, n_hosts, n_attr_cols, hosts, n_groups, groups, n_users, users,
                         max_preemption, min_dru_diff, safe_dru_threshold, host_lifetime_mins, out_decisions,
                         out_decision_job_id, out_victim_task_id, victim_cap, out_n);
}
/* stateRebalance with the groups' cot lists derived on the device over `hosts` (those columns are not read) */
JFN(jint, stateRebalanceDerived)(JNIEnv* env, jclass k, jlong pool, jint n_hosts, jint n_attr_cols, jobjectArray hosts,
                                 jint n_groups, jobjectArray groups, jint n_users, jobjectArray users, jint max_preemption,
                                 jdouble min_dru_diff, jdouble safe_dru_threshold, jint host_lifetime_mins,
                                 jobject out_decisions, jobject out_decision_job_id, jobject out_victim_task_id,
                                 jint victim_cap, jintArray out_n) {
  return state_rebalance(cook_state_rebalance_derived, env, pool, n_hosts, n_attr_cols, hosts, n_groups, groups, n_users,
                         users, max_preemption, min_dru_diff, safe_dru_threshold, host_lifetime_mins, out_decisions,
                         out_decision_job_id, out_victim_task_id, victim_cap, out_n);
}
/* stateRebalanceDerived with the hosts' spare columns derived from the live offers (those columns are not read) */
JFN(jint, stateRebalanceOffers)(JNIEnv* env, jclass k, jlong pool, jint n_hosts, jint n_attr_cols, jobjectArray hosts,
                                jint n_groups, jobjectArray groups, jint n_users, jobjectArray users, jint max_preemption,
                                jdouble min_dru_diff, jdouble safe_dru_threshold, jint host_lifetime_mins,
                                jobject out_decisions, jobject out_decision_job_id, jobject out_victim_task_id,
                                jint victim_cap, jintArray out_n) {
  return state_rebalance(cook_state_rebalance_offers, env, pool, n_hosts, n_attr_cols, hosts, n_groups, groups, n_users,
                         users, max_preemption, min_dru_diff, safe_dru_threshold, host_lifetime_mins, out_decisions,
                         out_decision_job_id, out_victim_task_id, victim_cap, out_n);
}

/* ---- B1-B6 ------------------------------------------------------------------------------------ */
JFN(jint, rebalance)(JNIEnv* env, jclass k, jlong pool, jint n_running, jobjectArray running, jobject running_host,
                     jint n_pending, jobjectArray pending, jobject pending_job_id, jobject pending_priority, jint n_hosts,
                     jint n_attr_cols, jobjectArray hosts, jint n_groups, jobjectArray groups, jint n_users,
                     jobjectArray users, jint max_preemption, jdouble min_dru_diff, jdouble safe_dru_threshold,
                     jint host_lifetime_mins, jobject out_decisions, jobject out_victims, jintArray out_n) {
  cook_running_soa r; cook_jobs_soa p; cook_host_table h; cook_groups g; cook_user_table u; cook_rebalance_params prm;
  memset(&r, 0, sizeof(r)); memset(&p, 0, sizeof(p)); memset(&h, 0, sizeof(h)); memset(&g, 0, sizeof(g)); memset(&u, 0, sizeof(u));
  tasks_from(env, n_running, running, &r.t); r.host = one(env, running_host);
  jobs_from(env, n_pending, pending, &p); hosts_from(env, n_hosts, n_attr_cols, hosts, &h);
  int have_g = groups_from(env, n_groups, groups, &g); users_from(env, n_users, users, &u);
  prm.max_preemption = max_preemption; prm.min_dru_diff = min_dru_diff; prm.safe_dru_threshold = safe_dru_threshold;
  prm.host_lifetime_mins = host_lifetime_mins;
  int32_t n = 0;
  jint rc = cook_rebalance((cook_pool*)(intptr_t)pool, &r, &p, one(env, pending_job_id), one(env, pending_priority), &h,
                           have_g ? &g : NULL, &u, &prm, (cook_decision*)one(env, out_decisions), one(env, out_victims), &n);
  (*env)->SetIntArrayRegion(env, out_n, 0, 1, (jint*)&n);
  return rc;
}

/* ---- phase timing / multi-GPU ------------------------------------------------------------------ */
JFN(jint, lastStats)(JNIEnv* env, jclass k, jlong pool, jint phase, jobject out /* sizeof(cook_phase_stats) */) {
  return cook_last_stats((cook_pool*)(intptr_t)pool, phase, (cook_phase_stats*)one(env, out));
}
JFN(jint, commUniqueId)(JNIEnv* env, jclass k, jobject out128) { return cook_comm_unique_id(one(env, out128)); }
JFN(jint, commInit)(JNIEnv* env, jclass k, jobject id128, jint rank, jint world, jint device, jlongArray out_comm) {
  void* c = NULL;
  jint rc = cook_comm_init(one(env, id128), rank, world, device, &c);
  jlong h = (jlong)(intptr_t)c; (*env)->SetLongArrayRegion(env, out_comm, 0, 1, &h);
  return rc;
}
JFN(jint, commDestroy)(JNIEnv* env, jclass k, jlong comm) { return cook_comm_destroy((void*)(intptr_t)comm); }
JFN(jint, exchangeUsage)(JNIEnv* env, jclass k, jlong pool, jlong comm, jint world, jint n_pad, jobject out_all) {
  return cook_exchange_usage((cook_pool*)(intptr_t)pool, (void*)(intptr_t)comm, world, n_pad, one(env, out_all));
}
/* all of this JVM's pools in one call: `pools` is a long[] of handles (one all-gather per cycle) */
JFN(jint, exchangeUsageBatch)(JNIEnv* env, jclass k, jlongArray pools, jlong comm, jint world, jint n_pad, jint n_slots,
                              jobject out_all) {
  jsize n = (*env)->GetArrayLength(env, pools);
  jlong* h = (*env)->GetLongArrayElements(env, pools, NULL);
  cook_pool* p[64];
  if (n > 64) n = 64;
  for (jsize i = 0; i < n; i++) p[i] = (cook_pool*)(intptr_t)h[i];
  (*env)->ReleaseLongArrayElements(env, pools, h, JNI_ABORT);
  return cook_exchange_usage_batch(p, (int32_t)n, (void*)(intptr_t)comm, world, n_pad, n_slots, one(env, out_all));
}
