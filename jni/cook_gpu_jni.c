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
