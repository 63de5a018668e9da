/* minimal.c -- the ydsched C ABI from plain C: register two servants, decide a small queue,
 * renew and free the leases.  Links against any library that speaks the ABI:
 *
 *     gcc -std=c99 -Iinclude examples/minimal.c -o minimal -Lyadcc_b200 -lydsched      (H100)
 *
 * (the test-suite builds it against the CPU oracle to check that the headers are plain C and
 * that the calls behave as documented).  Mirrors what SchedulerServiceImpl does with
 * TaskDispatcher (yadcc/scheduler/scheduler_service_impl.cc:171-315). */
#include <stdio.h>
#include <string.h>

#include "ydsched.h"

#define NS 1000000000ll

int main(void) {
  yd_config cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.abi_version = YD_ABI_VERSION;
  cfg.servant_min_memory_for_accepting_new_task = "10G";
  yd_sched* s = yd_create(&cfg);
  if (!s) {
    fprintf(stderr, "yd_create failed (backend %s)\n", yd_backend_name());
    return 2;
  }
  const char* digest = "0123456789abcdef0123456789abcdef0123456789abcdef0123456789abcdef";
  const char* envs[1];
  envs[0] = digest;
  {
    int i;
    for (i = 0; i < 2; ++i) {
      char loc[32];
      yd_servant sv;
      memset(&sv, 0, sizeof sv);
      snprintf(loc, sizeof loc, "10.0.0.%d:8335", i + 1);
      sv.version = 8;
      sv.priority = YD_PRIORITY_USER;
      sv.num_envs = 1;
      sv.observed_location = loc;
      sv.reported_location = loc;
      sv.env_digests = envs;
      sv.num_processors = 16;
      sv.current_load = 0;
      sv.max_tasks = 2;
      sv.total_memory_in_bytes = 64ull << 30;
      sv.memory_available_in_bytes = 40ull << 30;
      yd_keep_servant_alive(s, 0, &sv, 10 * NS);
    }
  }
  /* five requests from one machine: four slots exist, the fifth times out */
  yd_task_req reqs[5];
  yd_grant grants[5];
  {
    int i;
    for (i = 0; i < 5; ++i) {
      reqs[i].env_id = yd_intern_env(s, digest, strlen(digest));
      reqs[i].min_version = 8;
      reqs[i].requestor_ip = yd_intern_ip(s, "10.9.9.9", 8);
      reqs[i].flags = 0;
      reqs[i].expires_in_ns = 15 * NS;
    }
  }
  yd_wait_for_starting_new_tasks(s, 1 * NS, reqs, 5, grants);
  {
    int i, granted = 0;
    for (i = 0; i < 5; ++i) {
      if (grants[i].status == YD_STATUS_GRANTED) {
        printf("request %d -> task %llu on %s\n", i, (unsigned long long)grants[i].task_id,
               yd_servant_location(s, grants[i].servant_index));
        ++granted;
      } else {
        printf("request %d -> %s\n", i, grants[i].status == YD_STATUS_TIMEOUT ? "timeout" : "environment not found");
      }
    }
    if (granted != 4 || grants[4].status != YD_STATUS_TIMEOUT) return 1;
  }
  {
    uint64_t ids[2];
    uint8_t ok[2];
    ids[0] = grants[0].task_id;
    ids[1] = 12345; /* unknown */
    yd_keep_task_alive(s, 2 * NS, ids, 2, 15 * NS, ok);
    printf("keep-alive: %d %d\n", ok[0], ok[1]);
    if (ok[0] != 1 || ok[1] != 0) return 1;
    yd_free_tasks(s, ids, 1);
  }
  /* one slot is free again */
  yd_wait_for_starting_new_tasks(s, 3 * NS, reqs, 1, grants);
  printf("after free: %s, %llu live leases\n", grants[0].status == YD_STATUS_GRANTED ? "granted" : "not granted",
         (unsigned long long)yd_num_tasks(s));
  if (grants[0].status != YD_STATUS_GRANTED || yd_num_tasks(s) != 4) return 1;
  /* the packed form of the same call: 16-byte requests (lease in milliseconds), 8-byte grants, ids by ordinal */
  {
    yd_task_req16 r16[2];
    yd_grant8 g8[2];
    yd_packed_ids ids;
    uint64_t gone = grants[0].task_id;
    yd_grant g;
    int i;
    for (i = 0; i < 2; ++i) {
      r16[i].env_id = reqs[0].env_id;
      r16[i].min_version = 8;
      r16[i].requestor_ip = reqs[0].requestor_ip;
      r16[i].lease = 15000u | (i == 1 ? YD_LEASE_PREFETCH : 0u);
    }
    yd_wait_for_starting_new_tasks_packed(s, 4 * NS, r16, 2, g8, &ids); /* every slot is taken */
    if (yd_unpack_grant(g8[0], ids).status != YD_STATUS_TIMEOUT || yd_unpack_grant(g8[1], ids).status != YD_STATUS_TIMEOUT) return 1;
    yd_free_tasks(s, &gone, 1);
    yd_wait_for_starting_new_tasks_packed(s, 5 * NS, r16, 2, g8, &ids); /* one slot came back */
    g = yd_unpack_grant(g8[0], ids);
    printf("packed: task %llu on %s, then %s\n", (unsigned long long)g.task_id, yd_servant_location(s, g.servant_index),
           yd_unpack_grant(g8[1], ids).status == YD_STATUS_TIMEOUT ? "timeout" : "?");
    if (g.status != YD_STATUS_GRANTED || g.task_id != ids.first_task_id || yd_unpack_grant(g8[1], ids).status != YD_STATUS_TIMEOUT ||
        yd_next_task_id(s) != g.task_id + 1 || yd_num_tasks(s) != 4) return 1;
  }
  yd_destroy(s);
  puts("ok");
  return 0;
}
