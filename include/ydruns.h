/* ydruns.h -- runs of Heartbeat, KeepTaskAlive and FreeTask RPCs served as one batch each, and the dispatcher call they
 * need: KeepTaskAlive with a lease length per id.  yd_wire_handle_frames (ydwire.h) hands each run of consecutive frames
 * of one of these methods to the service call below.  Exported by the CUDA library; the CPU checkers export it from
 * builds of their own (yd_keep_tasks_alive as the loop of single calls, include/ydsched_keep_impl.inc; the service
 * calls from include/ydservice_impl.inc).  The range-sharded group's yd_shard_keep_tasks_alive is in ydshard.h. */
#ifndef YDRUNS_H_
#define YDRUNS_H_

#include "ydservice.h"

#ifdef __cplusplus
extern "C" {
#endif

/* n TaskDispatcher::KeepTaskAlive calls (cc:142-165) in array order, call i with its own lease length
 * new_expires_in_ns[i]; ok_out[i] is call i's bool.  KeepTaskAlive changes nothing but the expiry, so
 * every occurrence of a repeated id gets the same answer, and a lease's expiry afterwards is now_ns plus
 * the length of the id's last occurrence. */
void yd_keep_tasks_alive(yd_sched* s, int64_t now_ns, const uint64_t* task_ids, const int64_t* new_expires_in_ns,
                         size_t n, uint8_t* ok_out);

/* Heartbeat x n, in array order: statuses[i] and resps[i] (may be NULL) are exactly what n
 * yd_service_heartbeat calls would return, and the dispatcher's state afterwards is theirs.  Each
 * request is checked as by the single call and a rejected one does nothing.  The accepted ones are
 * registered with one yd_keep_servants_alive and notified with one yd_notify_servants_running_tasks
 * (one collective on a group).  That equals the interleaved order because registering a servant
 * touches no lease and no running task, and a notification reads of the registry only whether its
 * location is registered.  One case differs: heartbeat i notifies under its reported location, and a
 * later heartbeat j that registers exactly that location would be found by i in a batch but not in
 * the interleaved order.  The run is cut before such a j and continues as a second batch. */
void yd_service_heartbeats(yd_service* svc, int64_t now_ns, const yd_heartbeat_request* reqs, size_t n,
                           yd_heartbeat_response* resps, int* statuses);

/* One KeepTaskAliveRequest (scheduler.proto:208-212). */
typedef struct yd_keep_task_alive_request {
  const char* token;
  uint32_t next_keep_alive_in_ms;
  const uint64_t* task_grant_ids;
  size_t n;
  uint8_t* statuses; /* caller's buffer of n: 0/1 per id, written if the request is accepted */
} yd_keep_task_alive_request;

/* KeepTaskAlive x n, in array order, with the answers of n yd_service_keep_task_alive calls
 * (statuses[i] is request i's status).  Each request is checked as by the single call; the ids of
 * the accepted ones, each with its request's lease length, go to one yd_keep_tasks_alive (one
 * yd_shard_keep_tasks_alive on a group). */
void yd_service_keep_tasks_alive(yd_service* svc, int64_t now_ns, const yd_keep_task_alive_request* reqs, size_t n,
                                 int* statuses);

/* One FreeTaskRequest (scheduler.proto:219-222). */
typedef struct yd_free_task_request {
  const char* token;
  const uint64_t* task_grant_ids;
  size_t n;
} yd_free_task_request;

/* FreeTask x n, in array order, with the answers of n yd_service_free_task calls.  The ids of the
 * accepted requests go to one yd_free_tasks (one collective free on a group): of several frees of
 * one lease the first releases it and the others find none, as in the sequence of single calls. */
void yd_service_free_tasks(yd_service* svc, const yd_free_task_request* reqs, size_t n, int* statuses);

#ifdef __cplusplus
}
#endif
#endif /* YDRUNS_H_ */
