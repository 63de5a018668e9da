// port_state.cc -- TEST INFRASTRUCTURE: the CPU port (oracle/port.cc) plus yd_export_state /
// yd_import_state (include/ydstate.h), built as checkers/libydport_state.so.
//
// oracle/port.cc is the pinned checker every other test compares against and stays as it is; its
// handle type is private to that file, so this file compiles it into the same translation unit and
// adds the two state calls on top.  Apart from them the library is the port, call for call.
#include "../oracle/port.cc"

#include "ydstate.h"
#include "ydstate_codec.inc"

namespace {

bool IsFresh(const yd_sched* s) {
  return s->servants.empty() && s->tasks.empty() && s->next_task_id == 0 && s->running_tasks.empty() &&
         s->running_tasks.bucket_count() == 1 && s->envs.empty() && s->ips.size() == 1;
}

}  // namespace

extern "C" size_t yd_export_state(yd_sched* s, int64_t now_ns, uint8_t* out, size_t cap) {
  ydstate::StateImage im;
  im.id_stride = (uint32_t)s->id_stride;
  im.id_offset = (uint32_t)s->id_offset;
  im.min_mem = s->min_memory_for_new_task;
  im.next_task_id = yd_next_task_id(s);
  im.envs = s->envs;
  im.ips = s->ips;
  std::unordered_map<const ServantRec*, uint32_t> pos;
  for (auto&& p : s->servants) {
    const ServantRec& v = *p;
    pos.emplace(&v, (uint32_t)im.servants.size());
    ydstate::Servant o;
    o.version = v.version; o.priority = v.priority; o.reason = v.reason;
    o.nproc = (uint32_t)v.num_processors; o.load = (uint32_t)v.current_load; o.max_tasks = (uint32_t)v.max_tasks;
    o.total_mem = v.total_memory; o.avail_mem = v.memory_available;
    o.expires_rel = v.expires_at - now_ns;
    o.ever = v.ever_assigned_tasks;
    o.observed = v.observed_location; o.reported = v.reported_location;
    o.envs = v.environments;
    im.servants.push_back(std::move(o));
  }
  im.leases.reserve(s->tasks.size());
  for (auto&& [id, t] : s->tasks) {
    // Orphans are swept in the same timer tick that drops their servant, so every lease has one.
    auto it = pos.find(t.servant.get());
    if (it == pos.end()) std::abort();
    im.leases.push_back(ydstate::Lease{id, it->second,
                                       (t.is_prefetch ? YD_STATE_LEASE_PREFETCH : 0u) | (t.zombie ? YD_STATE_LEASE_ZOMBIE : 0u),
                                       t.expires_at - now_ns});
  }
  std::sort(im.leases.begin(), im.leases.end(), [](auto& a, auto& b) { return a.id < b.id; });
  im.bucket_count = s->running_tasks.bucket_count();
  for (auto&& [loc, v] : s->running_tasks) {
    ydstate::Group g;
    g.location = loc;
    for (auto&& t : v) g.tasks.push_back(ydstate::Task{t.servant_task_id, t.task_grant_id, t.servant_location, t.task_digest});
    im.groups.push_back(std::move(g));
  }
  return ydstate::EncodeState(im, out, cap);
}

extern "C" int yd_import_state(yd_sched* s, int64_t now_ns, const uint8_t* blob, size_t len) {
  if (!IsFresh(s)) return YD_STATE_NOT_FRESH;
  ydstate::StateImage im;
  if (int rc = ydstate::DecodeState(blob, len, &im)) return rc;
  if (im.id_stride != s->id_stride || im.id_offset != s->id_offset || im.min_mem != s->min_memory_for_new_task) {
    return YD_STATE_CONFIG_MISMATCH;
  }
  s->next_task_id = (im.next_task_id - im.id_offset) / im.id_stride;
  s->envs = im.envs;
  s->ips = im.ips;
  s->env_ids.clear();
  s->ip_ids.clear();
  for (uint32_t i = 0; i != s->envs.size(); ++i) s->env_ids.emplace(s->envs[i], i);
  for (uint32_t i = 0; i != s->ips.size(); ++i) s->ip_ids.emplace(s->ips[i], i);
  for (auto&& v : im.servants) {
    auto& rec = *s->servants.emplace_back(std::make_shared<ServantRec>());
    rec.version = v.version; rec.priority = v.priority; rec.reason = v.reason;
    rec.observed_location = v.observed; rec.reported_location = v.reported;
    rec.environments = v.envs;
    rec.num_processors = v.nproc; rec.current_load = v.load; rec.max_tasks = v.max_tasks;
    rec.total_memory = v.total_mem; rec.memory_available = v.avail_mem;
    rec.discovered_at = now_ns;
    rec.expires_at = now_ns + v.expires_rel;
    rec.ever_assigned_tasks = v.ever;
  }
  s->tasks.reserve(im.leases.size());
  for (auto&& l : im.leases) {
    TaskRec& t = s->tasks[l.id];
    t.servant = s->servants[l.servant];
    ++t.servant->running_tasks;  // running_tasks == leases on the servant, zombies included
    t.started_at = now_ns;
    t.expires_at = now_ns + l.expires_rel;
    t.is_prefetch = (l.flags & YD_STATE_LEASE_PREFETCH) != 0;
    t.zombie = (l.flags & YD_STATE_LEASE_ZOMBIE) != 0;
  }
  // The bookkeeper's iteration order: same bucket count, groups inserted last-first (ydstate.h).
  if (im.bucket_count != 1) s->running_tasks.rehash(im.bucket_count);
  for (auto g = im.groups.rbegin(); g != im.groups.rend(); ++g) {
    std::vector<RunningTaskRec> v;
    for (auto&& t : g->tasks) v.push_back(RunningTaskRec{t.servant_task_id, t.task_grant_id, t.servant_location, t.task_digest});
    s->running_tasks.emplace(g->location, std::move(v));
  }
  return YD_STATE_OK;
}
