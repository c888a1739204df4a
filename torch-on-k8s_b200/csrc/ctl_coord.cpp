// ctl_coord.cpp — job coordinator: tenant queues + plugin pipeline of pkg/coordinator, re-targeted
// from ResourceQuota objects to the GPU slots of one 8-GPU H100 box.
//
//   schedule cycle      pkg/coordinator/core/coordinator.go:310-366
//   queue selection     RR  core/policy.go:31-76 ; WRR core/policy.go:80-230 (default here: the
//                       reference hard-wires RR with "TODO: test the weighted rr selector",
//                       coordinator.go:62, and its WRR constructor leaves its maps nil — §2.3)
//   tenant / filter / pre-dequeue   Quota plugin, plugins/quota.go:82-277
//   score               Priority plugin, plugins/priority.go:48-85
//   select              max score, uniform random tie-break, coordinator.go:456-476
//
// Deviations that implement the intent (SURVEY.md §2.3): queue units are always owned (the
// reference never wires SetQueueUnitOwner, so nothing would ever dequeue); queues are scanned in
// insertion order (Go map order is random); WRR weight = pending replicas (mode 0) or the number of
// task types, i.e. what calculateQueueWeight literally computes (mode 1, reference-compat).
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "ctl_common.h"

using namespace tok;
using json::Value;

namespace {

struct Unit {
  std::string uid, key, tenant;
  bool has_priority = false;
  int64_t priority = 0;
  int64_t slots = 0;        // non-spot replicas x GPU slots (pkg/utils/resources/resources.go:90-109)
  int64_t spot_slots = 0;
  int64_t task_types = 0;   // len(qu.Tasks)
  int64_t replicas = 0;     // sum of numTasks
  bool marked_enqueued = false;
};

struct Queue {
  std::string name;
  std::vector<Unit> units;  // insertion order
  int weight(int mode) const {  // calculateQueueWeight, policy.go:224-230
    int64_t w = 0;
    for (const Unit& u : units) w += (mode == TOK_WRR_WEIGHT_TASK_TYPES) ? u.task_types : u.replicas;
    return static_cast<int>(w);
  }
};

struct Assumed {
  int64_t slots;
  double ts;
};

int gcd(int a, int b) { return b == 0 ? a : gcd(b, a % b); }

// splitmix64: deterministic tie-break RNG (the reference uses math/rand's global source)
struct Rng {
  uint64_t s;
  uint64_t next() {
    uint64_t z = (s += 0x9e3779b97f4a7c15ull);
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
  }
  int intn(int n) { return static_cast<int>(next() % static_cast<uint64_t>(n)); }
};

}  // namespace

struct tok_coord {
  int policy = TOK_POLICY_WRR;
  int weight_mode = TOK_WRR_WEIGHT_REPLICAS;
  Rng rng{1};
  std::vector<Queue> queues;                    // creation order
  std::map<std::string, std::string> index;     // uid -> tenant (queueIndexer)
  // RR state (policy.go:37-40)
  std::vector<std::string> rr_names;
  long rr_last = -1;
  // WRR state (policy.go:89-102)
  std::vector<std::string> wrr_names;
  std::map<std::string, int> wrr_weight;
  std::vector<int> wrr_slice;
  std::map<std::string, int> wrr_index;
  int wrr_cur = -1, wrr_cw = 0;
  // quota in GPU slots
  std::map<std::string, int64_t> hard, used;
  std::map<std::string, std::map<std::string, Assumed>> assumed;  // tenant -> key -> assumption
  std::map<std::string, bool> settled;                           // key -> Running/Failed/Succeeded

  Queue* find_queue(const std::string& name) {
    for (Queue& q : queues)
      if (q.name == name) return &q;
    return nullptr;
  }
};

namespace {

constexpr double kAssumeTimeout = 60.0;  // defaultQuotaAssumedTimeoutSeconds, quota.go:48

Queue* rr_next(tok_coord* c, std::string* name) {  // policy.go:42-76
  if (c->rr_names.empty() || c->rr_names.size() != c->queues.size())
    for (const Queue& q : c->queues)
      if (std::find(c->rr_names.begin(), c->rr_names.end(), q.name) == c->rr_names.end())
        c->rr_names.push_back(q.name);
  if (c->rr_names.empty()) return nullptr;
  const size_t idx = static_cast<size_t>((c->rr_last + 1) % static_cast<long>(c->rr_names.size()));
  *name = c->rr_names[idx];
  c->rr_last++;
  return c->find_queue(*name);
}

Queue* wrr_next(tok_coord* c, std::string* name) {  // policy.go:104-221
  bool changed = c->wrr_names.empty() || c->wrr_names.size() != c->queues.size();
  if (!changed)
    for (const Queue& q : c->queues)
      if (c->wrr_weight[q.name] != q.weight(c->weight_mode)) {
        changed = true;
        break;
      }
  if (changed) {  // appendNewQueuesOrUpdate (:142-170); (curSelected, curWeight) are NOT reset
    for (const Queue& q : c->queues) {
      const int w = q.weight(c->weight_mode);
      auto it = c->wrr_index.find(q.name);
      if (it == c->wrr_index.end()) {
        c->wrr_names.push_back(q.name);
        c->wrr_weight[q.name] = w;
        c->wrr_slice.push_back(w);
        c->wrr_index[q.name] = static_cast<int>(c->wrr_names.size()) - 1;
      } else if (c->wrr_weight[q.name] != w) {
        c->wrr_weight[q.name] = w;
        c->wrr_slice[static_cast<size_t>(it->second)] = w;
      }
    }
  }
  if (c->wrr_names.empty()) return nullptr;
  int g = c->wrr_slice[0], mx = -1;
  for (size_t i = 1; i < c->wrr_slice.size(); ++i) g = gcd(g, c->wrr_slice[i]);
  for (int w : c->wrr_slice) mx = std::max(mx, w);
  // every queue drained: the reference would spin forever here (gcd == 0 never lowers curWeight)
  if (mx <= 0) return nullptr;
  // nextQueueIndex (:203-221)
  const int n = static_cast<int>(c->wrr_slice.size());
  for (;;) {
    c->wrr_cur = (c->wrr_cur + 1) % n;
    if (c->wrr_cur == 0) {
      c->wrr_cw -= g;
      if (c->wrr_cw <= 0) {
        c->wrr_cw = mx;
        if (c->wrr_cw == 0) return nullptr;  // every queue is empty (the reference would index -1)
      }
    }
    if (c->wrr_slice[static_cast<size_t>(c->wrr_cur)] >= c->wrr_cw) break;
  }
  *name = c->wrr_names[static_cast<size_t>(c->wrr_cur)];
  return c->find_queue(*name);
}

// Quota filter (quota.go:97-131): Wait unless the tenant's free GPU slots cover the request.
// The quota object a tenant is accounted against: its own ResourceQuota when one was set, else the
// default ("" = the whole box).  Usage and 60 s assumptions live under the SAME key as the hard limit:
// tenants that share the default quota see each other's GPUs (a job of tenant A holding every GPU
// keeps tenant B's job queued, as ResourceQuota.used would in the reference, quota.go:97-131).
const std::string& quota_key(const tok_coord* c, const Unit& u) {
  static const std::string kDefault;
  return c->hard.count(u.tenant) ? u.tenant : kDefault;
}

bool quota_ok(tok_coord* c, const Unit& u, double now, std::string* why) {
  const std::string& qk = quota_key(c, u);
  auto h = c->hard.find(qk);
  if (h == c->hard.end()) return true;  // no quota object in this namespace: nothing to check
  const int64_t used = c->used.count(qk) ? c->used[qk] : 0;
  if (used > h->second) {  // availableQuota: exceed (:134-143)
    *why = "queue " + u.tenant + " guaranteed quota has exceed";
    return false;
  }
  int64_t available = h->second - used;
  // accumulateAssumedQuota: drop stale assumptions first (:146-173, 256-277)
  auto& as = c->assumed[qk];
  for (auto it = as.begin(); it != as.end();) {
    const bool expired = (now - it->second.ts) > kAssumeTimeout || c->settled.count(it->first);
    it = expired ? as.erase(it) : std::next(it);
  }
  int64_t assumed = 0;
  for (const auto& kv : as) assumed += kv.second.slots;
  available = std::max<int64_t>(0, available - assumed);  // SubtractWithNonNegativeResult
  if (available < u.slots) {
    *why = "resource nvidia.com/gpu request exceeds available quota " + u.tenant + ", available: " +
           std::to_string(available) + ", requests: " + std::to_string(u.slots) +
           ", assumed: " + std::to_string(assumed);
    return false;
  }
  return true;
}

Unit make_unit(const tok_job* j, const char* uid) {  // ToQueueUnit, pkg/coordinator/types.go:65-79
  Unit u;
  u.uid = uid;
  u.key = "TorchJob/" + job_namespace(j) + "/" + job_name(j);
  const Value* sched = j->doc.path({"spec", "schedulingPolicy"});
  const Value* q = sched ? sched->find("queue") : nullptr;
  u.tenant = (q && !q->as_string().empty()) ? q->as_string() : job_namespace(j);  // quota.go:82-92
  const Value* p = sched ? sched->find("priority") : nullptr;
  if (p && p->is_number()) {
    u.has_priority = true;
    u.priority = p->as_int();
  }
  const Value* specs = task_specs(j);
  if (specs)
    for (const auto& kv : specs->o) {
      const int64_t per = replica_slots(kv.first, kv.second);
      int64_t n = num_tasks(kv.second);
      u.task_types++;
      u.replicas += n;
      const Value* spot = kv.second.find("spotTaskSpec");
      const int64_t ns = (spot && spot->find("numSpotTasks")) ? spot->find("numSpotTasks")->as_int() : 0;
      if (ns > 0) {
        n = std::max<int64_t>(0, n - ns);
        u.spot_slots += ns * per;
      }
      u.slots += n * per;
    }
  return u;
}

}  // namespace

extern "C" {

int tok_coord_create(int policy, int weight_mode, uint64_t seed, tok_coord_t** out) {
  if (!out) return fail(TOK_ERR_INVALID, "coordinator out pointer is null");
  if (policy != TOK_POLICY_RR && policy != TOK_POLICY_WRR)
    return fail(TOK_ERR_INVALID, "unknown queue selection policy %d", policy);
  tok_coord* c = new tok_coord();
  c->policy = policy;
  c->weight_mode = weight_mode;
  c->rng.s = seed ? seed : 1;
  *out = c;
  return TOK_OK;
}

void tok_coord_destroy(tok_coord_t* c) { delete c; }

int tok_coord_set_quota(tok_coord_t* c, const char* tenant, int hard_slots) {
  if (!c) return fail(TOK_ERR_INVALID, "coordinator is null");
  if (hard_slots < 0)
    c->hard.erase(tenant ? tenant : "");
  else
    c->hard[tenant ? tenant : ""] = hard_slots;
  return TOK_OK;
}

int tok_coord_set_used(tok_coord_t* c, const char* tenant, int used_slots) {
  if (!c || !tenant) return fail(TOK_ERR_INVALID, "coordinator / tenant is null");
  c->used[tenant] = used_slots;
  return TOK_OK;
}

// EnqueueOrUpdate (coordinator.go:195-223)
int tok_coord_enqueue(tok_coord_t* c, const tok_job_t* job, const char* uid) {
  if (!c || !job || !uid) return fail(TOK_ERR_INVALID, "coordinator / job / uid is null");
  Unit u = make_unit(job, uid);
  Queue* q = c->find_queue(u.tenant);
  if (!q) {
    c->queues.push_back(Queue{u.tenant, {}});
    q = &c->queues.back();
  }
  c->index[u.uid] = u.tenant;
  c->settled.erase(u.uid);
  for (Unit& e : q->units)
    if (e.uid == u.uid) {  // update in place
      u.marked_enqueued = e.marked_enqueued;
      e = u;
      return TOK_OK;
    }
  u.marked_enqueued = true;  // queueStateMarker(qu, JobEnqueued) is the caller's condition write
  q->units.push_back(u);
  return TOK_OK;
}

int tok_coord_is_queuing(tok_coord_t* c, const char* uid, int* queuing) {
  if (!c || !uid || !queuing) return fail(TOK_ERR_INVALID, "coordinator / uid / out is null");
  *queuing = 0;
  auto it = c->index.find(uid);
  if (it == c->index.end()) return TOK_OK;
  Queue* q = c->find_queue(it->second);
  if (q)
    for (const Unit& u : q->units)
      if (u.uid == uid) *queuing = 1;
  return TOK_OK;
}

// Dequeue / popQueueUnitFromQueue (coordinator.go:226-270)
int tok_coord_dequeue(tok_coord_t* c, const char* uid) {
  if (!c || !uid) return fail(TOK_ERR_INVALID, "coordinator / uid is null");
  auto it = c->index.find(uid);
  if (it == c->index.end()) return fail(TOK_ERR_NOT_FOUND, "queue unit %s has already been dequeued", uid);
  Queue* q = c->find_queue(it->second);
  if (q)
    q->units.erase(std::remove_if(q->units.begin(), q->units.end(),
                                  [&](const Unit& u) { return u.uid == uid; }),
                   q->units.end());
  c->index.erase(it);
  return TOK_OK;
}

int tok_coord_job_settled(tok_coord_t* c, const char* uid_or_key) {
  if (!c || !uid_or_key) return fail(TOK_ERR_INVALID, "coordinator / key is null");
  c->settled[uid_or_key] = true;
  // assumptions are keyed by QueueUnit.Key(); also accept the uid the caller enqueued with
  for (auto& t : c->assumed)
    for (auto it = t.second.begin(); it != t.second.end();)
      it = (it->first == uid_or_key) ? t.second.erase(it) : std::next(it);
  return TOK_OK;
}

int tok_coord_pending(tok_coord_t* c, const char* tenant, int* pending) {
  if (!c || !pending) return fail(TOK_ERR_INVALID, "coordinator / out is null");
  *pending = 0;
  for (const Queue& q : c->queues)
    if (!tenant || !*tenant || q.name == tenant) *pending += static_cast<int>(q.units.size());
  return TOK_OK;
}

// schedule (coordinator.go:310-366)
int tok_coord_tick(tok_coord_t* c, double now, char** out) {
  if (!c) return fail(TOK_ERR_INVALID, "coordinator is null");
  Value res = Value::object();
  std::string tenant;
  Queue* q = (c->policy == TOK_POLICY_RR) ? rr_next(c, &tenant) : wrr_next(c, &tenant);
  if (!q) {
    res["queue"] = Value();
    res["dequeued"] = Value();
    res["reason"] = Value::str("no queue available yet");
    return out_json(res, out);
  }
  res["queue"] = Value::str(tenant);
  res["pending"] = Value::integer(static_cast<int64_t>(q->units.size()));
  Value mark = Value::array();
  Value waits = Value::array();
  std::vector<std::pair<const Unit*, int64_t>> candidates;
  for (Unit& u : q->units) {
    if (!u.marked_enqueued) {  // !IsEnqueued -> queueStateMarker(JobEnqueued)
      u.marked_enqueued = true;
      mark.a.push_back(Value::str(u.uid));
    }
    std::string why;
    if (quota_ok(c, u, now, &why)) {
      candidates.emplace_back(&u, u.has_priority ? u.priority : 0);  // priority.go:48-65
    } else {
      Value w = Value::object();
      w["uid"] = Value::str(u.uid);
      w["status"] = Value::str("Wait");
      w["reason"] = Value::str(why);
      waits.a.push_back(std::move(w));
    }
  }
  res["markEnqueued"] = std::move(mark);
  res["waiting"] = std::move(waits);
  if (candidates.empty()) {
    res["dequeued"] = Value();
    res["reason"] = Value::str("empty feasible queue unit after filtering and scoring");
    return out_json(res, out);
  }
  // selectQueueUnit (:456-476): max score, reservoir-style uniform tie-break
  int64_t best = candidates[0].second;
  size_t sel = 0;
  int ties = 1;
  for (size_t i = 1; i < candidates.size(); ++i) {
    if (candidates[i].second > best) {
      best = candidates[i].second;
      sel = i;
      ties = 1;
    } else if (candidates[i].second == best) {
      ties++;
      if (c->rng.intn(ties) == 0) sel = i;
    }
  }
  const Unit chosen = *candidates[sel].first;
  // PreDequeue: assume the quota (quota.go:176-181, 229-241)
  c->assumed[quota_key(c, chosen)][chosen.uid] = Assumed{chosen.slots, now};
  tok_coord_dequeue(c, chosen.uid.c_str());
  res["dequeued"] = Value::str(chosen.uid);
  res["key"] = Value::str(chosen.key);
  res["score"] = Value::integer(best);
  res["slots"] = Value::integer(chosen.slots);
  res["reason"] = Value::str("JobDequeued");
  return out_json(res, out);
}

}  // extern "C"
