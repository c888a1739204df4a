// ctl_job.cpp — the TorchJob surface of the single-box controller, behind the C ABI:
// manifest parse, SetDefaults_TorchJob, SetClusterSpec (replica rendezvous identity), DAG gating,
// MinMember gang admission over GPU slots, failover truth table, job condition machine.
//
// A TorchJob is kept as a JSON document (apis/train/v1alpha1 wire names, incl. the reference's
// `clenPodPolicy`), so unknown fields of the embedded PodTemplateSpec survive a round trip.
// Reference files are cited per function; where the reference has a latent defect the INTENDED
// behaviour is implemented (SURVEY.md §2.3) and said so.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include <algorithm>
#include <atomic>
#include <map>
#include <string>
#include <vector>

#include "ctl_common.h"

namespace tok {

std::atomic<unsigned> g_gates{TOK_GATES_DEFAULT};

bool gate(unsigned g) { return (g_gates.load() & g) != 0; }

std::string lower(const std::string& s) {
  std::string r = s;
  for (char& c : r) c = static_cast<char>(tolower(static_cast<unsigned char>(c)));
  return r;
}

bool equal_fold(const std::string& a, const std::string& b) { return lower(a) == lower(b); }

char* dup_cstr(const std::string& s) {
  char* p = static_cast<char*>(malloc(s.size() + 1));
  if (p) memcpy(p, s.c_str(), s.size() + 1);
  return p;
}

int out_json(const json::Value& v, char** out) {
  if (!out) return fail(TOK_ERR_INVALID, "output pointer is null");
  *out = dup_cstr(json::dump(v));
  return *out ? TOK_OK : fail(TOK_ERR_INVALID, "out of memory");
}

// pkg/utils/utils.go:75-77
std::string gen_general_name(const std::string& job, const std::string& task_type,
                             const std::string& index) {
  std::string s = job + "-" + task_type + "-" + index;
  std::replace(s.begin(), s.end(), '/', '-');
  return s;
}

json::Value* task_specs(tok_job* j) {
  json::Value* spec = j->doc.find("spec");
  return spec ? spec->find("torchTaskSpecs") : nullptr;
}
const json::Value* task_specs(const tok_job* j) { return task_specs(const_cast<tok_job*>(j)); }

// `*ts.NumTasks` with the nil-safe default of pkg/utils/resources/resources.go:75-78
int64_t num_tasks(const json::Value& ts) {
  const json::Value* n = ts.find("numTasks");
  return (n && n->is_number()) ? n->as_int() : 1;
}

// canonical task-type key present in the spec for a (possibly lower-cased) name
const std::string* find_task_key(const json::Value& specs, const std::string& name) {
  for (const auto& kv : specs.o)
    if (equal_fold(kv.first, name)) return &kv.first;
  return nullptr;
}

// pkg/utils/utils.go:49-63 GetTotalExcludedTasks(tasks, AIMaster)
int64_t total_tasks_excluding_aimaster(const json::Value& specs) {
  int64_t n = 0;
  for (const auto& kv : specs.o)
    if (kv.first != "AIMaster") n += num_tasks(kv.second);
  return n;
}

std::string job_name(const tok_job* j) {
  const json::Value* n = j->doc.path({"metadata", "name"});
  return n ? n->as_string() : "";
}
std::string job_namespace(const tok_job* j) {
  const json::Value* n = j->doc.path({"metadata", "namespace"});
  std::string s = n ? n->as_string() : "";
  return s.empty() ? "default" : s;
}

// GPU slots one replica of this task type occupies on the box.  The reference sums container
// resource requests (pkg/utils/resources/resources.go:56-72); on one 8-GPU H100 box the only resource is
// nvidia.com/gpu (apis/train/v1alpha1/constants.go:28) and every training replica is bound to exactly
// one GPU unless the template asks for more.  AIMaster defaults to zero (it does not train).
int64_t replica_slots(const std::string& task_type, const json::Value& ts) {
  int64_t sum = 0;
  const json::Value* containers = ts.path({"template", "spec", "containers"});
  if (containers && containers->is_array()) {
    for (const json::Value& c : containers->a) {
      const json::Value* r = c.path({"resources", "requests", "nvidia.com/gpu"});
      if (!r) r = c.path({"resources", "limits", "nvidia.com/gpu"});
      if (!r) continue;
      if (r->is_number())
        sum += r->as_int();
      else if (r->is_string())
        sum += strtoll(r->s.c_str(), nullptr, 10);
    }
  }
  if (sum == 0 && task_type != "AIMaster") sum = 1;
  return sum;
}

// ---- conditions (pkg/utils/utils.go:100-243) --------------------------------------------------------
json::Value& status_of(tok_job* j) {
  json::Value& st = j->doc["status"];
  if (!st.is_object()) st = json::Value::object();
  return st;
}

bool has_condition(const json::Value& status, const std::string& type) {
  const json::Value* cs = status.find("conditions");
  if (!cs || !cs->is_array()) return false;
  for (const json::Value& c : cs->a) {
    const json::Value* t = c.find("type");
    const json::Value* s = c.find("status");
    if (t && s && t->as_string() == type && s->as_string() == "True") return true;
  }
  return false;
}

// setCondition + filterOutCondition (utils.go:186-243)
void set_condition(json::Value& status, const std::string& type, const std::string& reason,
                   const std::string& message, const std::string& now) {
  if (has_condition(status, "Failed") || has_condition(status, "Succeeded")) return;
  json::Value& conds = status["conditions"];
  if (!conds.is_array()) conds = json::Value::array();
  const json::Value* current = nullptr;
  for (const json::Value& c : conds.a) {
    const json::Value* t = c.find("type");
    if (t && t->as_string() == type) {
      current = &c;
      break;
    }
  }
  std::string transition = now;
  if (current) {
    const json::Value* s = current->find("status");
    const json::Value* r = current->find("reason");
    const bool same_status = s && s->as_string() == "True";
    if (same_status && r && r->as_string() == reason) return;  // nothing changed
    if (same_status) {
      const json::Value* lt = current->find("lastTransitionTime");
      if (lt) transition = lt->as_string();
    }
  }
  json::Value kept = json::Value::array();
  for (json::Value c : conds.a) {
    const std::string ct = c.find("type") ? c.find("type")->as_string() : "";
    if (type == "Restarting" && ct == "Running") continue;
    if (type == "Running" && ct == "Restarting") continue;
    if (ct == type) continue;
    if ((type == "Failed" || type == "Succeeded") && ct == "Running") c["status"] = json::Value::str("False");
    kept.a.push_back(std::move(c));
  }
  json::Value nc = json::Value::object();
  nc["type"] = json::Value::str(type);
  nc["status"] = json::Value::str("True");
  nc["lastUpdateTime"] = json::Value::str(now);
  nc["lastTransitionTime"] = json::Value::str(transition);
  nc["reason"] = json::Value::str(reason);
  nc["message"] = json::Value::str(message);
  kept.a.push_back(std::move(nc));
  conds = std::move(kept);
}

}  // namespace tok

using namespace tok;
using json::Value;

extern "C" {

int tok_set_feature_gates(unsigned gates) {
  g_gates.store(gates);
  return TOK_OK;
}
unsigned tok_get_feature_gates(void) { return g_gates.load(); }

// ---- parse ----------------------------------------------------------------------------------------
int tok_job_parse(const char* text, tok_job_t** out) {
  if (!out) return fail(TOK_ERR_INVALID, "job out pointer is null");
  *out = nullptr;
  Value doc;
  std::string err;
  if (!json::parse(text, &doc, &err)) return fail(TOK_ERR_INVALID, "%s", err.c_str());
  if (!doc.is_object()) return fail(TOK_ERR_INVALID, "TorchJob manifest must be a JSON object");
  const Value* kind = doc.find("kind");
  if (kind && kind->is_string() && !kind->s.empty() && kind->s != "TorchJob")
    return fail(TOK_ERR_INVALID, "kind is %s, expected TorchJob", kind->s.c_str());
  const Value* name = doc.path({"metadata", "name"});
  if (!name || !name->is_string() || name->s.empty())
    return fail(TOK_ERR_INVALID, "metadata.name is required");
  const Value* specs = doc.path({"spec", "torchTaskSpecs"});
  if (!specs || !specs->is_object())
    return fail(TOK_ERR_INVALID, "spec.torchTaskSpecs (map of task type -> task spec) is required");
  for (const auto& kv : specs->o) {
    if (!kv.second.is_object())
      return fail(TOK_ERR_INVALID, "spec.torchTaskSpecs.%s must be an object", kv.first.c_str());
    const Value* n = kv.second.find("numTasks");
    if (n && (!n->is_number() || n->as_int() < 0))
      return fail(TOK_ERR_INVALID, "spec.torchTaskSpecs.%s.numTasks must be a non-negative integer",
                  kv.first.c_str());
    const Value* rp = kv.second.find("restartPolicy");
    if (rp && rp->is_string() && !rp->s.empty() && rp->s != "Always" && rp->s != "OnFailure" &&
        rp->s != "ExitCode" && rp->s != "Never")
      return fail(TOK_ERR_INVALID, "spec.torchTaskSpecs.%s.restartPolicy %s is not one of "
                  "Always|OnFailure|ExitCode", kv.first.c_str(), rp->s.c_str());
  }
  tok_job* j = new tok_job();
  j->doc = std::move(doc);
  *out = j;
  return TOK_OK;
}

void tok_job_free(tok_job_t* job) { delete job; }

int tok_job_to_json(const tok_job_t* job, char** out) {
  if (!job) return fail(TOK_ERR_INVALID, "job is null");
  return out_json(job->doc, out);
}

// ---- SetDefaults_TorchJob (apis/train/v1alpha1/torchjob_defaults.go:29-74) ---------------------------
static void default_port(Value& ts) {  // setDefaults_TorchJobPort, :150-178
  Value* containers = ts["template"]["spec"].find("containers");
  if (!containers || !containers->is_array()) return;
  for (Value& c : containers->a) {
    const Value* n = c.find("name");
    if (!n || n->as_string() != "torch") continue;  // TorchJobDefaultContainerName
    Value& ports = c["ports"];
    if (!ports.is_array()) ports = Value::array();
    for (const Value& p : ports.a) {
      const Value* pn = p.find("name");
      if (pn && pn->as_string() == "torchjob-port") return;
    }
    Value p = Value::object();
    p["name"] = Value::str("torchjob-port");
    p["containerPort"] = Value::integer(23456);
    ports.a.push_back(std::move(p));
    return;  // first container named "torch" only (:152-158)
  }
}

int tok_job_default(tok_job_t* j) {
  if (!j) return fail(TOK_ERR_INVALID, "job is null");
  // 6. apiVersion / kind (:60-65) — done first: inserting top-level members may reallocate the
  //    document's member vector, which would invalidate references into `spec` taken below
  if (j->doc["apiVersion"].as_string().empty())
    j->doc["apiVersion"] = Value::str("train.distributed.io/v1alpha1");
  if (j->doc["kind"].as_string().empty()) j->doc["kind"] = Value::str("TorchJob");
  Value& spec = j->doc["spec"];
  // 1. cleanPodPolicy <- None (:31-34); wire name keeps the reference's typo
  if (!spec.find("clenPodPolicy") || spec.find("clenPodPolicy")->is_null())
    spec["clenPodPolicy"] = Value::str("None");
  Value* specs = task_specs(j);
  if (!specs) return fail(TOK_ERR_INVALID, "spec.torchTaskSpecs is missing");
  // 2. normalise the task-type keys to "Master" / "Worker" (:77-92); AIMaster is NOT normalised
  for (const char* canon : {"Master", "Worker"}) {
    for (auto& kv : specs->o) {
      if (equal_fold(kv.first, canon) && kv.first != canon) {
        if (specs->find(canon)) break;  // canonical key already present: keep it
        kv.first = canon;
        break;
      }
    }
  }
  // 3. DAG conditions (:95-124): Master waits for AIMaster Running, Worker for Master Running
  j->depends.clear();
  if (gate(TOK_GATE_DAG_SCHEDULING)) {
    if (specs->find("AIMaster") && specs->find("Master"))
      j->depends["Master"] = {{"AIMaster", "Running"}};
    if (specs->find("Worker") && specs->find("Master"))
      j->depends["Worker"] = {{"Master", "Running"}};
  }
  // 4./5. per task type (:46-59)
  for (auto& kv : specs->o) {
    Value& ts = kv.second;
    if (kv.first == "Worker") {
      if (!ts.find("numTasks") || ts.find("numTasks")->is_null()) ts["numTasks"] = Value::integer(1);
      if (ts["restartPolicy"].as_string().empty()) ts["restartPolicy"] = Value::str("OnFailure");
    }
    if (kv.first == "Master") {
      if (!ts.find("numTasks") || ts.find("numTasks")->is_null()) ts["numTasks"] = Value::integer(1);
      if (ts["restartPolicy"].as_string().empty()) ts["restartPolicy"] = Value::str("ExitCode");
      if (ts.path({"template", "spec"})) default_port(ts);
    }
    Value* containers = ts.find("template") && ts.find("template")->find("spec")
                            ? ts["template"]["spec"].find("containers")
                            : nullptr;
    if (containers && containers->is_array())
      for (Value& c : containers->a)  // setDefaults_TerminationMessagePolicy (:181-188)
        if (c.is_object() && c["terminationMessagePolicy"].as_string().empty())
          c["terminationMessagePolicy"] = Value::str("FallbackToLogsOnError");
  }
  // 7. MinMembers (:69-73, 192-197).  The reference iterates the nil map it guards (a no-op);
  //    intended (field doc torchjob_types.go:192-195): minMembers[tt] = numTasks[tt].
  if (gate(TOK_GATE_DAG_SCHEDULING) && gate(TOK_GATE_GANG_SCHEDULING) &&
      (!spec.find("minMembers") || spec.find("minMembers")->is_null())) {
    Value mm = Value::object();
    for (const auto& kv : specs->o) mm[kv.first] = Value::integer(num_tasks(kv.second));
    spec["minMembers"] = std::move(mm);
  }
  j->defaulted = true;
  return TOK_OK;
}

// ---- SetClusterSpec (controllers/train/torchjob_controller.go:314-449) -------------------------------
static int master_port(const Value& specs, int64_t* port) {  // getPortFromJob, :508-521
  const Value* master = specs.find("Master");
  if (!master) return fail(TOK_ERR_INVALID, "invalid config: job has no Master task (failed to found the port)");
  const Value* containers = master->path({"template", "spec", "containers"});
  if (containers && containers->is_array())
    for (const Value& c : containers->a) {
      const Value* n = c.find("name");
      if (!n || n->as_string() != "torch") continue;
      const Value* ports = c.find("ports");
      if (!ports || !ports->is_array()) continue;
      for (const Value& p : ports->a) {
        const Value* pn = p.find("name");
        if (pn && pn->as_string() == "torchjob-port") {
          *port = p.find("containerPort") ? p.find("containerPort")->as_int() : 0;
          return TOK_OK;
        }
      }
    }
  return fail(TOK_ERR_INVALID, "failed to found the port (Master container `torch` has no port "
              "named torchjob-port; run tok_job_default first)");
}

int tok_job_cluster_spec(const tok_job_t* j, const char* task_type, int index, char** out) {
  if (!j || !task_type) return fail(TOK_ERR_INVALID, "job / task_type is null");
  const Value* specs = task_specs(j);
  if (!specs) return fail(TOK_ERR_INVALID, "spec.torchTaskSpecs is missing");
  const std::string tt = lower(task_type);
  const std::string* key = find_task_key(*specs, tt);
  if (!key) return fail(TOK_ERR_NOT_FOUND, "task type %s is not in spec.torchTaskSpecs", task_type);
  const Value& ts = *specs->find(*key);
  if (index < 0) return fail(TOK_ERR_INVALID, "negative task index %d", index);
  const std::string name = job_name(j);
  int64_t port = 0;
  int rc = master_port(*specs, &port);
  if (rc != TOK_OK) return rc;

  const bool master_role = (tt == "master");
  std::string master_addr = gen_general_name(name, "master", "0");
  int rank = index;
  if (master_role) {
    if (rank != 0)
      return fail(TOK_ERR_INVALID, "invalid config: There should be only a single master with index=0");
    if (gate(TOK_GATE_TORCH_LOCAL_MASTER_ADDR)) master_addr = "localhost";
  } else {
    rank++;  // workers (and AIMaster, as in the reference) are shifted by the master
  }
  const int64_t world = total_tasks_excluding_aimaster(*specs);
  const Value* ann = j->doc.path({"metadata", "annotations"});
  const Value* el = ann ? ann->find("distributed.io/enable-elastic-training") : nullptr;
  const bool elastic = el && el->as_string() == "true";

  Value res = Value::object();
  res["name"] = Value::str(gen_general_name(name, tt, std::to_string(index)));
  res["taskType"] = Value::str(*key);
  res["index"] = Value::integer(index);
  res["rank"] = Value::integer(rank);
  res["worldSize"] = Value::integer(world);
  Value env = Value::array();
  auto add_env = [&](const char* n, const std::string& v) {
    Value e = Value::object();
    e["name"] = Value::str(n);
    e["value"] = Value::str(v);
    env.a.push_back(std::move(e));
  };
  add_env("MASTER_PORT", std::to_string(port));  // order of :398-413
  add_env("MASTER_ADDR", master_addr);
  add_env("RANK", std::to_string(rank));
  add_env("PYTHONUNBUFFERED", "0");
  Value annotations = Value::object();
  Value labels = Value::object();
  labels["group-name"] = Value::str("train.distributed.io");  // controllers/common/pod.go:519-524
  labels["job-name"] = Value::str([&] { std::string s = name; std::replace(s.begin(), s.end(), '/', '-'); return s; }());
  labels["task-type"] = Value::str(tt);
  labels["task-index"] = Value::str(std::to_string(index));
  if (master_role) labels["task-role"] = Value::str("master");

  // restart policy of the replica process (pod.go:556-561): ExitCode is decided by the controller
  std::string task_rp = ts.find("restartPolicy") ? ts.find("restartPolicy")->as_string() : "";
  std::string pod_rp = task_rp == "ExitCode" ? "Never" : task_rp;

  Value init = Value::array();
  if (elastic && tt != "aimaster") {
    // :419-439 — WORLD_SIZE is read from an annotation so that an in-place restart sees the new size
    annotations["distributed.io/world-size"] = Value::str(std::to_string(world));
    Value e = Value::object();
    e["name"] = Value::str("WORLD_SIZE");
    e["value"] = Value::str(std::to_string(world));
    e["valueFrom"] = Value::str("metadata.annotations['distributed.io/world-size']");
    env.a.push_back(std::move(e));
    pod_rp = "OnFailure";
    const Value* gen = j->doc.path({"metadata", "generation"});
    labels["distributed.io/job-generation"] = Value::str(std::to_string(gen ? gen->as_int() : 0));
    res["finalizers"] = Value::array();
    res["finalizers"].a.push_back(Value::str("distributed.io/preempt-protector"));
    if (!master_role) {  // :351-361 warm-up + master-waiter init containers (no-ops on one box)
      init.a.push_back(Value::str("warmup"));
      init.a.push_back(Value::str("master-waiter"));
    }
  } else {
    add_env("WORLD_SIZE", std::to_string(world));
  }
  res["env"] = std::move(env);

  // torchelastic args (:364-392, 415-417); guarded on the policy being present (SURVEY §2.3)
  Value args = Value::array();
  const Value* spec = j->doc.find("spec");
  const Value* ete = spec ? spec->find("enableTorchElastic") : nullptr;
  const Value* pol = spec ? spec->find("torchElasticPolicy") : nullptr;
  if (ete && ete->as_bool() && pol && pol->is_object()) {
    // getDesiredReplicas returns the MASTER count in the reference (:524-530); intended: workers
    const Value* w = specs->find("Worker");
    const int64_t desired = w ? num_tasks(*w) : 1;
    const Value* mn = pol->find("numMinReplicas");
    const Value* mx = pol->find("numMaxReplicas");
    const Value* np = pol->find("numWorkersPerNodePolicy");
    const int64_t vmin = (mn && mn->is_number()) ? mn->as_int() : desired;
    const int64_t vmax = (mx && mx->is_number()) ? mx->as_int() : desired;
    const int64_t vnp = (np && np->is_number()) ? np->as_int() : 1;
    args.a.push_back(Value::str("--rdzv_backend=" + (pol->find("rendezvousBackend") ? pol->find("rendezvousBackend")->as_string() : "")));
    args.a.push_back(Value::str("--rdzv_endpoint=" + (pol->find("rendezvousEndpoint") ? pol->find("rendezvousEndpoint")->as_string() : "")));
    args.a.push_back(Value::str("--rdzv_id=" + name));
    args.a.push_back(Value::str("--nproc_per_node=" + std::to_string(vnp)));
    args.a.push_back(Value::str("--nnodes=" + std::to_string(vmin) + ":" + std::to_string(vmax)));
  }
  res["args"] = std::move(args);

  // gang binding (pkg/gangscheduler/volcano/volcano.go:238-287, pod.go:569-589)
  if (gate(TOK_GATE_GANG_SCHEDULING) && tt != "aimaster") {
    const std::string pg = gate(TOK_GATE_DAG_SCHEDULING) ? name + "-" + tt : name;
    annotations["scheduling.k8s.io/group-name"] = Value::str(pg);
    res["schedulerName"] = Value::str("volcano");
  } else if (tt == "aimaster") {
    res["schedulerName"] = Value::str("default-scheduler");
  }
  // spot replicas (pod.go:592-603)
  const Value* spot = ts.find("spotTaskSpec");
  if (spot && spot->is_object()) {
    const int64_t nspot = spot->find("numSpotTasks") ? spot->find("numSpotTasks")->as_int() : 0;
    if (index >= num_tasks(ts) - nspot) {
      res["spot"] = Value::boolean(true);
      const Value* sl = spot->find("labels");
      if (sl && sl->is_object())
        for (const auto& kv : sl->o) labels[kv.first] = kv.second;
      if (spot->find("priorityClassName"))
        res["priorityClassName"] = *spot->find("priorityClassName");
    }
  }
  res["labels"] = std::move(labels);
  res["annotations"] = std::move(annotations);
  res["initContainers"] = std::move(init);
  res["restartPolicy"] = Value::str(pod_rp);
  res["taskRestartPolicy"] = Value::str(task_rp);
  res["gpuSlots"] = Value::integer(replica_slots(*key, ts));
  return out_json(res, out);
}

// ---- DAG gate (controllers/common/dag.go:30-116) -------------------------------------------------------
static int phase_code(const std::string& p) {
  if (p == "Pending") return 0;
  if (p == "Running") return 1;
  if (p == "Succeeded" || p == "Failed") return 2;
  return 0;  // unknown phases map to the zero value, like a missing Go map key
}

int tok_job_dag_ready(const tok_job_t* j, const char* task_type, const char* phases_json, int* ready) {
  if (!j || !task_type || !ready) return fail(TOK_ERR_INVALID, "job / task_type / ready is null");
  const Value* specs = task_specs(j);
  if (!specs) return fail(TOK_ERR_INVALID, "spec.torchTaskSpecs is missing");
  const std::string* key = find_task_key(*specs, task_type);
  if (!key) return fail(TOK_ERR_NOT_FOUND, "task type %s is not in spec.torchTaskSpecs", task_type);
  Value phases;
  std::string err;
  if (!json::parse(phases_json ? phases_json : "{}", &phases, &err) || !phases.is_object())
    return fail(TOK_ERR_INVALID, "phases must be a JSON object {taskType: [phase...]}: %s", err.c_str());
  *ready = 1;
  auto it = j->depends.find(*key);
  if (!gate(TOK_GATE_DAG_SCHEDULING) || it == j->depends.end()) return TOK_OK;
  for (const auto& cond : it->second) {
    const Value* up = specs->find(cond.first);
    if (!up) continue;  // upstream task does not exist: satisfied (dag.go:87-91)
    const Value* have = nullptr;
    for (const auto& kv : phases.o)
      if (equal_fold(kv.first, cond.first)) have = &kv.second;
    const size_t n = (have && have->is_array()) ? have->a.size() : 0;
    if (static_cast<int64_t>(n) < num_tasks(*up)) {
      *ready = 0;
      return TOK_OK;
    }
    if (!have || !have->is_array()) continue;  // upstream with numTasks 0 and no phase entry
    for (const Value& p : have->a)
      if (phase_code(p.as_string()) - phase_code(cond.second) < 0) {
        *ready = 0;
        return TOK_OK;
      }
  }
  return TOK_OK;
}

// ---- gang admission (pkg/gangscheduler/volcano/volcano.go:109-230) -----------------------------------
int tok_gang_admit(const tok_job_t* j, int free_slots, char** out) {
  if (!j) return fail(TOK_ERR_INVALID, "job is null");
  const Value* specs = task_specs(j);
  if (!specs) return fail(TOK_ERR_INVALID, "spec.torchTaskSpecs is missing");
  const std::string name = job_name(j);
  Value res = Value::object();
  Value groups = Value::array();
  int64_t need = 0;
  if (!gate(TOK_GATE_GANG_SCHEDULING)) {
    res["admitted"] = Value::boolean(true);
    res["groups"] = std::move(groups);
    res["slotsNeeded"] = Value::integer(0);
    res["reason"] = Value::str("gang scheduling disabled: replicas start as GPU slots free up");
    return out_json(res, out);
  }
  const Value* spec = j->doc.find("spec");
  const Value* sched = spec ? spec->find("schedulingPolicy") : nullptr;
  const std::string queue = (sched && sched->find("queue")) ? sched->find("queue")->as_string() : "";
  const std::string pclass = (sched && sched->find("priorityClassName")) ? sched->find("priorityClassName")->as_string() : "";
  if (gate(TOK_GATE_DAG_SCHEDULING)) {  // generatePodGroupsByRole: one group per task type
    const Value* mm = spec ? spec->find("minMembers") : nullptr;
    for (const auto& kv : specs->o) {
      if (kv.first == "AIMaster") continue;
      const int64_t n = num_tasks(kv.second);
      int64_t min_member = n;
      const Value* m = (mm && mm->is_object()) ? mm->find(kv.first) : nullptr;
      if (m && m->is_number()) {
        if (m->as_int() > n)
          return fail(TOK_ERR_INVALID,
                      "the mimMember provided for task type %s is larger than NumTasks, minMember "
                      "provided: %lld, NumTasks: %lld", kv.first.c_str(), (long long)m->as_int(), (long long)n);
        min_member = m->as_int();
      }
      Value g = Value::object();
      g["name"] = Value::str(name + "-" + lower(kv.first));
      g["taskType"] = Value::str(kv.first);
      g["minMember"] = Value::integer(min_member);
      const int64_t slots = min_member * replica_slots(kv.first, kv.second);
      g["slots"] = Value::integer(slots);
      g["queue"] = Value::str(queue);
      g["priorityClassName"] = Value::str(pclass);
      need += slots;
      groups.a.push_back(std::move(g));
    }
  } else {  // generatePodGroupsByJob: one group for the whole job
    int64_t min_member = 0, slots = 0;
    for (const auto& kv : specs->o) {
      if (kv.first == "AIMaster") continue;
      min_member += num_tasks(kv.second);
      slots += num_tasks(kv.second) * replica_slots(kv.first, kv.second);
    }
    const Value* ma = sched ? sched->find("minAvailable") : nullptr;
    if (ma && ma->is_number() && ma->as_int() > 0) {
      // the reference keeps MinResources at the whole-job request here (known inconsistency,
      // volcano.go:223-227); on one box a replica is one GPU, so slots follow MinMember
      const int64_t total = min_member;
      min_member = ma->as_int();
      if (total > 0) slots = slots * min_member / total;
    }
    Value g = Value::object();
    g["name"] = Value::str(name);
    g["taskType"] = Value::str("");
    g["minMember"] = Value::integer(min_member);
    g["slots"] = Value::integer(slots);
    g["queue"] = Value::str(queue);
    g["priorityClassName"] = Value::str(pclass);
    need = slots;
    groups.a.push_back(std::move(g));
  }
  const bool ok = need <= free_slots;
  res["admitted"] = Value::boolean(ok);
  res["groups"] = std::move(groups);
  res["slotsNeeded"] = Value::integer(need);
  res["freeSlots"] = Value::integer(free_slots);
  res["reason"] = Value::str(ok ? "all MinMember groups fit" : "not enough free GPU slots for the MinMember groups (all-or-nothing)");
  return out_json(res, out);
}

// ---- failover truth table (controllers/common/failover.go:52-113) -------------------------------------
int tok_failover_decide(const char* restart_policy, int exit_code, const char* reason, int* should) {
  if (!restart_policy || !should) return fail(TOK_ERR_INVALID, "restart_policy / out is null");
  *should = 0;
  if (strcmp(restart_policy, "ExitCode") != 0) return TOK_OK;  // :57-60
  const bool retryable_code = exit_code == 130 || exit_code == 137 || exit_code == 143 || exit_code == 138;
  const std::string r = reason ? reason : "";
  const bool retryable_reason = r == "OOMKilled" || r == "Killed" || r == "Evicted" || r == "UnexpectedAdmissionError";
  *should = (retryable_code || retryable_reason) ? 1 : 0;
  return TOK_OK;
}

// ---- conditions -------------------------------------------------------------------------------------
int tok_job_set_condition(tok_job_t* j, const char* type, const char* reason, const char* message,
                          const char* now) {
  if (!j || !type) return fail(TOK_ERR_INVALID, "job / type is null");
  static const char* kTypes[] = {"Created", "Queuing", "Running", "Restarting", "Succeeded", "Failed"};
  bool known = false;
  for (const char* t : kTypes) known = known || strcmp(t, type) == 0;
  if (!known) return fail(TOK_ERR_INVALID, "unknown job condition type %s", type);
  set_condition(status_of(j), type, reason ? reason : "", message ? message : "", now ? now : "");
  return TOK_OK;
}

int tok_job_need_enqueue(const tok_job_t* j, int* need) {  // utils.go:138-149
  if (!j || !need) return fail(TOK_ERR_INVALID, "job / need is null");
  const Value* cs = j->doc.path({"status", "conditions"});
  if (!cs || !cs->is_array() || cs->a.empty()) {
    *need = 1;
    return TOK_OK;
  }
  const Value& last = cs->a.back();
  const std::string t = last.find("type") ? last.find("type")->as_string() : "";
  const std::string r = last.find("reason") ? last.find("reason")->as_string() : "";
  *need = (t == "Created" || (t == "Queuing" && r == "JobEnqueued")) ? 1 : 0;
  return TOK_OK;
}

// ---- job status machine (controllers/common/pod.go:690-714, controllers/train/job.go:99-207) ----------
int tok_job_update_status(tok_job_t* j, const char* replicas_json, int restarting, const char* now_c,
                          char** out) {
  if (!j) return fail(TOK_ERR_INVALID, "job is null");
  status_of(j);  // create .status BEFORE taking pointers into the document (insertion reallocates)
  const Value* specs = task_specs(j);
  if (!specs) return fail(TOK_ERR_INVALID, "spec.torchTaskSpecs is missing");
  Value reps;
  std::string err;
  if (!json::parse(replicas_json ? replicas_json : "{}", &reps, &err) || !reps.is_object())
    return fail(TOK_ERR_INVALID, "replicas must be a JSON object {taskType: [{phase,...}]}: %s", err.c_str());
  const std::string now = now_c ? now_c : "";
  const std::string name = job_name(j);
  Value& status = status_of(j);
  // task counters are recomputed from scratch on every pass (pod.go:391)
  Value ts_all = Value::object();
  for (const auto& kv : specs->o) {
    int64_t active = 0, succeeded = 0, failed = 0, evicted = 0;
    const Value* list = nullptr;
    for (const auto& rk : reps.o)
      if (equal_fold(rk.first, kv.first)) list = &rk.second;
    if (list && list->is_array())
      for (const Value& r : list->a) {
        const std::string ph = r.find("phase") ? r.find("phase")->as_string() : "";
        if (ph == "Pending") {
          // active only once scheduled (bound to a GPU slot) and past its init steps (pod.go:705-714)
          const bool scheduled = r.find("scheduled") ? r.find("scheduled")->as_bool() : false;
          const bool init_ok = r.find("initPassed") ? r.find("initPassed")->as_bool() : true;
          if (scheduled && init_ok) active++;
        } else if (ph == "Running") {
          active++;
        } else if (ph == "Succeeded") {
          succeeded++;
        } else if (ph == "Failed") {
          failed++;
          if (r.find("reason") && r.find("reason")->as_string() == "Evicted") evicted++;
        }
      }
    Value t = Value::object();
    t["active"] = Value::integer(active);
    t["succeed"] = Value::integer(succeeded);
    t["failed"] = Value::integer(failed);
    if (evicted) t["evicted"] = Value::integer(evicted);
    ts_all[kv.first] = std::move(t);
  }
  status["taskStatuses"] = ts_all;
  if (!status.find("startTime") || status.find("startTime")->is_null())
    status["startTime"] = Value::str(now);  // job.go:104-108

  const bool has_master_kind = specs->find("Master") || specs->find("AIMaster");
  const Value* wspec = specs->find("Worker");
  bool all_workers_ok = false;
  if (wspec) {
    const Value* w = ts_all.find("Worker");
    all_workers_ok = num_tasks(*wspec) == (w ? w->find("succeed")->as_int() : 0);
  }
  // deterministic order: AIMaster, Master, Worker, then the rest (Go iterates the map randomly)
  std::vector<std::string> order;
  for (const char* k : {"AIMaster", "Master", "Worker"})
    if (specs->find(k)) order.push_back(k);
  for (const auto& kv : specs->o)
    if (std::find(order.begin(), order.end(), kv.first) == order.end()) order.push_back(kv.first);
  for (const std::string& tt : order) {
    const Value& tspec = *specs->find(tt);
    const Value& t = *ts_all.find(tt);
    const int64_t n = num_tasks(tspec);
    const int64_t expected = n - t.find("succeed")->as_int();
    const int64_t running = t.find("active")->as_int();
    const int64_t failed = t.find("failed")->as_int();
    if (!has_master_kind)
      return fail(TOK_ERR_INVALID, "invalid config: Job must contain master replica spec");
    if (tt == "Master" || tt == "AIMaster") {
      if (running > 0)
        set_condition(status, "Running", "JobRunning", "TorchJob " + name + " is running.", now);
      bool succeed = n > 0 && expected == 0;
      if (tt != "AIMaster" && wspec) succeed = succeed && all_workers_ok;
      if (succeed) {
        if (!status.find("completionTime") || status.find("completionTime")->is_null())
          status["completionTime"] = Value::str(now);
        set_condition(status, "Succeeded", "JobSucceeded",
                      "TorchJob " + name + " is successfully completed.", now);
      }
    }
    if (failed > 0) {
      if (restarting && tt != "AIMaster") {
        set_condition(status, "Restarting", "JobRestarting",
                      "TorchJob " + name + " is restarting because " + std::to_string(failed) + " " +
                          tt + " task(s) failed.", now);
      } else {
        if (!status.find("completionTime") || status.find("completionTime")->is_null())
          status["completionTime"] = Value::str(now);
        set_condition(status, "Failed", "JobFailed",
                      "TorchJob " + name + " is failed because " + std::to_string(failed) + " " + tt +
                          " task(s) failed.", now);
      }
    }
  }
  return out ? out_json(status, out) : TOK_OK;
}

// ---- termination policies (controllers/common/job.go:100-200, 385-460, 511-539) -------------------------
static bool parse_rfc3339(const std::string& t, double* out) {
  int Y, M, D, h, m, sec;
  if (sscanf(t.c_str(), "%d-%d-%dT%d:%d:%d", &Y, &M, &D, &h, &m, &sec) != 6) return false;
  struct tm tmv;
  memset(&tmv, 0, sizeof(tmv));
  tmv.tm_year = Y - 1900;
  tmv.tm_mon = M - 1;
  tmv.tm_mday = D;
  tmv.tm_hour = h;
  tmv.tm_min = m;
  tmv.tm_sec = sec;
  *out = static_cast<double>(timegm(&tmv));
  return true;
}

int tok_job_check_termination(tok_job_t* j, const char* replicas_json, int prev_retries,
                              const char* now_c, char** out) {
  if (!j || !now_c) return fail(TOK_ERR_INVALID, "job / now is null");
  status_of(j);
  const Value* specs = task_specs(j);
  if (!specs) return fail(TOK_ERR_INVALID, "spec.torchTaskSpecs is missing");
  Value reps;
  std::string err;
  if (!json::parse(replicas_json ? replicas_json : "{}", &reps, &err) || !reps.is_object())
    return fail(TOK_ERR_INVALID, "replicas must be a JSON object {taskType: [{phase,restartCount}]}: %s", err.c_str());
  double now = 0;
  if (!parse_rfc3339(now_c, &now)) return fail(TOK_ERR_INVALID, "now must be RFC3339 (YYYY-MM-DDTHH:MM:SSZ): %s", now_c);
  const std::string name = job_name(j);
  const Value* spec = j->doc.find("spec");
  Value& status = status_of(j);

  int64_t expected = 0, active = 0, failed = 0, restarts = 0, prev_failed = 0;
  for (const auto& kv : specs->o) {
    expected += num_tasks(kv.second);  // GetTotalTasks (pkg/utils/utils.go:30-37)
    const std::string rp = kv.second.find("restartPolicy") ? kv.second.find("restartPolicy")->as_string() : "";
    const Value* list = nullptr;
    for (const auto& rk : reps.o)
      if (equal_fold(rk.first, kv.first)) list = &rk.second;
    if (!list || !list->is_array()) continue;
    for (const Value& r : list->a) {
      const std::string ph = r.find("phase") ? r.find("phase")->as_string() : "";
      if (ph == "Pending" || ph == "Running") active++;  // k8scontroller.IsPodActive
      if (ph == "Failed") failed++;
      if (ph == "Running" && (rp == "OnFailure" || rp == "Always"))  // pastBackoffLimit :385-419
        restarts += r.find("restartCount") ? r.find("restartCount")->as_int() : 0;
    }
  }
  const Value* ts = status.find("taskStatuses");
  if (ts && ts->is_object())
    for (const auto& kv : ts->o)
      prev_failed += kv.second.find("failed") ? kv.second.find("failed")->as_int() : 0;

  bool exceeds = false, past = false, deadline = false;
  const Value* bl = spec ? spec->find("backoffLimit") : nullptr;
  if (bl && bl->is_number()) {
    const int64_t limit = bl->as_int();
    exceeds = failed > prev_failed && active != expected && (static_cast<int64_t>(prev_retries) + 1) > limit;
    past = limit == 0 ? restarts > 0 : restarts >= limit;
  }
  std::string failure;
  bool exceeds_limit = false;
  if (exceeds || past) {
    exceeds_limit = true;
    failure = "Job " + name + " has failed because it has reached the specified backoff limit";
  } else {
    const Value* ad = spec ? spec->find("activeDurations") : nullptr;
    const Value* st = status.find("startTime");
    double start = 0;
    if (ad && ad->is_number() && st && st->is_string() && parse_rfc3339(st->s, &start) &&
        now - start >= static_cast<double>(ad->as_int())) {  // pastActiveDeadline :422-430
      deadline = true;
      exceeds_limit = true;
      failure = "Job " + name + " has failed because it was no longer active";
      // the reference overwrites CompletionTime on EVERY pass past the deadline (job.go:131-132), so
      // its TTL clock never starts; intended: stamp it once
      if (!status.find("completionTime") || status.find("completionTime")->is_null())
        status["completionTime"] = Value::str(now_c);
    }
  }
  const bool terminate = has_condition(status, "Succeeded") || has_condition(status, "Failed") || exceeds_limit;
  Value res = Value::object();
  res["terminate"] = Value::boolean(terminate);
  res["exceedsBackoffLimit"] = Value::boolean(exceeds);
  res["pastBackoffLimit"] = Value::boolean(past);
  res["pastActiveDeadline"] = Value::boolean(deadline);
  if (terminate) {
    const std::string policy = (spec && spec->find("clenPodPolicy")) ? spec->find("clenPodPolicy")->as_string() : "None";
    res["deletePods"] = Value::str(policy == "None" || policy.empty() ? "None" : (policy == "Running" ? "Running" : "All"));
    if (exceeds_limit) {
      if (!status.find("completionTime") || status.find("completionTime")->is_null())
        status["completionTime"] = Value::str(now_c);
      set_condition(status, "Failed", "JobFailed", failure, now_c);
      res["message"] = Value::str(failure);
    }
    if (has_condition(status, "Succeeded")) {  // job.go:176-184: fold still-active replicas into succeed
      Value* tsm = status.find("taskStatuses");
      if (tsm && tsm->is_object())
        for (auto& kv : tsm->o) {
          const int64_t a = kv.second.find("active") ? kv.second.find("active")->as_int() : 0;
          const int64_t sc = kv.second.find("succeed") ? kv.second.find("succeed")->as_int() : 0;
          kv.second["succeed"] = Value::integer(sc + a);
          kv.second["active"] = Value::integer(0);
        }
    }
    // cleanupJob (:511-539): TTL after the completion time
    const Value* ttl = spec ? spec->find("TTLSecondsAfterFinished") : nullptr;
    const Value* ct = status.find("completionTime");
    double done = 0;
    if (ttl && ttl->is_number() && ct && ct->is_string() && parse_rfc3339(ct->s, &done)) {
      const double del = done + static_cast<double>(ttl->as_int());
      res["deleteJob"] = Value::boolean(now > del);
      res["requeueAfter"] = Value::number(now > del ? 0.0 : del - now);
    }
  }
  res["status"] = status;
  return out_json(res, out);
}

}  // extern "C"
