"""Single-box TorchJob controller: the reference operator's reconcile loop for the data-parallel
path, with "pod" = OS process bound to one GPU of the 8-GPU H100 box.

  reference                                            here
  -------------------------------------------------    ------------------------------------------------
  OnOwnerCreateFunc: default, Created, enqueue         submit(): TorchJob defaults, Created, coordinator
    (controllers/common/eventhandler.go:38-64)           .enqueue (held until dequeued — §2.3 intent)
  Coordinator.schedule every 100 ms                     tick(): Coordinator.tick (C ABI)
    (pkg/coordinator/core/coordinator.go:310-366)
  ReconcileJobs: PodGroup, DAG order, ReconcilePods     _reconcile(): gang admission over free GPU slots
    (controllers/common/job.go:55-342)                   (all-or-nothing MinMember), AIMaster -> Master
                                                         -> Worker with the DAG gate, one process per
                                                         missing index
  createNewPod + SetClusterSpec                         _start_replica(): env from tok_job_cluster_spec
    (controllers/common/pod.go:503-637)                  + TOK8S_GPU / TOK8S_JOB / TOK8S_RDZV
  reconcileOnePod + failover table                      _poll(): exit codes -> should_failover ->
    (pod.go:640-687, failover.go:52-172)                 restart same index (same RANK), Restarting
  updateGeneralJobStatus                                TorchJob.update_status (C ABI)

All decisions are made by libtok8s' C++ control plane through the C ABI; this module only owns the
processes.  Nothing here touches the data path.
"""
from __future__ import annotations

import os
import shlex
import signal
import subprocess
import sys
import time
from dataclasses import dataclass, field
from typing import Dict, List, Optional

from .coordinator import SCHEDULING_PERIOD_S, Coordinator
from .elastic import LOOP_PERIOD_S, ElasticPolicy, parse_log_line
from .job import TASK_ORDER, TorchJob, should_failover
from .metrics import KIND, Metrics


def _now() -> str:
    return time.strftime("%Y-%m-%dT%H:%M:%SZ", time.gmtime())


@dataclass
class ReplicaProc:
    task_type: str
    index: int
    gpu: Optional[int]
    proc: Optional[subprocess.Popen] = None
    phase: str = "Pending"      # Pending | Running | Succeeded | Failed
    exit_code: Optional[int] = None
    restarts: int = 0
    log_path: Optional[str] = None
    epoch: int = 0              # membership epoch at which this replica was started
    log_pos: int = 0            # bytes of the log already scraped for TOK8S_METRIC records


@dataclass
class ManagedJob:
    job: TorchJob
    uid: str
    command: Optional[List[str]] = None
    replicas: Dict[str, Dict[int, ReplicaProc]] = field(default_factory=dict)
    admitted: bool = False
    dequeued: bool = False
    gpus: List[int] = field(default_factory=list)
    done: bool = False
    retries: int = 0          # BackoffStatesQueue.NumRequeues stand-in (failover passes so far)
    epoch: int = 0            # membership epoch of the job's peer group (bumped on every rescale)
    elastic: Optional[ElasticPolicy] = None
    elastic_due: float = 0.0
    membership_dirty: bool = False     # the replica set changed since the last published epoch
    published: Optional[dict] = None   # last membership document written
    draining: List[tuple] = field(default_factory=list)   # (replica, name, deadline) leaving by itself


class Controller:
    def __init__(self, num_gpus: int = 8, *, policy: str = "wrr", log_dir: Optional[str] = None,
                 rdzv_dir: str = "/tmp", state_dir: Optional[str] = None,
                 elastic_period: float = LOOP_PERIOD_S, drain_grace_s: float = 0.0,
                 gpu_map: Optional[List[int]] = None, wait_ready: bool = False):
        """num_gpus GPU slots (one replica each).  gpu_map[slot] = physical CUDA ordinal (default:
        identity; a test box with one GPU maps every slot to 0).  drain_grace_s > 0: a replica that
        is scaled in is first dropped from the published membership and given that long to leave at
        a step boundary of its own accord (in-place scale-in: its peers must not find it dead in the
        middle of a gradient exchange); 0 = delete immediately (reconcileOnePod, pod.go:648-651)."""
        self.drain_grace_s = drain_grace_s
        self.gpu_map = gpu_map
        # wait_ready: announce a scale-out only when every joiner has written its readiness marker
        # (worker.init_replica does, once CUDA is up and the script's model is built): the survivors
        # then pause for the re-form and the state hand-over only, not for the joiners' start-up
        self.wait_ready = wait_ready
        self.free_gpus = list(range(num_gpus))
        self.num_gpus = num_gpus
        self.coord = Coordinator(policy=policy)
        self.coord.set_quota("", num_gpus)      # the box is the (only) quota
        self.jobs: Dict[str, ManagedJob] = {}
        self.log_dir = log_dir
        self.rdzv_dir = rdzv_dir
        self.events: List[tuple] = []
        self.metrics = Metrics()
        self._t_created: Dict[str, float] = {}
        self.state_dir = state_dir
        self.elastic_period = elastic_period

    # ---- submit (owner create) -------------------------------------------------------------------
    def submit(self, manifest, command: Optional[List[str]] = None) -> str:
        job = manifest if isinstance(manifest, TorchJob) else TorchJob(manifest)
        d = job.to_dict()
        uid = d["metadata"].get("uid") or "%s/%s" % (d["metadata"].get("namespace", "default"),
                                                       d["metadata"]["name"])
        job.set_condition("Created", "JobCreated", "TorchJob %s is created." % job.name, _now())
        mj = ManagedJob(job=job, uid=uid, command=command)
        self.jobs[uid] = mj
        self._t_created[uid] = time.time()
        if job.need_enqueue():
            self.coord.enqueue(job, uid)
            job.set_condition("Queuing", "JobEnqueued",
                              "Job %s is queuing and waiting for being scheduled." % uid, _now())
        self._event(uid, "JobEnqueued")
        self.metrics.created.labels(KIND).inc()
        return uid

    def _event(self, uid, reason, msg=""):
        self.events.append((time.time(), uid, reason, msg))
        self._persist(uid)

    def _persist(self, uid) -> None:
        """Job object + status for `python -m torch_on_k8s_b200 get/describe` (cli.py)."""
        if not self.state_dir or uid not in self.jobs:
            return
        import json
        os.makedirs(self.state_dir, exist_ok=True)
        d = self.jobs[uid].job.to_dict()
        d["metadata"].setdefault("creationTimestamp", time.strftime(
            "%Y-%m-%dT%H:%M:%SZ", time.gmtime(self._t_created.get(uid, time.time()))))
        d["x-events"] = [(time.strftime("%H:%M:%S", time.gmtime(t)), r, m)
                         for t, u, r, m in self.events if u == uid][-20:]
        tmp = os.path.join(self.state_dir, uid.replace("/", ".") + ".json")
        with open(tmp + ".tmp", "w") as f:
            json.dump(d, f)
        os.replace(tmp + ".tmp", tmp)

    # ---- one controller pass ------------------------------------------------------------------------
    def tick(self, now: Optional[float] = None) -> None:
        now = time.monotonic() if now is None else now
        # ResourceQuota.used stand-in: GPUs held per tenant (for tenants with their own quota) and by
        # the whole box (the default quota "" every other tenant is accounted against)
        held: Dict[str, int] = {}
        for m in self.jobs.values():
            held[self._tenant(m)] = held.get(self._tenant(m), 0) + len(m.gpus)
        for tenant, n in held.items():
            self.coord.set_used(tenant, n)
        self.coord.set_used("", self.num_gpus - len(self.free_gpus))
        out = self.coord.tick(now)
        if out.get("dequeued"):
            mj = self.jobs[out["dequeued"]]
            mj.dequeued = True
            mj.job.set_condition("Queuing", "JobDequeued",
                                 "Job %s is being dequeued and waiting for reconciling." % mj.uid, _now())
            self._event(mj.uid, "JobDequeued")
        for mj in list(self.jobs.values()):
            if mj.dequeued and not mj.done:
                self._reconcile(mj)
        states = [m.job.last_condition() for m in self.jobs.values() if not m.done]
        self.metrics.running.labels(KIND).set(sum(s in ("Running", "Restarting") for s in states))
        self.metrics.pending.labels(KIND).set(sum(s in ("Created", "Queuing") for s in states))
        for tenant in {self._tenant(m) for m in self.jobs.values()}:
            self.metrics.queue_pending.labels(tenant).set(self.coord.pending(tenant))

    @staticmethod
    def _tenant(mj: ManagedJob) -> str:
        d = mj.job.to_dict()
        return (d["spec"].get("schedulingPolicy") or {}).get("queue") or \
            d["metadata"].get("namespace", "default")

    # ---- reconcile -------------------------------------------------------------------------------------
    def _reconcile(self, mj: ManagedJob) -> None:
        job = mj.job
        if not mj.admitted:
            g = job.gang_admit(len(self.free_gpus))
            if not g["admitted"]:
                return  # all-or-nothing: wait for MinMember slots
            mj.admitted = True
            self._event(mj.uid, "GangAdmitted", "slots=%d" % g["slotsNeeded"])
        restarting = self._poll(mj)
        if restarting:
            mj.retries += 1
        self._scrape_metrics(mj)
        # termination policies first, as ReconcileJobs does (controllers/common/job.go:100-200)
        pods = {tt: [dict(phase=r.phase, restartCount=r.restarts) for r in v.values()]
                for tt, v in mj.replicas.items()}
        term = job.check_termination(pods, mj.retries, _now())
        if term["terminate"]:
            if term.get("message"):
                self._event(mj.uid, "JobFailed", term["message"])
            self.coord.job_settled(mj.uid)
            self._finish(mj, term.get("deletePods", "None"))
            return
        self._elastic_pass(mj)
        specs = job.task_specs
        # replicas whose index fell out of [0, numTasks) are scaled down (reconcileOnePod,
        # controllers/common/pod.go:648-651)
        changed = False
        for r, name, deadline in list(mj.draining):
            gone = r.proc is None or r.proc.poll() is not None
            if not gone and time.monotonic() > deadline:
                self._kill(r)
                gone = True
            if gone:
                mj.draining.remove((r, name, deadline))
                self._release(mj, r)
                self._event(mj.uid, "SuccessfulDeletePod", name)
        for tt, have in mj.replicas.items():
            n = int(specs.get(tt, {}).get("numTasks", 1)) if tt in specs else 0
            for idx in [i for i in have if i >= n]:
                r = have.pop(idx)
                name = "%s-%s-%d" % (job.name, tt.lower(), idx)
                changed = True
                if r.proc and r.proc.poll() is None and self.drain_grace_s > 0:
                    mj.draining.append((r, name, time.monotonic() + self.drain_grace_s))
                    self._event(mj.uid, "DrainingPod", name)
                    continue
                self._kill(r)
                self._release(mj, r)
                self._event(mj.uid, "SuccessfulDeletePod", name)
        before = sum(len(v) for v in mj.replicas.values())
        for tt in TASK_ORDER + [k for k in specs if k not in TASK_ORDER]:
            if tt not in specs:
                continue
            phases = {k: [r.phase for r in v.values()] for k, v in mj.replicas.items()}
            if not job.dag_ready(tt, phases):
                continue
            have = mj.replicas.setdefault(tt, {})
            for idx in range(int(specs[tt].get("numTasks", 1))):
                if idx not in have:
                    self._start_replica(mj, tt, idx)
        if changed or sum(len(v) for v in mj.replicas.values()) != before:
            mj.membership_dirty = True
        if mj.epoch > 0 and mj.membership_dirty:
            self._publish_membership(mj)     # deferred while a listed replica has no process yet
        reps = {tt: [dict(phase=r.phase, scheduled=r.gpu is not None or tt == "AIMaster",
                          exitCode=r.exit_code) for r in v.values()]
                for tt, v in mj.replicas.items()}
        job.update_status(reps, restarting, _now())
        last = job.last_condition()
        if last in ("Running", "Failed", "Succeeded"):
            self.coord.job_settled(mj.uid)
        if last in ("Failed", "Succeeded"):
            term = job.check_termination(pods, mj.retries, _now())
            self._finish(mj, term.get("deletePods", "None"))

    def _scrape_metrics(self, mj: ManagedJob) -> None:
        """New `TOK8S_METRIC {...}` lines of the master / first worker log -> Prometheus series."""
        import json
        for tt in ("Master", "Worker"):
            r = mj.replicas.get(tt, {}).get(0)
            if r is None or not r.log_path:
                continue
            try:
                with open(r.log_path, "rb") as f:
                    f.seek(r.log_pos)
                    chunk = f.read()
            except OSError:
                continue
            cut = chunk.rfind(b"\n") + 1          # only whole lines
            r.log_pos += cut
            for ln in chunk[:cut].decode("utf-8", "replace").splitlines():
                if ln.startswith("TOK8S_METRIC "):
                    try:
                        self.metrics.feed(mj.job.name, json.loads(ln[13:]))
                    except ValueError:
                        pass

    # ---- torchelastic (controllers/train/torchelastic/elastictorchjob_controller.go:142-166) -------
    def _elastic_pass(self, mj: ManagedJob) -> None:
        """One decision pass per `elastic_period` for jobs with enableTorchElastic: read the last
        progress line of <job>-worker-0 (observation.go:40-85), feed the policy, let the normal
        reconcile create / delete replicas for the new Worker.numTasks.  Survivors are not restarted:
        they learn the new membership from the epoch file (see _publish_membership)."""
        spec = mj.job.to_dict()["spec"]
        if not spec.get("enableTorchElastic") or not spec.get("torchElasticPolicy"):
            return
        now = time.monotonic()
        if now < mj.elastic_due:
            return
        mj.elastic_due = now + self.elastic_period
        if mj.elastic is None:
            mj.elastic = ElasticPolicy()
        workers = mj.replicas.get("Worker", {})
        latency = -1.0
        w0 = workers.get(0)
        if w0 is not None and w0.log_path and os.path.exists(w0.log_path):
            with open(w0.log_path, "rb") as f:
                lines = f.read().decode("utf-8", "replace").strip().splitlines()
            if lines:
                try:
                    latency = float(parse_log_line(lines[-1])["latency"])
                except Exception:  # noqa: BLE001 — not a progress line / latency > 1 s: skip the tick
                    latency = -1.0
        before = mj.job.num_tasks("Worker")
        out = mj.elastic.observe(mj.job, latency,
                                 has_pending=any(r.phase == "Pending" for r in workers.values()),
                                 has_failed=any(r.phase == "Failed" for r in workers.values()))
        if out["action"] in ("scale", "revert"):
            mj.epoch += 1
            self._event(mj.uid, "ElasticScale", "%s: Worker %d -> %d (%s)" %
                        (out["action"], before, out["replicas"], out["condition"]))
        elif out["action"] in ("forget", "stop_managing"):
            mj.elastic_due = float("inf")

    # ---- user-driven rescale (row a7) ---------------------------------------------------------------
    def scale(self, uid: str, task_type: str, num_tasks: int) -> int:
        """A spec update of torchTaskSpecs[task_type].numTasks on a running job — what the reference
        answers by restarting every stale pod with a new WORLD_SIZE (controllers/train/
        elastic_scale.go:210-397).  Here the next reconcile creates / deletes the replicas and a new
        membership epoch lets the survivors re-form in place.  Returns the new epoch."""
        from ._ffi import TOK_MAX_WORLD
        mj = self.jobs[uid]
        others = sum(int(ts.get("numTasks", 1)) for tt, ts in mj.job.task_specs.items()
                     if tt not in ("AIMaster", task_type))
        if others + num_tasks > TOK_MAX_WORLD:
            raise ValueError("world %d exceeds the box (%d replicas)" % (others + num_tasks, TOK_MAX_WORLD))
        before = mj.job.num_tasks(task_type)
        if before == num_tasks:
            return mj.epoch
        mj.job.scale(task_type, num_tasks)
        mj.epoch += 1
        mj.membership_dirty = True
        self._event(uid, "Scale", "%s %d -> %d (epoch %d)" % (task_type, before, num_tasks, mj.epoch))
        return mj.epoch

    def _publish_membership(self, mj: ManagedJob) -> bool:
        """Membership epoch file next to the job's rendezvous socket: the in-place replacement of the
        reference's `distributed.io/world-size` annotation + kruise container restart
        (controllers/train/elastic_scale.go:303-397).  Replicas poll it (worker.Replica.poll_membership)
        and call tok_comm_reform / join at the announced epoch.

        Only a membership every member of which has a live process is announced: survivors that
        re-formed towards a replica that is still Pending (no free GPU) would block in the rendezvous
        until it times out — the reference's has_pending branch reverts such a scale-out instead, and
        so does the next torchelastic pass here.  Returns True when a document was written."""
        import json
        from ._ffi import TOK_MAX_WORLD
        members, mask = {}, 0
        for tt in TASK_ORDER:
            for idx in sorted(mj.replicas.get(tt, {})):
                if tt == "AIMaster":
                    continue
                r = mj.replicas[tt][idx]
                if r.proc is None or r.proc.poll() is not None:
                    return False            # Pending / exited: wait for the reconcile to settle
                spec = mj.job.cluster_spec(tt.lower(), idx)
                known = mj.published["ranks"] if mj.published is not None else None
                joiner = (known is not None and spec["name"] not in known) or \
                    (known is None and r.epoch > 0)
                if self.wait_ready and joiner and not os.path.exists(
                        "%s.ready.%s" % (self._rdzv_path(mj), spec["name"])):
                    return False            # still starting up: the survivors keep training
                members[spec["name"]] = spec["rank"]
                # a replica's rank is a function of (task type, index), so a survivor keeps its rank:
                # bit i set <=> the replica that held rank i in the membership the group currently
                # runs with (the last PUBLISHED one, or the initial one) is still a member
                # (tok_comm_reform's member_mask).  Replicas started since then are joiners, whatever
                # epoch they were started at: they wait for this document and join at ITS epoch.
                if not joiner:
                    mask |= 1 << spec["rank"]
        world = mj.job.world_size
        if len(members) != world or sorted(members.values()) != list(range(world)):
            return False                    # replicas of the new spec are not all created yet
        if world > TOK_MAX_WORLD:
            self._event(mj.uid, "MembershipRejected", "world %d > %d" % (world, TOK_MAX_WORLD))
            return False
        mj.membership_dirty = False
        if mj.published is not None and mj.published["ranks"] == members:
            return False                    # e.g. a scale-out that was reverted before it happened
        path = self._rdzv_path(mj) + ".members"
        doc = {"epoch": mj.epoch, "world": world, "ranks": members, "survivor_mask": mask}
        with open(path + ".tmp", "w") as f:
            json.dump(doc, f)
        os.replace(path + ".tmp", path)
        mj.published = doc
        self._event(mj.uid, "MembershipPublished", json.dumps(doc))
        return True

    def _rdzv_path(self, mj: ManagedJob) -> str:
        port = mj.job.cluster_spec("master", 0)["env"][0]["value"]
        return os.path.join(self.rdzv_dir, "tok8s-%s-%s" % (mj.job.name.replace("/", "-"), port))

    def _start_replica(self, mj: ManagedJob, tt: str, idx: int, restarts: int = 0) -> None:
        spec = mj.job.cluster_spec(tt.lower(), idx)
        gpu = None
        if spec["gpuSlots"] > 0:
            if not self.free_gpus:
                mj.replicas[tt][idx] = ReplicaProc(tt, idx, None)   # Pending, unscheduled
                return
            gpu = self.free_gpus.pop(0)
            mj.gpus.append(gpu)
        env = dict(os.environ)
        env.update({e["name"]: e["value"] for e in spec["env"]})
        if env.get("MASTER_ADDR") not in ("localhost", "127.0.0.1"):
            env["MASTER_ADDR"] = "127.0.0.1"   # single box: the master's name resolves to loopback
        env.update(TOK8S_JOB=mj.job.name, TOK8S_REPLICA=spec["name"], TOK8S_TASK_TYPE=tt,
                   TOK8S_TASK_INDEX=str(idx), TOK8S_EPOCH=str(mj.epoch),
                   TOK8S_RDZV=os.path.join(self.rdzv_dir, "tok8s-%s-%s" %
                                           (mj.job.name.replace("/", "-"), env["MASTER_PORT"])))
        if gpu is not None:
            phys = self.gpu_map[gpu] if self.gpu_map else gpu
            env.update(TOK8S_GPU=str(phys), LOCAL_RANK=str(phys), TOK8S_SLOT=str(gpu))
        cmd = mj.command or self._container_command(mj, tt)
        cmd = list(cmd) + spec["args"] if spec["args"] and mj.command is None else list(cmd)
        log = None
        if self.log_dir:
            os.makedirs(self.log_dir, exist_ok=True)
            path = os.path.join(self.log_dir, spec["name"] + ".log")
            log = open(path, "ab")
        proc = subprocess.Popen(cmd, env=env, stdout=log or None, stderr=subprocess.STDOUT if log else None,
                                start_new_session=True)
        mj.replicas[tt][idx] = ReplicaProc(tt, idx, gpu, proc, "Running", restarts=restarts,
                                           log_path=log.name if log else None, epoch=mj.epoch)
        self._event(mj.uid, "SuccessfulCreatePod", spec["name"])
        d = mj.job.to_dict()["metadata"]
        lbl = (KIND, d["name"], d.get("namespace", "default"), mj.uid)
        created = sum(len(v) for v in mj.replicas.values())
        if created == 1 and restarts == 0:
            self.metrics.first_pod_delay.labels(*lbl).observe(time.time() - self._t_created.get(mj.uid, time.time()))
        if created == mj.job.world_size + mj.job.num_tasks("AIMaster") and restarts == 0:
            self.metrics.all_pods_delay.labels(*lbl).observe(time.time() - self._t_created.get(mj.uid, time.time()))

    def _container_command(self, mj: ManagedJob, tt: str) -> List[str]:
        c = None
        for cand in mj.job.task_specs[tt].get("template", {}).get("spec", {}).get("containers", []):
            if cand.get("name") == "torch":
                c = cand
        if not c or not (c.get("command") or c.get("args")):
            raise ValueError("replica template of %s has no `torch` container command" % tt)
        return list(c.get("command") or []) + list(c.get("args") or [])

    def _poll(self, mj: ManagedJob) -> bool:
        """reconcileOnePod for every replica; returns True when a failover was triggered."""
        restarting = False
        for tt, reps in mj.replicas.items():
            policy = mj.job.task_specs[tt].get("restartPolicy", "")
            for idx, r in list(reps.items()):
                if r.proc is None:
                    if r.gpu is None and self.free_gpus and r.phase == "Pending":
                        del reps[idx]          # a GPU slot freed up: recreate the replica
                    continue
                rc = r.proc.poll()
                if rc is None or r.phase in ("Succeeded", "Failed"):
                    continue
                code = rc if rc >= 0 else 128 - rc     # killed by signal n -> 128 + n
                r.exit_code = code
                r.phase = "Succeeded" if code == 0 else "Failed"
                self._release(mj, r)
                self._event(mj.uid, "ExitedWithCode", "%s-%s-%d: %d" % (mj.job.name, tt, idx, code))
                if code != 0 and should_failover(policy, code, ""):
                    del reps[idx]              # recreated next pass with the same index => same RANK
                    restarting = True
                    self.metrics.restarted.labels(KIND).inc()
                    self._event(mj.uid, "FailoverRecreate", "%s-%d" % (tt, idx))
                elif code != 0 and policy in ("OnFailure", "Always"):
                    limit = (mj.job.to_dict()["spec"].get("backoffLimit"))
                    if limit is None or r.restarts < int(limit):
                        n = r.restarts + 1
                        del reps[idx]
                        self._start_replica(mj, tt, idx, restarts=n)   # kubelet-style in-place restart
        return restarting

    @staticmethod
    def _kill(r: ReplicaProc) -> None:
        if r.proc and r.proc.poll() is None:
            try:
                os.killpg(r.proc.pid, signal.SIGTERM)
                r.proc.wait(timeout=10)
            except (ProcessLookupError, subprocess.TimeoutExpired):
                pass

    def _release(self, mj: ManagedJob, r: ReplicaProc) -> None:
        if r.gpu is not None and r.gpu in mj.gpus:
            mj.gpus.remove(r.gpu)
            self.free_gpus.append(r.gpu)
            self.free_gpus.sort()
            r.gpu = None

    def _finish(self, mj: ManagedJob, delete_pods: str = "None") -> None:
        # deletePodsAndServices (job.go:433-460): cleanPodPolicy None keeps everything, Running / All
        # stop what is still running (finished processes have nothing left to delete on one box)
        for r, name, _ in mj.draining:
            self._kill(r)
            self._release(mj, r)
        mj.draining = []
        for reps in mj.replicas.values():
            for r in reps.values():
                if r.proc and r.proc.poll() is None and delete_pods in ("Running", "All"):
                    try:
                        os.killpg(r.proc.pid, signal.SIGTERM)
                        r.proc.wait(timeout=10)
                    except (ProcessLookupError, subprocess.TimeoutExpired):
                        pass
                if r.proc and r.proc.poll() is not None:
                    self._release(mj, r)
        mj.done = True
        self._event(mj.uid, "Job" + (mj.job.last_condition() or ""))
        (self.metrics.successful if mj.job.last_condition() == "Succeeded" else self.metrics.failed) \
            .labels(KIND).inc()

    # ---- helpers ------------------------------------------------------------------------------------------
    def run_until_done(self, timeout: float = 600.0, period: float = SCHEDULING_PERIOD_S) -> Dict[str, str]:
        deadline = time.time() + timeout
        while time.time() < deadline and not all(m.done for m in self.jobs.values()):
            self.tick()
            time.sleep(period)
        for mj in self.jobs.values():
            if not mj.done:
                for reps in mj.replicas.values():
                    for r in reps.values():
                        if r.proc and r.proc.poll() is None:
                            try:
                                os.killpg(r.proc.pid, signal.SIGKILL)
                            except ProcessLookupError:
                                pass
        return {uid: (m.job.last_condition() or "") for uid, m in self.jobs.items()}


def main(argv=None) -> int:
    import argparse
    import json
    from .job import load_manifest
    ap = argparse.ArgumentParser(prog="tok8s-controller",
                                 description="run TorchJob manifests on this box (one replica per GPU)")
    ap.add_argument("manifests", nargs="+")
    ap.add_argument("--gpus", type=int, default=8)
    ap.add_argument("--policy", default="wrr", choices=["rr", "wrr"])
    ap.add_argument("--command", default=None, help="override the replica command (shell-split)")
    ap.add_argument("--log-dir", default=None)
    ap.add_argument("--state-dir", default=os.environ.get("TOK8S_STATE_DIR"))
    ap.add_argument("--timeout", type=float, default=3600)
    ap.add_argument("--metrics-port", type=int, default=0,
                    help="serve GET /metrics here (the reference's default is 8443; 0 = off)")
    a = ap.parse_args(argv)
    ctl = Controller(a.gpus, policy=a.policy, log_dir=a.log_dir, state_dir=a.state_dir)
    if a.metrics_port:
        ctl.metrics.serve(a.metrics_port)
    for m in a.manifests:
        ctl.submit(load_manifest(m), shlex.split(a.command) if a.command else None)
    res = ctl.run_until_done(a.timeout)
    print(json.dumps(res))
    return 0 if all(v == "Succeeded" for v in res.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
