"""Observability parity (SURVEY.md §5 / §8f-3): the reference's Prometheus metric NAMES
(pkg/metrics/metrics.go:33-125, pkg/coordinator/core/metrics.go:25-28) kept verbatim, fed by the
single-box controller, plus two series for the new path (allreduce bus bandwidth, re-form latency).
Rendering uses prometheus_client's text exposition; nothing here is on the data path."""
from __future__ import annotations

from typing import Optional

from prometheus_client import CollectorRegistry, Counter, Gauge, Histogram, generate_latest

KIND = "TorchJob"


class Metrics:
    def __init__(self, registry: Optional[CollectorRegistry] = None):
        self.registry = registry or CollectorRegistry()
        r = self.registry

        def counter(name, doc):
            return Counter(name, doc, ["kind"], registry=r)
        # counters by `kind` (metrics.go:33-66)
        self.created = counter("torch_on_k8s_jobs_created", "Counts number of jobs created")
        self.deleted = counter("torch_on_k8s_jobs_deleted", "Counts number of jobs deleted")
        self.successful = counter("torch_on_k8s_jobs_successful", "Counts number of jobs successfully finished")
        self.failed = counter("torch_on_k8s_jobs_failed", "Counts number of jobs failed")
        self.restarted = counter("torch_on_k8s_jobs_restarted", "Counts number of jobs restarted")
        # gauges (metrics.go:97-122)
        self.running = Gauge("torch_on_k8s_jobs_running", "Counts number of jobs running currently",
                             ["kind"], registry=r)
        self.pending = Gauge("torch_on_k8s_jobs_pending", "Counts number of jobs pending currently",
                             ["kind"], registry=r)
        # launch-delay histograms (metrics.go:67-96)
        self.first_pod_delay = Histogram("torch_on_k8s_jobs_first_pod_launch_delay_seconds",
                                         "Histogram for recording launch delay duration(from job created to first pod running).",
                                         ["kind", "name", "namespace", "uid"], registry=r)
        self.all_pods_delay = Histogram("torch_on_k8s_jobs_all_pods_launch_delay_seconds",
                                        "Histogram for recording launch delay duration(from job created to all pods running).",
                                        ["kind", "name", "namespace", "uid"], registry=r)
        # coordinator (core/metrics.go:25-28)
        self.queue_pending = Gauge("torch_on_k8s_tenant_queue_jobs_pending_count",
                                   "Counts number of jobs pending in queue", ["queue"], registry=r)
        # new series for the H100 path
        self.busbw = Gauge("torch_on_k8s_allreduce_busbw_gbps",
                           "Achieved allreduce bus bandwidth of the last step (GB/s)", ["job"], registry=r)
        self.reform_latency = Histogram("torch_on_k8s_reform_latency_seconds",
                                        "Peer-group re-form latency (elastic add/drop in place)",
                                        ["job"], registry=r)

    def render(self) -> str:
        return generate_latest(self.registry).decode()

    def serve(self, port: int = 8443, addr: str = "127.0.0.1"):
        """GET /metrics on the reference's default port (main.go:59 `--metrics-addr 8443`,
        metrics.StartMonitoringForDefaultRegistry).  Returns (server, thread)."""
        from prometheus_client import start_http_server
        return start_http_server(port, addr=addr, registry=self.registry)

    def feed(self, job: str, record: dict) -> None:
        """One `TOK8S_METRIC {...}` record printed by a replica (worker.report_metric): the two
        series of the new path."""
        if "busbw_gbps" in record:
            self.busbw.labels(job).set(float(record["busbw_gbps"]))
        if "reform_s" in record:
            self.reform_latency.labels(job).observe(float(record["reform_s"]))
