"""Fake torchelastic replica for the CPU controller tests: prints the progress line the torchelastic
controller scrapes (observation.go:54-76) every 50 ms for $RUN_S seconds, then exits 0.  With
ADAPTIVE=1 the printed batch latency follows the membership epoch file the controller publishes
(0.1 s x workers^2: scaling out makes the per-replica latency worse, so the policy must revert).
With EXIT_WHEN_DROPPED=1 it leaves on its own (exit 0) as soon as a published membership no longer
lists it — what a real replica does at a step boundary (Replica.poll_membership_collective)."""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from torch_on_k8s_b200 import membership  # noqa: E402

t_end = time.time() + float(os.environ.get("RUN_S", "6"))
rdzv = os.environ.get("TOK8S_RDZV", "")
step = 0
while time.time() < t_end:
    step += 10
    lat = 0.100
    if os.environ.get("ADAPTIVE"):
        doc = membership.read(rdzv)
        if doc is not None:
            workers = doc["world"] - 1
            lat = min(0.999, 0.1 * workers * workers)
    sys.stdout.write("Epoch: [0][%4d/5000]\tTime %6.3f (%6.3f)\tData  0.000 ( 0.000)\tLoss 6.9e+00\t"
                     "Acc@1   0.10 (  0.10)\tAcc@5  10.00 ( 10.00)\n" % (step, lat, lat))
    sys.stdout.flush()
    if os.environ.get("EXIT_WHEN_DROPPED"):
        doc = membership.read(rdzv)
        if doc is not None and os.environ.get("TOK8S_REPLICA") not in doc.get("ranks", {}):
            sys.exit(0)
    time.sleep(0.05)
