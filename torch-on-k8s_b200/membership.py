"""The membership file protocol between the controller and a job's replicas.

Next to the job's rendezvous socket path the controller publishes `<rendezvous>.members`, a JSON
document {"epoch", "world", "ranks": {replica name: rank}, "survivor_mask"}: the in-place
replacement of the reference's `distributed.io/world-size` annotation + kruise container restart
(controllers/train/elastic_scale.go:303-397).  A replica started into a running job writes
`<rendezvous>.ready.<replica name>` once it is up, so that the controller announces a scale-out only
when the survivors will not have to wait for anybody's start-up.

Standard library only: the controller and the CPU fake replicas of the tests use it without torch.
"""
from __future__ import annotations

import json
import os
import time
from typing import Optional


def _members(rdzv_path: str) -> str:
    return rdzv_path + ".members"


def publish(rdzv_path: str, doc: dict) -> None:
    """Write the membership document atomically: a reader sees the old one or the new one."""
    path = _members(rdzv_path)
    with open(path + ".tmp", "w") as f:
        json.dump(doc, f)
    os.replace(path + ".tmp", path)


def read(rdzv_path: str) -> Optional[dict]:
    """The published membership document, or None when there is none (yet) or it is partly written."""
    try:
        with open(_members(rdzv_path)) as f:
            return json.load(f)
    except (OSError, ValueError):
        return None


def mark_ready(rdzv_path: str, replica_name: str, epoch: int) -> None:
    with open("%s.ready.%s" % (rdzv_path, replica_name), "w") as f:
        f.write(str(epoch))


def is_ready(rdzv_path: str, replica_name: str) -> bool:
    return os.path.exists("%s.ready.%s" % (rdzv_path, replica_name))


def membership_update(doc: dict, replica_name: str, current_epoch: int):
    """Pure decision behind Replica.poll_membership_collective: (new_world, new_rank, member_mask,
    epoch) for tok_comm_reform, or None when the published epoch is not newer / this replica was
    dropped."""
    if int(doc.get("epoch", 0)) <= current_epoch or replica_name not in doc.get("ranks", {}):
        return None
    return int(doc["world"]), int(doc["ranks"][replica_name]), int(doc.get("survivor_mask", 0)), \
        int(doc["epoch"])


def wait_for_membership(rdzv_path: str, replica_name: str, min_epoch: int,
                        timeout_s: Optional[float] = None):
    """(rank, world, epoch) of the first published membership with epoch >= min_epoch that lists
    `replica_name`."""
    deadline = time.time() + (timeout_s if timeout_s is not None else
                              float(os.environ.get("TOK_RDZV_TIMEOUT_S", "120")))
    while True:
        doc = read(rdzv_path)
        if doc is not None and int(doc.get("epoch", 0)) >= min_epoch and \
                replica_name in doc.get("ranks", {}):
            return int(doc["ranks"][replica_name]), int(doc["world"]), int(doc["epoch"])
        if time.time() > deadline:
            raise TimeoutError("no membership listing %s at epoch >= %d was published under %s" %
                               (replica_name, min_epoch, _members(rdzv_path)))
        time.sleep(0.02)
