"""The constructed contamination trace (DESIGN.md 1.5) shared by the CPU and GPU tests: the simulator's LockBit trace
with its files seeded by an application process (pid 300), a backup agent A that archives ciphertext and a backup
agent B that archived the files before the attack."""
from datetime import datetime, timedelta

from nerrf_b200 import trace_sim

APP, A, B = 300, 600, 601
NIGHTLY, OLD, NOTE = "/backup/nightly.tar", "/backup/old.tar", "/app/uploads/README_LOCKBIT.txt"


def _ts(e):
    return datetime.fromisoformat(e["timestamp"])


def constructed_trace(bystanders=0, n_files=12, benign_files=4, seed=0, a_reads=4):
    """-> (events, A's openat events, A's write event)"""
    ev = [dict(e) for e in trace_sim.lockbit_trace(n_files=n_files, benign_files=benign_files, seed=seed, bystanders=bystanders)]
    for e in ev:
        if e["event"] == "file_created":
            e["pid"] = APP                                   # an application seeds the files, not the attacker
    done = [e for e in ev if e["event"] == "file_encrypt_complete"]
    extra, a_open = [], []
    for k, e in enumerate(done[:a_reads]):                   # A reads ciphertext after it was written ...
        o = {"timestamp": (_ts(e) + timedelta(seconds=0.05)).isoformat(), "event": "openat", "path": e["path"], "size": 0,
             "pid": A, "phase": "benign", "flags": 0}
        extra.append(o); a_open.append(o)
    last = max(_ts(e) for e in ev)
    a_write = {"timestamp": (last + timedelta(seconds=1.0)).isoformat(), "event": "write", "path": NIGHTLY, "size": 4096,
               "pid": A, "phase": "benign"}
    extra.append(a_write)                                    # ... and archives it
    seeded = max(_ts(e) for e in ev if e["event"] == "seed_complete")
    created = [e for e in ev if e["event"] == "file_created"]
    for k, e in enumerate(created[:3]):                      # B reads the plaintext before the attack and archives it
        extra.append({"timestamp": (seeded + timedelta(seconds=0.1 + 0.1 * k)).isoformat(), "event": "openat",
                      "path": e["path"], "size": 0, "pid": B, "phase": "benign", "flags": 0})
    extra.append({"timestamp": (seeded + timedelta(seconds=0.9)).isoformat(), "event": "write", "path": OLD, "size": 4096,
                  "pid": B, "phase": "benign"})
    ev = sorted(ev + extra, key=_ts)
    return ev, a_open, a_write
