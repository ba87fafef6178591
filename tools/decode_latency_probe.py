#!/usr/bin/env python
"""Where does a single 4 MiB decode launch spend its time?  Runs bench.c2_single_request_latency under a few library switches
(each in its own process) and prints launch times + how the records were served.

    python tools/decode_latency_probe.py
"""
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r"""
import json, os, sys, ctypes as C
sys.path[:0] = [os.path.join(%(repo)r, "min-tfs-client_b200"), %(repo)r]
import bench
class W: local_rank = 0
out = bench.c2_single_request_latency(W())
print(json.dumps({k: (round(v["launch_us"], 3) if isinstance(v, dict) and "launch_us" in v else v) for k, v in out.items() if k != "how"}))
"""

VARIANTS = [
    ("default", {}),
    ("no inline template", {"B200TFS_NO_INLINE_TEMPLATE": "1"}),
    ("16 KB tiles (272 CTAs)", {"B200TFS_TILE_BYTES": "16384"}),
    ("8 KB tiles (544 CTAs)", {"B200TFS_TILE_BYTES": "8192"}),
    ("64 KB tiles (72 CTAs)", {"B200TFS_TILE_BYTES": "65536"}),
]


def main():
    if "--one" in sys.argv:       # in-process, default switches: the thing to run under ncu
        sys.path[:0] = [os.path.join(REPO, "min-tfs-client_b200"), REPO]
        import bench

        class W:
            local_rank = 0
        print(json.dumps(bench.c2_single_request_latency(W())))
        return
    rows = {}
    for name, env in VARIANTS:
        e = dict(os.environ, **env)
        r = subprocess.run([sys.executable, "-c", CHILD % {"repo": REPO}], capture_output=True, text=True, env=e, timeout=600)
        line = [l for l in r.stdout.strip().splitlines() if l.startswith("{")]
        rows[name] = json.loads(line[-1]) if line else {"error": (r.stderr or r.stdout)[-400:]}
        print(name, rows[name], flush=True)
    print(json.dumps(rows))


if __name__ == "__main__":
    main()
