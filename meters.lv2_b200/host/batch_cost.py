"""Per-instance cost of the LV2 façade's batched plugins (B200M_LV2_BATCH) against private instances.

Runs lv2_host (built next to this file by build.py) for each plugin and mode, alternating the libraries given with --lib so that
two builds can be compared in one session, and prints one JSON line per run, then the min-max of `us_per_instance` per plugin,
mode and library.  The GPU's name and power limit are read at the start and printed with the results.

    python meters.lv2_b200/host/batch_cost.py [--lib meters.lv2_b200/libb200meters.so ...] [--uri COR ...] [--runs 3] [--instances 512]
                                              [--ui 1]
"""
import json
import os
import subprocess
import sys

import _cost
from _cost import B

HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    ap = _cost.parser(__doc__, lib=True, instances=512, nframes=1024, runs=3)
    ap.add_argument("--uri", action="append")
    ap.add_argument("--cycles", type=int, default=100)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--ui", type=int, default=0)                 # 1: a GUI is attached to every instance (lv2_host --ui)
    a = ap.parse_args()
    libs = a.lib or [B.LIB_PATH]
    uris = a.uri or ["spectr30stereo", "BBCM6", "surround5", "COR", "phasewheel", "goniometer"]
    gpu = _cost.gpu()
    print(json.dumps({"gpu": gpu}), flush=True)
    res = {}
    for r in range(a.runs):
        for uri in uris:
            for batch in (a.batch, 0):
                for lib in libs:
                    env = dict(os.environ)
                    env.pop("B200M_LV2_BATCH", None)
                    if batch:
                        env["B200M_LV2_BATCH"] = str(batch)
                    out = subprocess.run([os.path.join(HERE, "lv2_host"), "--lib", lib, "--uri", uri, "--instances", str(a.instances),
                                          "--cycles", str(a.cycles), "--nframes", str(a.nframes), "--ui", str(a.ui)], env=env, capture_output=True, text=True)
                    if out.returncode:
                        sys.exit("lv2_host failed: %s" % out.stderr)
                    j = json.loads(out.stdout.strip().splitlines()[-1])
                    print(json.dumps(j), flush=True)
                    res.setdefault((uri, batch, lib), []).append(j["us_per_instance"])
    for (uri, batch, lib), v in res.items():
        print(json.dumps({"uri": uri, "batch_slots": batch or None, "lib": lib, "gpu": gpu,
                          "us_per_instance_min": min(v), "us_per_instance_max": max(v)}))


if __name__ == "__main__":
    main()
