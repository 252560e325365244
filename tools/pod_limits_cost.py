"""What RespectNodePodLimits costs one C3 round on the device (dev tooling; needs a GPU):
    python tools/pod_limits_cost.py [--scale S]   ->  one JSON line per configuration

Configurations: C3 as it is; C3 with the knob on and 110 pods per node (the kubelet's default), where the pods field
takes the best-fit key's fields from 25 to 32 bits and so past the 32-bit compare keys of the assignment loop; and a
C3 variant where pods bind first (8 per 32-cpu node, 16 per 64-cpu gpu node).  Each is uploaded once and run three
times, one round at a time like tools/time_configs.py; reported: the assignment loop's form (from the upload's layout
line), the best `ms_per_round` (device time), SM cycles per placement (the kernel's cycle count from
ARMADA_PRINT_STATS over the placements) and the number of outputs that differ from the oracle."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import oracle_lib  # noqa: E402
import shape_cases  # noqa: E402
from armada_b200 import synth  # noqa: E402
from armada_b200.scheduler import DeviceRound  # noqa: E402


def configs(scale):
    def c3():
        return synth.config_c3() if scale == 1.0 else synth.scaled("C3", scale)

    def binding():
        r = c3()
        return synth.with_pod_limits(r, np.where(np.asarray(r.node_type) == 1, 16, 8))

    return [("C3", c3), ("C3+pods110", lambda: synth.with_pod_limits(c3(), 110)), ("C3+pods8", binding)]


class captured_stderr:
    """The process's stderr (file descriptor 2, where the library prints) while the block runs, in `.text`."""

    def __enter__(self):
        sys.stderr.flush()
        self.tmp = tempfile.TemporaryFile(mode="w+")
        self.saved = os.dup(2)
        os.dup2(self.tmp.fileno(), 2)
        return self

    def __exit__(self, *exc):
        sys.stderr.flush()
        os.dup2(self.saved, 2)
        os.close(self.saved)
        self.tmp.seek(0)
        self.text = self.tmp.read()
        self.tmp.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0, help="C3 at this fraction of its size (1: 100k nodes, 1M jobs)")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": card}), flush=True)
    os.environ["ARMADA_TIME_UPLOAD"] = "1"
    os.environ["ARMADA_PRINT_STATS"] = "1"
    with DeviceRound(0) as dev:
        for name, make in configs(args.scale):
            inp = make().to_input()
            with captured_stderr() as up:
                dev.upload(inp)
            lay = shape_cases.layout_of(up.text)
            best = best_cycles = None
            for _ in range(3):
                with captured_stderr() as run:
                    st = dev.run()
                if best is None or st.device_ms < best.device_ms:
                    best, best_cycles = st, int(re.findall(r"kernel_cycles=(\d+)", run.text)[-1])
            got = dev.download()
            diffs = got.diff(oracle_lib.round_schedule(inp))
            print(json.dumps({"config": name, "form": shape_cases.form_of(lay, inp), "key_bits_above_node": lay["key_total_bits"] - lay["node_bits"],
                              "ms_per_round": round(best.device_ms, 3), "placements": int(best.placements),
                              "sm_cycles_per_placement": round(best_cycles / max(1, int(best.placements)), 1),
                              "parity_diffs": len(diffs)}), flush=True)


if __name__ == "__main__":
    main()
