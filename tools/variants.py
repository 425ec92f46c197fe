#!/usr/bin/env python
"""Build experiment variants of the library next to the default one and (on a GPU box) compare them.

    python tools/variants.py build e8=-DIRBPP_ENVS_PER_CTA=8 tpl2=-DIRBPP_TASKS_PER_LANE=2 fine=-DIRBPP_PROBE_FINE
        -> irbpp_b200/lib/libirbpp_e8.so, libirbpp_tpl2.so, libirbpp_fine.so   (they travel with gpurun like the default .so;
           several -D flags of one variant are separated by commas)
    python tools/variants.py bench e8 tpl2         # GPU: parity tests of the episode goldens + bench.py per variant
    IRBPP_LIB=irbpp_b200/lib/libirbpp_e8.so python tools/kbench.py    # or time one build on several workloads (tools/gpu/call19.sh)

Known build switches (csrc/): IRBPP_PROBE_FINE   slots 4-7 of the phase counters time the sub-phases of phase C
                              IRBPP_PROBE_TRACE  per-CTA timelines of the candidates kernel (tools/cta_trace.py)
                              IRBPP_TASKS_PER_LANE / IRBPP_ENVS_PER_CTA / IRBPP_ENVS_PER_CTA_WIDE / IRBPP_WIDE_MIN_R / IRBPP_SCAN_MIN_CTAS   CTA shapes
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
LIB_DIR = os.path.join(ROOT, "irbpp_b200", "lib")


def lib_path(name):
    return os.path.join(LIB_DIR, "libirbpp.so" if name == "default" else "libirbpp_%s.so" % name)


def main():
    if len(sys.argv) < 2:
        raise SystemExit(__doc__)
    cmd, args = sys.argv[1], sys.argv[2:]
    if cmd == "build":
        from irbpp_b200 import build as b
        for spec in args:
            name, defs = spec.split("=", 1)
            print(b.build(out=lib_path(name), defs=defs.split(",")))
        return 0
    if cmd == "bench":
        for name in ["default"] + args:
            env = dict(os.environ, IRBPP_LIB=lib_path(name))
            t = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_parity.py"), "-q", "-x",
                                "-m", "gpu", "-k", "episode or random or hull"], env=env, capture_output=True, text=True)
            r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "100", "--warmup", "5",
                                "--no-cpu-baseline"], env=env, capture_output=True, text=True)
            line = json.loads(r.stdout.strip().splitlines()[-1])
            print(json.dumps({"variant": name, "tests": t.stdout.strip().splitlines()[-1], "ms_per_step": line["ms_per_step"],
                              "e2e_ms": line["e2e"]["ms_per_step"]}))
        return 0
    raise SystemExit(__doc__)


if __name__ == "__main__":
    sys.exit(main())
