#!/usr/bin/env python
"""ThreadSanitizer over the kernels under the CUDA emulator (tests/host_harness/cuda_emu.h): a CPU-side
race check of shared-memory / global hand-overs between the threads of a block (barriers and atomics of
the emulator are visible to TSan).  No GPU needed.

    LD_PRELOAD=$(gcc -print-file-name=libtsan.so) TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0" \\
        python tools/tsan_emulated.py episode_irregular 2>&1 | grep -E "SUMMARY|replayed"

Known report: irbpp_scan_kernel, `any_sh = 1` written by lane 0 of several warps (same value, idempotent).
"""
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import test_kernels_emulated as t  # noqa: E402

lib = t.build_emulated(tempfile.mkdtemp(), defs=sys.argv[2:] + ["-fsanitize=thread", "-g"])
t._replay(lib, sys.argv[1], 3)
print("replayed")
