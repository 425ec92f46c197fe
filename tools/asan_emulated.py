#!/usr/bin/env python
"""AddressSanitizer over the kernels under the CUDA emulator: a CPU-side memcheck of every shared / global
access (dynamic shared memory is a heap block of exactly the launch's size, so a wrong size shows up).

    LD_PRELOAD=$(gcc -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 \\
        python tools/asan_emulated.py 2>&1 | grep -E "ERROR|SUMMARY| ok"
"""
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import test_kernels_emulated as t  # noqa: E402
import test_narrow_spill  # noqa: E402
import test_item_sources  # noqa: E402
import test_scan_warp  # noqa: E402

emu = t.build_emulated(tempfile.mkdtemp(), defs=sys.argv[1:] + ["-fsanitize=address", "-g", "-fno-omit-frame-pointer"])
test_narrow_spill.test_emulated_narrow_shape_list_spill(emu); print("narrow-shape list spill ok")
for k in (1, 5):
    test_item_sources.test_emulated_trajectories_match_oracle_until_idle(emu, k); print("trajectories k=%d ok" % k)
test_item_sources.test_emulated_grouped_stream_matches_mirror(emu); print("grouped draws ok")
test_item_sources.test_emulated_trajectory_end_is_error_5(emu); print("trajectory end ok")
test_item_sources.test_emulated_bad_tables_are_rejected(emu); print("bad tables ok")
t.test_emulated_hull_actions_match_reference_golden(emu); print("hull goldens ok")
t.test_emulated_survey_known_answers(emu); print("known answers ok")
t.test_emulated_many_start_pixels(emu); print("many start pixels ok")
t.test_emulated_heuristics_match_reference_golden(emu); print("heuristics ok")
for tag in ("blockout", "irregular", "cube"):
    t.test_emulated_scan_matches_reference_golden(emu, tag); print("scan", tag, "ok")
for name, steps in (("episode_blockout", 12), ("episode_irregular", 4), ("episode_truncate", 4), ("episode_buffered", 5),
                    ("episode_rot24", 2)):
    t._replay(emu, name, steps); print(name, "ok")
for edge, steps in ((0.08, 14), (0.02, 3)):
    test_scan_warp.test_emulated_warp_scan_episodes_and_invalid_actions(emu, edge, steps); print("warp scan edge", edge, "ok")
