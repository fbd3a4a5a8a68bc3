"""CPU tier: the retained batcher (gm_retain_batcher_create / gm_retain_batcher_probe, rmqtt_b200/csrc/retain_batcher.cpp over
batcher.cpp's queue and dispatchers) against a stubbed gm_retain_match_batch, under ThreadSanitizer and under AddressSanitizer +
UBSan: every cookie answered exactly once with its own filter's handles from several producers and batcher settings, the
per-filter invalid status, the capacity retry, a failing batch, destroy with queued work, gm_submit_publish refused, and the
PUBLISH engine call never reached."""
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "rmqtt_b200" / "csrc"


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
@pytest.mark.parametrize("san", ["address,undefined", "thread"])
def test_retained_batcher_under_sanitizers(tmp_path, san):
    exe = tmp_path / ("retain_batcher_" + san.split(",")[0])
    flags = [f"-fsanitize={san}"] + (["-fno-sanitize-recover=undefined"] if "undefined" in san else [])
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-pthread", *flags, "-fno-omit-frame-pointer", "-o", str(exe),
           str(ROOT / "tests" / "native" / "retain_batcher_stress.cpp"), str(CSRC / "batcher.cpp"), str(CSRC / "retain_batcher.cpp")]
    build = subprocess.run(cmd, capture_output=True, text=True)
    if build.returncode != 0 and "sanitize" in build.stderr and "cannot find" in build.stderr:
        pytest.skip("sanitizer runtime not installed")
    assert build.returncode == 0, build.stderr[-2000:]
    env = {"PATH": "/usr/bin:/bin", "ASAN_OPTIONS": "detect_leaks=1", "TSAN_OPTIONS": "halt_on_error=1"}
    run = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600, env=env)
    assert run.returncode == 0, (run.stdout[-2000:], run.stderr[-3000:])
    assert run.stdout.count("-> ok:") == 7 and "FAILED" not in run.stdout and "WARNING: ThreadSanitizer" not in run.stderr
