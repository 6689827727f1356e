"""GPU: svo::streams::addKeyframes / detect / detectFeatures of the C++ host layer (rpg_svo_b200/host/svo_host.h), run by
host_detect_streams_demo against the same objects' own DepthFilter::addKeyframe / FastDetector::detect /
initialization::detectFeatures: the digest of every object's state after the batched run equals the digest after the
per-object run (seed ids and batch ids included), and every refusal throws with the objects unchanged."""
import re
import subprocess

import pytest

from tests.test_host_cpp_gpu import build_demo

pytestmark = pytest.mark.gpu


def test_detect_streams_host_digests_equal():
    out = subprocess.run([build_demo("host_detect_streams_demo")], capture_output=True, text=True, timeout=600)
    print(out.stdout, out.stderr)
    rows = {}
    refusal = None
    for line in out.stdout.splitlines():
        m = re.match(r"(keyframes|detect|init) (per-object|batched)\s+([0-9a-f]{16}) (?:seeds|features) (\d+)$", line)
        if m:
            rows[(m.group(1), m.group(2))] = (m.group(3), int(m.group(4)))
            continue
        m = re.match(r"refusals thrown (\d+) of (\d+) objects (unchanged|changed) seeds-before (\d+) [0-9a-f]{16}$", line)
        assert m, line
        refusal = (int(m.group(1)), int(m.group(2)), m.group(3), int(m.group(4)))
    assert len(rows) == 6
    for stage in ("keyframes", "detect", "init"):
        assert rows[(stage, "batched")] == rows[(stage, "per-object")], stage
        assert rows[(stage, "per-object")][1] > 0, stage
    thrown, n, state, seeds_before = refusal
    assert n == 5 and thrown == n and state == "unchanged" and seeds_before == 0
    assert out.returncode == 0
