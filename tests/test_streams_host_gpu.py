"""GPU: svo::streams::updateSeeds / reprojectMap of the C++ host layer (rpg_svo_b200/host/svo_host.h), run by
host_streams_demo against the same objects' own DepthFilter::updateSeeds / Reprojector::reprojectMap: the digest of every
object's state after the batched run equals the digest after the per-object run."""
import re
import subprocess

import pytest

from tests.test_host_cpp_gpu import build_demo

pytestmark = pytest.mark.gpu


def test_streams_host_digests_equal():
    out = subprocess.run([build_demo("host_streams_demo")], capture_output=True, text=True, timeout=600)
    print(out.stdout, out.stderr)
    rows = {}
    for line in out.stdout.splitlines():
        m = re.match(r"(depth|reproject) (per-object|batched)\s+([0-9a-f]{16}) \w+ (\d+) [\w ]+? (\d+)$", line)
        assert m, line
        rows[(m.group(1), m.group(2))] = (m.group(3), int(m.group(4)), int(m.group(5)))
    assert len(rows) == 4
    for stage in ("depth", "reproject"):
        assert rows[(stage, "batched")] == rows[(stage, "per-object")], stage
    _, seeds, candidates = rows[("depth", "per-object")]
    assert seeds > 0 and candidates > 0            # seeds were kept and others converged into candidates
    _, matches, new = rows[("reproject", "per-object")]
    assert matches > 0 and new > 0
    assert out.returncode == 0
