"""CPU: the layout of the full-batch alignment kernel's patch arrays (rpg_svo_b200/csrc/sia_patch_layout.h), compiled with
the host compiler.  For every slot count a sia_kernel instantiation allocates, every (slot, chunk) has its own 16-byte
position inside the set's 192 bytes per slot, and the 8 slots of a quarter-warp phase of a 128-bit shared-memory access
to one chunk fall into 8 distinct 16-byte bank groups (conflict-free)."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHUNKS = 12  # 4 value rows + 8 gradient chunks per slot
# kSiaThroughputSlots and MAXT * FPT of the other instantiations
SLOT_COUNTS = (96, 192, 304, 320, 384, 512, 1024)

PROGRAM = r"""
#include <cstdio>
#include <cstdlib>
#include "sia_patch_layout.h"
int main(int argc, char** argv) {
  const int SA = std::atoi(argv[1]);
  for (int s = 0; s < SA; ++s)
    for (int c = 0; c < %d; ++c) std::printf("%%u\n", sia_patch_chunk(SA, s, c));
  return 0;
}
""" % CHUNKS


@pytest.fixture(scope="module")
def layout_exe(tmp_path_factory):
    d = tmp_path_factory.mktemp("sia_patch_layout")
    src, exe = d / "layout.cpp", d / "layout"
    src.write_text(PROGRAM)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "rpg_svo_b200", "csrc"),
                           "-o", str(exe), str(src)])
    return str(exe)


def _offsets(exe, sa):
    out = subprocess.run([exe, str(sa)], check=True, capture_output=True, text=True).stdout
    return np.array(out.split(), dtype=np.int64).reshape(sa, CHUNKS)


@pytest.mark.parametrize("sa", SLOT_COUNTS)
def test_every_chunk_has_its_own_16_byte_position_in_the_set(layout_exe, sa):
    off = _offsets(layout_exe, sa)
    assert (off % 16 == 0).all()
    assert off.min() >= 0 and off.max() + 16 <= 192 * sa
    assert len(np.unique(off)) == off.size


@pytest.mark.parametrize("sa", SLOT_COUNTS)
def test_a_quarter_warp_phase_reading_one_chunk_is_conflict_free(layout_exe, sa):
    off = _offsets(layout_exe, sa)
    assert sa % 8 == 0  # the slots of a warp's lanes start at a multiple of 32
    groups = (off // 16) % 8  # 32 banks of 4 bytes = 8 groups of 16 bytes
    for s0 in range(0, sa, 8):
        for c in range(CHUNKS):
            assert len(set(groups[s0:s0 + 8, c].tolist())) == 8, (s0, c)
