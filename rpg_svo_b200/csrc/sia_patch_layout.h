// Layout of one patch array set of the full-batch alignment kernel (sia_kernel): the 4x4 reference patch (f32) and its
// gradients (float2) of SA feature slots, 192 bytes per slot.  Plain C++ so that a host compiler can check it.
#pragma once

#include <stdint.h>

#ifdef __CUDACC__
#define SIA_PATCH_HD __host__ __device__
#else
#define SIA_PATCH_HD
#endif

// Byte offset of 16-byte chunk c of slot s in a set of SA slots.  Chunks 0..3: patch row c (4 values); chunks 4..11:
// the gradients (dx, dy of two pixels each), patch row y in chunks 4 + 2y and 5 + 2y.  A thread reads a patch row with
// three 128-bit accesses.  Chunk-major ([12][SA] chunks): the 8 consecutive slots of one quarter-warp phase that access
// the same chunk read 128 contiguous bytes, conflict-free, and every chunk of a slot is at an immediate offset from the
// slot's first one.  (A slot-major record with swizzled chunks is conflict-free too, but costs two integer instructions
// per access to form the address.)
SIA_PATCH_HD constexpr uint32_t sia_patch_chunk(int SA, int s, int c) { return ((uint32_t)c * (uint32_t)SA + (uint32_t)s) * 16u; }
