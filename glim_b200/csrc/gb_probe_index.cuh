// gb_probe_index.cuh -- the probe index of a built voxel map: a second, read-only lookup structure beside the bucket table that
// k_vgicp_sweep3 probes instead of the buckets (gb_sweep_steps.cuh).  It answers every coordinate exactly as gb_lookup does,
// in one dependent 16-byte gather for all but a few lookups, where the bucket table's clustered XOR-of-primes hash and linear
// probing need two or more (DESIGN.md 4.1).  Like gb_vgicp_math.cuh this text also compiles for the host:
// tests/cpp/probe_index_host.cpp builds and probes the index with it on the CPU (tests/test_probe_index_host.py,
// scripts/probe_stats.py --index).
//
// Layout (built by k_table_clear / k_table_insert / k_table_finalize, gb_kernels_voxelmap.cu):
//   entry (8 B)   voxel index (21 bits) << 43 | key (42 bits) << 1 | overflow (1 bit); key = dx | dy << 14 | dz << 28, the voxel's
//                 coordinates less the box minimum (14 bits per axis).  Empty: every bit but the overflow bit (kPiEmpty).
//   set (16 B)    two entries, one LDG.128.  The home set of a coordinate is pi_home & set_mask.
//   slot order    linear probing over the entries (set s entry 0, set s entry 1, set s + 1 entry 0, ...), filled as a
//                 sequential insertion in ascending voxel index would fill it (k_table_insert's rule): deterministic.
//   overflow      the bit of a set's entry 0: some key homed at that set lives in a later set.  A lookup leaves its home set
//                 only when the key is absent and the bit is set, and then walks on while the sets it reads are full.
//   box           the voxels' coordinate box {min, max - min}; a coordinate outside it is a miss without a gather.  A map
//                 gets an index only when every extent fits 14 bits (<= kPiMaxExtent) and it has fewer than 2^21 voxels.
#pragma once
#include "gb_vgicp_math.cuh"  // GB_HD, int4 / float4 on the host

#ifdef __CUDACC__
#define PI_LDG(p) __ldg(p)
#define PI_HHD __host__ __device__ __forceinline__
#else
struct uint4 { unsigned x, y, z, w; };
#define PI_LDG(p) (*(p))
#define PI_HHD static inline
#endif

constexpr int kPiAxisBits = 14;
// max - min per axis: the key of every in-box coordinate then differs from the empty entry's all-ones key
constexpr unsigned kPiMaxExtent = (1u << kPiAxisBits) - 2u;
constexpr int kPiVoxelBits = 21;
constexpr unsigned long long kPiEmpty = ~1ull;
// sets = buckets >> kPiSetShift: 8 bytes of index per bucket, half the bucket table (DESIGN.md 4.1 has the statistics)
constexpr int kPiSetShift = 1;

// the voxel coordinate box of a map: min and max - min per axis
struct PiBox {
  int x, y, z;
  unsigned ex, ey, ez;
};

// The box of V voxels from their reduced coordinates mm = {min x y z, max x y z}, and whether the index can pack them: fewer
// than 2^21 voxels and every extent <= kPiMaxExtent.  A map without voxels gets the box {0, 0, 0} of extent 0.
PI_HHD bool pi_box(const int* mm, int V, PiBox& B) {
  B = PiBox{0, 0, 0, 0u, 0u, 0u};
  if (V <= 0) return true;
  if (V >= (1 << kPiVoxelBits)) return false;
  const long long ex = (long long)mm[3] - mm[0], ey = (long long)mm[4] - mm[1], ez = (long long)mm[5] - mm[2];
  if (ex < 0 || ey < 0 || ez < 0 || ex > kPiMaxExtent || ey > kPiMaxExtent || ez > kPiMaxExtent) return false;
  B = PiBox{mm[0], mm[1], mm[2], (unsigned)ex, (unsigned)ey, (unsigned)ez};
  return true;
}

// The home hash: a sum of odd multiples of the coordinates and a 32-bit finalizer.  gb_hash (the XOR of three prime multiples)
// is not used: its clustering survives a finalizer (scripts/probe_stats.py --index: 2-6x the overflow walks, DESIGN.md 4.1).
GB_HD uint32_t pi_home(int x, int y, int z) {
  uint32_t h = (uint32_t)x * 0x9E3779B1u + (uint32_t)y * 0x85EBCA77u + (uint32_t)z * 0xC2B2AE3Du;
  h ^= h >> 16; h *= 0x85ebca6bu;
  h ^= h >> 13; h *= 0xc2b2ae35u;
  return h ^ (h >> 16);
}

// the bits of key << 1 as two words (lo: entry bits 0-31, hi: entry bits 32-42) and whether (x, y, z) lies in the box
GB_HD bool pi_key(const PiBox& B, int x, int y, int z, uint32_t& lo, uint32_t& hi) {
  const uint32_t dx = (uint32_t)x - (uint32_t)B.x, dy = (uint32_t)y - (uint32_t)B.y, dz = (uint32_t)z - (uint32_t)B.z;
  lo = (dx << 1) | (dy << 15) | (dz << 29);
  hi = dz >> 3;
  return dx <= B.ex && dy <= B.ey && dz <= B.ez;
}

// the voxel of entry (elo, ehi) when it holds key (lo, hi), else -1.  An empty entry matches no in-box key.
GB_HD int pi_match(uint32_t elo, uint32_t ehi, uint32_t lo, uint32_t hi) {
  return ((elo ^ lo) >> 1) == 0u && ((ehi ^ hi) & 0x7ffu) == 0u ? (int)(ehi >> 11) : -1;
}

// a set's two entries against a key
GB_HD int pi_match_set(const uint4 e, uint32_t lo, uint32_t hi) {
  const int v = pi_match(e.x, e.y, lo, hi);
  return v >= 0 ? v : pi_match(e.z, e.w, lo, hi);
}

// the overflow walk of a key absent from its home set s whose overflow bit is set: the sets after s, while they are full
GB_HD int pi_walk(const uint4* __restrict__ sets, uint32_t set_mask, uint32_t s, uint32_t lo, uint32_t hi) {
  for (uint32_t k = 0; k < set_mask; k++) {
    s = (s + 1u) & set_mask;
    const uint4 e = PI_LDG(&sets[s]);
    const int v = pi_match_set(e, lo, hi);
    if (v >= 0) return v;
    if (e.z == (uint32_t)kPiEmpty && e.w == (uint32_t)(kPiEmpty >> 32)) return -1;  // entry 1 empty: the run ends here
  }
  return -1;
}

// the whole lookup, as gb_lookup answers it: the voxel index of (x, y, z), -1 if absent.  rounds (optional): the dependent
// set gathers it took (0: outside the box).
GB_HD int pi_lookup(const uint4* __restrict__ sets, uint32_t set_mask, const PiBox& B, int x, int y, int z, int* rounds = nullptr) {
  uint32_t lo, hi;
  if (rounds) *rounds = 0;
  if (!pi_key(B, x, y, z, lo, hi)) return -1;
  const uint32_t s = pi_home(x, y, z) & set_mask;
  const uint4 e = PI_LDG(&sets[s]);
  if (rounds) *rounds = 1;
  const int v = pi_match_set(e, lo, hi);
  if (v >= 0 || !(e.x & 1u)) return v;
  if (rounds) {  // count the walk's gathers
    uint32_t t = s;
    for (uint32_t k = 0; k < set_mask; k++) {
      t = (t + 1u) & set_mask;
      ++*rounds;
      const uint4 f = PI_LDG(&sets[t]);
      if (pi_match_set(f, lo, hi) >= 0 || (f.z == (uint32_t)kPiEmpty && f.w == (uint32_t)(kPiEmpty >> 32))) break;
    }
  }
  return pi_walk(sets, set_mask, s, lo, hi);
}

// Inserts voxel v at (x, y, z) (in the box) into the entries (2 (set_mask + 1) of them).  cas(slot, expected, desired) returns the
// slot's previous value and stores desired when it equalled expected; mark(slot) sets the slot's overflow bit.  An entry takes
// a slot that is empty or holds a larger voxel index, and carries the entry it displaced onward, keeping the slot's overflow
// bit; so concurrent inserts (atomicCAS, atomicOr) reach the table a sequential insertion in ascending voxel index builds.
template <class Cas, class Mark>
GB_HD void pi_insert(const PiBox& B, uint32_t set_mask, int v, int x, int y, int z, Cas&& cas, Mark&& mark) {
  uint32_t lo, hi;
  pi_key(B, x, y, z, lo, hi);
  unsigned long long w = ((unsigned long long)(uint32_t)v << 43) | ((unsigned long long)hi << 32) | lo;
  uint32_t home = pi_home(x, y, z) & set_mask;
  const uint32_t slot_mask = 2u * set_mask + 1u;
  uint32_t slot = 2u * home;
  for (;;) {
    unsigned long long prev = cas(slot, kPiEmpty, w);
    bool placed = prev == kPiEmpty, carry = false;
    while (!placed && (prev & ~1ull) > w) {  // a larger voxel index: take its slot, keep the slot's overflow bit
      const unsigned long long got = cas(slot, prev, w | (prev & 1ull));
      if (got == prev) placed = carry = true;
      else prev = got;
    }
    if (placed) {
      if ((slot >> 1) != home) mark(2u * home);
      if (!carry) return;
      w = prev & ~1ull;  // the displaced entry moves on: recover its coordinates for its home set
      const uint32_t ek = (uint32_t)(w >> 1);  // key bits 0-31
      const uint32_t dz = (uint32_t)(w >> 29) & ((1u << kPiAxisBits) - 1u);
      home = pi_home(B.x + (int)(ek & 0x3fffu), B.y + (int)((ek >> 14) & 0x3fffu), B.z + (int)dz) & set_mask;
    }
    slot = (slot + 1u) & slot_mask;
  }
}
