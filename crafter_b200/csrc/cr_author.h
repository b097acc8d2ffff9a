// crafter_b200: cr_author_levels, caller-made worlds into level cache rows (semantics: include/crafter_b200.h,
// cr_author_levels).  Device code only, like cr_kernels.h, so that tests/simt compiles the very same kernels.
//
// One call is four launches on the caller's stream, each behind the one before:
//   k_author_check  one CTA per world: the world's bytes, its entry, and a claim on the entry (a duplicate is
//                   found by the second claim); any rejection sets the scratch's `rejected` word
//   k_author_copy   one CTA per world: nothing when rejected, else the world's bytes into its row's terrain, and
//                   the number of worlds k_wg_obj is to build (0 when rejected: all or nothing)
//   k_wg_obj        the step's own creature pass, on a State whose next_mat / next_ents are the cache rows and
//                   whose next_meta is the scratch (author_state): it strips bits 4-5 off the terrain and writes
//                   the creatures in x-major cell order with the records generation gives them, and n
//   k_author_tag    one thread per world: the row's meta (n, 1 | 4) and last its tag, when accepted; the claims are
//                   released either way
// cr_mutate_levels is k_mutate (below: the children of parent rows into the caller's worlds) and then these four.
#pragma once
#include "cr_kernels.h"

namespace cr {
namespace kernels {

enum AuthorStatus : int {  // cr_author_levels' status bits, per world
  AUTHOR_BYTE = 1,      // a byte out of range: material 0 or above M_FURNACE, or bit 6 or 7 set
  AUTHOR_CREATURE = 2,  // a creature on a cell that is not grass, sand or path
  AUTHOR_START = 4,     // the start cell (W/2, H/2) is not grass, sand or path, or holds a creature
  AUTHOR_SLOTS = 8,     // more than slot_capacity - 2 creatures
  AUTHOR_ENTRY = 16,    // the entry lies outside the table's and the cache's capacity, or appears twice in the call
};
constexpr int32_t CACHE_AUTHORED = 4;  // bit 2 of a cache row's meta[1]: the row holds an authored world

// The library-owned scratch of cr_author_levels (crafter_kernels.cu), one allocation of author_words(cap) int32:
// [0] rejected, [1] worlds k_wg_obj builds, then claim[cap] (the call index that holds each entry, -1: none; all
// -1 between calls), then meta[cap][NM_COUNT] (what k_wg_obj writes for the row of each entry).
constexpr int AUTHOR_THREADS = 256;
__host__ __device__ inline size_t author_words(int cap) { return 2 + (size_t)cap + (size_t)cap * NM_COUNT; }
__host__ __device__ inline int32_t *author_claim(int32_t *scratch) { return scratch + 2; }
__host__ __device__ inline int32_t *author_meta(int32_t *scratch, int cap) { return scratch + 2 + cap; }

// The State k_wg_obj builds the authored rows on: env index = table entry.
__host__ __device__ inline State author_state(const State &st, int32_t *scratch, int cap) {
  State as = st;
  as.next_mat = st.lc_mat;
  as.next_ents = st.lc_ents;
  as.next_meta = author_meta(scratch, cap);
  as.lc_row = nullptr;  // nothing is copied from the cache while it is written
  return as;
}

CR_DEV bool author_walkable(int m) { return (WALKABLE >> m) & 1u; }

// k_author_check: CTA i checks world i.  Every thread folds the bytes it reads into status bits and a creature
// count; ballots and a warp sum gather them, thread 0 adds the slot and entry checks.  `status` is zeroed before.
__global__ void __launch_bounds__(AUTHOR_THREADS)
k_author_check(Geom g, State st, const int32_t *__restrict__ entries, const uint8_t *__restrict__ worlds, int cap,
               int32_t *status, int32_t *scratch) {
  __shared__ unsigned s_bits[AUTHOR_THREADS / 32];
  __shared__ int s_count[AUTHOR_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int i = blockIdx.x;
  const uint8_t *w = worlds + (size_t)i * g.NC;
  const int start = (g.W / 2) * g.H + g.H / 2;
  unsigned bits = 0;
  int count = 0;
  for (int c = tid; c < g.NC; c += AUTHOR_THREADS) {
    const int b = w[c], m = b & 0x0F, creature = (b >> 4) & 3;
    if ((b & 0xC0) || m == M_NONE || m > M_FURNACE) bits |= AUTHOR_BYTE;
    if (creature && !author_walkable(m)) bits |= AUTHOR_CREATURE;
    if (c == start && (creature || !author_walkable(m))) bits |= AUTHOR_START;
    count += creature != 0;
  }
  unsigned warp_bits = 0;
  for (int k = 0; k < 3; ++k)
    if (__ballot_sync(0xffffffffu, (bits >> k) & 1)) warp_bits |= 1u << k;
  int incl = count;  // warp sum (inclusive scan: lane 31 holds it)
  for (int d = 1; d < 32; d <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += v;
  }
  if (lane == 31) { s_bits[warp] = warp_bits; s_count[warp] = incl; }
  __syncthreads();
  if (tid != 0) return;
  unsigned all = 0;
  int creatures = 0;
  for (int k = 0; k < AUTHOR_THREADS / 32; ++k) { all |= s_bits[k]; creatures += s_count[k]; }
  if (creatures > g.CAP - 2) all |= AUTHOR_SLOTS;
  const int32_t e = entries[i];
  if (e < 0 || e >= cap) {
    all |= AUTHOR_ENTRY;
  } else {
    const int32_t held = atomicCAS(author_claim(scratch) + e, -1, i);
    if (held >= 0) {  // the entry appears twice: both worlds carry the bit
      all |= AUTHOR_ENTRY;
      atomicOr(reinterpret_cast<unsigned *>(status + held), (unsigned)AUTHOR_ENTRY);
    }
  }
  if (all) {
    atomicOr(reinterpret_cast<unsigned *>(status + i), all);
    atomicOr(reinterpret_cast<unsigned *>(scratch), 1u);
  }
}

// k_author_copy: CTA i copies world i into its row's terrain, creature bits included (k_wg_obj takes them off),
// unless any world was rejected.  CTA 0 sets the number of worlds k_wg_obj builds.
__global__ void __launch_bounds__(AUTHOR_THREADS)
k_author_copy(Geom g, State st, const int32_t *__restrict__ entries, const uint8_t *__restrict__ worlds, int count,
              int32_t *scratch) {
  const int i = blockIdx.x, tid = threadIdx.x;
  const bool rejected = scratch[0] != 0;
  if (i == 0 && tid == 0) scratch[1] = rejected ? 0 : count;
  if (rejected) return;
  const uint8_t *src = worlds + (size_t)i * g.NC;
  uint8_t *dst = st.lc_mat + (size_t)entries[i] * g.NC;
  if ((g.NC & 7) == 0 && (reinterpret_cast<uintptr_t>(worlds) & 7) == 0) {  // rows stay 8-byte aligned
    const uint64_t *s8 = reinterpret_cast<const uint64_t *>(src);
    uint64_t *d8 = reinterpret_cast<uint64_t *>(dst);
    for (int k = tid; k < g.NC / 8; k += AUTHOR_THREADS) d8[k] = s8[k];
  } else {
    for (int c = tid; c < g.NC; c += AUTHOR_THREADS) dst[c] = src[c];
  }
}

// cr_mutate_levels (include/crafter_b200.h): k_mutate writes the children into the caller's `worlds` in front of
// the four launches above, which install them.  Its status bit comes beside AuthorStatus'.
constexpr int MUTATE_PARENT = 32;  // the parent lies outside the capacity, or its row's tag is not seeds[parent]
constexpr int MUTATE_OPS = 16;     // 0..11 set material o + 1, 12..14 place a cow / zombie / skeleton, 15 remove
constexpr int MUTATE_CHUNK = AUTHOR_THREADS;  // edits drawn per round, one per thread
struct MutateOps {
  uint32_t cum[MUTATE_OPS];  // inclusive cumulative weights; cum[MUTATE_OPS - 1] is the total
};

// k_mutate: CTA i makes child i.  Thread 0 checks the parent row; the CTA copies its terrain (bits 0-3) into the
// child's bytes and scatters the creatures of slots [2, n) into bits 4-5, counting them with a block sum.  Then, by
// rounds of MUTATE_CHUNK edits, every thread draws one edit (cell and op) into shared memory and thread 0 applies
// the round in order: edits are sequential by definition (one may undo, or make room for, the next).  A rejected
// parent leaves a grass world behind, so its child's status names only the reasons that apply to it.  Parents are
// only read: nothing writes a row before the launches behind this one.
__global__ void __launch_bounds__(AUTHOR_THREADS)
k_mutate(Geom g, State st, const int32_t *__restrict__ parents, const int32_t *__restrict__ children, int edits,
         MutateOps ops, uint32_t key, int cap, uint8_t *__restrict__ worlds, int32_t *status, int32_t *scratch) {
  __shared__ int s_ok, s_creatures;
  __shared__ uint32_t s_cell[MUTATE_CHUNK];
  __shared__ uint8_t s_op[MUTATE_CHUNK];
  const int tid = threadIdx.x, i = blockIdx.x;
  const int32_t p = parents[i];
  if (tid == 0) {
    const bool ok = p >= 0 && p < cap && st.lc_tag[p] == st.lt_seeds[p];
    if (!ok) {
      status[i] = MUTATE_PARENT;  // (zeroed before; this CTA is its only writer so far)
      atomicOr(reinterpret_cast<unsigned *>(scratch), 1u);
    }
    s_ok = ok;
    s_creatures = 0;
  }
  __syncthreads();
  uint8_t *w = worlds + (size_t)i * g.NC;
  const bool wide = (g.NC & 7) == 0 && (reinterpret_cast<uintptr_t>(worlds) & 7) == 0;  // rows stay 8-byte aligned
  if (!s_ok) {
    for (int c = tid; c < g.NC; c += AUTHOR_THREADS) w[c] = M_GRASS;
    return;
  }
  const uint8_t *src = st.lc_mat + (size_t)p * g.NC;
  if (wide) {
    const uint64_t *s8 = reinterpret_cast<const uint64_t *>(src);
    uint64_t *d8 = reinterpret_cast<uint64_t *>(w);
    for (int k = tid; k < g.NC / 8; k += AUTHOR_THREADS) d8[k] = s8[k] & 0x0F0F0F0F0F0F0F0FULL;
  } else {
    for (int c = tid; c < g.NC; c += AUTHOR_THREADS) w[c] = src[c] & 0x0F;
  }
  __syncthreads();
  const int n = st.lc_meta[(size_t)p * 2];
  const Ent *ents = st.lc_ents + (size_t)p * g.CAP;
  int count = 0;
  for (int s = 2 + tid; s < n; s += AUTHOR_THREADS) {
    const Ent e = ents[s];
    if (e.type >= T_COW && e.type <= T_SKELETON) {
      w[e.x * g.H + e.y] |= (uint8_t)((e.type - 1) << 4);
      ++count;
    }
  }
  if (count) atomicAdd(&s_creatures, count);
  __syncthreads();  // the child's bytes and the count are complete, and visible to thread 0
  int creatures = s_creatures;
  const int start = (g.W / 2) * g.H + g.H / 2;
  const uint32_t child = (uint32_t)children[i];
  for (int base = 0; base < edits; base += MUTATE_CHUNK) {
    const int j = base + tid;
    if (j < edits) {
      Rng r = rng_ctx(key, D_MUTATE, child);
      r.k = 2u * (uint32_t)j;
      const uint32_t c = rng_randint(r, (uint32_t)g.NC - 1u);
      const uint32_t t = rng_randint(r, ops.cum[MUTATE_OPS - 1]);
      int o = 0;  // the first o with t < cum[o]: the number of cum[k] <= t (cum is non-decreasing, t < total)
#pragma unroll
      for (int k = 0; k < MUTATE_OPS - 1; ++k) o += ops.cum[k] <= t;
      s_cell[tid] = c + (c >= (uint32_t)start);
      s_op[tid] = (uint8_t)o;
    }
    __syncthreads();
    if (tid == 0) {
      const int m = edits - base < MUTATE_CHUNK ? edits - base : MUTATE_CHUNK;
      for (int k = 0; k < m; ++k) {
        const int cell = (int)s_cell[k], o = s_op[k];
        const int b = w[cell], mat = b & 0x0F, cre = b >> 4;
        if (o < 12) {  // a material; a creature stays only on grass, sand or path
          const bool keep = cre && author_walkable(o + 1);
          creatures -= cre && !keep;
          w[cell] = (uint8_t)((o + 1) | (keep ? cre << 4 : 0));
        } else if (o < 15) {  // a creature of kind o - 11, on a walkable cell, within the slots
          if (author_walkable(mat) && (cre || creatures < g.CAP - 2)) {
            creatures += !cre;
            w[cell] = (uint8_t)(mat | (o - 11) << 4);
          }
        } else if (cre) {  // remove the creature
          --creatures;
          w[cell] = (uint8_t)mat;
        }
      }
    }
    __syncthreads();  // the round's draws are applied before the next round overwrites them
  }
}

// k_author_tag: behind k_wg_obj, thread i writes the meta and last the tag of world i's row, when no world was
// rejected; it releases the entry's claim either way.
// `cap`: the entries' bound, as k_author_check had it; `scratch_cap`: the scratch's (author_meta).
__global__ void k_author_tag(State st, const int32_t *__restrict__ entries, int count, int cap, int32_t *scratch,
                             int scratch_cap) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const int32_t e = entries[i];
  if (e < 0 || e >= cap) return;
  if (scratch[0] == 0) {
    const int32_t *nm = author_meta(scratch, scratch_cap) + (size_t)e * NM_COUNT;
    st.lc_meta[(size_t)e * 2] = nm[NM_NSLOTS];
    st.lc_meta[(size_t)e * 2 + 1] = nm[NM_VALID] | CACHE_AUTHORED;
    st.lc_tag[e] = st.lt_seeds[e];
  }
  author_claim(scratch)[e] = -1;
}

}  // namespace kernels
}  // namespace cr
