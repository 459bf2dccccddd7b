// estk_sort.cuh -- stable LSD radix sort of (key, uint32 value) pairs across all CTAs of a
// cooperative grid (sm_90a).  Used by the rank phase of rank_grad_kernel for P > 8192 and by
// the offsets kernel for more than 4096 pairs.
//
// One pass per 8-bit digit, three grid-wide steps each:
//   1. every CTA counts the digits of its contiguous tile of the input   -> hist[digit][cta]
//   2. one warp per digit turns its row of hist into an exclusive scan over the CTAs
//      (and the digit's total)
//   3. every CTA scatters its tile, in input order, to
//        (totals of the smaller digits) + (the same digit in earlier CTAs) + (earlier in this tile)
// The positions are pure functions of the input: no atomic whose order could change the output
// (the shared-memory digit counts of step 1 are commutative sums), so the sort is deterministic.
// Elements with equal keys keep their input order (stable), which is what breaks ties by index
// when the input is in index order and the value is the index.
#pragma once
#include "estk_common.cuh"
#include <cooperative_groups.h>

namespace estk_sort {

constexpr int kDigitBits = 8;
constexpr int kDigits = 1 << kDigitBits;

// Buffers of one sort; all of them live in the context workspace (estk_ctx_reserve).
struct Workspace {
  void* keys[2];       // ping-pong key buffers, [n] Key each
  uint32_t* vals[2];   // ping-pong value buffers, [n]
  uint32_t* hist;      // [kDigits * gridDim.x]: per-CTA digit counts, then their scans
  uint32_t* total;     // [kDigits]: elements per digit
};

// Workspace bytes for n elements with keys of `key_bytes` bytes on a grid of at most `max_grid` CTAs.
inline size_t workspace_bytes(int64_t n, int key_bytes, int max_grid) {
  return (size_t)n * (2 * key_bytes + 2 * sizeof(uint32_t)) + sizeof(uint32_t) * (size_t)kDigits * (max_grid + 1);
}

// The context's sort buffers: up to c->members 4-byte keys, or c->members / 2 8-byte keys.
inline Workspace workspace_of(const estk_ctx* c) {
  unsigned char* b = static_cast<unsigned char*>(c->sort_ws);
  const size_t m = (size_t)c->members;
  Workspace w;
  w.keys[0] = b;
  w.keys[1] = b + 4 * m;
  w.vals[0] = reinterpret_cast<uint32_t*>(b + 8 * m);
  w.vals[1] = reinterpret_cast<uint32_t*>(b + 12 * m);
  w.hist = reinterpret_cast<uint32_t*>(b + 16 * m);
  w.total = w.hist + (size_t)kDigits * c->max_grid;
  return w;
}

// Dynamic shared memory of grid_sort per CTA of T threads: running digit bases, scan scratch, and
// one digit-count row per warp.
__host__ __device__ constexpr size_t smem_bytes(int T) {
  return sizeof(uint32_t) * ((size_t)2 * kDigits + (size_t)(T / 32) * kDigits);
}

#ifdef __CUDACC__
// Sorts n elements of keys[0, key_bits) bits.  Pass 0 reads element i as (load_key(i), i); later
// passes read the previous pass's buffer.  Returns the index b of the buffers holding the result
// (ws.keys[b], ws.vals[b]); every CTA has passed a grid.sync after the last store.  Called by
// every thread of the grid with the same arguments; `smem` is smem_bytes(T) of dynamic shared memory.
template <typename Key, int T, class LoadKey>
__device__ __forceinline__ int grid_sort(cooperative_groups::grid_group& grid, const Workspace& ws, int n,
                                         int key_bits, LoadKey load_key, uint32_t* smem) {
  static_assert(T >= kDigits && T % 32 == 0, "one thread per digit");
  constexpr int kWarps = T / 32;
  uint32_t* run = smem;                    // [kDigits] next output position of each digit (this CTA)
  uint32_t* scan = smem + kDigits;         // [kDigits] digit counts of the tile / scan scratch
  uint32_t* wcnt = smem + 2 * kDigits;     // [kWarps][kDigits] digit counts of one round, per warp
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int G = gridDim.x, cta = blockIdx.x;
  const int tile = (n + G - 1) / G;
  const int b0 = min(n, cta * tile), b1 = min(n, b0 + tile);
  const int passes = key_bits > kDigitBits ? (key_bits + kDigitBits - 1) / kDigitBits : 1;
  for (int pass = 0; pass < passes; ++pass) {
    const int shift = pass * kDigitBits;
    const bool odd = pass & 1;               // (selects, not indexes: the buffer arrays stay in registers)
    const Key* kin = static_cast<const Key*>(odd ? ws.keys[0] : ws.keys[1]);
    const uint32_t* vin = odd ? ws.vals[0] : ws.vals[1];
    Key* kout = static_cast<Key*>(odd ? ws.keys[1] : ws.keys[0]);
    uint32_t* vout = odd ? ws.vals[1] : ws.vals[0];
    auto key_at = [&](int i) -> Key { return pass == 0 ? (Key)load_key(i) : __ldcg(kin + i); };
    auto digit_of = [&](Key k) { return (uint32_t)(k >> shift) & (kDigits - 1); };

    // ---- 1. digit counts of this CTA's tile
    for (int d = tid; d < kDigits; d += T) scan[d] = 0u;
    __syncthreads();
    for (int i = b0 + tid; i < b1; i += T) atomicAdd(&scan[digit_of(key_at(i))], 1u);
    __syncthreads();
    for (int d = tid; d < kDigits; d += T) ws.hist[(size_t)d * G + cta] = scan[d];
    __threadfence();
    grid.sync();

    // ---- 2. exclusive scan of each digit's row over the CTAs, one warp per digit
    {
      const int nwarps = G * kWarps;
      for (int d = cta * kWarps + warp; d < kDigits; d += nwarps) {
        uint32_t* row = ws.hist + (size_t)d * G;
        uint32_t carry = 0;
        for (int c0 = 0; c0 < G; c0 += 32) {
          const uint32_t v = c0 + lane < G ? __ldcg(row + c0 + lane) : 0u;
          uint32_t incl = v;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const uint32_t up = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += up;
          }
          if (c0 + lane < G) row[c0 + lane] = carry + incl - v;
          carry += __shfl_sync(0xffffffffu, incl, 31);
        }
        if (lane == 0) ws.total[d] = carry;
      }
    }
    __threadfence();
    grid.sync();

    // ---- 3. stable scatter.  run[d] = (elements of smaller digits) + (digit d in earlier CTAs)
    for (int d = tid; d < kDigits; d += T) scan[d] = __ldcg(ws.total + d);
    __syncthreads();
    if (warp == 0) {
      constexpr int kPer = kDigits / 32;
      uint32_t v[kPer], s = 0;
#pragma unroll
      for (int e = 0; e < kPer; ++e) { v[e] = scan[lane * kPer + e]; s += v[e]; }
      uint32_t incl = s;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t up = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += up;
      }
      uint32_t base = incl - s;
#pragma unroll
      for (int e = 0; e < kPer; ++e) {
        const int d = lane * kPer + e;
        run[d] = base + __ldcg(ws.hist + (size_t)d * G + cta);
        base += v[e];
      }
    }
    // rounds of T consecutive elements: rank among equal digits = earlier warps of the round
    // (per-warp counts) + earlier lanes of the warp (match mask)
    for (int r0 = b0; r0 < b1; r0 += T) {
      for (int k = tid; k < kWarps * kDigits; k += T) wcnt[k] = 0u;
      __syncthreads();                                   // also: run[] ready, previous round consumed
      const int i = r0 + tid;
      const bool valid = i < b1;
      Key key = 0;
      uint32_t val = 0, d = kDigits;
      if (valid) {
        key = key_at(i);
        val = pass == 0 ? (uint32_t)i : __ldcg(vin + i);
        d = digit_of(key);
      }
      const uint32_t peers = __match_any_sync(0xffffffffu, d);
      const uint32_t below = peers & ((1u << lane) - 1u);
      if (valid && below == 0u) wcnt[warp * kDigits + d] = __popc(peers);
      __syncthreads();
      for (int dd = tid; dd < kDigits; dd += T) {        // exclusive prefix over the warps, in place
        uint32_t s = run[dd];
#pragma unroll
        for (int w = 0; w < kWarps; ++w) {
          const uint32_t c = wcnt[w * kDigits + dd];
          wcnt[w * kDigits + dd] = s;
          s += c;
        }
        run[dd] = s;
      }
      __syncthreads();
      if (valid) {
        const uint32_t pos = wcnt[warp * kDigits + d] + __popc(below);
        kout[pos] = key;
        vout[pos] = val;
      }
      __syncthreads();                                   // wcnt is cleared by the next round
    }
    __threadfence();
    grid.sync();
  }
  return (passes - 1) & 1;
}
#endif

}  // namespace estk_sort
