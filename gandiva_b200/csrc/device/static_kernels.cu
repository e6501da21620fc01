// static_kernels.cu — kernels that do not depend on the expression: the synthetic TPC-H
// lineitem column generator used by bench.py / tests (SURVEY.md §8d concretisation) and an
// L2 flush.  Compiled by nvcc to an sm_90a cubin at build time and embedded in
// libgandiva_b200.so; loaded through the driver API.  Including the device library here
// also makes nvcc type-check every function in it (the build-time gate for code that
// NVRTC otherwise only sees at Make()).
#include "gdv_device_lib.cuh"

// Counter-based generator: value = mix(seed, rng column, row).  oracle/lineitem.h restates
// the same arithmetic on the CPU so host- and device-generated columns are identical.
__device__ __forceinline__ u64 gdv_mix64(u64 x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__device__ __forceinline__ u64 gdv_rng(u64 seed, u32 col, i64 row) {
  return gdv_mix64(gdv_mix64(seed ^ ((u64)(col + 1u) * 0xD6E8FEB86659FD93ull)) +
                   (u64)row * 0x9E3779B97F4A7C15ull);
}

// column kinds (rng column in brackets):
//  0 l_shipdate  date32  uniform 1992-01-01 .. 1998-12-01            [0]
//  1 l_discount  f64     {0.00 .. 0.10} step 0.01                    [5]
//  2 l_quantity  f64     {1 .. 50}                                   [2]
//  3 l_quantity  int64   {1 .. 50}                                   [2]
//  4 l_extendedprice decimal128(15,2)  cents in [90000, 10500000)     [4]
//  5 l_discount  decimal128(15,2)  cents {0 .. 10}                    [5]
//  6 l_tax       decimal128(15,2)  cents {0 .. 8}                     [6]
//  7 l_extendedprice f64 = cents / 100.0                             [4]
//  8 l_tax       f64 = cents / 100.0                                 [6]
//  9 int32 uniform in [-2^30, 2^30)                                   [9]
// 10 int32 uniform in [-2^30, 2^30)                                   [10]
// validity: null iff mix(rng ^ NULLSALT) % 1000 < null_permille
extern "C" __global__ void __launch_bounds__(256)
gdv_gen_lineitem(int kind, u64 seed, i64 first_row, i64 num_rows, void* values, u32* validity,
                 int null_permille) {
  const u32 lane = threadIdx.x & 31u;
  const i64 warp = (i64)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const i64 nwarps = (i64)gridDim.x * (blockDim.x >> 5);
  const i64 n_w = (num_rows + 31) / 32;
  for (i64 w = warp; w < n_w; w += nwarps) {
    const i64 i = w * 32 + lane;
    const bool in = i < num_rows;
    const i64 row = first_row + i;
    u32 col;
    switch (kind) {
      case 0: col = 0; break;
      case 1: case 5: col = 5; break;
      case 2: case 3: col = 2; break;
      case 4: case 7: col = 4; break;
      case 6: case 8: col = 6; break;
      default: col = (u32)kind; break;
    }
    const u64 r = gdv_rng(seed, col, row);
    if (in) {
      switch (kind) {
        case 0: reinterpret_cast<i32*>(values)[i] = (i32)(8035 + (i64)(r % 2527ull)); break;
        case 1: reinterpret_cast<f64*>(values)[i] = (f64)(r % 11ull) / 100.0; break;
        case 2: reinterpret_cast<f64*>(values)[i] = (f64)(1ull + r % 50ull); break;
        case 3: reinterpret_cast<i64*>(values)[i] = (i64)(1ull + r % 50ull); break;
        case 4: gdv_st<i128>(values, i, (i128)(90000ull + r % 10410000ull)); break;
        case 5: gdv_st<i128>(values, i, (i128)(r % 11ull)); break;
        case 6: gdv_st<i128>(values, i, (i128)(r % 9ull)); break;
        case 7: reinterpret_cast<f64*>(values)[i] = (f64)(90000ull + r % 10410000ull) / 100.0; break;
        case 8: reinterpret_cast<f64*>(values)[i] = (f64)(r % 9ull) / 100.0; break;
        default:
          reinterpret_cast<i32*>(values)[i] = (i32)((i64)(r % 2147483648ull) - 1073741824ll);
          break;
      }
    }
    if (validity != nullptr) {
      const bool ok = in && (gdv_mix64(r ^ 0xA5A5A5A55A5A5A5Aull) % 1000ull) >= (u64)null_permille;
      const u32 m = __ballot_sync(GDV_FULL, ok);
      if (lane == 0u && w * 32 < num_rows) validity[w] = m;
    }
  }
}

// Writes `words` 32-bit words: used to flush L2 between timed iterations.
extern "C" __global__ void __launch_bounds__(256) gdv_fill_u32(u32* p, i64 words, u32 v) {
  const i64 stride = (i64)gridDim.x * blockDim.x;
  for (i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += stride) p[i] = v;
}

// ---- string-producing projections: exclusive scan of the per-tile byte counts -------------------
// One CTA of 1024 threads walks the tile array in blocks of 1024 (a 1e9-row batch has ~2M tiles of
// 512 rows: a few hundred microseconds next to the two passes over the string bytes).  Writes the
// total to *total and raises GDV_ERR_OFFSET_OVERFLOW when it exceeds `limit` (int32 offsets).
extern "C" __global__ void __launch_bounds__(1024)
gdv_scan_tiles(u64* tiles, i64 n_tiles, u64* total, int* err, u64 limit) {
  __shared__ u64 s_warp[32];
  __shared__ u64 s_carry;
  const u32 lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_carry = 0ull;
  __syncthreads();
  for (i64 b = 0; b < n_tiles; b += 1024) {
    const i64 i = b + (i64)threadIdx.x;
    const u64 v = i < n_tiles ? tiles[i] : 0ull;
    u64 x = v;
    for (int o = 1; o < 32; o <<= 1) {
      const u64 t = __shfl_up_sync(GDV_FULL, x, o);
      if (lane >= (u32)o) x += t;
    }
    if (lane == 31u) s_warp[wid] = x;
    __syncthreads();
    if (wid == 0u) {
      u64 w = s_warp[lane];
      for (int o = 1; o < 32; o <<= 1) {
        const u64 t = __shfl_up_sync(GDV_FULL, w, o);
        if (lane >= (u32)o) w += t;
      }
      s_warp[lane] = w;  // inclusive over warps
    }
    __syncthreads();
    const u64 carry = s_carry;
    const u64 wexcl = wid == 0u ? 0ull : s_warp[wid - 1];
    if (i < n_tiles) tiles[i] = carry + wexcl + x - v;
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = carry + wexcl + x;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    *total = s_carry;
    if (s_carry > limit && err != nullptr) atomicCAS(err, 0, GDV_ERR_OFFSET_OVERFLOW);
  }
}

// ---- SelectionVector reassembly across row-range shards (DESIGN.md "Multi-GPU") ------------
// One process per GPU filters its row range into a LOCAL index run (global row numbers).  This
// kernel, launched on a side stream next to the following batch's filter kernel, moves the run
// into its final position of the root's SelectionVector with plain stores over NVLink (the root
// buffer is peer-mapped through CUDA IPC).  The only thing the ranks exchange besides the runs
// is a "board" of 64-bit words in the root's memory:
//   count[q]  = (seq << 40) | rows selected by rank q in step seq   (published at kernel start)
//   done[q]   = seq once rank q's run has landed in the root buffer
//   consumed  = seq of the last step whose vector the root has released for reuse
// seq increases by one per step, so no word is ever reset and no host round trip is needed:
// rank r's offset is the sum of count[q], q < r, read with acquire loads once they carry seq.
#define GDV_BOARD_SEQ_SHIFT 40
#define GDV_BOARD_COUNT_MASK ((1ull << GDV_BOARD_SEQ_SHIFT) - 1ull)
#ifndef GDV_HOST_EMU
__device__ __forceinline__ u64 gdv_ld_acquire_sys(const u64* p) {
  u64 v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void gdv_st_release_sys(u64* p, u64 v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
#endif

// Moves one index run into peer memory.  16-byte peer stores move more per instruction than 8-byte
// ones, and what limits a FEW CTAs is bytes in flight per thread, so every thread keeps eight 16-byte
// stores in flight (tools/p2p_store_bench.cu measures both on a pair of GPUs).  The CTAs are 256 threads wide because they must
// fit the slots the persistent filter kernel (256-thread CTAs) leaves free (gdv_config_t.sm_reserve).
template <typename T>
__device__ __forceinline__ void gdv_copy_run_scalar(const T* __restrict__ src, T* dst, u64 n) {
  const u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) dst[i] = src[i];
}
// 8-byte elements: the destination (run offset in the root's vector) is only 8-byte aligned, so the
// first element goes alone when needed; after that every store is one aligned 16-byte peer store fed
// by two local 8-byte loads (the source is then off by one element, which local loads do not mind).
__device__ __forceinline__ void gdv_copy_run_u64(const u64* __restrict__ src, u64* dst, u64 n) {
  const u64 tid = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  const u64 stride = (u64)gridDim.x * blockDim.x;
  const u64 head = (((unsigned long long)dst & 15ull) != 0ull && n > 0) ? 1ull : 0ull;
  if (head != 0ull && tid == 0) dst[0] = src[0];
  const u64* s = src + head;
  ulonglong2* d = reinterpret_cast<ulonglong2*>(dst + head);
  const u64 pairs = (n - head) >> 1;
  u64 i = tid;
  for (; i + 7 * stride < pairs; i += 8 * stride) {
    ulonglong2 v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const u64 e = 2 * (i + k * stride);
      v[k].x = __ldcs(s + e);
      v[k].y = __ldcs(s + e + 1);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) d[i + k * stride] = v[k];
  }
  for (; i < pairs; i += stride) {
    ulonglong2 v;
    v.x = s[2 * i];
    v.y = s[2 * i + 1];
    d[i] = v;
  }
  if (((n - head) & 1ull) != 0ull && tid == 0) dst[n - 1] = src[n - 1];
}

// One rank's part of the SelectionVector reassembly on the root (C-ABI gdv_selection_push).
//  base == nullptr: the vector is one run per rank.  The root's filter wrote its run in place at
//                   offset 0; every other rank stores its run behind the lower ranks' runs.
//  base != nullptr: the vector is built from several WAVES (the batch is filtered in slices so that
//                   the transfer of slice j hides under the filter kernel of slice j+1 and only the
//                   last slice's transfer is exposed).  Every rank, the root included, stores the
//                   run of this wave at  *base + runs of the lower ranks in this wave ; the last CTA
//                   of the push then adds the wave's total (all ranks) to *base, a device word owned
//                   by the calling rank.  GDV_WAVE_FIRST starts a vector (*base is taken as 0),
//                   GDV_WAVE_LAST makes the root wait for every rank's stores and write the total.
#define GDV_WAVE_FIRST 1
#define GDV_WAVE_LAST 2
extern "C" __global__ void __launch_bounds__(256)
gdv_sel_push(const void* src, const u64* d_count, void* dst, i64 dst_cap, u64* board_count,
             u64* board_done, u64* board_consumed, u64* board_err, int rank, int world, u64 seq,
             u64 need_consumed, int elem_bytes, u64* local_ctr, u64 done_target, u64* total_out,
             u64* base, int wave_flags) {
  __shared__ u64 s_off, s_cnt, s_base;
  const bool waves = base != nullptr;
  if (threadIdx.x == 0) {
    const u64 cnt = *d_count;
    if (blockIdx.x == 0) gdv_st_release_sys(&board_count[rank], (seq << GDV_BOARD_SEQ_SHIFT) | cnt);
    if (need_consumed != 0ull)
      while (gdv_ld_acquire_sys(board_consumed) < need_consumed) {
      }
    // *base was written by the previous wave's push, a kernel earlier on this stream
    const u64 b0 = (waves && (wave_flags & GDV_WAVE_FIRST) == 0) ? *base : 0ull;
    u64 off = b0;
    for (int q = 0; q < rank; ++q) {
      u64 v;
      do {
        v = gdv_ld_acquire_sys(&board_count[q]);
      } while ((v >> GDV_BOARD_SEQ_SHIFT) != seq);
      off += v & GDV_BOARD_COUNT_MASK;
    }
    s_off = off;
    s_cnt = cnt;
    s_base = b0;
  }
  __syncthreads();
  const u64 off = s_off, cnt = s_cnt;
  if (rank != 0 || waves) {
    if (off + cnt <= (u64)dst_cap) {
      if (elem_bytes == 8)
        gdv_copy_run_u64(reinterpret_cast<const u64*>(src), reinterpret_cast<u64*>(dst) + off, cnt);
      else if (elem_bytes == 4)
        gdv_copy_run_scalar(reinterpret_cast<const u32*>(src), reinterpret_cast<u32*>(dst) + off, cnt);
      else
        gdv_copy_run_scalar(reinterpret_cast<const u16*>(src), reinterpret_cast<u16*>(dst) + off, cnt);
    } else if (threadIdx.x == 0 && blockIdx.x == 0) {
      gdv_st_release_sys(board_err, seq);
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
      const u64 prev = atomicAdd(reinterpret_cast<unsigned long long*>(local_ctr), 1ull);
      if (prev + 1ull == done_target) {  // the last CTA of this push: every store of the rank is out
        if (waves) {
          u64 total = s_base;
          for (int q = 0; q < world; ++q) {
            u64 v;
            do {
              v = gdv_ld_acquire_sys(&board_count[q]);
            } while ((v >> GDV_BOARD_SEQ_SHIFT) != seq);
            total += v & GDV_BOARD_COUNT_MASK;
          }
          *base = total;
          gdv_st_release_sys(&board_done[rank], seq);
          if (rank == 0 && (wave_flags & GDV_WAVE_LAST) != 0) {
            for (int q = 1; q < world; ++q)
              while (gdv_ld_acquire_sys(&board_done[q]) != seq) {
              }
            if (total_out != nullptr) *total_out = total;
          }
        } else {
          gdv_st_release_sys(&board_done[rank], seq);
        }
      }
    }
  } else if (blockIdx.x == 0 && threadIdx.x == 0) {
    // root, one run per rank: its own run was written in place by the filter kernel (offset 0)
    if (cnt > (u64)dst_cap) gdv_st_release_sys(board_err, seq);
    gdv_st_release_sys(&board_done[0], seq);
    u64 total = cnt;
    for (int q = 1; q < world; ++q) {
      while (gdv_ld_acquire_sys(&board_done[q]) != seq) {
      }
      total += gdv_ld_acquire_sys(&board_count[q]) & GDV_BOARD_COUNT_MASK;
    }
    if (total_out != nullptr) *total_out = total;
  }
}

// root: stamps `consumed` once the consumer of step seq's vector is done with it.
extern "C" __global__ void gdv_sel_release(u64* board_consumed, u64 seq) {
  if (threadIdx.x == 0 && blockIdx.x == 0) gdv_st_release_sys(board_consumed, seq);
}
