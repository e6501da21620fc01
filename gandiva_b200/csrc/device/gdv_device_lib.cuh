// gdv_device_lib.cuh — device-side function library of the H100 expression engine.
//
// Replaces the reference's precompiled-bitcode function library (BASELINE.json
// north_star: "a device-side function library that replaces the precompiled-bitcode
// function_registry").  This header is prepended to every kernel the fuser emits and
// compiled by NVRTC for sm_90a at Projector/Filter::Make(); every function is
// __forceinline__ so the per-row body becomes straight-line SASS.  It is also compiled
// by nvcc in __graft_entry__.build() (static_kernels.cu includes it) as a syntax gate.
//
// Naming follows the reference library: <base>_<param suffix>..., e.g. add_int32_int32.
// Semantics decisions (the reference has no source in the mount, SURVEY.md §8c) are
// listed in DESIGN.md §"Semantics table"; oracle/gdv_oracle.cc restates each in scalar C++.
#pragma once

typedef signed char i8;
typedef short i16;
typedef int i32;
typedef long long i64;
typedef unsigned char u8;
typedef unsigned short u16;
typedef unsigned int u32;
typedef unsigned long long u64;
typedef float f32;
typedef double f64;
typedef __int128 i128;
typedef unsigned __int128 u128;

#define GDV_FULL 0xffffffffu
#define GDV_DEV __device__ __forceinline__
// big, rarely hot helpers (digests, parsers, decimal rounding): one copy per kernel instead of one
// per call site keeps Make() latency (ptxas time) in check
#define GDV_DEV_BIG __device__ __noinline__

// ---- error reporting (ExecutionError, P/include/arrow/status.h:100) -----------------
#define GDV_ERR_NONE 0
#define GDV_ERR_DIV_ZERO 1
#define GDV_ERR_OFFSET_OVERFLOW 2  /* a utf8/binary output needs more than 2^31 - 1 bytes */
#define GDV_ERR_VAR_CAPACITY 3     /* the caller's var_data buffer is too small */
#define GDV_ERR_CAST_INT 4         /* castINT / castBIGINT of a string that is not an integer */
#define GDV_ERR_CAST_DATE 5        /* castDATE / castTIMESTAMP of a string that is not a date / timestamp */
#define GDV_ERR_SPLIT_INDEX 6      /* split_part with an index < 1 */
#define GDV_ERR_CAST_DECIMAL 7     /* castDECIMAL of a string that is not a decimal number */
#define GDV_ERR_CAST_FLOAT 8       /* castFLOAT4 / castFLOAT8 of a string that is not a number */
#define GDV_ERR_CAST_BOOL 9        /* castBIT / castBOOLEAN of a string that is not true / false / 1 / 0 */
#define GDV_ERR_NEG_LENGTH 10      /* castVARCHAR(x, n) with n < 0 */
#define GDV_ERR_LOCATE_START 11    /* locate(sub, s, start) with start < 1 */
#define GDV_ERR_FACTORIAL_NEG 12   /* factorial of a negative number */
#define GDV_ERR_FACTORIAL_BIG 13   /* factorial of a number above 20 (does not fit int64) */
#define GDV_ERR_TO_DATE 14         /* to_date: the text does not match the format (and errors are not suppressed) */
struct gdv_ctx {
  int* err;
};
GDV_DEV void gdv_set_error(gdv_ctx* c, int code) {
  if (c->err != nullptr) atomicCAS(c->err, 0, code);
}
// Argument checks of castVARCHAR(x, n) and locate(sub, s, start): the reference raises on a negative
// length / a start position below 1.  Called only on rows where every argument is valid.
GDV_DEV long long gdv_check_len(gdv_ctx* c, long long n) {
  if (n < 0) {
    gdv_set_error(c, GDV_ERR_NEG_LENGTH);
    return 0;
  }
  return n;
}
GDV_DEV int gdv_check_start(gdv_ctx* c, int start) {
  if (start < 1) {
    gdv_set_error(c, GDV_ERR_LOCATE_START);
    return 1;
  }
  return start;
}

// ---- strings: a view on Arrow bytes plus a lazy ASCII case map ------------------------
// upper()/lower()/substr()/trim() never materialise: they return a view, and consumers read
// bytes through gdv_ch().  xf bits 0-1: 0 = as stored, 1 = upper-cased, 2 = lower-cased,
// 3 = initcap (a letter is upper-cased at the start of the view or after a byte that is not part of a
// word, lower-cased inside a word; the fuser never narrows a view from the left after initcap);
// GDV_XF_ASCII: every stored byte of the row is known to be < 0x80 (set by the cooperative
// scan of the staged bytes), so glyph positions are byte positions.
#define GDV_XF_CASE 3u
#define GDV_XF_ASCII 0x100u
#define GDV_XF_LOCAL 0x200u  /* bytes live in the producing thread's scratch slot: only that thread may read them */
#define GDV_XF_REP 0x400u    /* periodic: byte i is p[i % (xf >> 12)]; only the string write pass reads these */
#define GDV_XF_REPL 0x4u     /* replace(): the view is the SOURCE text, (xf >> 12) & 0xff the call site whose
                                literals gdv_repl_len / gdv_repl_copy (generated per kernel) apply */
#define GDV_XF_REV 0x800u    /* glyph-reversed: copied by the owning lane in the string write pass */
#define GDV_SCRATCH_SLOT 64  /* bytes per (row, call site) of a function that writes its result as text */
struct gdv_str {
  const u8* p;
  i32 len;
  u32 xf;
};
// Part of a word for initcap: ASCII letters and digits, and every byte of a multi-byte glyph (the case
// maps are ASCII-only, DESIGN.md §5: a non-ASCII letter continues a word but is never re-cased itself).
GDV_DEV bool gdv_is_word_byte(u8 c) {
  return (u32)((c | 0x20u) - (u32)'a') <= 25u || (u32)(c - (u32)'0') <= 9u || c >= 0x80u;
}
GDV_DEV u8 gdv_ch(const gdv_str& s, i32 i) {
  u8 c = s.p[i];
  const u32 cm = s.xf & GDV_XF_CASE;
  if (cm == 1u) {
    if (c >= (u8)'a' && c <= (u8)'z') c = (u8)(c - 32);
  } else if (cm == 2u) {
    if (c >= (u8)'A' && c <= (u8)'Z') c = (u8)(c + 32);
  } else if (cm == 3u) {
    const u32 low = (u32)c | 0x20u;
    if (low - (u32)'a' <= 25u) c = (i > 0 && gdv_is_word_byte(s.p[i - 1])) ? (u8)low : (u8)(low - 32u);
  }
  return c;
}
// gdv_ch(s, i) == lit for an immediate `lit`: under a case map the comparison is folded into
// the constant instead of transforming the text byte (2 instructions instead of 4).
GDV_DEV bool gdv_ch_eq(const gdv_str& s, i32 i, u32 lit) {
  const u32 c = s.p[i];
  const u32 cm = s.xf & GDV_XF_CASE;
  if (cm == 3u) return (u32)gdv_ch(s, i) == lit;
  if (cm == 1u) {
    if (lit >= (u32)'a' && lit <= (u32)'z') return false;  // upper-cased text has no a-z
    if (lit >= (u32)'A' && lit <= (u32)'Z') return (c | 0x20u) == (lit | 0x20u);
  } else if (cm == 2u) {
    if (lit >= (u32)'A' && lit <= (u32)'Z') return false;
    if (lit >= (u32)'a' && lit <= (u32)'z') return (c | 0x20u) == lit;
  }
  return c == lit;
}
// True when the first n bytes at p are all ASCII (< 0x80).
GDV_DEV bool gdv_all_ascii(const u8* p, i32 n) {
  i32 i = 0;
  u32 acc = 0u;
  while (i < n && ((unsigned long long)(p + i) & 3ull) != 0ull) acc |= p[i++];
  while (i + 4 <= n) {
    acc |= *reinterpret_cast<const u32*>(p + i);
    i += 4;
  }
  while (i < n) acc |= p[i++];
  return (acc & 0x80808080u) == 0u;
}
GDV_DEV gdv_str gdv_make_str(const u8* p, i32 len) {
  gdv_str s;
  s.p = p;
  s.len = len;
  s.xf = 0u;
  return s;
}
// Length in bytes of the UTF-8 glyph that starts with byte c (malformed lead bytes count 1).
GDV_DEV i32 gdv_glyph_len(u8 c) {
  if (c < 0x80u) return 1;
  if ((c & 0xE0u) == 0xC0u) return 2;
  if ((c & 0xF0u) == 0xE0u) return 3;
  if ((c & 0xF8u) == 0xF0u) return 4;
  return 1;
}

// ---- streaming loads / stores ----------------------------------------------------------
// Inputs are read once and outputs written once: evict-first policy on both sides.
template <typename T>
GDV_DEV void gdv_st(void* base, i64 i, T v) {
  __stcs(reinterpret_cast<T*>(base) + i, v);
}
template <>
GDV_DEV void gdv_st<i128>(void* base, i64 i, i128 v) {
  longlong2 w;
  w.x = (i64)(u64)(u128)v;
  w.y = (i64)(u64)((u128)v >> 64);
  __stcs(reinterpret_cast<longlong2*>(base) + i, w);
}
template <>
GDV_DEV void gdv_st<i8>(void* base, i64 i, i8 v) {
  __stcs(reinterpret_cast<signed char*>(base) + i, (signed char)v);
}
// Pointer-based streaming load / store used by the fast path (one pointer per column, steps at
// immediate offsets).
template <typename T>
GDV_DEV T gdv_ldp(const T* p) {
  return __ldcs(p);
}
template <>
GDV_DEV i128 gdv_ldp<i128>(const i128* p) {
  const longlong2 v = __ldcs(reinterpret_cast<const longlong2*>(p));
  return (i128)(((u128)(u64)v.y << 64) | (u128)(u64)v.x);
}
template <typename T>
GDV_DEV void gdv_stp(T* p, T v) {
  __stcs(p, v);
}
template <>
GDV_DEV void gdv_stp<i128>(i128* p, i128 v) {
  longlong2 w;
  w.x = (i64)(u64)(u128)v;
  w.y = (i64)(u64)((u128)v >> 64);
  __stcs(reinterpret_cast<longlong2*>(p), w);
}
// What a column without a validity bitmap reads on the branch-free fast path (index 0, and
// index 1 when the column's bit shift is not 0).
__device__ const u32 gdv_all_ones[2] = {0xffffffffu, 0xffffffffu};
// 32 bitmap bits starting at bit (32 * widx + sh), sh in [0, 31], from a 4-byte aligned word
// pointer.  Warp-uniform address: one broadcast transaction for the 32 rows of a step.
GDV_DEV u32 gdv_ldwin(const u32* p, i64 widx, u32 sh) {
  const u32 lo = __ldg(p + widx);
  u32 hi = 0u;
  if (sh != 0u) hi = __ldg(p + widx + 1);  // a predicated load: the word after the last one is never touched
  return __funnelshift_r(lo, hi, sh);      // sh == 0 yields lo
}
// Bit `i` (LSB-first, Arrow validity layout, P/include/arrow/util/bit_util.h:158) of a
// bitmap that starts `sh` bits into byte *p.  p == nullptr means "all set".
GDV_DEV bool gdv_ldbit(const u8* p, u32 sh, i64 i) {
  if (p == nullptr) return true;
  const i64 b = i + (i64)sh;
  return ((p[b >> 3] >> (u32)(b & 7)) & 1u) != 0u;
}
// The 32 bitmap bits of rows [rb, rb + 32), rb % 32 == 0, of a bitmap whose row 0 is bit `sh` of the
// 4-byte aligned word *p; rows >= n read as 0 and no byte past the one that holds row n - 1 is touched.
// (Filter epilogue: one word per lane and 1024-row chunk, ColumnSlot::hoist.)
GDV_DEV u32 gdv_ldwin_rows(const u32* p, u32 sh, i64 rb, i64 n) {
  if (rb + 64 <= n) return gdv_ldwin(p, rb >> 5, sh);  // word rb / 32 + 1 still holds rows < n
  u32 w = 0u;
  const u8* b = reinterpret_cast<const u8*>(p);
  for (int i = 0; i < 32 && rb + i < n; ++i) w |= (u32)gdv_ldbit(b, sh, rb + i) << i;
  return w;
}
// ---- TMA bulk copies into shared memory (cp.async.bulk + mbarrier) ------------------------
// Wide projectors stage each CTA tile of every input column through shared memory with one
// bulk copy per column (SASS UBLKCP): the loads of the next tiles are in flight while the
// current tile computes, at no register cost.  Source and destination must be 16-byte aligned
// and the size a multiple of 16; the codegen aligns column pointers down and keeps the
// misalignment as a constant byte offset into the stage.
#ifndef GDV_HOST_EMU  // tests/emu/gdv_emu.h restates these primitives for the host-side simulator
GDV_DEV u32 gdv_smem_addr(const void* p) { return (u32)__cvta_generic_to_shared(p); }
GDV_DEV void gdv_mbar_init(u64* bar, u32 count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(gdv_smem_addr(bar)), "r"(count)
               : "memory");
}
GDV_DEV void gdv_fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
GDV_DEV void gdv_mbar_expect_tx(u64* bar, u32 bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(gdv_smem_addr(bar)),
               "r"(bytes)
               : "memory");
}
GDV_DEV u64 gdv_policy_evict_first() {
  u64 pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
GDV_DEV void gdv_bulk_g2s(void* dst, const void* src, u32 bytes, u64* bar, u64 policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint "
      "[%0], [%1], %2, [%3], %4;" ::"r"(gdv_smem_addr(dst)),
      "l"(src), "r"(bytes), "r"(gdv_smem_addr(bar)), "l"(policy)
      : "memory");
}
GDV_DEV bool gdv_mbar_try_wait(u64* bar, u32 parity) {
  u32 ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}"
      : "=r"(ok)
      : "r"(gdv_smem_addr(bar)), "r"(parity)
      : "memory");
  return ok != 0u;
}
GDV_DEV void gdv_mbar_wait(u64* bar, u32 parity) {
  while (!gdv_mbar_try_wait(bar, parity)) {
  }
}
// 16-byte asynchronous global -> shared copies (LDGSTS): the filter's string stage is filled one
// group ahead with these, so the copy needs no registers and overlaps the scan of the current group.
GDV_DEV void gdv_cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(gdv_smem_addr(smem_dst)), "l"(gsrc)
               : "memory");
}
GDV_DEV void gdv_cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
GDV_DEV void gdv_cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
#endif  // GDV_HOST_EMU
// Shared-memory element load (i128 as one LDS.128).
template <typename T>
GDV_DEV T gdv_lds(const T* p) {
  return *p;
}
template <>
GDV_DEV i128 gdv_lds<i128>(const i128* p) {
  const longlong2 v = *reinterpret_cast<const longlong2*>(p);
  return (i128)(((u128)(u64)v.y << 64) | (u128)(u64)v.x);
}
// gdv_ldwin() over a bitmap window that was staged into shared memory.
GDV_DEV u32 gdv_ldwin_s(const u32* p, u32 widx, u32 sh) {
  const u32 lo = p[widx];
  if (sh == 0u) return lo;
  return __funnelshift_r(lo, p[widx + 1], sh);
}

// Halfwords of x equal to the matching halfword of pat, as 0x8000 in that halfword (the upper one
// can be flagged falsely when the lower one matches: callers verify candidates).
GDV_DEV u32 gdv_eqhalf_msb(u32 x, u32 pat) {
  const u32 z = x ^ pat;
  return (z - 0x00010001u) & ~z & 0x80008000u;
}
// Digram hit masks of the four words of a chunk (e: pair starts at byte 0 / 2 of the word, o: at
// byte 1 / 3) -> one bit per start byte of the 16-byte chunk.
GDV_DEV u32 gdv_nib_half(u32 e, u32 o) {
  return ((e >> 15) & 1u) | ((o >> 14) & 2u) | ((e >> 29) & 4u) | ((o >> 28) & 8u);
}
GDV_DEV u32 gdv_mask16_half(u32 e0, u32 o0, u32 e1, u32 o1, u32 e2, u32 o2, u32 e3, u32 o3) {
  return gdv_nib_half(e0, o0) | (gdv_nib_half(e1, o1) << 4) | (gdv_nib_half(e2, o2) << 8) |
         (gdv_nib_half(e3, o3) << 12);
}
#ifndef GDV_HOST_EMU
GDV_DEV u32 gdv_lanemask_lt() {
  u32 m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}
#endif

// ---- arithmetic ------------------------------------------------------------------------
// Integer add/subtract/multiply wrap in two's complement (SURVEY.md §8a row a8).
#define GDV_INT_ARITH(T, UT, S)                                                              \
  GDV_DEV T add_##S##_##S(T a, T b) { return (T)((UT)a + (UT)b); }                           \
  GDV_DEV T subtract_##S##_##S(T a, T b) { return (T)((UT)a - (UT)b); }                      \
  GDV_DEV T multiply_##S##_##S(T a, T b) { return (T)((UT)a * (UT)b); }
GDV_INT_ARITH(i8, u32, int8)
GDV_INT_ARITH(i16, u32, int16)
GDV_INT_ARITH(i32, u32, int32)
GDV_INT_ARITH(i64, u64, int64)
GDV_INT_ARITH(u8, u32, uint8)
GDV_INT_ARITH(u16, u32, uint16)
GDV_INT_ARITH(u32, u32, uint32)
GDV_INT_ARITH(u64, u64, uint64)
#define GDV_SDIV(T, UT, S)                                        \
  GDV_DEV T divide_##S##_##S(gdv_ctx* c, T a, T b) {              \
    if (b == 0) {                                                 \
      gdv_set_error(c, GDV_ERR_DIV_ZERO);                         \
      return 0;                                                   \
    }                                                             \
    if (b == (T)-1) return (T)((UT)0 - (UT)a);                    \
    return (T)(a / b);                                            \
  }
#define GDV_UDIV(T, S)                                            \
  GDV_DEV T divide_##S##_##S(gdv_ctx* c, T a, T b) {              \
    if (b == 0) {                                                 \
      gdv_set_error(c, GDV_ERR_DIV_ZERO);                         \
      return 0;                                                   \
    }                                                             \
    return (T)(a / b);                                            \
  }
GDV_SDIV(i8, u32, int8)
GDV_SDIV(i16, u32, int16)
GDV_SDIV(i32, u32, int32)
GDV_SDIV(i64, u64, int64)
GDV_UDIV(u8, uint8)
GDV_UDIV(u16, uint16)
GDV_UDIV(u32, uint32)
GDV_UDIV(u64, uint64)
// IEEE arithmetic, no contraction (the engine passes --fmad=false to NVRTC).
#define GDV_FLT_ARITH(T, S)                                       \
  GDV_DEV T add_##S##_##S(T a, T b) { return a + b; }             \
  GDV_DEV T subtract_##S##_##S(T a, T b) { return a - b; }        \
  GDV_DEV T multiply_##S##_##S(T a, T b) { return a * b; }        \
  GDV_DEV T divide_##S##_##S(gdv_ctx* c, T a, T b) {              \
    if (b == (T)0) {                                              \
      gdv_set_error(c, GDV_ERR_DIV_ZERO);                         \
      return (T)0;                                                \
    }                                                             \
    return a / b;                                                 \
  }
GDV_FLT_ARITH(f32, float32)
GDV_FLT_ARITH(f64, float64)

GDV_DEV i32 mod_int64_int32(i64 a, i32 b) {
  if (b == 0) return (i32)a;
  if (b == -1) return 0;
  return (i32)(a % (i64)b);
}
GDV_DEV i32 mod_int32_int32(i32 a, i32 b) {
  if (b == 0) return a;
  if (b == -1) return 0;
  return a % b;
}
// mod of doubles: the exact IEEE remainder with the sign of x (fmod); a zero divisor raises like `divide`
GDV_DEV f64 mod_float64_float64(gdv_ctx* c, f64 x, f64 y) {
  if (y == 0.0) {
    gdv_set_error(c, GDV_ERR_DIV_ZERO);
    return 0.0;
  }
  const f64 r = fmod(x, y);
  return r != r ? __longlong_as_double(0x7ff8000000000000ll) : r;
}
GDV_DEV i64 mod_int64_int64(i64 a, i64 b) {
  if (b == 0) return a;
  if (b == -1) return 0;
  return a % b;
}
GDV_DEV i32 abs_int32(i32 a) { return a < 0 ? (i32)(0u - (u32)a) : a; }
GDV_DEV i64 abs_int64(i64 a) { return a < 0 ? (i64)(0ull - (u64)a) : a; }
GDV_DEV f32 abs_float32(f32 a) { return fabsf(a); }
GDV_DEV f64 abs_float64(f64 a) { return fabs(a); }
GDV_DEV i32 negative_int32(i32 a) { return (i32)(0u - (u32)a); }
GDV_DEV i64 negative_int64(i64 a) { return (i64)(0ull - (u64)a); }
GDV_DEV f32 negative_float32(f32 a) { return -a; }
GDV_DEV f64 negative_float64(f64 a) { return -a; }
GDV_DEV f64 sqrt_float64(f64 a) { return sqrt(a); }
#define GDV_BITWISE(T, S)                                                   \
  GDV_DEV T bitwise_and_##S##_##S(T a, T b) { return a & b; }               \
  GDV_DEV T bitwise_or_##S##_##S(T a, T b) { return a | b; }                \
  GDV_DEV T bitwise_xor_##S##_##S(T a, T b) { return a ^ b; }               \
  GDV_DEV T bitwise_not_##S(T a) { return ~a; }
GDV_BITWISE(i32, int32)
GDV_BITWISE(i64, int64)

// div: truncating integer division (x / 0 raises like divide); pmod: modulo with the sign of the
// divisor (Hive's ((x % y) + y) % y), pmod(x, 0) = x like mod; sign: -1 / 0 / 1 (floats: +-0 and
// NaN pass through).
#define GDV_INTDIV(T, UT, S)                                      \
  GDV_DEV T div_##S##_##S(gdv_ctx* c, T a, T b) {                 \
    if (b == 0) {                                                 \
      gdv_set_error(c, GDV_ERR_DIV_ZERO);                         \
      return (T)0;                                                \
    }                                                             \
    if (b == (T)-1) return (T)((UT)0 - (UT)a);                    \
    return (T)(a / b);                                            \
  }                                                               \
  GDV_DEV T pmod_##S##_##S(T a, T b) {                            \
    if (b == 0) return a;                                         \
    if (b == (T)-1) return (T)0;                                  \
    T r = (T)(a % b);                                             \
    if (r != 0 && ((r < 0) != (b < 0))) r = (T)(r + b);           \
    return r;                                                     \
  }                                                               \
  GDV_DEV T sign_##S(T a) { return (T)((a > 0) - (a < 0)); }
GDV_INTDIV(i32, u32, int32)
GDV_INTDIV(i64, u64, int64)
GDV_DEV f32 sign_float32(f32 a) { return a > 0.0f ? 1.0f : (a < 0.0f ? -1.0f : a); }
GDV_DEV f64 sign_float64(f64 a) { return a > 0.0 ? 1.0 : (a < 0.0 ? -1.0 : a); }
// bround: round half to even (the IEEE default rounding of rint)
GDV_DEV f64 bround_float64(f64 a) { return rint(a); }
// factorial(n), 0 <= n <= 20 (21! does not fit int64); anything else raises as the reference does
GDV_DEV i64 factorial_int64(gdv_ctx* c, i64 n) {
  if (n < 0) {
    gdv_set_error(c, GDV_ERR_FACTORIAL_NEG);
    return 0;
  }
  if (n > 20) {
    gdv_set_error(c, GDV_ERR_FACTORIAL_BIG);
    return 0;
  }
  i64 r = 1;
  for (i64 k = 2; k <= n; ++k) r *= k;
  return r;
}
GDV_DEV i64 factorial_int32(gdv_ctx* c, i32 n) { return factorial_int64(c, (i64)n); }
// greatest / least of 2..4 arguments, folded left to right with > / <: a NaN that is not the
// first argument never wins, a leading NaN is only displaced by a comparison that is true.
#define GDV_GREATEST_LEAST(T, S)                                                                  \
  GDV_DEV T greatest_##S##_##S(T a, T b) { return b > a ? b : a; }                                \
  GDV_DEV T greatest_##S##_##S##_##S(T a, T b, T c) {                                             \
    return greatest_##S##_##S(greatest_##S##_##S(a, b), c);                                       \
  }                                                                                               \
  GDV_DEV T greatest_##S##_##S##_##S##_##S(T a, T b, T c, T d) {                                  \
    return greatest_##S##_##S(greatest_##S##_##S##_##S(a, b, c), d);                              \
  }                                                                                               \
  GDV_DEV T least_##S##_##S(T a, T b) { return b < a ? b : a; }                                   \
  GDV_DEV T least_##S##_##S##_##S(T a, T b, T c) { return least_##S##_##S(least_##S##_##S(a, b), c); } \
  GDV_DEV T least_##S##_##S##_##S##_##S(T a, T b, T c, T d) {                                     \
    return least_##S##_##S(least_##S##_##S##_##S(a, b, c), d);                                    \
  }
GDV_GREATEST_LEAST(i32, int32)
GDV_GREATEST_LEAST(i64, int64)
GDV_GREATEST_LEAST(f32, float32)
GDV_GREATEST_LEAST(f64, float64)

// ---- exp / log / log10 / cbrt: explicit IEEE sequences ------------------------------------------------
// CUDA's libm and the host's differ in the last bit(s), so these are not library calls: each is the
// classic fdlibm (Sun Microsystems, 1993, freely usable) argument reduction + polynomial written out
// as a fixed sequence of IEEE double operations, which oracle/gdv_oracle.cc repeats operation for
// operation (the engine compiles with --fmad=false, the oracle with -ffp-contract=off): bit-exact
// parity, < 1 ULP from the exact result (measured against the host libm in tests/).
GDV_DEV f64 gdv_f64_from_bits(u64 b) { return __longlong_as_double((i64)b); }
GDV_DEV u64 gdv_f64_bits(f64 d) { return (u64)__double_as_longlong(d); }
GDV_DEV f64 exp_float64(f64 x) {
  const f64 ln2hi = 6.93147180369123816490e-01, ln2lo = 1.90821492927058770002e-10, invln2 = 1.44269504088896338700e+00;
  const f64 P1 = 1.66666666666666019037e-01, P2 = -2.77777777770155933842e-03, P3 = 6.61375632143793436117e-05,
            P4 = -1.65339022054652515390e-06, P5 = 4.13813679705723846039e-08;
  if (x != x) return x;
  if (x > 7.09782712893383973096e+02) return gdv_f64_from_bits(0x7ff0000000000000ull);
  if (x < -7.45133219101941108420e+02) return 0.0;
  const f64 ax = x < 0.0 ? -x : x;
  f64 hi = 0.0, lo = 0.0;
  i32 k = 0;
  if (ax > 0.34657359027997264) {          // |x| > 0.5 ln2
    if (ax < 1.0397207708399179) {         // |x| < 1.5 ln2
      k = x < 0.0 ? -1 : 1;
    } else {
      k = (i32)(invln2 * x + (x < 0.0 ? -0.5 : 0.5));
    }
    hi = x - (f64)k * ln2hi;
    lo = (f64)k * ln2lo;
    x = hi - lo;
  } else if (ax < 3.7252902984619141e-09) {  // |x| < 2^-28
    return 1.0 + x;
  }
  const f64 t = x * x;
  const f64 c = x - t * (P1 + t * (P2 + t * (P3 + t * (P4 + t * P5))));
  if (k == 0) return 1.0 - ((x * c) / (c - 2.0) - x);
  const f64 y = 1.0 - ((lo - (x * c) / (2.0 - c)) - hi);
  // y * 2^k through the exponent field (y is in [0.5, 2))
  if (k == 1024) return (y * 2.0) * 8.98846567431157953865e+307;  // 2^1023: the field would overflow
  if (k >= -1021) return gdv_f64_from_bits(gdv_f64_bits(y) + ((u64)(i64)k << 52));
  return gdv_f64_from_bits(gdv_f64_bits(y) + ((u64)(i64)(k + 1000) << 52)) * 9.33263618503218878990e-302;  // 2^-1000
}
GDV_DEV f64 log_float64(f64 x) {
  const f64 ln2hi = 6.93147180369123816490e-01, ln2lo = 1.90821492927058770002e-10;
  const f64 Lg1 = 6.666666666666735130e-01, Lg2 = 3.999999999940941908e-01, Lg3 = 2.857142874366239149e-01,
            Lg4 = 2.222219843214978396e-01, Lg5 = 1.818357216161805012e-01, Lg6 = 1.531383769920937332e-01,
            Lg7 = 1.479819860511658591e-01;
  if (x != x) return x;
  if (x < 0.0) return gdv_f64_from_bits(0x7ff8000000000000ull);
  if (x == 0.0) return gdv_f64_from_bits(0xfff0000000000000ull);
  u64 bits = gdv_f64_bits(x);
  if (bits == 0x7ff0000000000000ull) return x;
  i32 k = 0;
  if ((bits >> 52) == 0ull) {  // subnormal: scale up by 2^54
    x = x * 18014398509481984.0;
    bits = gdv_f64_bits(x);
    k = -54;
  }
  i32 hx = (i32)(bits >> 32);
  k += (hx >> 20) - 1023;
  hx &= 0x000fffff;
  const i32 i = (hx + 0x95f64) & 0x100000;
  x = gdv_f64_from_bits(((u64)(u32)(hx | (i ^ 0x3ff00000)) << 32) | (bits & 0xffffffffull));  // x in [sqrt(2)/2, sqrt(2))
  k += i >> 20;
  const f64 f = x - 1.0;
  const f64 dk = (f64)k;
  if ((0x000fffff & (2 + hx)) < 3) {  // |f| < 2^-20
    if (f == 0.0) return k == 0 ? 0.0 : dk * ln2hi + dk * ln2lo;
    const f64 R = f * f * (0.5 - 0.33333333333333333 * f);
    if (k == 0) return f - R;
    return dk * ln2hi - ((R - dk * ln2lo) - f);
  }
  const f64 s = f / (2.0 + f);
  const f64 z = s * s;
  const f64 w = z * z;
  const f64 t1 = w * (Lg2 + w * (Lg4 + w * Lg6));
  const f64 t2 = z * (Lg1 + w * (Lg3 + w * (Lg5 + w * Lg7)));
  const f64 R = t2 + t1;
  if (((hx - 0x6147a) | (0x6b851 - hx)) > 0) {
    const f64 hfsq = 0.5 * f * f;
    if (k == 0) return f - (hfsq - s * (hfsq + R));
    return dk * ln2hi - ((hfsq - (s * (hfsq + R) + dk * ln2lo)) - f);
  }
  if (k == 0) return f - s * (f - R);
  return dk * ln2hi - ((s * (f - R) - dk * ln2lo) - f);
}
// log(base, value) = ln(value) / ln(base); a base whose logarithm is zero (1) raises "divide by zero"
GDV_DEV f64 log_float64_float64(gdv_ctx* c, f64 base, f64 v) {
  const f64 lb = log_float64(base);
  if (lb == 0.0) {
    gdv_set_error(c, GDV_ERR_DIV_ZERO);
    return 0.0;
  }
  return log_float64(v) / lb;
}
GDV_DEV f64 log10_float64(f64 x) {
  // FreeBSD msun's e_log10: log(1 + f) kept as a hi + lo pair, multiplied by 1 / ln 10 (hi + lo too)
  const f64 ivln10hi = 4.34294481878168880939e-01, ivln10lo = 2.50829467116452752298e-11;
  const f64 log10_2hi = 3.01029995663611771306e-01, log10_2lo = 3.69423907715893078616e-13;
  const f64 Lg1 = 6.666666666666735130e-01, Lg2 = 3.999999999940941908e-01, Lg3 = 2.857142874366239149e-01,
            Lg4 = 2.222219843214978396e-01, Lg5 = 1.818357216161805012e-01, Lg6 = 1.531383769920937332e-01,
            Lg7 = 1.479819860511658591e-01;
  if (x != x) return x;
  if (x < 0.0) return gdv_f64_from_bits(0x7ff8000000000000ull);
  if (x == 0.0) return gdv_f64_from_bits(0xfff0000000000000ull);
  u64 bits = gdv_f64_bits(x);
  if (bits == 0x7ff0000000000000ull) return x;
  if (x == 1.0) return 0.0;
  i32 k = 0;
  if ((bits >> 52) == 0ull) {
    x = x * 18014398509481984.0;
    bits = gdv_f64_bits(x);
    k = -54;
  }
  i32 hx = (i32)(bits >> 32);
  k += (hx >> 20) - 1023;
  hx &= 0x000fffff;
  const i32 i = (hx + 0x95f64) & 0x100000;
  x = gdv_f64_from_bits(((u64)(u32)(hx | (i ^ 0x3ff00000)) << 32) | (bits & 0xffffffffull));
  k += i >> 20;
  const f64 dk = (f64)k;
  const f64 f = x - 1.0;
  const f64 hfsq = 0.5 * f * f;
  const f64 s = f / (2.0 + f);
  const f64 z = s * s;
  const f64 w = z * z;
  const f64 t1 = w * (Lg2 + w * (Lg4 + w * Lg6));
  const f64 t2 = z * (Lg1 + w * (Lg3 + w * (Lg5 + w * Lg7)));
  const f64 r = s * (hfsq + (t2 + t1));  // log(1 + f) - f + f * f / 2
  f64 hi = f - hfsq;
  hi = gdv_f64_from_bits(gdv_f64_bits(hi) & 0xffffffff00000000ull);
  const f64 lo = (f - hi) - hfsq + r;
  f64 val_hi = hi * ivln10hi;
  const f64 y2 = dk * log10_2hi;
  f64 val_lo = dk * log10_2lo + (lo + hi) * ivln10lo + lo * ivln10hi;
  const f64 ww = y2 + val_hi;
  val_lo += (y2 - ww) + val_hi;
  val_hi = ww;
  return val_lo + val_hi;
}
GDV_DEV f64 cbrt_float64(f64 x) {
  const f64 P0 = 1.87595182427177009643, P1 = -1.88497979543377169875, P2 = 1.621429720105354466140,
            P3 = -0.758397934778766047437, P4 = 0.145996192886612446982;
  const u64 bits = gdv_f64_bits(x);
  const u64 sign = bits & 0x8000000000000000ull;
  const u32 hx = (u32)(bits >> 32) & 0x7fffffffu;
  if (hx >= 0x7ff00000u) return x + x;  // inf / NaN
  f64 t;
  if (hx < 0x00100000u) {               // zero or subnormal
    if ((bits & 0x7fffffffffffffffull) == 0ull) return x;
    const f64 sc = gdv_f64_from_bits(bits & 0x7fffffffffffffffull) * 18014398509481984.0;  // |x| * 2^54
    const u32 h2 = (u32)(gdv_f64_bits(sc) >> 32) & 0x7fffffffu;
    t = gdv_f64_from_bits(sign | ((u64)(h2 / 3u + 696219795u) << 32));
  } else {
    t = gdv_f64_from_bits(sign | ((u64)(hx / 3u + 715094163u) << 32));
  }
  f64 r = (t * t) * (t / x);
  t = t * ((P0 + r * (P1 + r * P2)) + ((r * r) * r) * (P3 + r * P4));
  t = gdv_f64_from_bits((gdv_f64_bits(t) + 0x80000000ull) & 0xffffffffc0000000ull);  // 23 significant bits
  const f64 s2 = t * t;
  r = x / s2;
  const f64 w = t + t;
  r = (r - t) / (w + r);
  return t + t * r;
}

// ---- sin / cos / tan / cot: explicit IEEE sequences -------------------------------------------------
// Argument reduction in integers (Payne-Hanek): |x| = M * 2^e times 192 bits of 2/pi picked so that
// everything above the quadrant bits is a multiple of 4; the product gives the quadrant and a
// 128+ bit fraction, which becomes a double-double multiple of pi/2 in [-pi/4, pi/4].  Then Taylor
// polynomials through x^17 / x^18 (truncation < 2^-63) with the leading terms carried as
// double-doubles: sin and cos are one rounding of those (0.55 ULP measured), tan and cot their
// double-double quotient (0.56 ULP).  Constants: tools/derive_trig_constants.py.  < 1 ULP from the
// exact result; the oracle repeats every operation, so kernel == oracle bit for bit.
__device__ const u64 gdv_two_over_pi[20] = {
    0xa2f9836e4e441529ull, 0xfc2757d1f534ddc0ull, 0xdb6295993c439041ull, 0xfe5163abdebbc561ull,
    0xb7246e3a424dd2e0ull, 0x06492eea09d1921cull, 0xfe1deb1cb129a73eull, 0xe88235f52ebb4484ull,
    0xe99c7026b45f7e41ull, 0x3991d639835339f4ull, 0x9c845f8bbdf9283bull, 0x1ff897ffde05980full,
    0xef2f118b5a0a6d1full, 0x6d367ecf27cb09b7ull, 0x4f463f669e5fea2dull, 0x7527bac7ebe5f17bull,
    0x3d0739f78a5292eaull, 0x6bfb5fb11f8d5d08ull, 0x56033046fc7b6babull, 0xf0cfbc209af4361dull};
// ax finite, > pi/4: ax = quad * pi/2 + (y0 + y1), |y0 + y1| <= pi/4
GDV_DEV_BIG void gdv_rem_pio2(f64 ax, f64* y0, f64* y1, i32* quad) {
  const u64 bits = gdv_f64_bits(ax);
  const i32 e = (i32)(bits >> 52) - 1075;  // ax = M * 2^e, M in [2^52, 2^53)
  const u64 M = (bits & 0x000fffffffffffffull) | 0x0010000000000000ull;
  const i32 i0 = e >= 2 ? e - 1 : 1;       // first bit of 2/pi (1 = the 2^-1 bit) that matters mod 4
  const i32 s = e >= 2 ? 190 : 192 - e;    // the product below is (ax * 2/pi mod 4) * 2^s
  const i32 j = (i0 - 1) >> 6, sh = (i0 - 1) & 63;
  u64 w[3];
  for (i32 k = 0; k < 3; ++k)
    w[k] = sh ? (gdv_two_over_pi[j + k] << sh) | (gdv_two_over_pi[j + k + 1] >> (64 - sh)) : gdv_two_over_pi[j + k];
  const u128 p2 = (u128)M * w[2], p1 = (u128)M * w[1], p0 = (u128)M * w[0];
  u64 P[4];
  P[0] = (u64)p2;
  u128 acc = (p2 >> 64) + (u128)(u64)p1;
  P[1] = (u64)acc;
  acc = (acc >> 64) + (p1 >> 64) + (u128)(u64)p0;
  P[2] = (u64)acc;
  acc = (acc >> 64) + (p0 >> 64);
  P[3] = (u64)acc;
  i32 q = (i32)((P[s >> 6] >> (s & 63)) & 1ull) | ((i32)((P[(s + 1) >> 6] >> ((s + 1) & 63)) & 1ull) << 1);
  const bool half = ((P[(s - 1) >> 6] >> ((s - 1) & 63)) & 1ull) != 0ull;
  // keep the s fraction bits; past one half, go to the next quadrant and negate the fraction
  const u64 top_mask = (1ull << (s & 63)) - 1ull;
  for (i32 k = 0; k < 4; ++k) {
    if (half) P[k] = ~P[k];
    if (k == (s >> 6)) P[k] &= top_mask;
    if (k > (s >> 6)) P[k] = 0ull;
  }
  if (half) {  // two's complement: + 1 (cannot carry out of s bits: the fraction was not zero)
    ++q;
    for (i32 k = 0; k < 4; ++k) {
      P[k] += 1ull;
      if (P[k] != 0ull) break;
    }
  }
  *quad = q & 3;
  i32 p = -1;
  for (i32 k = 3; k >= 0 && p < 0; --k)
    if (P[k] != 0ull) p = k * 64 + 63 - __clzll((long long)P[k]);
  if (p < 0) {
    *y0 = 0.0;
    *y1 = 0.0;
    return;
  }
  // the top 106 bits of the fraction as two 53-bit integers
  const i32 up = 255 - p, uw = up >> 6, ub = up & 63;
  u64 G[4];
  for (i32 k = 3; k >= 0; --k) {
    const u64 hi = k - uw >= 0 ? P[k - uw] : 0ull;
    const u64 lo = k - uw - 1 >= 0 ? P[k - uw - 1] : 0ull;
    G[k] = ub ? (hi << ub) | (lo >> (64 - ub)) : hi;
  }
  const u64 H = G[3] >> 11, L = ((G[3] & 0x7ffull) << 42) | (G[2] >> 22);
  const f64 sc = gdv_f64_from_bits((u64)(i64)(1023 + p - 52 - s) << 52);
  const f64 fh = (f64)(i64)H * sc, fl = ((f64)(i64)L * sc) * 1.1102230246251565e-16;  // * 2^-53
  const f64 ph = 1.5707963267948966, pl = 6.123233995736766e-17;
  const f64 t = fh * ph;
  const f64 err = fma(fh, ph, -t);
  const f64 lo = err + (fh * pl + fl * ph);
  f64 r0 = t + lo;
  f64 r1 = (t - r0) + lo;
  if (half) {
    r0 = -r0;
    r1 = -r1;
  }
  *y0 = r0;
  *y1 = r1;
}
GDV_DEV f64 gdv_ksin_poly(f64 z) {  // (sin(x) - x + x^3/6) / x^5, z = x^2
  const f64 S2 = 0.008333333333333333, S3 = -0.0001984126984126984, S4 = 2.7557319223985893e-06,
            S5 = -2.505210838544172e-08, S6 = 1.6059043836821613e-10, S7 = -7.647163731819816e-13,
            S8 = 2.8114572543455206e-15;
  return S2 + z * (S3 + z * (S4 + z * (S5 + z * (S6 + z * (S7 + z * S8)))));
}
GDV_DEV f64 gdv_kcos_poly(f64 z) {
  const f64 C1 = 0.041666666666666664, C2 = -0.001388888888888889, C3 = 2.48015873015873e-05,
            C4 = -2.755731922398589e-07, C5 = 2.08767569878681e-09, C6 = -1.1470745597729725e-11,
            C7 = 4.779477332387385e-14, C8 = -1.5619206968586225e-16;
  return z * (C1 + z * (C2 + z * (C3 + z * (C4 + z * (C5 + z * (C6 + z * (C7 + z * C8)))))));
}
// fn: 0 sin, 1 cos, 2 tan, 3 cot
GDV_DEV_BIG f64 gdv_trig(f64 x, i32 fn) {
  const u64 bits = gdv_f64_bits(x);
  const u64 ab = bits & 0x7fffffffffffffffull;
  if (ab >= 0x7ff0000000000000ull) return gdv_f64_from_bits(0x7ff8000000000000ull);  // inf, nan -> the canonical nan
  const bool neg = (bits >> 63) != 0ull;
  const f64 ax = gdv_f64_from_bits(ab);
  if (ab < 0x3e40000000000000ull) {  // |x| < 2^-27
    if (fn == 1) return 1.0;
    if (fn == 3) return 1.0 / x;
    return x;
  }
  f64 y0 = ax, y1 = 0.0;
  i32 q = 0;
  if (ax > 0.7853981633974483) gdv_rem_pio2(ax, &y0, &y1, &q);
  // sin = y0 - (y0 + y1)^3 / 6 + ..., cos = 1 - (y0 + y1)^2 / 2 + ...: the squares, the cube and 1/6
  // carry their rounding errors along, so that both come out as double-doubles good to ~2^-58
  const f64 S1 = -0.16666666666666666, S1L = -9.25185853854297e-18;
  const f64 z = y0 * y0;
  const f64 zl = fma(y0, y0, -z) + (2.0 * y0) * y1;
  const f64 v = z * y0;
  const f64 vl = fma(z, y0, -v) + (zl * y0 + z * y1);
  const f64 t3 = v * S1;
  const f64 t3l = (fma(v, S1, -t3) + v * S1L) + vl * S1;
  const f64 s_rest = (t3l + y1) + ((z * z) * y0) * gdv_ksin_poly(z);
  const f64 s_a = y0 + t3, s_b = ((y0 - s_a) + t3) + s_rest;
  const f64 s_hi = s_a + s_b, s_lo = (s_a - s_hi) + s_b;
  const f64 ch = -0.5 * z;
  const f64 c_rest = z * gdv_kcos_poly(z) - 0.5 * zl;
  const f64 c_a = 1.0 + ch, c_b = ((1.0 - c_a) + ch) + c_rest;
  const f64 c_hi = c_a + c_b, c_lo = (c_a - c_hi) + c_b;
  f64 res;
  if (fn <= 1) {
    const i32 k = (q + fn) & 3;  // cos(t) = sin(t + pi/2)
    res = (k & 1) ? c_hi : s_hi;
    if (k & 2) res = -res;
    if (fn == 0 && neg) res = -res;
    return res;
  }
  // tan / cot: one double-double divided by the other
  const bool sin_over_cos = ((q & 1) != 0) == (fn == 3);
  const f64 n_hi = sin_over_cos ? s_hi : c_hi, n_lo = sin_over_cos ? s_lo : c_lo;
  const f64 d_hi = sin_over_cos ? c_hi : s_hi, d_lo = sin_over_cos ? c_lo : s_lo;
  const f64 q0 = n_hi / d_hi;
  const f64 rem = fma(-q0, d_hi, n_hi);
  const f64 q1 = ((rem + n_lo) - q0 * d_lo) / d_hi;
  res = q0 + q1;
  if (q & 1) res = -res;
  return neg ? -res : res;
}
GDV_DEV f64 sin_float64(f64 x) { return gdv_trig(x, 0); }
GDV_DEV f64 cos_float64(f64 x) { return gdv_trig(x, 1); }
GDV_DEV f64 tan_float64(f64 x) { return gdv_trig(x, 2); }
GDV_DEV f64 cot_float64(f64 x) { return gdv_trig(x, 3); }
#define GDV_TRIG_OF(T, S)                                              \
  GDV_DEV f64 sin_##S(T x) { return gdv_trig((f64)x, 0); }             \
  GDV_DEV f64 cos_##S(T x) { return gdv_trig((f64)x, 1); }             \
  GDV_DEV f64 tan_##S(T x) { return gdv_trig((f64)x, 2); }             \
  GDV_DEV f64 cot_##S(T x) { return gdv_trig((f64)x, 3); }
GDV_TRIG_OF(i32, int32)
GDV_TRIG_OF(i64, int64)
GDV_TRIG_OF(f32, float32)

// ---- comparisons -----------------------------------------------------------------------
#define GDV_RELOP(T, S)                                                               \
  GDV_DEV bool equal_##S##_##S(T a, T b) { return a == b; }                           \
  GDV_DEV bool not_equal_##S##_##S(T a, T b) { return a != b; }                       \
  GDV_DEV bool less_than_##S##_##S(T a, T b) { return a < b; }                        \
  GDV_DEV bool less_than_or_equal_to_##S##_##S(T a, T b) { return a <= b; }           \
  GDV_DEV bool greater_than_##S##_##S(T a, T b) { return a > b; }                     \
  GDV_DEV bool greater_than_or_equal_to_##S##_##S(T a, T b) { return a >= b; }
GDV_RELOP(i8, int8)
GDV_RELOP(i16, int16)
GDV_RELOP(i32, int32)
GDV_RELOP(i64, int64)
GDV_RELOP(u8, uint8)
GDV_RELOP(u16, uint16)
GDV_RELOP(u32, uint32)
GDV_RELOP(u64, uint64)
GDV_RELOP(f32, float32)
GDV_RELOP(f64, float64)
GDV_RELOP(i32, date32)
GDV_RELOP(i64, date64)
GDV_RELOP(i64, timestamp)
GDV_RELOP(i32, time32)
GDV_DEV bool equal_boolean_boolean(bool a, bool b) { return a == b; }
GDV_DEV bool not_equal_boolean_boolean(bool a, bool b) { return a != b; }
GDV_DEV bool not_boolean(bool a) { return !a; }

// Lexicographic byte comparison, shorter string first on a common prefix.
GDV_DEV i32 gdv_mem_compare(const gdv_str& a, const gdv_str& b) {
  const i32 n = a.len < b.len ? a.len : b.len;
  for (i32 i = 0; i < n; ++i) {
    const u8 x = gdv_ch(a, i), y = gdv_ch(b, i);
    if (x != y) return x < y ? -1 : 1;
  }
  return a.len == b.len ? 0 : (a.len < b.len ? -1 : 1);
}
#define GDV_STR_RELOP(S)                                                                           \
  GDV_DEV bool equal_##S##_##S(gdv_str a, gdv_str b) {                                             \
    return a.len == b.len && gdv_mem_compare(a, b) == 0;                                           \
  }                                                                                                \
  GDV_DEV bool not_equal_##S##_##S(gdv_str a, gdv_str b) {                                         \
    return !(a.len == b.len && gdv_mem_compare(a, b) == 0);                                        \
  }                                                                                                \
  GDV_DEV bool less_than_##S##_##S(gdv_str a, gdv_str b) { return gdv_mem_compare(a, b) < 0; }     \
  GDV_DEV bool less_than_or_equal_to_##S##_##S(gdv_str a, gdv_str b) {                             \
    return gdv_mem_compare(a, b) <= 0;                                                             \
  }                                                                                                \
  GDV_DEV bool greater_than_##S##_##S(gdv_str a, gdv_str b) { return gdv_mem_compare(a, b) > 0; }  \
  GDV_DEV bool greater_than_or_equal_to_##S##_##S(gdv_str a, gdv_str b) {                          \
    return gdv_mem_compare(a, b) >= 0;                                                             \
  }
GDV_STR_RELOP(utf8)
GDV_STR_RELOP(binary)

// ---- null tests (NullMode::kNever: receive value + validity) -----------------------------
#define GDV_NULLTEST(T, S)                                                   \
  GDV_DEV bool isnull_##S(T, bool ok) { return !ok; }                        \
  GDV_DEV bool isnotnull_##S(T, bool ok) { return ok; }
GDV_NULLTEST(i8, int8)
GDV_NULLTEST(i16, int16)
GDV_NULLTEST(i32, int32)
GDV_NULLTEST(i64, int64)
GDV_NULLTEST(u8, uint8)
GDV_NULLTEST(u16, uint16)
GDV_NULLTEST(u32, uint32)
GDV_NULLTEST(u64, uint64)
GDV_NULLTEST(f32, float32)
GDV_NULLTEST(f64, float64)
GDV_NULLTEST(i32, date32)
GDV_NULLTEST(i64, date64)
GDV_NULLTEST(i64, timestamp)
GDV_NULLTEST(i32, time32)
GDV_NULLTEST(bool, boolean)
GDV_NULLTEST(i128, decimal128)
GDV_NULLTEST(gdv_str, utf8)
GDV_NULLTEST(gdv_str, binary)
GDV_DEV bool istrue_boolean(bool v, bool ok) { return ok && v; }
GDV_DEV bool isfalse_boolean(bool v, bool ok) { return ok && !v; }
GDV_DEV bool isnottrue_boolean(bool v, bool ok) { return !(ok && v); }
GDV_DEV bool isnotfalse_boolean(bool v, bool ok) { return !(ok && !v); }
#define GDV_DISTINCT(T, S)                                                                   \
  GDV_DEV bool is_distinct_from_##S##_##S(T a, bool aok, T b, bool bok) {                    \
    if (aok != bok) return true;                                                             \
    if (!aok) return false;                                                                  \
    return a != b;                                                                           \
  }                                                                                          \
  GDV_DEV bool is_not_distinct_from_##S##_##S(T a, bool aok, T b, bool bok) {                \
    return !is_distinct_from_##S##_##S(a, aok, b, bok);                                      \
  }
GDV_DISTINCT(i8, int8)
GDV_DISTINCT(i16, int16)
GDV_DISTINCT(i32, int32)
GDV_DISTINCT(i64, int64)
GDV_DISTINCT(u8, uint8)
GDV_DISTINCT(u16, uint16)
GDV_DISTINCT(u32, uint32)
GDV_DISTINCT(u64, uint64)
GDV_DISTINCT(f32, float32)
GDV_DISTINCT(f64, float64)
GDV_DISTINCT(i32, date32)
GDV_DISTINCT(i64, date64)
GDV_DISTINCT(i64, timestamp)
GDV_DISTINCT(i32, time32)
GDV_DISTINCT(bool, boolean)

// ---- casts -----------------------------------------------------------------------------
GDV_DEV i64 castBIGINT_int32(i32 a) { return (i64)a; }
GDV_DEV i32 castINT_int64(i64 a) { return (i32)(u32)(u64)a; }
GDV_DEV f32 castFLOAT4_int32(i32 a) { return (f32)a; }
GDV_DEV f32 castFLOAT4_int64(i64 a) { return (f32)a; }
GDV_DEV f32 castFLOAT4_float64(f64 a) { return (f32)a; }
GDV_DEV f64 castFLOAT8_int32(i32 a) { return (f64)a; }
GDV_DEV f64 castFLOAT8_int64(i64 a) { return (f64)a; }
GDV_DEV f64 castFLOAT8_float32(f32 a) { return (f64)a; }
GDV_DEV i64 castDATE_int64(i64 a) { return a; }
GDV_DEV i64 castTIMESTAMP_int64(i64 a) { return a; }
GDV_DEV i64 castTIMESTAMP_date64(i64 a) { return a; }
GDV_DEV i64 castBIGINT_date64(i64 a) { return a; }
GDV_DEV i64 castBIGINT_timestamp(i64 a) { return a; }
GDV_DEV i32 castINT_date32(i32 a) { return a; }
GDV_DEV i32 castDATE_int32(i32 a) { return a; }
// floor-divide helper for negative epochs
GDV_DEV i64 gdv_floordiv(i64 a, i64 b) {
  i64 q = a / b;
  if ((a % b != 0) && ((a < 0) != (b < 0))) --q;
  return q;
}
// days -> milliseconds with two's-complement wrap (dates within 86400 s of the int64 limits have
// month / year starts outside the range: the result is then defined, and the oracle's, not UB)
GDV_DEV i64 gdv_days_to_ms(i64 days) { return (i64)((u64)days * 86400000ull); }
GDV_DEV i64 castDATE_timestamp(i64 ms) { return gdv_days_to_ms(gdv_floordiv(ms, 86400000ll)); }

// ---- date / time extraction (proleptic Gregorian, days-from-civil inverse) ---------------
struct gdv_ymd {
  i64 y;
  i32 m, d, doy;
};
GDV_DEV gdv_ymd gdv_civil_from_days(i64 z) {
  z += 719468;
  const i64 era = gdv_floordiv(z, 146097);
  const i64 doe = z - era * 146097;
  const i64 yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
  const i64 y = yoe + era * 400;
  const i64 doy_mar = doe - (365 * yoe + yoe / 4 - yoe / 100);
  const i64 mp = (5 * doy_mar + 2) / 153;
  gdv_ymd r;
  r.d = (i32)(doy_mar - (153 * mp + 2) / 5 + 1);
  r.m = (i32)(mp < 10 ? mp + 3 : mp - 9);
  r.y = y + (r.m <= 2 ? 1 : 0);
  const bool leap = (r.y % 4 == 0) && ((r.y % 100 != 0) || (r.y % 400 == 0));
  const i32 cum[12] = {0, 31, 59, 90, 120, 151, 181, 212, 243, 273, 304, 334};
  r.doy = cum[r.m - 1] + r.d + ((leap && r.m > 2) ? 1 : 0);
  return r;
}
#define GDV_EXTRACT_MS(S)                                                                       \
  GDV_DEV i64 extractYear_##S(i64 ms) {                                                         \
    return gdv_civil_from_days(gdv_floordiv(ms, 86400000ll)).y;                                 \
  }                                                                                             \
  GDV_DEV i64 extractMonth_##S(i64 ms) {                                                        \
    return gdv_civil_from_days(gdv_floordiv(ms, 86400000ll)).m;                                 \
  }                                                                                             \
  GDV_DEV i64 extractDay_##S(i64 ms) {                                                          \
    return gdv_civil_from_days(gdv_floordiv(ms, 86400000ll)).d;                                 \
  }                                                                                             \
  GDV_DEV i64 extractDoy_##S(i64 ms) {                                                          \
    return gdv_civil_from_days(gdv_floordiv(ms, 86400000ll)).doy;                               \
  }                                                                                             \
  GDV_DEV i64 extractQuarter_##S(i64 ms) {                                                      \
    return (gdv_civil_from_days(gdv_floordiv(ms, 86400000ll)).m - 1) / 3 + 1;                   \
  }                                                                                             \
  GDV_DEV i64 extractDow_##S(i64 ms) {                                                          \
    const i64 days = gdv_floordiv(ms, 86400000ll);                                              \
    i64 w = (days + 4) % 7; /* 1970-01-01 was a Thursday; Sunday = 1 */                         \
    if (w < 0) w += 7;                                                                          \
    return w + 1;                                                                               \
  }                                                                                             \
  GDV_DEV i64 extractHour_##S(i64 ms) {                                                         \
    return (ms - gdv_floordiv(ms, 86400000ll) * 86400000ll) / 3600000ll;                        \
  }                                                                                             \
  GDV_DEV i64 extractMinute_##S(i64 ms) {                                                       \
    return ((ms - gdv_floordiv(ms, 86400000ll) * 86400000ll) / 60000ll) % 60;                   \
  }                                                                                             \
  GDV_DEV i64 extractSecond_##S(i64 ms) {                                                       \
    return ((ms - gdv_floordiv(ms, 86400000ll) * 86400000ll) / 1000ll) % 60;                    \
  }                                                                                             \
  GDV_DEV i64 extractEpoch_##S(i64 ms) { return gdv_floordiv(ms, 1000ll); }
GDV_EXTRACT_MS(date64)
GDV_EXTRACT_MS(timestamp)
GDV_DEV i64 extractYear_date32(i32 d) { return gdv_civil_from_days((i64)d).y; }
GDV_DEV i64 extractMonth_date32(i32 d) { return gdv_civil_from_days((i64)d).m; }
GDV_DEV i64 extractDay_date32(i32 d) { return gdv_civil_from_days((i64)d).d; }

// ---- rounding (exact IEEE operations; half away from zero like C's round()) ------------------
GDV_DEV f64 round_float64(f64 a) { return round(a); }
GDV_DEV f32 round_float32(f32 a) { return roundf(a); }
GDV_DEV f64 ceil_float64(f64 a) { return ceil(a); }
GDV_DEV f64 floor_float64(f64 a) { return floor(a); }
GDV_DEV f64 truncate_float64(f64 a) { return trunc(a); }
GDV_DEV i32 round_int32(i32 a) { return a; }
GDV_DEV i64 round_int64(i64 a) { return a; }
// round(x, s): s >= 0: round(x * 10^s) / 10^s; s < 0: round(x / 10^-s) * 10^-s; a value that is
// already a multiple of 10^-s is returned unchanged; the power is built by repeated
// multiplication (exact up to 10^22); |s| is clamped to 308.
GDV_DEV f64 gdv_pow10_f64(i32 e) {
  f64 p = 1.0;
  for (i32 i = 0; i < e; ++i) p = p * 10.0;
  return p;
}
GDV_DEV f64 round_float64_int32(f64 a, i32 s) {
  s = s > 308 ? 308 : (s < -308 ? -308 : s);  // clamp first: -s must not overflow for INT32_MIN
  if (s >= 0) {
    const f64 p = gdv_pow10_f64(s);
    const f64 v = a * p;
    if (!(fabs(v) < 1.7976931348623157e308)) return a;  // overflow or NaN: nothing to round
    if (v == floor(v)) return a;  // already a multiple of 10^-s: do not disturb the value
    return round(v) / p;
  }
  const f64 p = gdv_pow10_f64(-s);
  const f64 q = a / p;
  if (q == floor(q)) return a;
  return round(q) * p;
}

// truncate(x, s): like round(x, s) with trunc() in place of round().
GDV_DEV f64 truncate_float64_int32(f64 a, i32 s) {
  s = s > 308 ? 308 : (s < -308 ? -308 : s);
  if (s >= 0) {
    const f64 p = gdv_pow10_f64(s);
    const f64 v = a * p;
    if (!(fabs(v) < 1.7976931348623157e308)) return a;
    if (v == floor(v)) return a;
    return trunc(v) / p;
  }
  const f64 p = gdv_pow10_f64(-s);
  const f64 q = a / p;
  if (q == floor(q)) return a;
  return trunc(q) * p;
}
// round / truncate of an integer to 10^-s, s < 0 (s >= 0: unchanged); half away from zero; the
// arithmetic is done in 128 bits and the result wraps into the output type like a cast.
GDV_DEV i128 gdv_round_int128(i128 x, i32 s, bool half_away) {
  if (s >= 0) return x;
  if (s < -38) return (i128)0;
  i128 p = 1;
  for (i32 i = 0; i < -s; ++i) p = p * 10;
  const i128 r = x % p;
  i128 base = x - r;
  if (half_away) {
    const i128 ar = r < 0 ? -r : r;
    if (ar >= p - ar) base = base + (x < 0 ? -p : p);
  }
  return base;
}
GDV_DEV i32 round_int32_int32(i32 a, i32 s) { return (i32)(u32)(u128)gdv_round_int128((i128)a, s, true); }
GDV_DEV i64 round_int64_int32(i64 a, i32 s) { return (i64)(u64)(u128)gdv_round_int128((i128)a, s, true); }
GDV_DEV i32 truncate_int32_int32(i32 a, i32 s) { return (i32)(u32)(u128)gdv_round_int128((i128)a, s, false); }
GDV_DEV i64 truncate_int64_int32(i64 a, i32 s) { return (i64)(u64)(u128)gdv_round_int128((i128)a, s, false); }

// ---- date / time arithmetic (date64 and timestamp are milliseconds since the epoch) -----------
GDV_DEV i64 gdv_days_from_civil(i64 y, i32 m, i32 d) {
  y -= m <= 2 ? 1 : 0;
  const i64 era = gdv_floordiv(y, 400);
  const i64 yoe = y - era * 400;
  const i64 doy = (153 * (i64)(m + (m > 2 ? -3 : 9)) + 2) / 5 + (i64)d - 1;
  const i64 doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
  return era * 146097 + doe - 719468;
}
// Calendar month arithmetic: the day of month is clamped to the length of the target month
// (Jan 31 + 1 month = Feb 28/29); the time of day is kept.
GDV_DEV i64 gdv_add_months(i64 ms, i64 months) {
  const i64 days = gdv_floordiv(ms, 86400000ll);
  const i64 in_day = ms - days * 86400000ll;
  const gdv_ymd c = gdv_civil_from_days(days);
  const i64 total = c.y * 12 + (i64)(c.m - 1) + months;
  const i64 ny = gdv_floordiv(total, 12);
  const i32 nm = (i32)(total - ny * 12) + 1;
  const bool leap = (ny % 4 == 0) && ((ny % 100 != 0) || (ny % 400 == 0));
  const i32 mlen[12] = {31, leap ? 29 : 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31};
  const i32 nd = c.d < mlen[nm - 1] ? c.d : mlen[nm - 1];
  return (i64)((u64)gdv_days_to_ms(gdv_days_from_civil(ny, nm, nd)) + (u64)in_day);
}
#define GDV_TSADD(NAME, UNIT_MS)                                                                  \
  GDV_DEV i64 NAME##_int32_timestamp(i32 n, i64 ts) { return (i64)((u64)ts + (u64)((i64)n * (UNIT_MS))); } \
  GDV_DEV i64 NAME##_int64_timestamp(i64 n, i64 ts) { return (i64)((u64)ts + (u64)n * (u64)(UNIT_MS)); } \
  GDV_DEV i64 NAME##_timestamp_int32(i64 ts, i32 n) { return NAME##_int32_timestamp(n, ts); }     \
  GDV_DEV i64 NAME##_timestamp_int64(i64 ts, i64 n) { return NAME##_int64_timestamp(n, ts); }
GDV_TSADD(timestampaddSecond, 1000ll)
GDV_TSADD(timestampaddMinute, 60000ll)
GDV_TSADD(timestampaddHour, 3600000ll)
GDV_TSADD(timestampaddDay, 86400000ll)
GDV_TSADD(timestampaddWeek, 604800000ll)
// calendar units: month counts wrap in 64 bits (an int64 count times 3 or 12), like the millisecond units
#define GDV_TSADD_MONTHS(NAME, K)                                                                 \
  GDV_DEV i64 NAME##_int32_timestamp(i32 n, i64 ts) { return gdv_add_months(ts, (K) * (i64)n); }  \
  GDV_DEV i64 NAME##_int64_timestamp(i64 n, i64 ts) { return gdv_add_months(ts, (i64)((u64)(K) * (u64)n)); } \
  GDV_DEV i64 NAME##_timestamp_int32(i64 ts, i32 n) { return NAME##_int32_timestamp(n, ts); }     \
  GDV_DEV i64 NAME##_timestamp_int64(i64 ts, i64 n) { return NAME##_int64_timestamp(n, ts); }
GDV_TSADD_MONTHS(timestampaddMonth, 1ll)
GDV_TSADD_MONTHS(timestampaddQuarter, 3ll)
GDV_TSADD_MONTHS(timestampaddYear, 12ll)
// add_months(date | timestamp, n): timestampaddMonth with the arguments the other way round
GDV_DEV i64 add_months_date64_int32(i64 d, i32 n) { return gdv_add_months(d, (i64)n); }
GDV_DEV i64 add_months_date64_int64(i64 d, i64 n) { return gdv_add_months(d, n); }
GDV_DEV i64 add_months_timestamp_int32(i64 d, i32 n) { return gdv_add_months(d, (i64)n); }
GDV_DEV i64 add_months_timestamp_int64(i64 d, i64 n) { return gdv_add_months(d, n); }
GDV_DEV i64 date_add_date64_int32(i64 d, i32 n) { return (i64)((u64)d + (u64)((i64)n * 86400000ll)); }
GDV_DEV i64 date_sub_date64_int32(i64 d, i32 n) { return (i64)((u64)d - (u64)((i64)n * 86400000ll)); }
GDV_DEV i64 date_add_timestamp_int32(i64 d, i32 n) { return date_add_date64_int32(d, n); }
GDV_DEV i64 date_sub_timestamp_int32(i64 d, i32 n) { return date_sub_date64_int32(d, n); }
#define GDV_TSDIFF(NAME, UNIT_MS)                                                                 \
  GDV_DEV i32 NAME##_timestamp_timestamp(i64 a, i64 b) {                                          \
    return (i32)(u32)(u64)((i64)((u64)b - (u64)a) / (UNIT_MS));                                   \
  }
GDV_TSDIFF(timestampdiffSecond, 1000ll)
GDV_TSDIFF(timestampdiffMinute, 60000ll)
GDV_TSDIFF(timestampdiffHour, 3600000ll)
GDV_TSDIFF(timestampdiffDay, 86400000ll)
GDV_TSDIFF(timestampdiffWeek, 604800000ll)

// timestampdiff{Month,Quarter,Year}(a, b): whole calendar months from a to b, consistent with
// timestampaddMonth: the largest |k| such that a + k months (day clamped to the month's length,
// time of day kept) does not pass b; quarters and years are that count / 3 and / 12, truncated.
GDV_DEV_BIG i64 gdv_months_between_whole(i64 a, i64 b) {
  const gdv_ymd ca = gdv_civil_from_days(gdv_floordiv(a, 86400000ll));
  const gdv_ymd cb = gdv_civil_from_days(gdv_floordiv(b, 86400000ll));
  i64 k = (cb.y - ca.y) * 12 + (i64)(cb.m - ca.m);
  if (b >= a) {
    if (k > 0 && gdv_add_months(a, k) > b) --k;
    if (k < 0) k = 0;
  } else {
    if (k < 0 && gdv_add_months(a, k) < b) ++k;
    if (k > 0) k = 0;
  }
  return k;
}
GDV_DEV i32 timestampdiffMonth_timestamp_timestamp(i64 a, i64 b) { return (i32)gdv_months_between_whole(a, b); }
GDV_DEV i32 timestampdiffQuarter_timestamp_timestamp(i64 a, i64 b) { return (i32)(gdv_months_between_whole(a, b) / 3); }
GDV_DEV i32 timestampdiffYear_timestamp_timestamp(i64 a, i64 b) { return (i32)(gdv_months_between_whole(a, b) / 12); }
// months_between(a, b) (Hive / Oracle): a - b in months; whole when both are the same day of the
// month or both the last day of theirs, else the month difference plus (day and time of day
// difference) / 31 days; IEEE double operations in a fixed order.
GDV_DEV_BIG f64 gdv_months_between(i64 a, i64 b) {
  const i64 da = gdv_floordiv(a, 86400000ll), db = gdv_floordiv(b, 86400000ll);
  const gdv_ymd ca = gdv_civil_from_days(da), cb = gdv_civil_from_days(db);
  const f64 months = (f64)((ca.y - cb.y) * 12 + (i64)(ca.m - cb.m));
  const bool last_a = gdv_civil_from_days(da + 1).d == 1, last_b = gdv_civil_from_days(db + 1).d == 1;
  if (ca.d == cb.d || (last_a && last_b)) return months;
  const i64 ta = a - da * 86400000ll, tb = b - db * 86400000ll;
  const f64 secs = (f64)((i64)(ca.d - cb.d) * 86400ll) + (f64)(ta - tb) / 1000.0;
  return months + secs / 2678400.0;
}
GDV_DEV f64 months_between_timestamp_timestamp(i64 a, i64 b) { return gdv_months_between(a, b); }
GDV_DEV f64 months_between_date64_date64(i64 a, i64 b) { return gdv_months_between(a, b); }

// ---- calendar fields and truncation -------------------------------------------------------------
// ISO 8601 week of the year (weeks start on Monday, week 1 holds the year's first Thursday).
GDV_DEV i64 gdv_iso_week(i64 days) {
  const gdv_ymd c = gdv_civil_from_days(days);
  i64 wd = (days + 3) % 7;  // 1970-01-01 was a Thursday: Monday = 0
  if (wd < 0) wd += 7;
  const i64 week = ((i64)c.doy - (wd + 1) + 10) / 7;
  if (week >= 1 && week <= 52) return week;
  // weekday of Jan 1 of year y (Monday = 0), and whether y has 53 ISO weeks
  const i64 jan1 = days - ((i64)c.doy - 1);
  if (week < 1) {
    const i64 py = c.y - 1;
    const bool pleap = (py % 4 == 0) && ((py % 100 != 0) || (py % 400 == 0));
    const i64 pjan1 = jan1 - (pleap ? 366 : 365);
    i64 pw = (pjan1 + 3) % 7;
    if (pw < 0) pw += 7;
    return (pw == 3 || (pleap && pw == 2)) ? 53 : 52;
  }
  const bool leap = (c.y % 4 == 0) && ((c.y % 100 != 0) || (c.y % 400 == 0));
  i64 jw = (jan1 + 3) % 7;
  if (jw < 0) jw += 7;
  return (jw == 3 || (leap && jw == 2)) ? 53 : 1;
}
// date_trunc: the first instant of the enclosing unit; weeks start on Monday; decades start in
// years divisible by 10, centuries / millennia in years ...01 (C truncating division on the year).
GDV_DEV i64 gdv_trunc_year_to(i64 ms, i64 span, i64 first) {
  const gdv_ymd c = gdv_civil_from_days(gdv_floordiv(ms, 86400000ll));
  const i64 y = span == 10 ? (c.y / 10) * 10 : ((c.y - 1) / span) * span + first;
  return gdv_days_to_ms(gdv_days_from_civil(span == 1 ? c.y : y, 1, 1));
}
#define GDV_CALENDAR(S)                                                                           \
  GDV_DEV i64 extractWeek_##S(i64 ms) { return gdv_iso_week(gdv_floordiv(ms, 86400000ll)); }      \
  GDV_DEV i64 extractDecade_##S(i64 ms) {                                                         \
    return gdv_civil_from_days(gdv_floordiv(ms, 86400000ll)).y / 10;                              \
  }                                                                                               \
  GDV_DEV i64 extractCentury_##S(i64 ms) {                                                        \
    return (gdv_civil_from_days(gdv_floordiv(ms, 86400000ll)).y - 1) / 100 + 1;                   \
  }                                                                                               \
  GDV_DEV i64 extractMillennium_##S(i64 ms) {                                                     \
    return (gdv_civil_from_days(gdv_floordiv(ms, 86400000ll)).y - 1) / 1000 + 1;                  \
  }                                                                                               \
  GDV_DEV i64 date_trunc_Second_##S(i64 ms) { return gdv_floordiv(ms, 1000ll) * 1000ll; }         \
  GDV_DEV i64 date_trunc_Minute_##S(i64 ms) { return gdv_floordiv(ms, 60000ll) * 60000ll; }       \
  GDV_DEV i64 date_trunc_Hour_##S(i64 ms) { return gdv_floordiv(ms, 3600000ll) * 3600000ll; }     \
  GDV_DEV i64 date_trunc_Day_##S(i64 ms) { return gdv_days_to_ms(gdv_floordiv(ms, 86400000ll)); } \
  GDV_DEV i64 date_trunc_Week_##S(i64 ms) {                                                       \
    const i64 days = gdv_floordiv(ms, 86400000ll);                                                \
    i64 wd = (days + 3) % 7;                                                                      \
    if (wd < 0) wd += 7;                                                                          \
    return gdv_days_to_ms(days - wd);                                                             \
  }                                                                                               \
  GDV_DEV i64 date_trunc_Month_##S(i64 ms) {                                                      \
    const gdv_ymd c = gdv_civil_from_days(gdv_floordiv(ms, 86400000ll));                          \
    return gdv_days_to_ms(gdv_days_from_civil(c.y, c.m, 1));                                      \
  }                                                                                               \
  GDV_DEV i64 date_trunc_Quarter_##S(i64 ms) {                                                    \
    const gdv_ymd c = gdv_civil_from_days(gdv_floordiv(ms, 86400000ll));                          \
    return gdv_days_to_ms(gdv_days_from_civil(c.y, ((c.m - 1) / 3) * 3 + 1, 1));                  \
  }                                                                                               \
  GDV_DEV i64 date_trunc_Year_##S(i64 ms) { return gdv_trunc_year_to(ms, 1, 0); }                 \
  GDV_DEV i64 date_trunc_Decade_##S(i64 ms) { return gdv_trunc_year_to(ms, 10, 0); }              \
  GDV_DEV i64 date_trunc_Century_##S(i64 ms) { return gdv_trunc_year_to(ms, 100, 1); }            \
  GDV_DEV i64 date_trunc_Millennium_##S(i64 ms) { return gdv_trunc_year_to(ms, 1000, 1); }        \
  GDV_DEV i64 last_day_##S(i64 ms) {                                                              \
    const gdv_ymd c = gdv_civil_from_days(gdv_floordiv(ms, 86400000ll));                          \
    const i64 ny = c.m == 12 ? c.y + 1 : c.y;                                                     \
    const i32 nm = c.m == 12 ? 1 : c.m + 1;                                                       \
    return gdv_days_to_ms(gdv_days_from_civil(ny, nm, 1) - 1);                                    \
  }
GDV_CALENDAR(date64)
GDV_CALENDAR(timestamp)
// float -> integer casts: round half away from zero, then saturate at the ends of the type; NaN -> 0
GDV_DEV i64 castBIGINT_float64(f64 x) {
  if (x != x) return 0ll;
  const f64 r = round(x);
  if (r >= 9223372036854775808.0) return 0x7fffffffffffffffll;
  if (r <= -9223372036854775808.0) return (i64)0x8000000000000000ull;
  return (i64)r;
}
GDV_DEV i64 castBIGINT_float32(f32 x) { return castBIGINT_float64((f64)x); }
GDV_DEV i32 castINT_float64(f64 x) {
  if (x != x) return 0;
  const f64 r = round(x);
  if (r >= 2147483647.0) return 2147483647;
  if (r <= -2147483648.0) return (i32)0x80000000u;
  return (i32)r;
}
GDV_DEV i32 castINT_float32(f32 x) { return castINT_float64((f64)x); }
// to_timestamp(seconds since the epoch) / to_time(seconds): milliseconds, fractions truncated toward
// zero; to_time keeps the time of day in [0, 86 400 000)
GDV_DEV i64 to_timestamp_int64(i64 sec) { return (i64)((u64)sec * 1000ull); }
GDV_DEV i64 to_timestamp_int32(i32 sec) { return (i64)sec * 1000ll; }
GDV_DEV i64 to_timestamp_float64(f64 sec) { return castBIGINT_float64(trunc(sec * 1000.0)); }
GDV_DEV i64 to_timestamp_float32(f32 sec) { return to_timestamp_float64((f64)sec); }
GDV_DEV i32 gdv_ms_of_day(i64 ms) { return (i32)(ms - gdv_floordiv(ms, 86400000ll) * 86400000ll); }
GDV_DEV i32 to_time_int64(i64 sec) { return gdv_ms_of_day(to_timestamp_int64(sec)); }
GDV_DEV i32 to_time_int32(i32 sec) { return gdv_ms_of_day(to_timestamp_int32(sec)); }
GDV_DEV i32 to_time_float64(f64 sec) { return gdv_ms_of_day(to_timestamp_float64(sec)); }
GDV_DEV i32 to_time_float32(f32 sec) { return gdv_ms_of_day(to_timestamp_float64((f64)sec)); }
// time of day (time32[ms]) of a timestamp, and its fields
GDV_DEV i32 castTIME_timestamp(i64 ms) { return (i32)(ms - gdv_floordiv(ms, 86400000ll) * 86400000ll); }
GDV_DEV i64 extractHour_time32(i32 t) { return (i64)(t / 3600000); }
GDV_DEV i64 extractMinute_time32(i32 t) { return (i64)((t / 60000) % 60); }
GDV_DEV i64 extractSecond_time32(i32 t) { return (i64)((t / 1000) % 60); }

// ---- decimal128 ------------------------------------------------------------------------
// Values are two's-complement 128-bit integers scaled by 10^scale (Arrow decimal128).
// Rounding on scale reduction is half away from zero; a result that does not fit 38
// digits yields 0 (the reference ignores the overflow flag of its decimal ops).
GDV_DEV u128 gdv_pow10_u128(i32 e) {  // 0 <= e <= 38
  const u64 p19 = 10000000000000000000ull;
  const u64 t[20] = {1ull, 10ull, 100ull, 1000ull, 10000ull, 100000ull, 1000000ull, 10000000ull,
                     100000000ull, 1000000000ull, 10000000000ull, 100000000000ull,
                     1000000000000ull, 10000000000000ull, 100000000000000ull,
                     1000000000000000ull, 10000000000000000ull, 100000000000000000ull,
                     1000000000000000000ull, 10000000000000000000ull};
  if (e <= 19) return (u128)t[e];
  return (u128)t[e - 19] * (u128)p19;
}
// 256-bit magnitude as four 64-bit limbs, little-endian.
struct gdv_u256 {
  u64 w[4];
};
GDV_DEV gdv_u256 gdv_mul_u128(u128 a, u128 b) {
  const u64 a0 = (u64)a, a1 = (u64)(a >> 64), b0 = (u64)b, b1 = (u64)(b >> 64);
  const u128 p00 = (u128)a0 * b0, p01 = (u128)a0 * b1, p10 = (u128)a1 * b0, p11 = (u128)a1 * b1;
  gdv_u256 r;
  r.w[0] = (u64)p00;
  u128 mid = (p00 >> 64) + (u128)(u64)p01 + (u128)(u64)p10;
  r.w[1] = (u64)mid;
  u128 hi = (mid >> 64) + (p01 >> 64) + (p10 >> 64) + (u128)(u64)p11;
  r.w[2] = (u64)hi;
  r.w[3] = (u64)((hi >> 64) + (p11 >> 64));
  return r;
}
GDV_DEV gdv_u256 gdv_add_u256(const gdv_u256& a, const gdv_u256& b) {
  gdv_u256 r;
  u128 c = 0;
  for (int i = 0; i < 4; ++i) {
    c += (u128)a.w[i] + (u128)b.w[i];
    r.w[i] = (u64)c;
    c >>= 64;
  }
  return r;
}
// a - b, requires a >= b
GDV_DEV gdv_u256 gdv_sub_u256(const gdv_u256& a, const gdv_u256& b) {
  gdv_u256 r;
  u64 borrow = 0;
  for (int i = 0; i < 4; ++i) {
    const u64 bi = b.w[i];
    const u64 d = a.w[i] - bi - borrow;
    borrow = (a.w[i] < bi || (a.w[i] == bi && borrow)) ? 1ull : 0ull;
    r.w[i] = d;
  }
  return r;
}
GDV_DEV int gdv_cmp_u256(const gdv_u256& a, const gdv_u256& b) {
  for (int i = 3; i >= 0; --i) {
    if (a.w[i] != b.w[i]) return a.w[i] < b.w[i] ? -1 : 1;
  }
  return 0;
}
// Divide a 256-bit magnitude by a 64-bit divisor in place; returns the remainder.
GDV_DEV u64 gdv_divmod_u256_u64(gdv_u256& a, u64 d) {
  u128 rem = 0;
  for (int i = 3; i >= 0; --i) {
    const u128 cur = (rem << 64) | (u128)a.w[i];
    a.w[i] = (u64)(cur / d);
    rem = cur % d;
  }
  return (u64)rem;
}
// round-half-away(mag / 10^e), 0 <= e <= 38.
GDV_DEV gdv_u256 gdv_div_pow10_round(gdv_u256 mag, i32 e) {
  if (e == 0) return mag;
  // add half of the divisor first, then truncate
  const u128 half = gdv_pow10_u128(e) / 2u;  // 10^e is even for e >= 1
  gdv_u256 h;
  h.w[0] = (u64)half;
  h.w[1] = (u64)(half >> 64);
  h.w[2] = 0;
  h.w[3] = 0;
  mag = gdv_add_u256(mag, h);
  i32 left = e;
  while (left > 0) {
    const i32 step = left > 19 ? 19 : left;
    gdv_divmod_u256_u64(mag, (u64)gdv_pow10_u128(step));
    left -= step;
  }
  return mag;
}
// Signed result from a 256-bit magnitude; 0 when it needs more than 38 digits.
GDV_DEV i128 gdv_fit_decimal(const gdv_u256& mag, bool neg) {
  if (mag.w[2] != 0 || mag.w[3] != 0) return (i128)0;
  const u128 m = ((u128)mag.w[1] << 64) | (u128)mag.w[0];
  if (m >= gdv_pow10_u128(38)) return (i128)0;
  return neg ? (i128)(~m + 1) : (i128)m;
}
GDV_DEV u128 gdv_abs_u128(i128 v) { return v < 0 ? (~(u128)v + 1) : (u128)v; }
GDV_DEV gdv_u256 gdv_u256_from(u128 v) {
  gdv_u256 r;
  r.w[0] = (u64)v;
  r.w[1] = (u64)(v >> 64);
  r.w[2] = 0;
  r.w[3] = 0;
  return r;
}

// x (scale xs) + sign * y (scale ys) -> scale os.  Exact in 256 bits, then rounded.
GDV_DEV i128 gdv_decimal_addsub(i128 x, i32 xs, i128 y, i32 ys, i32 os, bool subtract,
                                bool headroom) {
  const i32 ms = xs > ys ? xs : ys;
  if (os == ms && xs == ys) {
    // fast path: no rescale (covers TPC-H Q1).  When the declared precisions leave headroom
    // (max(xp, yp) + 1 <= 38) the sum of two in-contract values cannot pass 38 digits and the
    // overflow test is dropped, as the reference's fast path does.
    const i128 r = subtract ? (i128)((u128)x - (u128)y) : (i128)((u128)x + (u128)y);
    if (headroom) return r;
    const u128 m = gdv_abs_u128(r);
    return m >= gdv_pow10_u128(38) ? (i128)0 : r;
  }
  const bool xneg = x < 0;
  bool yneg = y < 0;
  if (subtract) yneg = !yneg;
  const gdv_u256 xm = gdv_mul_u128(gdv_abs_u128(x), gdv_pow10_u128(ms - xs));
  const gdv_u256 ym = gdv_mul_u128(gdv_abs_u128(y), gdv_pow10_u128(ms - ys));
  gdv_u256 mag;
  bool neg;
  if (xneg == yneg) {
    mag = gdv_add_u256(xm, ym);
    neg = xneg;
  } else if (gdv_cmp_u256(xm, ym) >= 0) {
    mag = gdv_sub_u256(xm, ym);
    neg = xneg;
  } else {
    mag = gdv_sub_u256(ym, xm);
    neg = yneg;
  }
  if (os < ms) mag = gdv_div_pow10_round(mag, ms - os);
  // os > ms never happens with the reference's result-type rule; scale up if a caller asks
  if (os > ms) {
    if (mag.w[2] != 0 || mag.w[3] != 0) return (i128)0;
    mag = gdv_mul_u128(((u128)mag.w[1] << 64) | mag.w[0], gdv_pow10_u128(os - ms));
  }
  if (mag.w[0] == 0 && mag.w[1] == 0 && mag.w[2] == 0 && mag.w[3] == 0) neg = false;
  return gdv_fit_decimal(mag, neg);
}
GDV_DEV i128 add_decimal128_decimal128(i128 x, i32 xp, i32 xs, i128 y, i32 yp, i32 ys, i32 op,
                                       i32 os) {
  return gdv_decimal_addsub(x, xs, y, ys, os, false, (xp > yp ? xp : yp) + 1 <= 38);
}
GDV_DEV i128 subtract_decimal128_decimal128(i128 x, i32 xp, i32 xs, i128 y, i32 yp, i32 ys,
                                            i32 op, i32 os) {
  return gdv_decimal_addsub(x, xs, y, ys, os, true, (xp > yp ? xp : yp) + 1 <= 38);
}
GDV_DEV i128 multiply_decimal128_decimal128(i128 x, i32 xp, i32 xs, i128 y, i32 yp, i32 ys,
                                            i32 op, i32 os) {
  const bool neg = (x < 0) != (y < 0);
  const i32 delta = xs + ys - os;
  if (xp + yp <= 38 && delta == 0) {
    // |x| < 10^xp, |y| < 10^yp  =>  |x*y| < 10^38 < 2^127: one 128-bit multiply is exact
    return (i128)((u128)x * (u128)y);
  }
  if (delta == 0 && x == (i128)(i64)x && y == (i128)(i64)y) {
    // both operands fit 64 bits (the usual case whatever the declared precision):
    // |x*y| < 2^126 < 10^38, so one signed 64x64->128 multiply is exact and cannot overflow
    return (i128)(i64)x * (i128)(i64)y;
  }
  gdv_u256 mag = gdv_mul_u128(gdv_abs_u128(x), gdv_abs_u128(y));
  if (delta > 0) mag = gdv_div_pow10_round(mag, delta > 38 ? 38 : delta);
  if (delta < 0) {
    if (mag.w[2] != 0 || mag.w[3] != 0) return (i128)0;
    mag = gdv_mul_u128(((u128)mag.w[1] << 64) | mag.w[0], gdv_pow10_u128(-delta));
  }
  const bool zero = mag.w[0] == 0 && mag.w[1] == 0 && mag.w[2] == 0 && mag.w[3] == 0;
  return gdv_fit_decimal(mag, neg && !zero);
}
GDV_DEV i128 abs_decimal128(i128 x, i32 xp, i32 xs, i32 op, i32 os) {
  return x < 0 ? (i128)(~(u128)x + 1) : x;
}
GDV_DEV i128 negative_decimal128(i128 x, i32 xp, i32 xs, i32 op, i32 os) {
  return (i128)(~(u128)x + 1);
}
// Compare after bringing both sides to the larger scale (exact, 256-bit).
GDV_DEV i32 gdv_decimal_compare(i128 x, i32 xs, i128 y, i32 ys) {
  if (xs == ys) return x < y ? -1 : (x > y ? 1 : 0);
  const bool xneg = x < 0, yneg = y < 0;
  if (xneg != yneg) return xneg ? -1 : 1;
  const i32 ms = xs > ys ? xs : ys;
  const gdv_u256 xm = gdv_mul_u128(gdv_abs_u128(x), gdv_pow10_u128(ms - xs));
  const gdv_u256 ym = gdv_mul_u128(gdv_abs_u128(y), gdv_pow10_u128(ms - ys));
  const int c = gdv_cmp_u256(xm, ym);
  return xneg ? -c : c;
}
#define GDV_DEC_RELOP(NAME, OP)                                                                  \
  GDV_DEV bool NAME##_decimal128_decimal128(i128 x, i32 xp, i32 xs, i128 y, i32 yp, i32 ys) {    \
    return gdv_decimal_compare(x, xs, y, ys) OP 0;                                               \
  }
GDV_DEC_RELOP(equal, ==)
GDV_DEC_RELOP(not_equal, !=)
GDV_DEC_RELOP(less_than, <)
GDV_DEC_RELOP(less_than_or_equal_to, <=)
GDV_DEC_RELOP(greater_than, >)
GDV_DEC_RELOP(greater_than_or_equal_to, >=)
// Rescale x from scale xs to (op, os): round half away; does not fit op digits -> 0.
GDV_DEV i128 castDECIMAL_decimal128(i128 x, i32 xp, i32 xs, i32 op, i32 os) {
  const bool neg = x < 0;
  gdv_u256 mag = gdv_u256_from(gdv_abs_u128(x));
  if (os > xs) mag = gdv_mul_u128(gdv_abs_u128(x), gdv_pow10_u128(os - xs));
  if (os < xs) mag = gdv_div_pow10_round(mag, xs - os);
  if (mag.w[2] != 0 || mag.w[3] != 0) return (i128)0;
  const u128 m = ((u128)mag.w[1] << 64) | (u128)mag.w[0];
  if (m >= gdv_pow10_u128(op)) return (i128)0;
  return (neg && m != 0) ? (i128)(~m + 1) : (i128)m;
}
GDV_DEV i128 castDECIMAL_int64(i64 v, i32 op, i32 os) {
  return castDECIMAL_decimal128((i128)v, 19, 0, op, os);
}
GDV_DEV i128 castDECIMAL_int32(i32 v, i32 op, i32 os) {
  return castDECIMAL_decimal128((i128)v, 10, 0, op, os);
}
// decimal -> int64: round half away at scale 0, then two's-complement truncation to 64 bits.
GDV_DEV i64 castBIGINT_decimal128(i128 x, i32 xp, i32 xs) {
  const i128 r = castDECIMAL_decimal128(x, xp, xs, 38, 0);
  return (i64)(u64)(u128)r;
}
// decimal -> double: (hi * 2^64 + lo) / 10^scale with the IEEE operations written out,
// so the oracle computes the identical sequence.
GDV_DEV f64 castFLOAT8_decimal128(i128 x, i32 xp, i32 xs) {
  const bool neg = x < 0;
  const u128 m = gdv_abs_u128(x);
  const f64 hi = (f64)(u64)(m >> 64), lo = (f64)(u64)m;
  f64 v = hi * 18446744073709551616.0 + lo;
  f64 p = 1.0;
  for (i32 i = 0; i < xs; ++i) p = p * 10.0;
  v = v / p;
  return neg ? -v : v;
}

// ---- decimal128 divide / mod / from double ---------------------------------------------------
GDV_DEV bool gdv_u256_is_zero(const gdv_u256& a) { return (a.w[0] | a.w[1] | a.w[2] | a.w[3]) == 0ull; }
GDV_DEV bool gdv_u256_fits128(const gdv_u256& a) { return (a.w[2] | a.w[3]) == 0ull; }
GDV_DEV u128 gdv_u256_low128(const gdv_u256& a) { return ((u128)a.w[1] << 64) | (u128)a.w[0]; }
// a * b for a 256-bit a and a 128-bit b; *overflow when the product needs more than 256 bits.
GDV_DEV gdv_u256 gdv_mul_u256_u128(const gdv_u256& a, u128 b, bool* overflow) {
  const gdv_u256 lo = gdv_mul_u128(gdv_u256_low128(a), b);
  const gdv_u256 hi = gdv_mul_u128(((u128)a.w[3] << 64) | (u128)a.w[2], b);  // weight 2^128
  gdv_u256 r;
  r.w[0] = lo.w[0];
  r.w[1] = lo.w[1];
  u128 c = (u128)lo.w[2] + (u128)hi.w[0];
  r.w[2] = (u64)c;
  c = (c >> 64) + (u128)lo.w[3] + (u128)hi.w[1];
  r.w[3] = (u64)c;
  *overflow = (c >> 64) != 0 || hi.w[2] != 0ull || hi.w[3] != 0ull;
  return r;
}
// Restoring division, one bit per iteration: n = q * d + r, r < d.  d != 0 and d < 2^255.
GDV_DEV void gdv_divmod_u256(const gdv_u256& n, const gdv_u256& d, gdv_u256* q, gdv_u256* r) {
  if (gdv_u256_fits128(n) && gdv_u256_fits128(d)) {
    const u128 nn = gdv_u256_low128(n), dd = gdv_u256_low128(d);
    *q = gdv_u256_from(nn / dd);
    *r = gdv_u256_from(nn % dd);
    return;
  }
  gdv_u256 quo, rem;
  for (int i = 0; i < 4; ++i) quo.w[i] = rem.w[i] = 0ull;
  int top = 255;
  while (top > 0 && ((n.w[top >> 6] >> (top & 63)) & 1ull) == 0ull) --top;
  for (int b = top; b >= 0; --b) {
    rem.w[3] = (rem.w[3] << 1) | (rem.w[2] >> 63);
    rem.w[2] = (rem.w[2] << 1) | (rem.w[1] >> 63);
    rem.w[1] = (rem.w[1] << 1) | (rem.w[0] >> 63);
    rem.w[0] = (rem.w[0] << 1) | ((n.w[b >> 6] >> (b & 63)) & 1ull);
    if (gdv_cmp_u256(rem, d) >= 0) {
      rem = gdv_sub_u256(rem, d);
      quo.w[b >> 6] |= 1ull << (b & 63);
    }
  }
  *q = quo;
  *r = rem;
}
// |x| * 10^e in 256 bits (e >= 0, any size); *overflow when it does not fit.
GDV_DEV gdv_u256 gdv_scale_up_u256(u128 x, i32 e, bool* overflow) {
  *overflow = false;
  gdv_u256 r = gdv_mul_u128(x, gdv_pow10_u128(e > 38 ? 38 : e));
  i32 left = e > 38 ? e - 38 : 0;
  while (left > 0) {
    const i32 step = left > 38 ? 38 : left;
    bool o = false;
    r = gdv_mul_u256_u128(r, gdv_pow10_u128(step), &o);
    *overflow = *overflow || o;
    left -= step;
  }
  return r;
}
// castFLOAT8 / castFLOAT4(utf8): [spaces][+-]digits[.digits][(e|E)[+-]digits][spaces].  Up to 19
// significant digits m (further digits only make the value "inexact") and a decimal exponent e10.
// m * 10^e10 is carried as X * 2^exp2 with X a 256-bit integer: multiplied by 10^k (k <= 19) after
// X is cut to its top 192 bits, or divided by 10^k after X is shifted up to bit 255, so every step
// keeps >= 192 significant bits (relative error < 2^-190 after the <= 22 steps the double range
// needs) -- far below the 2^-120 by which a 64-bit decimal significand can approach a rounding
// boundary, and exact whenever the value is a dyadic rational.  One round-to-nearest-even at the end,
// subnormals, overflow to infinity and underflow to zero included: the result strtod / Python
// float() give.  The oracle does the same steps on 32-bit limbs, bit by bit and digit by digit.
GDV_DEV int gdv_u256_top(const gdv_u256& x) {  // index of the highest set bit (x != 0)
  for (int w = 3; w > 0; --w)
    if (x.w[w] != 0ull) return w * 64 + 63 - __clzll((long long)x.w[w]);
  return 63 - __clzll((long long)x.w[0]);
}
GDV_DEV void gdv_u256_shr_sticky(gdv_u256& x, int s, bool& sticky) {  // 0 <= s <= 255
  if (s <= 0) return;
  const int ws = s >> 6, bs = s & 63;
  gdv_u256 r;
  for (int i = 0; i < 4; ++i) {
    if (i < ws) sticky = sticky || x.w[i] != 0ull;
    const u64 lo = i + ws < 4 ? x.w[i + ws] : 0ull;
    const u64 hi = i + ws + 1 < 4 ? x.w[i + ws + 1] : 0ull;
    r.w[i] = bs ? (lo >> bs) | (hi << (64 - bs)) : lo;
  }
  if (bs) sticky = sticky || (x.w[ws] & ((1ull << bs) - 1ull)) != 0ull;
  x = r;
}
GDV_DEV void gdv_u256_shl(gdv_u256& x, int s) {  // 0 <= s <= 255, no bit is shifted out by callers
  if (s <= 0) return;
  const int ws = s >> 6, bs = s & 63;
  gdv_u256 r;
  for (int i = 3; i >= 0; --i) {
    const u64 hi = i - ws >= 0 ? x.w[i - ws] : 0ull;
    const u64 lo = i - ws - 1 >= 0 ? x.w[i - ws - 1] : 0ull;
    r.w[i] = bs ? (hi << bs) | (lo >> (64 - bs)) : hi;
  }
  x = r;
}
GDV_DEV f64 gdv_u256_to_f64(gdv_u256 x, bool sticky, i32 exp2) {  // x != 0: RNE(x * 2^exp2) as an IEEE double
  const int p = gdv_u256_top(x);
  const i32 be = p + exp2;  // x * 2^exp2 in [2^be, 2^(be+1))
  if (be > 1023) return gdv_f64_from_bits(0x7ff0000000000000ull);
  const i32 nb = be >= -1022 ? 53 : be + 1075;  // significand bits the format has at this magnitude
  if (nb < 0) return 0.0;
  const i32 drop = p + 1 - nb;
  u64 mant;
  bool round = false;
  if (drop <= 0) {
    mant = x.w[0] << (-drop);
  } else {
    gdv_u256_shr_sticky(x, drop - 1, sticky);  // nb + 1 bits left, all in w[0]
    round = (x.w[0] & 1ull) != 0ull;
    mant = x.w[0] >> 1;
  }
  if (round && (sticky || (mant & 1ull) != 0ull)) ++mant;
  // mant * 2^(exp2 + drop): normal numbers carry the hidden bit into the exponent field, subnormals
  // (exp2 + drop == -1074, mant < 2^52) come out as the bare fraction, 2^53 / 2^1024 carry upwards
  return gdv_f64_from_bits(((u64)(i64)(exp2 + drop + 1075) << 52) + mant - (1ull << 52));
}
// x * 2^exp2 times 10^rest, 19 decimal digits at a time, keeping >= 192 significant bits (see below)
GDV_DEV void gdv_scale_pow10(gdv_u256& x, i32& exp2, bool& sticky, i32 rest) {
  while (rest > 0) {
    const i32 k = rest > 19 ? 19 : rest;
    const int p = gdv_u256_top(x);
    if (p > 191) {
      gdv_u256_shr_sticky(x, p - 191, sticky);
      exp2 += p - 191;
    }
    bool o = false;
    x = gdv_mul_u256_u128(x, gdv_pow10_u128(k), &o);  // < 2^192 * 2^64
    rest -= k;
  }
  while (rest < 0) {
    const i32 k = -rest > 19 ? 19 : -rest;
    const int up = 255 - gdv_u256_top(x);
    gdv_u256_shl(x, up);
    exp2 -= up;
    sticky = (gdv_divmod_u256_u64(x, (u64)gdv_pow10_u128(k)) != 0ull) || sticky;
    rest += k;
  }
}
GDV_DEV_BIG f64 gdv_parse_f64(gdv_ctx* c, const gdv_str& s) {
  i32 b = 0, e = s.len;
  while (b < e && s.p[b] == (u8)' ') ++b;
  while (e > b && s.p[e - 1] == (u8)' ') --e;
  bool neg = false;
  if (b < e && (s.p[b] == (u8)'-' || s.p[b] == (u8)'+')) {
    neg = s.p[b] == (u8)'-';
    ++b;
  }
  u64 m = 0ull;
  i32 sig = 0, e10 = 0, ndig = 0;
  bool point = false, sticky = false, ok = true;
  i32 i = b;
  for (; i < e; ++i) {
    const u32 ch = (u32)s.p[i];
    if (ch == (u32)'.') {
      if (point) ok = false;
      point = true;
      continue;
    }
    const u32 d = ch - (u32)'0';
    if (d > 9u) break;
    ++ndig;
    if (sig < 19) {
      if (m != 0ull || d != 0u) {
        m = m * 10ull + d;
        ++sig;
      }
      if (point) --e10;
    } else {
      sticky = sticky || d != 0u;
      if (!point) ++e10;
    }
  }
  if (ok && ndig > 0 && i < e && (s.p[i] == (u8)'e' || s.p[i] == (u8)'E')) {
    ++i;
    bool eneg = false;
    if (i < e && (s.p[i] == (u8)'-' || s.p[i] == (u8)'+')) {
      eneg = s.p[i] == (u8)'-';
      ++i;
    }
    i32 ev = 0, edig = 0;
    for (; i < e; ++i) {
      const u32 d = (u32)s.p[i] - (u32)'0';
      if (d > 9u) break;
      if (ev < 100000) ev = ev * 10 + (i32)d;
      ++edig;
    }
    ok = ok && edig > 0;
    e10 += eneg ? -ev : ev;
  }
  if (!ok || ndig == 0 || i != e) {
    gdv_set_error(c, GDV_ERR_CAST_FLOAT);
    return 0.0;
  }
  if (m == 0ull) return neg ? -0.0 : 0.0;
  if (e10 > 400) e10 = 400;
  if (e10 < -400) e10 = -400;
  gdv_u256 x;
  x.w[0] = m;
  x.w[1] = 0ull;
  x.w[2] = 0ull;
  x.w[3] = 0ull;
  i32 exp2 = 0;
  gdv_scale_pow10(x, exp2, sticky, e10);
  const f64 d = gdv_u256_to_f64(x, sticky, exp2);
  return neg ? -d : d;
}
GDV_DEV f64 castFLOAT8_utf8(gdv_ctx* c, gdv_str s) { return gdv_parse_f64(c, s); }
GDV_DEV f32 castFLOAT4_utf8(gdv_ctx* c, gdv_str s) { return (f32)gdv_parse_f64(c, s); }

// ---- power(x, y) = 2^(y * log2 x), in integers -------------------------------------------------------
// log2 of the significand bit by bit (square; if >= 2, halve and emit a 1) in Q2.126 for 120 bits:
// absolute error < 2^-118, also when x is next to 1 and log2 x ~ 2^-53.  y * log2 x is an exact
// integer product (53 x 131 bits); its fraction F goes through e^(F ln 2) as a 34-term Taylor sum in
// Q1.127, and the 128-bit significand is rounded once (nearest-even, subnormals and overflow
// included) by gdv_u256_to_f64.  Total error before that rounding < 2^-57 relative: the result is the
// correctly rounded one except within 2^-57 of a tie.  IEEE 754 pow special cases up front.  The
// oracle repeats the same steps; both are checked against Python's decimal at 60 digits.
GDV_DEV u128 gdv_mulshr127(u128 a, u128 b) {  // (a * b) >> 127, the result fits 128 bits
  const gdv_u256 p = gdv_mul_u128(a, b);
  return ((u128)p.w[3] << 65) | ((u128)p.w[2] << 1) | (u128)(p.w[1] >> 63);
}
// 2^(+-(ip + fq / 2^128)) as a 128-bit significand: value = mant * 2^(e2 - 127), mant in [2^127, 2^128)
struct gdv_bigf {
  u128 mant;
  i32 e2;
};
GDV_DEV_BIG gdv_bigf gdv_exp2_q(bool tneg, i32 ip, u128 fq) {
  i32 e2 = ip;
  if (tneg) {
    if (fq != 0) {
      e2 = -e2 - 1;
      fq = (u128)0 - fq;
    } else {
      e2 = -e2;
    }
  }
  // 2^fq = e^z, z = fq * ln 2 in Q1.127
  const u128 ln2 = ((u128)0x58b90bfbe8e7bcd5ull << 64) | (u128)0xe4f1d9cc01f97b57ull;
  const gdv_u256 zp = gdv_mul_u128(fq, ln2);
  const u128 z = ((u128)zp.w[3] << 64) | (u128)zp.w[2];
  const u128 one = (u128)1 << 127;
  u128 acc = 0;
  for (u32 n = 34u; n >= 2u; --n) acc = gdv_mulshr127(one + acc, z) / (u128)n;
  gdv_bigf r;
  r.mant = one + gdv_mulshr127(one + acc, z);  // Q1.127 in [1, 2)
  r.e2 = e2;
  return r;
}
// |t| = P * 2^-s split into its integer part (false when it is >= 1100: certain overflow / underflow)
// and the top 128 bits of its fraction; 1 <= s <= 250
GDV_DEV bool gdv_split_fixed(const gdv_u256& P, i32 s, i32* ip, u128* fq) {
  gdv_u256 ipart = P;
  bool dropped = false;
  gdv_u256_shr_sticky(ipart, s, dropped);
  if ((ipart.w[1] | ipart.w[2] | ipart.w[3]) != 0ull || ipart.w[0] >= 1100ull) return false;
  gdv_u256 fr = P;
  gdv_u256_shl(fr, 256 - s);
  *fq = ((u128)fr.w[3] << 64) | (u128)fr.w[2];
  *ip = (i32)ipart.w[0];
  return true;
}
GDV_DEV_BIG f64 power_float64_float64(f64 x, f64 y) {
  const u64 xb = gdv_f64_bits(x), yb = gdv_f64_bits(y);
  const u64 xa = xb & 0x7fffffffffffffffull, ya = yb & 0x7fffffffffffffffull;
  const u64 inf = 0x7ff0000000000000ull;
  const bool xneg = (xb >> 63) != 0ull, yneg = (yb >> 63) != 0ull;
  if (ya == 0ull || xb == 0x3ff0000000000000ull) return 1.0;  // pow(x, +-0) = pow(1, y) = 1, NaNs included
  if (xa > inf || ya > inf) return gdv_f64_from_bits(0x7ff8000000000000ull);
  // y as an integer M_y * 2^ey; is it an integer, an odd one?
  const i32 yexp = (i32)(ya >> 52);
  const u64 my = yexp == 0 ? (ya & 0x000fffffffffffffull) : ((ya & 0x000fffffffffffffull) | 0x0010000000000000ull);
  const i32 ey = (yexp == 0 ? 1 : yexp) - 1075;
  bool y_int = false, y_odd = false;
  if (ya < inf) {
    if (ey >= 0) {
      y_int = true;
      y_odd = ey == 0 && (my & 1ull) != 0ull;
    } else if (ey >= -52) {
      y_int = (my & ((1ull << (-ey)) - 1ull)) == 0ull;
      y_odd = y_int && ((my >> (-ey)) & 1ull) != 0ull;
    }
  }
  const bool res_neg = xneg && y_odd;
  if (xa == 0ull) {  // +-0
    if (yneg) return gdv_f64_from_bits((res_neg ? 0x8000000000000000ull : 0ull) | inf);
    return gdv_f64_from_bits(res_neg ? 0x8000000000000000ull : 0ull);
  }
  if (ya == inf) {
    if (xa == 0x3ff0000000000000ull) return 1.0;  // pow(-1, +-inf)
    return ((xa > 0x3ff0000000000000ull) != yneg) ? gdv_f64_from_bits(inf) : 0.0;
  }
  if (xa == inf) {
    if (yneg) return gdv_f64_from_bits(res_neg ? 0x8000000000000000ull : 0ull);
    return gdv_f64_from_bits((res_neg ? 0x8000000000000000ull : 0ull) | inf);
  }
  if (xneg && !y_int) return gdv_f64_from_bits(0x7ff8000000000000ull);
  // |x| = m * 2^k, m in [1, 2)
  const i32 xexp = (i32)(xa >> 52);
  u64 mx = xexp == 0 ? (xa & 0x000fffffffffffffull) : ((xa & 0x000fffffffffffffull) | 0x0010000000000000ull);
  i32 k = (xexp == 0 ? 1 : xexp) - 1023;
  if (xexp == 0) {
    const i32 up = __clzll((long long)mx) - 11;
    mx <<= up;
    k -= up;
  }
  u128 m = (u128)mx << 74;  // Q2.126
  u128 frac = 0;            // 120 bits of log2 m
  for (i32 i = 0; i < 120; ++i) {
    const gdv_u256 p = gdv_mul_u128(m, m);
    const u128 sq = ((u128)p.w[3] << 66) | ((u128)p.w[2] << 2) | (u128)(p.w[1] >> 62);  // >> 126: in [1, 4)
    const bool two = (sq >> 127) != 0;
    m = two ? sq >> 1 : sq;
    frac = (frac << 1) | (two ? 1u : 0u);
  }
  // |log2 |x|| = ip + fp / 2^120
  const bool lneg = k < 0;
  u64 ip = (u64)(lneg ? -k : k);
  u128 fp = frac;
  if (lneg && frac != 0) {
    ip -= 1ull;
    fp = ((u128)1 << 120) - frac;
  }
  if (ip == 0ull && fp == 0) return res_neg ? -1.0 : 1.0;  // |x| = 1
  // P = M_y * (ip * 2^120 + fp);  |y log2|x|| = P * 2^(ey - 120)
  gdv_u256 P = gdv_mul_u128((u128)my, fp);
  {
    const u64 v = my * ip;  // < 2^53 * 2^11
    gdv_u256 add;
    add.w[0] = 0ull;
    add.w[1] = v << 56;
    add.w[2] = v >> 8;
    add.w[3] = 0ull;
    P = gdv_add_u256(P, add);
  }
  const bool tneg = lneg != yneg;
  const i32 s = 120 - ey;
  if (s > 250) return res_neg ? -1.0 : 1.0;  // |t| < 2^-66
  const f64 big = gdv_f64_from_bits((res_neg ? 0x8000000000000000ull : 0ull) | (tneg ? 0ull : inf));  // overflow / underflow
  if (s <= 0) return big;
  i32 ipow = 0;
  u128 fq = 0;
  if (!gdv_split_fixed(P, s, &ipow, &fq)) return big;
  const gdv_bigf v = gdv_exp2_q(tneg, ipow, fq);
  const f64 r = gdv_u256_to_f64(gdv_u256_from(v.mant), true, v.e2 - 127);
  return res_neg ? -r : r;
}
// sinh / cosh / tanh from the same pieces: a = e^|x| and b = e^-|x| as 128-bit significands (|x| log2 e
// is an exact 53 x 127-bit product), a +- b aligned in 256 bits, tanh as their 128-bit quotient; one
// rounding at the end.  fn: 0 sinh, 1 cosh, 2 tanh
GDV_DEV_BIG f64 gdv_hyperbolic(f64 x, i32 fn) {
  const u64 xb = gdv_f64_bits(x);
  const u64 xa = xb & 0x7fffffffffffffffull;
  const bool neg = (xb >> 63) != 0ull && fn != 1;
  if (xa > 0x7ff0000000000000ull) return gdv_f64_from_bits(0x7ff8000000000000ull);
  if (xa < 0x3e30000000000000ull) return fn == 1 ? 1.0 : x;  // |x| < 2^-28
  const f64 top = fn == 2 ? 1.0 : gdv_f64_from_bits(0x7ff0000000000000ull);
  if (xa == 0x7ff0000000000000ull) return neg ? -top : top;
  const u64 mx = (xa & 0x000fffffffffffffull) | 0x0010000000000000ull;
  const i32 ex = (i32)(xa >> 52) - 1075;  // |x| = mx * 2^ex, ex >= -80 here
  const u128 log2e = ((u128)0x5c551d94ae0bf85dull << 64) | (u128)0xdf43ff68348e9f44ull;  // Q2.126
  const gdv_u256 P = gdv_mul_u128((u128)mx, log2e);  // |x| log2 e = P * 2^(ex - 126)
  const i32 s = 126 - ex;
  i32 ip = 0;
  u128 fq = 0;
  if (s <= 0 || !gdv_split_fixed(P, s, &ip, &fq)) return neg ? -top : top;
  const gdv_bigf a = gdv_exp2_q(false, ip, fq), b = gdv_exp2_q(true, ip, fq);
  // A = a.mant * 2^126, B = b aligned to it: a + b < 2^255
  gdv_u256 A, B;
  A.w[0] = 0ull;
  A.w[1] = (u64)(a.mant << 62);
  A.w[2] = (u64)(a.mant >> 2);
  A.w[3] = (u64)(a.mant >> 66);
  B.w[0] = 0ull;
  B.w[1] = (u64)(b.mant << 62);
  B.w[2] = (u64)(b.mant >> 2);
  B.w[3] = (u64)(b.mant >> 66);
  bool sticky = true;  // a and b are themselves inexact
  const i32 d = a.e2 - b.e2;
  if (d > 255) {
    B.w[0] = B.w[1] = B.w[2] = B.w[3] = 0ull;
  } else {
    gdv_u256_shr_sticky(B, d, sticky);
  }
  const gdv_u256 sum = gdv_add_u256(A, B), dif = gdv_sub_u256(A, B);
  f64 r;
  if (fn == 2) {
    // (a - b) / (a + b) from the top 128 bits of each
    gdv_u256 num, den, q, rem;
    num.w[0] = 0ull;
    num.w[1] = 0ull;
    num.w[2] = (dif.w[1] >> 63) | (dif.w[2] << 1);  // (a - b) >> 127, times 2^128
    num.w[3] = (dif.w[2] >> 63) | (dif.w[3] << 1);
    den.w[0] = (sum.w[1] >> 63) | (sum.w[2] << 1);  // (a + b) >> 127 < 2^128
    den.w[1] = (sum.w[2] >> 63) | (sum.w[3] << 1);
    den.w[2] = 0ull;
    den.w[3] = 0ull;
    gdv_divmod_u256(num, den, &q, &rem);
    r = gdv_u256_is_zero(q) ? 0.0 : gdv_u256_to_f64(q, true, -128);
  } else {
    // value = (A +- B) * 2^(a.e2 - 127 - 126) / 2
    r = gdv_u256_to_f64(fn == 1 ? sum : dif, sticky, a.e2 - 254);
  }
  return neg ? -r : r;
}
GDV_DEV f64 sinh_float64(f64 x) { return gdv_hyperbolic(x, 0); }
GDV_DEV f64 cosh_float64(f64 x) { return gdv_hyperbolic(x, 1); }
GDV_DEV f64 tanh_float64(f64 x) { return gdv_hyperbolic(x, 2); }
// ---- atan / atan2 / asin / acos: CORDIC in 128-bit integers ---------------------------------------------
// The vector (X, Y) is rotated onto the x axis through the angles atan(2^-i), i = 0..119, accumulated
// in Q2.126 (table derived by tools/derive_trig_constants.py; below i = 42 the angle is 2^-i itself):
// absolute error < 2^-118, relative < 2^-86 for the smallest angles that come here (2^-32; smaller
// ones are y / x).  asin / acos feed it (sqrt(1 - v^2), v) with the square root taken exactly
// (digit by digit) of the 248-bit integer 2^248 - V^2.  One nearest-even rounding of the 128-bit angle.
__device__ const u64 gdv_atan_tab[43][2] = {
      {0x3243f6a8885a308dull, 0x313198a2e0370734ull},
      {0x1dac670561bb4f68ull, 0xadfc88bd978751a0ull},
      {0x0fadbafc96406eb1ull, 0x56dc79ef5f7a217eull},
      {0x07f56ea6ab0bdb71ull, 0x9644bcc4f9f44477ull},
      {0x03feab76e59fbd38ull, 0xdb2c9e4b7038b835ull},
      {0x01ffd55bba97624aull, 0x84ef3aeedbb518c4ull},
      {0x00fffaaadddb94d5ull, 0xbbe78c564015f760ull},
      {0x007fff5556eeea5cull, 0xb40311a8fddf3057ull},
      {0x003fffeaaab7776eull, 0x52ec4abedadb53dfull},
      {0x001ffffd5555bbbbull, 0xa9729ab7aac08947ull},
      {0x000fffffaaaaadddull, 0xddb94b968067ef3aull},
      {0x0007fffff555556eull, 0xeeeea5ca5d895892ull},
      {0x0003fffffeaaaaabull, 0x777776e52e5356f5ull},
      {0x0001ffffffd55555ull, 0x5bbbbbba972972d0ull},
      {0x0000fffffffaaaaaull, 0xaadddddddb94b94bull},
      {0x00007fffffff5555ull, 0x5556eeeeeeea5ca5ull},
      {0x00003fffffffeaaaull, 0xaaaab77777776e52ull},
      {0x00001ffffffffd55ull, 0x555555bbbbbbbba9ull},
      {0x00000fffffffffaaull, 0xaaaaaaadddddddddull},
      {0x000007fffffffff5ull, 0x555555556eeeeeeeull},
      {0x000003fffffffffeull, 0xaaaaaaaaab777777ull},
      {0x000001ffffffffffull, 0xd5555555555bbbbbull},
      {0x000000ffffffffffull, 0xfaaaaaaaaaaaddddull},
      {0x0000007fffffffffull, 0xff555555555556eeull},
      {0x0000003fffffffffull, 0xffeaaaaaaaaaaab7ull},
      {0x0000001fffffffffull, 0xfffd555555555555ull},
      {0x0000000fffffffffull, 0xffffaaaaaaaaaaaaull},
      {0x00000007ffffffffull, 0xfffff55555555555ull},
      {0x00000003ffffffffull, 0xfffffeaaaaaaaaaaull},
      {0x00000001ffffffffull, 0xffffffd555555555ull},
      {0x00000000ffffffffull, 0xfffffffaaaaaaaaaull},
      {0x000000007fffffffull, 0xffffffff55555555ull},
      {0x000000003fffffffull, 0xffffffffeaaaaaaaull},
      {0x000000001fffffffull, 0xfffffffffd555555ull},
      {0x000000000fffffffull, 0xffffffffffaaaaaaull},
      {0x0000000007ffffffull, 0xfffffffffff55555ull},
      {0x0000000003ffffffull, 0xfffffffffffeaaaaull},
      {0x0000000001ffffffull, 0xffffffffffffd555ull},
      {0x0000000000ffffffull, 0xfffffffffffffaaaull},
      {0x00000000007fffffull, 0xffffffffffffff55ull},
      {0x00000000003fffffull, 0xffffffffffffffeaull},
      {0x00000000001fffffull, 0xfffffffffffffffdull},
      {0x00000000000fffffull, 0xffffffffffffffffull}};
GDV_DEV u128 gdv_mul_hi128(u128 a, u128 b) {
  const gdv_u256 p = gdv_mul_u128(a, b);
  return ((u128)p.w[3] << 64) | (u128)p.w[2];
}
GDV_DEV u128 gdv_mul_lo128(u128 a, u128 b) {
  const gdv_u256 p = gdv_mul_u128(a, b);
  return ((u128)p.w[1] << 64) | (u128)p.w[0];
}
// atan(y0 / x0) in Q2.126 for 0 <= x0, y0 < 2^125, not both zero
GDV_DEV_BIG i128 gdv_cordic_atan(u128 x0, u128 y0) {
  i128 X = (i128)x0, Y = (i128)y0, Z = 0;
  for (i32 i = 0; i < 120; ++i) {
    const i128 dx = X >> i, dy = Y >> i;
    const i128 a = i < 43 ? (i128)(((u128)gdv_atan_tab[i][0] << 64) | (u128)gdv_atan_tab[i][1]) : (i128)1 << (126 - i);
    if (Y > 0) {
      X += dy;
      Y -= dx;
      Z += a;
    } else {
      X -= dy;
      Y += dx;
      Z -= a;
    }
  }
  return Z < 0 ? (i128)0 : Z;
}
GDV_DEV u128 gdv_pi_q126() { return ((u128)0xc90fdaa22168c234ull << 64) | (u128)0xc4c6628b80dc1cd1ull; }
GDV_DEV f64 gdv_angle_to_f64(u128 z, bool neg) {  // Q2.126 -> double
  if (z == 0) return neg ? -0.0 : 0.0;
  const f64 r = gdv_u256_to_f64(gdv_u256_from(z), true, -126);
  return neg ? -r : r;
}
// a finite nonzero double as M * 2^e with M in [2^52, 2^53)
GDV_DEV void gdv_split_f64(u64 abits, u64* m, i32* e) {
  const i32 ex = (i32)(abits >> 52);
  u64 mm = abits & 0x000fffffffffffffull;
  i32 ee = (ex == 0 ? 1 : ex) - 1075;
  if (ex != 0) {
    mm |= 0x0010000000000000ull;
  } else {
    while ((mm >> 52) == 0ull) {
      mm <<= 1;
      --ee;
    }
  }
  *m = mm;
  *e = ee;
}
GDV_DEV_BIG f64 atan2_float64_float64(f64 y, f64 x) {
  const u64 yb = gdv_f64_bits(y), xb = gdv_f64_bits(x);
  const u64 ya = yb & 0x7fffffffffffffffull, xa = xb & 0x7fffffffffffffffull, inf = 0x7ff0000000000000ull;
  const bool yneg = (yb >> 63) != 0ull, xneg = (xb >> 63) != 0ull;
  if (ya > inf || xa > inf) return gdv_f64_from_bits(0x7ff8000000000000ull);
  const f64 pi = 3.141592653589793, pi_lo = 1.2246467991473532e-16, pio2 = 1.5707963267948966, pio2_lo = 6.123233995736766e-17;
  f64 r;
  if (ya == 0ull) r = xneg ? pi : 0.0;
  else if (xa == 0ull) r = pio2;
  else if (ya == inf) r = xa == inf ? (xneg ? 2.356194490192345 : 0.7853981633974483) : pio2;
  else if (xa == inf) r = xneg ? pi : 0.0;
  else {
    u64 my, mx;
    i32 ey, ex;
    gdv_split_f64(ya, &my, &ey);
    gdv_split_f64(xa, &mx, &ex);
    const i32 d = ey - ex;
    if (d > 70) {
      const f64 t = x / (yneg ? -y : y);  // signed, tiny
      r = pio2 + (pio2_lo - t);
    } else if (d < -32) {
      const f64 t = (yneg ? -y : y) / (xneg ? -x : x);
      r = xneg ? pi + (pi_lo - t) : t;
    } else {
      u128 X0 = (u128)mx << 71, Y0 = (u128)my << 71;
      if (d > 0) X0 >>= d;
      else Y0 >>= -d;
      u128 z = (u128)gdv_cordic_atan(X0, Y0);
      if (xneg) z = gdv_pi_q126() - z;
      r = gdv_angle_to_f64(z, false);
    }
  }
  return yneg ? -r : r;
}
GDV_DEV f64 atan_float64(f64 v) { return atan2_float64_float64(v, 1.0); }
// fn: 0 asin, 1 acos
GDV_DEV_BIG f64 gdv_asin_acos(f64 v, i32 fn) {
  const u64 vb = gdv_f64_bits(v), va = vb & 0x7fffffffffffffffull;
  const bool neg = (vb >> 63) != 0ull;
  if (va > 0x3ff0000000000000ull) return gdv_f64_from_bits(0x7ff8000000000000ull);  // |v| > 1, nan
  const f64 pi = 3.141592653589793, pio2 = 1.5707963267948966, pio2_lo = 6.123233995736766e-17;
  if (va < 0x3e10000000000000ull) return fn == 0 ? v : pio2 + (pio2_lo - v);  // |v| < 2^-30
  u64 mv;
  i32 ev;
  gdv_split_f64(va, &mv, &ev);
  const u128 V = (u128)mv << (124 + ev);  // |v| in Q0.124
  // W = 2^248 - V^2, S = floor(sqrt(W)): sqrt(1 - v^2) in Q0.124
  const u128 sq_hi = gdv_mul_hi128(V, V), sq_lo = gdv_mul_lo128(V, V);
  const u128 w_lo = (u128)0 - sq_lo;
  const u128 w_hi = ((u128)1 << 120) - sq_hi - (sq_lo != 0 ? 1u : 0u);
  u128 res = 0, rem = 0;
  for (i32 i = 123; i >= 0; --i) {
    const i32 bit = 2 * i;  // the pair (bit + 1, bit) of W
    const u128 pair = bit >= 128 ? (w_hi >> (bit - 128)) & 3u : (w_lo >> bit) & 3u;
    rem = (rem << 2) | pair;
    const u128 trial = (res << 2) | 1u;
    if (rem >= trial) {
      rem -= trial;
      res = (res << 1) | 1u;
    } else {
      res <<= 1;
    }
  }
  if (res == 0) {  // |v| = 1
    if (fn == 0) return neg ? -pio2 : pio2;
    return neg ? pi : 0.0;
  }
  if (fn == 0) return gdv_angle_to_f64((u128)gdv_cordic_atan(res, V), neg);
  u128 z = (u128)gdv_cordic_atan(V, res);
  if (neg) z = gdv_pi_q126() - z;
  return gdv_angle_to_f64(z, false);
}
GDV_DEV f64 asin_float64(f64 v) { return gdv_asin_acos(v, 0); }
GDV_DEV f64 acos_float64(f64 v) { return gdv_asin_acos(v, 1); }

// round / truncate / ceil / floor of a decimal: drop `d` = xs - rs digits under `mode` (0 half away
// from zero, 1 toward zero, 2 toward +inf, 3 toward -inf), then express the result (scale rs) at the
// declared output (op, os).  rs >= xs: nothing to drop.  More than 38 digits -> 0, like the others.
GDV_DEV_BIG i128 gdv_decimal_round_to(i128 x, i32 xs, i32 rs, i32 mode, i32 op, i32 os) {
  const bool neg = x < 0;
  gdv_u256 mag = gdv_u256_from(gdv_abs_u128(x));
  i32 cur = xs;  // scale of `mag`
  if (rs < xs) {
    const i32 d = xs - rs;
    if (d > 39) {
      mag = gdv_u256_from((u128)0);
      if ((mode == 2 && !neg && x != 0) || (mode == 3 && neg)) mag = gdv_u256_from((u128)1);
    } else if (mode == 0) {
      mag = gdv_div_pow10_round(mag, d > 38 ? 38 : d);
      if (d > 38) gdv_divmod_u256_u64(mag, 10ull);  // 10^39 > any 38-digit magnitude: 0 (half of it too)
    } else {
      bool rem_any = false;
      i32 left = d;
      while (left > 0) {
        const i32 step = left > 19 ? 19 : left;
        rem_any = (gdv_divmod_u256_u64(mag, (u64)gdv_pow10_u128(step)) != 0ull) || rem_any;
        left -= step;
      }
      if (rem_any && ((mode == 2 && !neg) || (mode == 3 && neg))) mag = gdv_add_u256(mag, gdv_u256_from((u128)1));
    }
    cur = rs;
  }
  if (os > cur) {
    bool overflow = false;
    if (mag.w[2] != 0 || mag.w[3] != 0) return (i128)0;
    mag = gdv_scale_up_u256(gdv_u256_low128(mag), os - cur, &overflow);
    if (overflow) return (i128)0;
  } else if (os < cur) {
    mag = gdv_div_pow10_round(mag, cur - os > 38 ? 38 : cur - os);
  }
  if (mag.w[2] != 0 || mag.w[3] != 0) return (i128)0;
  const u128 m = ((u128)mag.w[1] << 64) | (u128)mag.w[0];
  if (m >= gdv_pow10_u128(op)) return (i128)0;
  return (neg && m != 0) ? (i128)(~m + 1) : (i128)m;
}
GDV_DEV i128 round_decimal128(i128 x, i32 xp, i32 xs, i32 op, i32 os) { return gdv_decimal_round_to(x, xs, 0, 0, op, os); }
GDV_DEV i128 round_decimal128_int32(i128 x, i32 xp, i32 xs, i32 rs, i32 op, i32 os) {
  return gdv_decimal_round_to(x, xs, rs < -38 ? -39 : rs, 0, op, os);
}
GDV_DEV i128 truncate_decimal128(i128 x, i32 xp, i32 xs, i32 op, i32 os) { return gdv_decimal_round_to(x, xs, 0, 1, op, os); }
GDV_DEV i128 truncate_decimal128_int32(i128 x, i32 xp, i32 xs, i32 rs, i32 op, i32 os) {
  return gdv_decimal_round_to(x, xs, rs < -38 ? -39 : rs, 1, op, os);
}
GDV_DEV i128 ceil_decimal128(i128 x, i32 xp, i32 xs, i32 op, i32 os) { return gdv_decimal_round_to(x, xs, 0, 2, op, os); }
GDV_DEV i128 floor_decimal128(i128 x, i32 xp, i32 xs, i32 op, i32 os) { return gdv_decimal_round_to(x, xs, 0, 3, op, os); }
// castDECIMAL(utf8): [spaces][+-]digits[.digits][spaces] (at least one digit), rounded half away
// from zero to the declared scale; anything else raises; a value that needs more than the declared
// precision yields 0 like the other decimal producers.  Digits beyond 76 are not accumulated
// (they cannot change a 38-digit result except through the sticky rounding digit, which is kept).
GDV_DEV_BIG i128 castDECIMAL_utf8(gdv_ctx* c, gdv_str s, i32 op, i32 os) {
  i32 b = 0, e = s.len;
  while (b < e && s.p[b] == (u8)' ') ++b;
  while (e > b && s.p[e - 1] == (u8)' ') --e;
  bool neg = false;
  if (b < e && (s.p[b] == (u8)'-' || s.p[b] == (u8)'+')) {
    neg = s.p[b] == (u8)'-';
    ++b;
  }
  gdv_u256 mag = gdv_u256_from((u128)0);
  i32 digits = 0, frac = 0;  // digits seen, fractional digits accumulated into mag
  bool seen_point = false, overflow = false, ok = true;
  u32 round_digit = 0u;      // first fractional digit beyond the target scale
  bool have_round = false;
  for (i32 i = b; i < e && ok; ++i) {
    const u32 ch = (u32)s.p[i];
    if (ch == (u32)'.') {
      ok = !seen_point;
      seen_point = true;
      continue;
    }
    const u32 d = ch - (u32)'0';
    if (d > 9u) {
      ok = false;
      break;
    }
    ++digits;
    if (seen_point && frac >= os) {
      if (!have_round) {
        round_digit = d;
        have_round = true;
      }
      continue;  // digits past the rounding digit cannot matter for half-away rounding
    }
    bool o = false;
    mag = gdv_mul_u256_u128(mag, (u128)10, &o);
    overflow = overflow || o;
    mag = gdv_add_u256(mag, gdv_u256_from((u128)d));
    if (seen_point) ++frac;
  }
  if (!ok || digits == 0) {
    gdv_set_error(c, GDV_ERR_CAST_DECIMAL);
    return (i128)0;
  }
  if (frac < os) {  // fewer fractional digits than the target scale: scale up
    bool o = false;
    mag = gdv_mul_u256_u128(mag, gdv_pow10_u128(os - frac), &o);
    overflow = overflow || o;
  }
  if (have_round && round_digit >= 5u) mag = gdv_add_u256(mag, gdv_u256_from((u128)1));
  if (overflow || mag.w[2] != 0 || mag.w[3] != 0) return (i128)0;
  const u128 m = ((u128)mag.w[1] << 64) | (u128)mag.w[0];
  if (m >= gdv_pow10_u128(op)) return (i128)0;
  return (neg && m != 0) ? (i128)(~m + 1) : (i128)m;
}
// x / y at the declared output scale: |x| * 10^(os - xs + ys) / |y|, rounded half away from zero;
// y == 0 raises "divide by zero error"; a quotient of more than 38 digits yields 0.
GDV_DEV i128 divide_decimal128_decimal128(gdv_ctx* c, i128 x, i32 xp, i32 xs, i128 y, i32 yp,
                                          i32 ys, i32 op, i32 os) {
  if (y == 0) {
    gdv_set_error(c, GDV_ERR_DIV_ZERO);
    return (i128)0;
  }
  const bool neg = (x < 0) != (y < 0);
  const i32 delta = os - xs + ys;
  bool overflow = false;
  gdv_u256 num = gdv_scale_up_u256(gdv_abs_u128(x), delta > 0 ? delta : 0, &overflow);
  if (overflow) return (i128)0;  // the quotient then has more than 38 digits whatever y is
  bool o2 = false;
  const gdv_u256 den = gdv_scale_up_u256(gdv_abs_u128(y), delta < 0 ? -delta : 0, &o2);
  if (o2) return (i128)0;  // |x / den| < 1/2: rounds to 0
  gdv_u256 q, r;
  gdv_divmod_u256(num, den, &q, &r);
  // round half away from zero: 2 * r >= den
  const gdv_u256 r2 = gdv_add_u256(r, r);
  if (gdv_cmp_u256(r2, den) >= 0) q = gdv_add_u256(q, gdv_u256_from((u128)1));
  return gdv_fit_decimal(q, neg && !gdv_u256_is_zero(q));
}
// x mod y with both sides brought to the larger scale; the sign follows the dividend (C's %).
GDV_DEV i128 mod_decimal128_decimal128(gdv_ctx* c, i128 x, i32 xp, i32 xs, i128 y, i32 yp, i32 ys,
                                       i32 op, i32 os) {
  if (y == 0) {
    gdv_set_error(c, GDV_ERR_DIV_ZERO);
    return (i128)0;
  }
  const i32 ms = xs > ys ? xs : ys;
  const gdv_u256 xm = gdv_mul_u128(gdv_abs_u128(x), gdv_pow10_u128(ms - xs));
  const gdv_u256 ym = gdv_mul_u128(gdv_abs_u128(y), gdv_pow10_u128(ms - ys));
  gdv_u256 q, r;
  gdv_divmod_u256(xm, ym, &q, &r);
  if (os < ms) r = gdv_div_pow10_round(r, ms - os);
  if (os > ms) {
    if (!gdv_u256_fits128(r)) return (i128)0;
    r = gdv_mul_u128(gdv_u256_low128(r), gdv_pow10_u128(os - ms));
  }
  return gdv_fit_decimal(r, x < 0 && !gdv_u256_is_zero(r));
}
// double -> decimal(op, os): v * 10^os (the power built by repeated IEEE multiplication, as in
// castFLOAT8_decimal128), rounded half away from zero; NaN, infinities and values of more than
// `op` digits yield 0.
GDV_DEV i128 castDECIMAL_float64(f64 v, i32 op, i32 os) {
  f64 p = 1.0;
  for (i32 i = 0; i < os; ++i) p = p * 10.0;
  const f64 s = v * p;
  const f64 a = fabs(s);
  if (!(a < 1.0e38)) return (i128)0;
  f64 t = floor(a);
  if (a - t >= 0.5) t = t + 1.0;
  u128 m;
  if (t < 18446744073709551616.0) {
    m = (u128)(u64)t;
  } else {
    const u64 bits = (u64)__double_as_longlong(t);
    const i32 e = (i32)((bits >> 52) & 0x7ffull) - 1075;  // >= 12 here
    const u64 mant = (bits & 0xfffffffffffffull) | 0x10000000000000ull;
    m = (u128)mant << e;
  }
  if (m >= gdv_pow10_u128(op)) return (i128)0;
  return (s < 0.0 && m != 0) ? (i128)(~m + 1) : (i128)m;
}
GDV_DEV i128 castDECIMAL_float32(f32 v, i32 op, i32 os) { return castDECIMAL_float64((f64)v, op, os); }

// ---- hashes (MurmurHash3; numeric values are hashed as the 8 bytes of their double) ------------
// hash32 = MurmurHash3_x86_32, hash64 = the low word of MurmurHash3_x64_128.  A null input yields
// the seed (0 without one); the result is never null.
GDV_DEV u64 gdv_rotl64(u64 v, int d) { return (v << d) | (v >> (64 - d)); }
GDV_DEV u32 gdv_rotl32(u32 v, int d) { return (v << d) | (v >> (32 - d)); }
GDV_DEV u64 gdv_fmix64(u64 k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdull;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ull;
  k ^= k >> 33;
  return k;
}
GDV_DEV u32 gdv_fmix32(u32 h) {
  h ^= h >> 16;
  h *= 0x85ebca6bu;
  h ^= h >> 13;
  h *= 0xc2b2ae35u;
  h ^= h >> 16;
  return h;
}
GDV_DEV u32 gdv_mm32_k(u32 k) { return gdv_rotl32(k * 0xcc9e2d51u, 15) * 0x1b873593u; }
GDV_DEV u32 gdv_mm32_h(u32 h, u32 k) { return gdv_rotl32(h ^ gdv_mm32_k(k), 13) * 5u + 0xe6546b64u; }
GDV_DEV u64 gdv_mm64_k1(u64 k) { return gdv_rotl64(k * 0x87c37b91114253d5ull, 31) * 0x4cf5ad432745937full; }
GDV_DEV u64 gdv_mm64_k2(u64 k) { return gdv_rotl64(k * 0x4cf5ad432745937full, 33) * 0x87c37b91114253d5ull; }
// one 8-byte key
GDV_DEV u32 gdv_murmur3_32(u64 val, i32 seed) {
  u32 h = (u32)seed;
  h = gdv_mm32_h(h, (u32)val);
  h = gdv_mm32_h(h, (u32)(val >> 32));
  return gdv_fmix32(h ^ 8u);
}
GDV_DEV u64 gdv_murmur3_64(u64 val, i32 seed) {
  u64 h1 = (u64)(i64)seed, h2 = (u64)(i64)seed;
  h1 ^= gdv_mm64_k1(val);
  h1 ^= 8ull;
  h2 ^= 8ull;
  h1 += h2;
  h2 += h1;
  h1 = gdv_fmix64(h1);
  h2 = gdv_fmix64(h2);
  return h1 + h2;
}
// byte strings (through the view's case map)
GDV_DEV u32 gdv_murmur3_32_buf(const gdv_str& s, i32 seed) {
  u32 h = (u32)seed;
  const i32 nb = s.len / 4;
  for (i32 b = 0; b < nb; ++b) {
    const u32 k = (u32)gdv_ch(s, 4 * b) | ((u32)gdv_ch(s, 4 * b + 1) << 8) |
                  ((u32)gdv_ch(s, 4 * b + 2) << 16) | ((u32)gdv_ch(s, 4 * b + 3) << 24);
    h = gdv_mm32_h(h, k);
  }
  u32 k = 0u;
  const i32 t = 4 * nb;
  switch (s.len & 3) {
    case 3: k ^= (u32)gdv_ch(s, t + 2) << 16;
    case 2: k ^= (u32)gdv_ch(s, t + 1) << 8;
    case 1: k ^= (u32)gdv_ch(s, t);
            h ^= gdv_mm32_k(k);
  }
  return gdv_fmix32(h ^ (u32)s.len);
}
GDV_DEV u64 gdv_ld64_str(const gdv_str& s, i32 at, i32 n) {  // n <= 8 bytes, little endian
  u64 k = 0ull;
  for (i32 i = 0; i < n; ++i) k |= (u64)gdv_ch(s, at + i) << (8 * i);
  return k;
}
GDV_DEV u64 gdv_murmur3_64_buf(const gdv_str& s, i32 seed) {
  u64 h1 = (u64)(i64)seed, h2 = (u64)(i64)seed;
  const i32 nb = s.len / 16;
  for (i32 b = 0; b < nb; ++b) {
    h1 ^= gdv_mm64_k1(gdv_ld64_str(s, 16 * b, 8));
    h1 = (gdv_rotl64(h1, 27) + h2) * 5ull + 0x52dce729ull;
    h2 ^= gdv_mm64_k2(gdv_ld64_str(s, 16 * b + 8, 8));
    h2 = (gdv_rotl64(h2, 31) + h1) * 5ull + 0x38495ab5ull;
  }
  const i32 t = 16 * nb, rest = s.len & 15;
  if (rest > 8) h2 ^= gdv_mm64_k2(gdv_ld64_str(s, t + 8, rest - 8));
  if (rest > 0) h1 ^= gdv_mm64_k1(gdv_ld64_str(s, t, rest > 8 ? 8 : rest));
  h1 ^= (u64)(u32)s.len;
  h2 ^= (u64)(u32)s.len;
  h1 += h2;
  h2 += h1;
  h1 = gdv_fmix64(h1);
  h2 = gdv_fmix64(h2);
  return h1 + h2;
}
#define GDV_HASH_NUM(T, S)                                                                        \
  GDV_DEV i32 hash32_##S(T v, bool ok) {                                                          \
    return ok ? (i32)gdv_murmur3_32((u64)__double_as_longlong((f64)v), 0) : 0;                    \
  }                                                                                               \
  GDV_DEV i32 hash32_##S##_int32(T v, bool ok, i32 seed, bool sok) {                              \
    const i32 sd = sok ? seed : 0;                                                                \
    return ok ? (i32)gdv_murmur3_32((u64)__double_as_longlong((f64)v), sd) : sd;                  \
  }                                                                                               \
  GDV_DEV i64 hash64_##S(T v, bool ok) {                                                          \
    return ok ? (i64)gdv_murmur3_64((u64)__double_as_longlong((f64)v), 0) : 0;                    \
  }                                                                                               \
  GDV_DEV i64 hash64_##S##_int64(T v, bool ok, i64 seed, bool sok) {                              \
    const i64 sd = sok ? seed : 0;                                                                \
    return ok ? (i64)gdv_murmur3_64((u64)__double_as_longlong((f64)v), (i32)(u32)(u64)sd) : sd;   \
  }
GDV_HASH_NUM(i8, int8)
GDV_HASH_NUM(i16, int16)
GDV_HASH_NUM(i32, int32)
GDV_HASH_NUM(i64, int64)
GDV_HASH_NUM(u8, uint8)
GDV_HASH_NUM(u16, uint16)
GDV_HASH_NUM(u32, uint32)
GDV_HASH_NUM(u64, uint64)
GDV_HASH_NUM(f32, float32)
GDV_HASH_NUM(f64, float64)
GDV_HASH_NUM(bool, boolean)
GDV_HASH_NUM(i32, date32)
GDV_HASH_NUM(i64, date64)
GDV_HASH_NUM(i64, timestamp)
GDV_HASH_NUM(i32, time32)
#define GDV_HASH_STR(S)                                                                           \
  GDV_DEV i32 hash32_##S(gdv_str v, bool ok) { return ok ? (i32)gdv_murmur3_32_buf(v, 0) : 0; }   \
  GDV_DEV i32 hash32_##S##_int32(gdv_str v, bool ok, i32 seed, bool sok) {                        \
    const i32 sd = sok ? seed : 0;                                                                \
    return ok ? (i32)gdv_murmur3_32_buf(v, sd) : sd;                                              \
  }                                                                                               \
  GDV_DEV i64 hash64_##S(gdv_str v, bool ok) { return ok ? (i64)gdv_murmur3_64_buf(v, 0) : 0; }   \
  GDV_DEV i64 hash64_##S##_int64(gdv_str v, bool ok, i64 seed, bool sok) {                        \
    const i64 sd = sok ? seed : 0;                                                                \
    return ok ? (i64)gdv_murmur3_64_buf(v, (i32)(u32)(u64)sd) : sd;                               \
  }
GDV_HASH_STR(utf8)
GDV_HASH_STR(binary)

// ---- strings ---------------------------------------------------------------------------
GDV_DEV gdv_str upper_utf8(gdv_str s) {
  s.xf = (s.xf & ~GDV_XF_CASE) | 1u;
  return s;
}
GDV_DEV gdv_str lower_utf8(gdv_str s) {
  s.xf = (s.xf & ~GDV_XF_CASE) | 2u;
  return s;
}
// ---- to_date(text, format): interpreter of the program csrc/gdv_datefmt.cc compiles from the format literal.
// The rules are glibc strptime's for %Y %y %m %d %H %I %M %S %b/%B %p, white space and literal bytes; trailing
// text is allowed, the time of day is parsed but ignored, the day defaults to 1 (gdv_datefmt.h).
GDV_DEV bool gdv_fmt_space(u8 c) { return c == (u8)' ' || (u32)(c - 9u) <= 4u; }
// up to `width` digits after optional white space, stopping early when another digit would exceed `hi`
GDV_DEV bool gdv_fmt_number(const gdv_str& s, i32* pos, i32 lo, i32 hi, i32 width, i32* out) {
  i32 i = *pos;
  while (i < s.len && gdv_fmt_space(gdv_ch(s, i))) ++i;
  if (i >= s.len || (u32)(gdv_ch(s, i) - (u32)'0') > 9u) return false;
  i32 val = 0;
  do {
    val = val * 10 + (i32)(gdv_ch(s, i) - (u32)'0');
    ++i;
  } while (--width > 0 && val * 10 <= hi && i < s.len && (u32)(gdv_ch(s, i) - (u32)'0') <= 9u);
  *pos = i;
  *out = val;
  return val >= lo && val <= hi;
}
// case-insensitive match of `word` (lower case, n bytes) at s[pos..]
GDV_DEV bool gdv_fmt_word(const gdv_str& s, i32 pos, const char* word, i32 n) {
  if (pos + n > s.len) return false;
  for (i32 k = 0; k < n; ++k)
    if (((u32)gdv_ch(s, pos + k) | 0x20u) != (u32)(u8)word[k]) return false;
  return true;
}
GDV_DEV i64 gdv_to_date_fmt(gdv_ctx* c, gdv_str s, const u8* prog, i32 nprog, bool suppress, bool* ok) {
  const char names[12][10] = {"january", "february", "march", "april", "may", "june", "july", "august", "september",
                              "october", "november", "december"};
  const int name_len[12] = {7, 8, 5, 5, 3, 4, 4, 6, 9, 7, 8, 8};
  i32 pos = 0, year = 1900, mon = 1, day = 0, tmp = 0;
  bool good = true;
  for (i32 k = 0; k < nprog && good; ++k) {
    const u32 op = prog[k];
    if (op == 11u) {  // white space in the format: any run of white space in the text
      while (pos < s.len && gdv_fmt_space(gdv_ch(s, pos))) ++pos;
    } else if (op == 12u) {  // literal byte
      ++k;
      good = pos < s.len && (u32)gdv_ch(s, pos) == (u32)prog[k];
      ++pos;
    } else if (op == 1u) {
      good = gdv_fmt_number(s, &pos, 0, 9999, 4, &year);
    } else if (op == 2u) {
      good = gdv_fmt_number(s, &pos, 0, 99, 2, &tmp);
      year = tmp >= 69 ? 1900 + tmp : 2000 + tmp;
    } else if (op == 3u) {
      good = gdv_fmt_number(s, &pos, 1, 12, 2, &mon);
    } else if (op == 4u) {
      good = gdv_fmt_number(s, &pos, 1, 31, 2, &day);
    } else if (op == 5u) {
      good = gdv_fmt_number(s, &pos, 0, 23, 2, &tmp);
    } else if (op == 6u) {
      good = gdv_fmt_number(s, &pos, 1, 12, 2, &tmp);
    } else if (op == 7u) {
      good = gdv_fmt_number(s, &pos, 0, 59, 2, &tmp);
    } else if (op == 8u) {
      good = gdv_fmt_number(s, &pos, 0, 61, 2, &tmp);
    } else if (op == 9u) {  // month name, full or three letters, any case
      good = false;
      for (i32 m = 0; m < 12 && !good; ++m) {
        if (gdv_fmt_word(s, pos, names[m], name_len[m])) {
          pos += name_len[m];
          good = true;
        } else if (gdv_fmt_word(s, pos, names[m], 3)) {
          pos += 3;
          good = true;
        }
        if (good) mon = m + 1;
      }
    } else {  // AM / PM
      good = gdv_fmt_word(s, pos, "am", 2) || gdv_fmt_word(s, pos, "pm", 2);
      pos += 2;
    }
  }
  *ok = good;
  if (!good) {
    if (!suppress) gdv_set_error(c, GDV_ERR_TO_DATE);
    return 0;
  }
  if (day < 1) day = 1;
  // midnight of year / month / day; a day past the month's end runs into the next month (plain day arithmetic)
  return (gdv_days_from_civil((i64)year, mon, 1) + (i64)(day - 1)) * 86400000ll;
}

GDV_DEV gdv_str initcap_utf8(gdv_str s) {
  s.xf = (s.xf & ~GDV_XF_CASE) | 3u;
  return s;
}
GDV_DEV i32 octet_length_utf8(gdv_str s) { return s.len; }
GDV_DEV i32 octet_length_binary(gdv_str s) { return s.len; }
GDV_DEV i32 bit_length_utf8(gdv_str s) { return s.len * 8; }
GDV_DEV i32 bit_length_binary(gdv_str s) { return s.len * 8; }
GDV_DEV i32 char_length_utf8(gdv_str s) {
  if ((s.xf & GDV_XF_ASCII) != 0u) return s.len;
  i32 n = 0;
  for (i32 i = 0; i < s.len; i += gdv_glyph_len(s.p[i])) ++n;
  return n;
}
// 1-based, counts UTF-8 glyphs; offset 0 behaves as 1; negative offsets count from the end.
GDV_DEV gdv_str substr_utf8_int64_int64(gdv_str s, i64 offset, i64 length) {
  gdv_str r = s;
  if (length <= 0 || s.len <= 0) {
    r.len = 0;
    return r;
  }
  // from the first glyph and at least as many glyphs as bytes: the whole string, no scan
  if ((offset == 0 || offset == 1) && length >= (i64)s.len) return s;
  // known-ASCII row: glyph positions are byte positions, pure arithmetic
  if ((s.xf & GDV_XF_ASCII) != 0u) {
    i64 from = 0;
    if (offset > 0) from = offset - 1;
    if (offset < 0) from = (i64)s.len + offset;
    if (from < 0 || from >= (i64)s.len) {
      r.len = 0;
      return r;
    }
    const i64 rest = (i64)s.len - from;
    r.p = s.p + from;
    r.len = (i32)(length < rest ? length : rest);
    return r;
  }
  // ASCII prefix: glyph positions are byte positions
  if ((offset == 0 || offset == 1) && gdv_all_ascii(s.p, (i32)length)) {
    r.len = (i32)length;
    return r;
  }
  i64 from_glyph;
  if (offset > 0) {
    from_glyph = offset - 1;
  } else if (offset < 0) {
    from_glyph = (i64)char_length_utf8(s) + offset;
    if (from_glyph < 0) {
      r.len = 0;
      return r;
    }
  } else {
    from_glyph = 0;
  }
  i32 pos = 0;
  i64 g = 0;
  while (pos < s.len && g < from_glyph) {
    pos += gdv_glyph_len(s.p[pos]);
    ++g;
  }
  if (pos >= s.len) {
    r.len = 0;
    return r;
  }
  const i32 start = pos;
  i64 taken = 0;
  while (pos < s.len && taken < length) {
    pos += gdv_glyph_len(s.p[pos]);
    ++taken;
  }
  if (pos > s.len) pos = s.len;
  r.p = s.p + start;
  r.len = pos - start;
  return r;
}
GDV_DEV gdv_str substr_utf8_int64(gdv_str s, i64 offset) {
  return substr_utf8_int64_int64(s, offset, (i64)s.len);
}
// castVARCHAR(s, n): the first n glyphs (n <= 0: empty).
GDV_DEV gdv_str castVARCHAR_utf8_int64(gdv_str s, i64 n) { return substr_utf8_int64_int64(s, 1, n); }
GDV_DEV bool starts_with_utf8_utf8(gdv_str s, gdv_str pre) {
  if (pre.len > s.len) return false;
  for (i32 i = 0; i < pre.len; ++i)
    if (gdv_ch(s, i) != gdv_ch(pre, i)) return false;
  return true;
}
GDV_DEV bool ends_with_utf8_utf8(gdv_str s, gdv_str suf) {
  if (suf.len > s.len) return false;
  const i32 d = s.len - suf.len;
  for (i32 i = 0; i < suf.len; ++i)
    if (gdv_ch(s, d + i) != gdv_ch(suf, i)) return false;
  return true;
}
GDV_DEV bool is_substr_utf8_utf8(gdv_str s, gdv_str sub) {
  if (sub.len == 0) return true;
  for (i32 i = 0; i + sub.len <= s.len; ++i) {
    i32 j = 0;
    while (j < sub.len && gdv_ch(s, i + j) == gdv_ch(sub, j)) ++j;
    if (j == sub.len) return true;
  }
  return false;
}
GDV_DEV gdv_str ltrim_utf8(gdv_str s) {
  while (s.len > 0 && s.p[0] == (u8)' ') {
    ++s.p;
    --s.len;
  }
  return s;
}
GDV_DEV gdv_str rtrim_utf8(gdv_str s) {
  while (s.len > 0 && s.p[s.len - 1] == (u8)' ') --s.len;
  return s;
}
GDV_DEV gdv_str btrim_utf8(gdv_str s) { return rtrim_utf8(ltrim_utf8(s)); }

// ascii(s): the first byte as seen through the case map (0 for the empty string).
GDV_DEV i32 ascii_utf8(gdv_str s) { return s.len > 0 ? (i32)gdv_ch(s, 0) : 0; }
// left(s, n): the first n glyphs, n < 0: all but the last |n|; right(s, n): the last n glyphs,
// n < 0: all but the first |n|.  Views, like substr.
GDV_DEV gdv_str left_utf8_int32(gdv_str s, i32 n) {
  if (n > 0) return substr_utf8_int64_int64(s, 1, (i64)n);
  gdv_str r = s;
  r.len = 0;
  if (n == 0) return r;
  const i64 keep = (i64)char_length_utf8(s) + (i64)n;
  if (keep <= 0) return r;
  return substr_utf8_int64_int64(s, 1, keep);
}
GDV_DEV gdv_str right_utf8_int32(gdv_str s, i32 n) {
  gdv_str r = s;
  r.len = 0;
  if (n == 0) return r;
  if (n < 0) return substr_utf8_int64_int64(s, 1 - (i64)n, (i64)s.len);
  const i64 g = (i64)char_length_utf8(s);
  if ((i64)n >= g) return s;
  return substr_utf8_int64_int64(s, g - (i64)n + 1, (i64)n);
}
// locate(sub, s[, start]): 1-based glyph position of the first occurrence of sub in s at or after
// glyph `start`, 0 when there is none; the empty string is found at `start` (start < 1 raises: the
// fuser checks it with gdv_check_start before this is called).
GDV_DEV i32 locate_utf8_utf8_int32(gdv_str sub, gdv_str s, i32 start) {
  if (start < 1) return 0;
  i32 pos = 0, g = 1;
  while (pos < s.len && g < start) {
    pos += gdv_glyph_len(s.p[pos]);
    ++g;
  }
  if (g < start) return 0;  // start lies beyond the end (start == length + 1 still finds "")
  if (pos > s.len) pos = s.len;
  while (true) {
    if (pos + sub.len <= s.len) {
      i32 j = 0;
      while (j < sub.len && gdv_ch(s, pos + j) == gdv_ch(sub, j)) ++j;
      if (j == sub.len) return g;
    } else {
      return 0;
    }
    if (pos >= s.len) return 0;
    pos += gdv_glyph_len(s.p[pos]);
    ++g;
  }
}
GDV_DEV i32 locate_utf8_utf8(gdv_str sub, gdv_str s) { return locate_utf8_utf8_int32(sub, s, 1); }
GDV_DEV i32 strpos_utf8_utf8(gdv_str s, gdv_str sub) { return locate_utf8_utf8_int32(sub, s, 1); }
// byte_substr(b, offset, length): substr over bytes (1-based, offset 0 acts as 1, negative offsets
// count from the end, out-of-range -> empty).
GDV_DEV gdv_str byte_substr_binary_int32_int32(gdv_str s, i32 offset, i32 length) {
  gdv_str r = s;
  r.len = 0;
  if (length <= 0 || s.len <= 0) return r;
  i64 from = 0;
  if (offset > 0) from = (i64)offset - 1;
  if (offset < 0) from = (i64)s.len + (i64)offset;
  if (from < 0 || from >= (i64)s.len) return r;
  const i64 rest = (i64)s.len - from;
  r.p = s.p + from;
  r.len = (i32)((i64)length < rest ? (i64)length : rest);
  return r;
}
// castINT / castBIGINT of a string: optional surrounding spaces, optional sign, decimal digits;
// anything else, or a value outside the type, raises an ExecutionError.
GDV_DEV_BIG i64 gdv_parse_int(gdv_ctx* c, const gdv_str& s, i64 lo, i64 hi) {
  i32 b = 0, e = s.len;
  while (b < e && s.p[b] == (u8)' ') ++b;
  while (e > b && s.p[e - 1] == (u8)' ') --e;
  bool neg = false;
  if (b < e && (s.p[b] == (u8)'-' || s.p[b] == (u8)'+')) {
    neg = s.p[b] == (u8)'-';
    ++b;
  }
  if (b >= e) {
    gdv_set_error(c, GDV_ERR_CAST_INT);
    return 0;
  }
  const u64 limit = neg ? (u64)0 - (u64)lo : (u64)hi;  // magnitude the type can hold
  u64 v = 0;
  for (i32 i = b; i < e; ++i) {
    const u32 d = (u32)s.p[i] - (u32)'0';
    if (d > 9u || v > (limit - d) / 10ull) {
      gdv_set_error(c, GDV_ERR_CAST_INT);
      return 0;
    }
    v = v * 10ull + d;
  }
  return neg ? (i64)((u64)0 - v) : (i64)v;
}
// castBIT / castBOOLEAN of a string: surrounding spaces ignored; "true" / "false" in any case, "1", "0";
// anything else raises an ExecutionError.
GDV_DEV_BIG bool castBIT_utf8(gdv_ctx* c, gdv_str s) {
  i32 b = 0, e = s.len;
  while (b < e && s.p[b] == (u8)' ') ++b;
  while (e > b && s.p[e - 1] == (u8)' ') --e;
  const i32 n = e - b;
  if (n == 1 && (s.p[b] == (u8)'1' || s.p[b] == (u8)'0')) return s.p[b] == (u8)'1';
  if (n == 4 && (s.p[b] | 0x20) == 't' && (s.p[b + 1] | 0x20) == 'r' && (s.p[b + 2] | 0x20) == 'u' && (s.p[b + 3] | 0x20) == 'e')
    return true;
  if (n == 5 && (s.p[b] | 0x20) == 'f' && (s.p[b + 1] | 0x20) == 'a' && (s.p[b + 2] | 0x20) == 'l' && (s.p[b + 3] | 0x20) == 's' &&
      (s.p[b + 4] | 0x20) == 'e')
    return false;
  gdv_set_error(c, GDV_ERR_CAST_BOOL);
  return false;
}
// find_in_set(s, list): 1-based index of s among the comma-separated items of list, 0 when it is
// not there or s itself contains a comma
GDV_DEV_BIG i32 find_in_set_utf8_utf8(gdv_str s, gdv_str list) {
  for (i32 i = 0; i < s.len; ++i)
    if (gdv_ch(s, i) == (u8)',') return 0;
  i32 item = 1, start = 0;
  for (i32 i = 0; i <= list.len; ++i) {
    if (i == list.len || gdv_ch(list, i) == (u8)',') {
      if (i - start == s.len) {
        bool same = true;
        for (i32 k = 0; k < s.len && same; ++k) same = gdv_ch(list, start + k) == gdv_ch(s, k);
        if (same) return item;
      }
      ++item;
      start = i + 1;
    }
  }
  return 0;
}
GDV_DEV i64 castBIGINT_utf8(gdv_ctx* c, gdv_str s) {
  return gdv_parse_int(c, s, (i64)0x8000000000000000ull, 0x7fffffffffffffffll);
}
GDV_DEV i32 castINT_utf8(gdv_ctx* c, gdv_str s) { return (i32)gdv_parse_int(c, s, -2147483648ll, 2147483647ll); }

// castDATE / castTIMESTAMP of a string: [spaces] Y-M-D [(' ' | 'T') h:m[:s[.fraction]]] [spaces],
// 1..9 digit year (optional leading '-'), 1..2 digit fields, fraction truncated to milliseconds;
// month 1..12, day valid for the month (proleptic Gregorian), h < 24, m < 60, s < 60.  castDATE
// drops the time of day.  Anything else raises an ExecutionError.
GDV_DEV bool gdv_parse_uint(const gdv_str& s, i32* pos, i32 end, i32 min_digits, i32 max_digits, i64* out) {
  i64 v = 0;
  i32 n = 0;
  while (*pos < end && n < max_digits) {
    const u32 d = (u32)s.p[*pos] - (u32)'0';
    if (d > 9u) break;
    v = v * 10 + (i64)d;
    ++*pos;
    ++n;
  }
  *out = v;
  return n >= min_digits;
}
GDV_DEV_BIG i64 gdv_parse_timestamp(gdv_ctx* c, const gdv_str& s, bool date_only) {
  i32 b = 0, e = s.len;
  while (b < e && s.p[b] == (u8)' ') ++b;
  while (e > b && s.p[e - 1] == (u8)' ') --e;
  bool ok = true, neg = false;
  if (b < e && s.p[b] == (u8)'-') {
    neg = true;
    ++b;
  }
  i64 y = 0, mo = 0, d = 0, hh = 0, mi = 0, ss = 0, ms = 0;
  ok = ok && gdv_parse_uint(s, &b, e, 1, 9, &y);
  ok = ok && b < e && s.p[b] == (u8)'-';
  ++b;
  ok = ok && gdv_parse_uint(s, &b, e, 1, 2, &mo);
  ok = ok && b < e && s.p[b] == (u8)'-';
  ++b;
  ok = ok && gdv_parse_uint(s, &b, e, 1, 2, &d);
  if (ok && b < e) {
    ok = s.p[b] == (u8)' ' || s.p[b] == (u8)'T';
    ++b;
    ok = ok && gdv_parse_uint(s, &b, e, 1, 2, &hh);
    ok = ok && b < e && s.p[b] == (u8)':';
    ++b;
    ok = ok && gdv_parse_uint(s, &b, e, 1, 2, &mi);
    if (ok && b < e) {
      ok = s.p[b] == (u8)':';
      ++b;
      ok = ok && gdv_parse_uint(s, &b, e, 1, 2, &ss);
      if (ok && b < e) {
        ok = s.p[b] == (u8)'.';
        ++b;
        i32 nd = 0;
        while (b < e && (u32)s.p[b] - (u32)'0' <= 9u) {
          if (nd < 3) ms = ms * 10 + (i64)((u32)s.p[b] - (u32)'0');
          ++nd;
          ++b;
        }
        ok = ok && nd >= 1 && b == e;
        for (; nd < 3; ++nd) ms *= 10;
      }
    }
  }
  if (neg) y = -y;
  ok = ok && b >= e && mo >= 1 && mo <= 12 && d >= 1 && hh < 24 && mi < 60 && ss < 60;
  if (ok) {
    const bool leap = (y % 4 == 0) && ((y % 100 != 0) || (y % 400 == 0));
    const i32 mdays[12] = {31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31};
    ok = d <= (i64)mdays[mo - 1] + ((mo == 2 && leap) ? 1 : 0);
  }
  if (!ok) {
    gdv_set_error(c, GDV_ERR_CAST_DATE);
    return 0;
  }
  const i64 day_ms = gdv_days_to_ms(gdv_days_from_civil(y, (i32)mo, (i32)d));
  if (date_only) return day_ms;
  return day_ms + ((hh * 60 + mi) * 60 + ss) * 1000 + ms;
}
GDV_DEV i64 castDATE_utf8(gdv_ctx* c, gdv_str s) { return gdv_parse_timestamp(c, s, true); }
GDV_DEV i64 castTIMESTAMP_utf8(gdv_ctx* c, gdv_str s) { return gdv_parse_timestamp(c, s, false); }

// ltrim / rtrim / btrim(s, chars): strips glyphs that occur in `chars` (both sides compared as
// stored bytes: case maps of the operands are ignored for the set test only when they differ per
// byte, i.e. bytes are read through gdv_ch).
GDV_DEV bool gdv_glyph_in_set(const gdv_str& s, i32 at, i32 glen, const gdv_str& set) {
  for (i32 j = 0; j < set.len;) {
    const i32 sl = gdv_glyph_len(set.p[j]);
    if (sl == glen && j + sl <= set.len) {
      i32 t = 0;
      while (t < glen && gdv_ch(s, at + t) == gdv_ch(set, j + t)) ++t;
      if (t == glen) return true;
    }
    j += sl;
  }
  return false;
}
GDV_DEV gdv_str ltrim_utf8_utf8(gdv_str s, gdv_str chars) {
  i32 at = 0;
  while (at < s.len) {
    i32 gl = gdv_glyph_len(s.p[at]);
    if (at + gl > s.len) gl = s.len - at;
    if (!gdv_glyph_in_set(s, at, gl, chars)) break;
    at += gl;
  }
  s.p += at;
  s.len -= at;
  return s;
}
GDV_DEV gdv_str rtrim_utf8_utf8(gdv_str s, gdv_str chars) {
  while (s.len > 0) {
    i32 st = s.len - 1;  // start of the last glyph: skip back over continuation bytes
    while (st > 0 && (s.p[st] & 0xC0u) == 0x80u && s.len - st < 4) --st;
    i32 gl = s.len - st;
    if (gdv_glyph_len(s.p[st]) != gl) {  // malformed tail: treat the last byte as a glyph of its own
      st = s.len - 1;
      gl = 1;
    }
    if (!gdv_glyph_in_set(s, st, gl, chars)) break;
    s.len = st;
  }
  return s;
}
GDV_DEV gdv_str btrim_utf8_utf8(gdv_str s, gdv_str chars) { return rtrim_utf8_utf8(ltrim_utf8_utf8(s, chars), chars); }
// split_part(s, delimiter, k): the k-th (1-based) piece of s split at every occurrence of the
// delimiter (leftmost, non-overlapping); empty when there are fewer pieces; k < 1 raises; an empty
// delimiter never matches (the whole string is piece 1).  A view.
GDV_DEV_BIG gdv_str split_part_utf8_utf8_int32(gdv_ctx* c, gdv_str s, gdv_str delim, i32 k) {
  gdv_str r = s;
  r.len = 0;
  if (k < 1) {
    gdv_set_error(c, GDV_ERR_SPLIT_INDEX);
    return r;
  }
  i32 piece = 1, start = 0, i = 0;
  while (delim.len > 0 && i + delim.len <= s.len) {
    i32 j = 0;
    while (j < delim.len && gdv_ch(s, i + j) == gdv_ch(delim, j)) ++j;
    if (j == delim.len) {
      if (piece == k) {
        r.p = s.p + start;
        r.len = i - start;
        return r;
      }
      ++piece;
      i += delim.len;
      start = i;
    } else {
      ++i;
    }
  }
  if (piece == k) {
    r.p = s.p + start;
    r.len = s.len - start;
  }
  return r;
}
// crc32 (IEEE 802.3, reflected polynomial 0xEDB88320) of the bytes seen through the view.
GDV_DEV i64 gdv_crc32(const gdv_str& s) {
  u32 crc = 0xffffffffu;
  for (i32 i = 0; i < s.len; ++i) {
    crc ^= (u32)gdv_ch(s, i);
    for (int b = 0; b < 8; ++b) crc = (crc >> 1) ^ (0xEDB88320u & (0u - (crc & 1u)));
  }
  return (i64)(crc ^ 0xffffffffu);
}
GDV_DEV i64 crc32_utf8(gdv_str s) { return gdv_crc32(s); }
GDV_DEV i64 crc32_binary(gdv_str s) { return gdv_crc32(s); }
GDV_DEV f64 degrees_float64(f64 a) { return a * 180.0 / 3.14159265358979323846; }
GDV_DEV f64 radians_float64(f64 a) { return a * 3.14159265358979323846 / 180.0; }
// datediff(a, b): whole days between the calendar days of a and b (a - b)
GDV_DEV i32 datediff_timestamp_timestamp(i64 a, i64 b) {
  return (i32)(gdv_floordiv(a, 86400000ll) - gdv_floordiv(b, 86400000ll));
}
GDV_DEV i32 datediff_date64_date64(i64 a, i64 b) { return datediff_timestamp_timestamp(a, b); }

// ---- virtual pieces: repeat / space / lpad / rpad / reverse ----------------------------------------
// A periodic view: `total` bytes that repeat the `period` bytes at p (period < 2^20).
GDV_DEV gdv_str gdv_rep_view(const u8* p, i64 period, i64 total) {
  gdv_str r = gdv_make_str(p, 0);
  if (period <= 0 || total <= 0 || period >= (1ll << 20)) return r;
  r.len = total > 0x7fffffffll ? 0x7fffffff : (i32)total;  // > 2^31 - 1 bytes: the tile scan raises
  r.xf = GDV_XF_REP | ((u32)period << 12);
  return r;
}
__device__ const u8 gdv_one_space[1] = {' '};
GDV_DEV gdv_str repeat_utf8_int32(gdv_str s, i32 n) {
  // the case map of s travels with the piece (xf low bits), its bytes repeat
  gdv_str r = gdv_rep_view(s.p, (i64)s.len, (i64)s.len * (i64)(n > 0 ? n : 0));
  r.xf |= s.xf & (GDV_XF_CASE | GDV_XF_LOCAL);
  return r;
}
GDV_DEV gdv_str space_int32(i32 n) { return gdv_rep_view(gdv_one_space, 1, (i64)(n > 0 ? n : 0)); }
GDV_DEV gdv_str reverse_utf8(gdv_str s) {
  s.xf = (s.xf & (GDV_XF_CASE | GDV_XF_LOCAL)) | GDV_XF_REV;
  return s;
}
// lpad / rpad(s, n, fill): the result has n glyphs: s cut to n glyphs, padded with the glyphs of
// `fill` repeated cyclically (an empty fill pads nothing; n <= 0 gives the empty string).
// gdv_pad_text = the text piece, gdv_pad_fill = the padding piece (a periodic view of fill).
GDV_DEV gdv_str gdv_pad_text(gdv_str s, i32 n) {
  gdv_str r = s;
  r.len = 0;
  if (n <= 0) return r;
  return substr_utf8_int64_int64(s, 1, (i64)n);
}
GDV_DEV gdv_str gdv_pad_fill(gdv_str s, i32 n, gdv_str fill) {
  gdv_str none = gdv_make_str(fill.p, 0);
  if (n <= 0 || fill.len <= 0) return none;
  const i64 need = (i64)n - (i64)char_length_utf8(s);  // glyphs of padding
  if (need <= 0) return none;
  const i64 fg = (i64)char_length_utf8(fill);
  if (fg <= 0) return none;
  i64 bytes = (need / fg) * (i64)fill.len;
  i64 rest = need % fg;
  for (i32 pos = 0; rest > 0 && pos < fill.len; --rest) {
    const i32 gl = gdv_glyph_len(fill.p[pos]);
    bytes += gl;
    pos += gl;
  }
  gdv_str r = gdv_rep_view(fill.p, (i64)fill.len, bytes);
  r.xf |= fill.xf & (GDV_XF_CASE | GDV_XF_LOCAL);
  return r;
}
// replace(s, from, to) with literal from / to: the piece is the source view; its output length and
// bytes come from these two (leftmost, non-overlapping occurrences; an empty `from` replaces
// nothing).  Bytes are compared and copied through the view's case map.
GDV_DEV_BIG i32 gdv_replace_len(const gdv_str& s, const u8* from, i32 fl, i32 tl) {
  if (fl <= 0) return s.len;
  i64 out = 0;
  for (i32 i = 0; i < s.len;) {
    bool hit = i + fl <= s.len;
    for (i32 j = 0; hit && j < fl; ++j) hit = gdv_ch(s, i + j) == from[j];
    if (hit) {
      out += tl;
      i += fl;
    } else {
      ++out;
      ++i;
    }
  }
  return out > 0x7fffffffll ? 0x7fffffff : (i32)out;
}
GDV_DEV_BIG void gdv_replace_copy(u8* dst, const gdv_str& s, const u8* from, i32 fl, const u8* to, i32 tl) {
  i64 out = 0;
  for (i32 i = 0; i < s.len;) {
    bool hit = fl > 0 && i + fl <= s.len;
    for (i32 j = 0; hit && j < fl; ++j) hit = gdv_ch(s, i + j) == from[j];
    if (hit) {
      for (i32 j = 0; j < tl; ++j) dst[out++] = to[j];
      i += fl;
    } else {
      dst[out++] = gdv_ch(s, i);
      ++i;
    }
  }
}
GDV_DEV gdv_str gdv_repl_view(gdv_str s, u32 site) {
  s.xf = (s.xf & (GDV_XF_CASE | GDV_XF_LOCAL)) | GDV_XF_REPL | (site << 12);
  return s;
}
#ifdef GDV_HAS_REPL  /* the fuser defines both after this header, one switch over the call sites */
GDV_DEV i32 gdv_repl_len(const gdv_str& v);
GDV_DEV void gdv_repl_copy(u8* dst, const gdv_str& v);
#else
GDV_DEV i32 gdv_repl_len(const gdv_str& v) { return v.len; }
GDV_DEV void gdv_repl_copy(u8*, const gdv_str&) {}
#endif
// Output bytes of a piece (everything but replace(): the view's own length).
GDV_DEV u32 gdv_piece_len(const gdv_str& v) {
  return (v.xf & GDV_XF_REPL) != 0u ? (u32)gdv_repl_len(v) : (u32)v.len;
}
// Byte i of a piece as the string write pass sees it (periodic pieces wrap around).
GDV_DEV u8 gdv_piece_byte(const gdv_str& v, i32 i) {
  if ((v.xf & GDV_XF_REP) != 0u) i = i % (i32)(v.xf >> 12);
  return gdv_ch(v, i);
}
// Copies a glyph-reversed piece (owner lane only): glyphs from the last to the first, the bytes
// of every glyph in their own order.
GDV_DEV void gdv_copy_reversed(u8* dst, const gdv_str& v) {
  i32 out = 0;
  for (i32 end = v.len; end > 0;) {
    i32 st = end - 1;
    while (st > 0 && (v.p[st] & 0xC0u) == 0x80u && end - st < 4) --st;
    if (gdv_glyph_len(v.p[st]) != end - st) st = end - 1;  // malformed: single bytes
    for (i32 i = st; i < end; ++i) dst[out++] = gdv_ch(v, i);
    end = st;
  }
}

// ---- numbers and dates as text (castVARCHAR): bytes are produced into a thread-private slot -----
GDV_DEV gdv_str gdv_scratch_str(u8* scr, i32 len, i64 maxlen) {
  gdv_str r;
  r.p = scr;
  r.len = maxlen <= 0 ? 0 : ((i64)len > maxlen ? (i32)maxlen : len);
  r.xf = GDV_XF_ASCII | GDV_XF_LOCAL;
  return r;
}
GDV_DEV i32 gdv_put_uint(u8* scr, i32 at, u64 v, i32 min_digits) {
  u8 tmp[20];
  i32 n = 0;
  do {
    tmp[n++] = (u8)((u32)'0' + (u32)(v % 10ull));
    v /= 10ull;
  } while (v != 0ull);
  for (i32 pad = n; pad < min_digits; ++pad) scr[at++] = (u8)'0';
  while (n > 0) scr[at++] = tmp[--n];
  return at;
}
GDV_DEV gdv_str castVARCHAR_int64_int64(i64 v, i64 maxlen, u8* scr) {
  i32 at = 0;
  if (v < 0) scr[at++] = (u8)'-';
  at = gdv_put_uint(scr, at, v < 0 ? (u64)0 - (u64)v : (u64)v, 1);
  return gdv_scratch_str(scr, at, maxlen);
}
GDV_DEV gdv_str castVARCHAR_int32_int64(i32 v, i64 maxlen, u8* scr) {
  return castVARCHAR_int64_int64((i64)v, maxlen, scr);
}
// castVARCHAR(float32 / float64, n): the SHORTEST decimal digits that read back as the same value
// (nearest to it when several do), laid out the way the reference's formatter does (Java's
// Double.toString): plain notation for 10^-3 <= |v| < 10^7 with at least one digit after the point,
// otherwise d.dddE[-]x; "NaN", "Infinity", "-Infinity", "0.0", "-0.0".
// v = M * 2^e is scaled to W = v * 10^(16 - k) in [10^16, 10^17) as a 57.128 fixed-point number (the
// 19-digit stepping of gdv_parse_f64: relative error < 2^-185); the rounding interval of v is
// W -+ W / (2M) (half of that below a power of two); for p = 1, 2, ... the multiples of 10^(17 - p)
// around W are tried against that interval -- end points count when M is even, as round-to-nearest-even
// reads them.  17 digits always suffice for a double, 9 for a float.
GDV_DEV_BIG void gdv_shortest_digits(u64 M, i32 e, bool lower_half, u64* digits, i32* ndig, i32* k10) {
  const int nb = 64 - __clzll((long long)M);
  i32 k = (i32)gdv_floordiv((i64)(e + nb - 1) * 1233ll, 4096ll);  // floor(log10 v) or one less
  gdv_u256 W;
  for (;;) {
    W.w[0] = M;
    W.w[1] = 0ull;
    W.w[2] = 0ull;
    W.w[3] = 0ull;
    i32 exp2 = e;
    bool sticky = false;
    gdv_scale_pow10(W, exp2, sticky, 16 - k);
    const i32 sh = exp2 + 128;  // W * 2^128 as an integer
    if (sh >= 0) gdv_u256_shl(W, sh);
    else gdv_u256_shr_sticky(W, -sh > 255 ? 255 : -sh, sticky);
    const u128 ip = ((u128)W.w[3] << 64) | (u128)W.w[2];
    if (ip < (u128)10000000000000000ull) {
      --k;
      continue;
    }
    if (ip >= (u128)100000000000000000ull) {
      ++k;
      continue;
    }
    break;
  }
  gdv_u256 h = W;
  gdv_divmod_u256_u64(h, 2ull * M);
  gdv_u256 hlo = h;
  if (lower_half) {
    bool unused = false;
    gdv_u256_shr_sticky(hlo, 1, unused);
  }
  const gdv_u256 whi = gdv_add_u256(W, h), wlo = gdv_sub_u256(W, hlo);
  const bool even = (M & 1ull) == 0ull;  // round-to-nearest-even reads the end points of the interval back as v
  // Integer parts (< 2^58: w[3] is 0) and 128-bit fractions.  The fixed-point values carry an error of a
  // few units of 2^-128, while a boundary that does not coincide with a candidate stays more than 2^-70
  // away from it (the 124-bit bound of shortest-digit printing): anything within 2^-104 is a coincidence.
  const u64 I = W.w[2], Il = wlo.w[2], Ih = whi.w[2];
  const u128 f = ((u128)W.w[1] << 64) | (u128)W.w[0];
  const u128 fl = ((u128)wlo.w[1] << 64) | (u128)wlo.w[0], fh = ((u128)whi.w[1] << 64) | (u128)whi.w[0];
  const u128 tol = (u128)1 << 24, near_one = (u128)0 - tol;
  u64 unit = 10000000000000000ull;
  for (i32 p = 1; p <= 17; ++p, unit /= 10ull) {
    const u64 cdn = (I / unit) * unit, cup = cdn + unit;
    bool dn_ok, up_ok;
    if ((cdn == Il && fl <= tol) || (cdn == Il + 1ull && fl >= near_one)) dn_ok = even;  // on the lower boundary
    else dn_ok = cdn > Il;
    if ((cup == Ih && fh <= tol) || (cup == Ih + 1ull && fh >= near_one)) up_ok = even;  // on the upper boundary
    else up_ok = cup <= Ih;
    if (!dn_ok && !up_ok) continue;
    u64 pick = dn_ok ? cdn : cup;
    if (dn_ok && up_ok) {
      // distances W - cdn and cup - W as (integer, 128-bit fraction)
      const u64 a_i = I - cdn;
      const u64 b_i = f == 0 ? cup - I : cup - I - 1ull;
      const u128 b_f = (u128)0 - f;
      const bool tie = a_i == b_i && (f > b_f ? f - b_f : b_f - f) <= tol;
      const bool up_closer = b_i < a_i || (b_i == a_i && b_f < f);
      if (tie ? ((cdn / unit) & 1ull) != 0ull : up_closer) pick = cup;
    }
    if (pick == 100000000000000000ull) {
      *digits = 1ull;
      *ndig = 1;
      *k10 = k + 1;
    } else {
      *digits = pick / unit;
      *ndig = p;
      *k10 = k;
    }
    return;
  }
  *digits = I;  // not reached: 17 digits always fit
  *ndig = 17;
  *k10 = k;
}
GDV_DEV_BIG i32 gdv_put_float(u8* scr, bool neg, u64 M, i32 e, bool lower_half) {
  u64 digits = 0ull;
  i32 nd = 0, k = 0;
  gdv_shortest_digits(M, e, lower_half, &digits, &nd, &k);
  u8 d[20];
  for (i32 i = nd - 1; i >= 0; --i) {
    d[i] = (u8)((u32)'0' + (u32)(digits % 10ull));
    digits /= 10ull;
  }
  i32 at = 0;
  if (neg) scr[at++] = (u8)'-';
  if (k >= -3 && k < 7) {
    if (k >= 0) {
      for (i32 i = 0; i <= k; ++i) scr[at++] = i < nd ? d[i] : (u8)'0';
      scr[at++] = (u8)'.';
      if (nd > k + 1) {
        for (i32 i = k + 1; i < nd; ++i) scr[at++] = d[i];
      } else {
        scr[at++] = (u8)'0';
      }
    } else {
      scr[at++] = (u8)'0';
      scr[at++] = (u8)'.';
      for (i32 i = 0; i < -k - 1; ++i) scr[at++] = (u8)'0';
      for (i32 i = 0; i < nd; ++i) scr[at++] = d[i];
    }
  } else {
    scr[at++] = d[0];
    scr[at++] = (u8)'.';
    if (nd > 1) {
      for (i32 i = 1; i < nd; ++i) scr[at++] = d[i];
    } else {
      scr[at++] = (u8)'0';
    }
    scr[at++] = (u8)'E';
    if (k < 0) scr[at++] = (u8)'-';
    at = gdv_put_uint(scr, at, (u64)(k < 0 ? -k : k), 1);
  }
  return at;
}
GDV_DEV i32 gdv_put_text(u8* scr, i32 at, const char* t, i32 n) {
  for (i32 i = 0; i < n; ++i) scr[at++] = (u8)t[i];
  return at;
}
GDV_DEV_BIG gdv_str castVARCHAR_float64_int64(f64 v, i64 maxlen, u8* scr) {
  const u64 b = gdv_f64_bits(v), a = b & 0x7fffffffffffffffull;
  const bool neg = (b >> 63) != 0ull;
  i32 at = 0;
  if (a > 0x7ff0000000000000ull) {
    at = gdv_put_text(scr, 0, "NaN", 3);
  } else if (a == 0x7ff0000000000000ull) {
    if (neg) scr[at++] = (u8)'-';
    at = gdv_put_text(scr, at, "Infinity", 8);
  } else if (a == 0ull) {
    if (neg) scr[at++] = (u8)'-';
    at = gdv_put_text(scr, at, "0.0", 3);
  } else {
    const i32 ex = (i32)(a >> 52);
    const u64 frac = a & 0x000fffffffffffffull;
    const u64 M = ex == 0 ? frac : (frac | 0x0010000000000000ull);
    at = gdv_put_float(scr, neg, M, (ex == 0 ? 1 : ex) - 1075, frac == 0ull && ex > 1);
  }
  return gdv_scratch_str(scr, at, maxlen);
}
GDV_DEV_BIG gdv_str castVARCHAR_float32_int64(f32 v, i64 maxlen, u8* scr) {
  const u32 b = (u32)__float_as_int(v), a = b & 0x7fffffffu;
  const bool neg = (b >> 31) != 0u;
  i32 at = 0;
  if (a > 0x7f800000u) {
    at = gdv_put_text(scr, 0, "NaN", 3);
  } else if (a == 0x7f800000u) {
    if (neg) scr[at++] = (u8)'-';
    at = gdv_put_text(scr, at, "Infinity", 8);
  } else if (a == 0u) {
    if (neg) scr[at++] = (u8)'-';
    at = gdv_put_text(scr, at, "0.0", 3);
  } else {
    const i32 ex = (i32)(a >> 23);
    const u32 frac = a & 0x007fffffu;
    const u64 M = ex == 0 ? (u64)frac : (u64)(frac | 0x00800000u);
    at = gdv_put_float(scr, neg, M, (ex == 0 ? 1 : ex) - 150, frac == 0u && ex > 1);
  }
  return gdv_scratch_str(scr, at, maxlen);
}
// castVARCHAR(decimal(p, s), n): [-]integer digits[.s fractional digits], then the first n characters
GDV_DEV_BIG gdv_str castVARCHAR_decimal128_int64(i128 x, i32 xp, i32 xs, i64 maxlen, u8* scr) {
  u8 tmp[40];
  i32 n = 0;
  u128 m = gdv_abs_u128(x);
  do {
    tmp[n++] = (u8)((u32)'0' + (u32)(m % 10u));
    m /= 10u;
  } while (m != 0u);
  while (n <= xs) tmp[n++] = (u8)'0';  // at least one digit before the point
  i32 at = 0;
  if (x < 0) scr[at++] = (u8)'-';
  for (i32 k = n - 1; k >= 0; --k) {
    scr[at++] = tmp[k];
    if (k == xs && xs > 0) scr[at++] = (u8)'.';
  }
  return gdv_scratch_str(scr, at, maxlen);
}
// to_hex(int): upper-case hexadecimal digits of the two's-complement bits, no leading zeros
GDV_DEV gdv_str gdv_to_hex(u64 v, u8* scr) {
  i32 n = 0;
  u8 tmp[16];
  do {
    const u32 d = (u32)(v & 15ull);
    tmp[n++] = (u8)(d < 10u ? (u32)'0' + d : (u32)'A' + d - 10u);
    v >>= 4;
  } while (v != 0ull);
  i32 at = 0;
  while (n > 0) scr[at++] = tmp[--n];
  return gdv_scratch_str(scr, at, 64);
}
GDV_DEV gdv_str to_hex_int64(i64 v, u8* scr) { return gdv_to_hex((u64)v, scr); }
GDV_DEV gdv_str to_hex_int32(i32 v, u8* scr) { return gdv_to_hex((u64)(u32)v, scr); }
// "YYYY-MM-DD" (years outside 0..9999: a leading '-' and / or more digits)
GDV_DEV i32 gdv_put_date(u8* scr, i64 days) {
  const gdv_ymd c = gdv_civil_from_days(days);
  i32 at = 0;
  if (c.y < 0) scr[at++] = (u8)'-';
  at = gdv_put_uint(scr, at, c.y < 0 ? (u64)0 - (u64)c.y : (u64)c.y, 4);
  scr[at++] = (u8)'-';
  at = gdv_put_uint(scr, at, (u64)c.m, 2);
  scr[at++] = (u8)'-';
  return gdv_put_uint(scr, at, (u64)c.d, 2);
}
GDV_DEV gdv_str castVARCHAR_date64_int64(i64 ms, i64 maxlen, u8* scr) {
  return gdv_scratch_str(scr, gdv_put_date(scr, gdv_floordiv(ms, 86400000ll)), maxlen);
}
// "YYYY-MM-DD hh:mm:ss.mmm"
GDV_DEV_BIG gdv_str castVARCHAR_timestamp_int64(i64 ms, i64 maxlen, u8* scr) {
  const i64 days = gdv_floordiv(ms, 86400000ll);
  const i64 in_day = (i64)((u64)ms - (u64)gdv_days_to_ms(days));
  i32 at = gdv_put_date(scr, days);
  scr[at++] = (u8)' ';
  at = gdv_put_uint(scr, at, (u64)(in_day / 3600000ll), 2);
  scr[at++] = (u8)':';
  at = gdv_put_uint(scr, at, (u64)((in_day / 60000ll) % 60), 2);
  scr[at++] = (u8)':';
  at = gdv_put_uint(scr, at, (u64)((in_day / 1000ll) % 60), 2);
  scr[at++] = (u8)'.';
  at = gdv_put_uint(scr, at, (u64)(in_day % 1000ll), 3);
  return gdv_scratch_str(scr, at, maxlen);
}
__device__ const u8 gdv_true_false[9] = {'t', 'r', 'u', 'e', 'f', 'a', 'l', 's', 'e'};
GDV_DEV gdv_str castVARCHAR_boolean_int64(bool v, i64 maxlen) {
  gdv_str r = gdv_make_str(v ? gdv_true_false : gdv_true_false + 4, v ? 4 : 5);
  if (maxlen <= 0) r.len = 0;
  else if ((i64)r.len > maxlen) r.len = (i32)maxlen;
  r.xf = GDV_XF_ASCII;
  return r;
}

// ---- message digests as lower-case hex text: hashMD5 / hashSHA1 / hashSHA256 (RFC 1321, FIPS 180-4) --
// Byte `pos` of the padded message: the text, 0x80, zeros, then the bit length in the last 8 bytes
// (little endian for MD5, big endian for SHA).
GDV_DEV u32 gdv_md_byte(const gdv_str& s, i64 pos, i64 padded, bool big_endian_len) {
  if (pos < (i64)s.len) return (u32)gdv_ch(s, (i32)pos);
  if (pos == (i64)s.len) return 0x80u;
  if (pos < padded - 8) return 0u;
  const u64 bits = (u64)s.len * 8ull;
  const int k = (int)(pos - (padded - 8));  // 0..7
  return (u32)((bits >> (big_endian_len ? 8 * (7 - k) : 8 * k)) & 0xffull);
}
GDV_DEV i32 gdv_put_hex32(u8* scr, i32 at, u32 v, bool big_endian) {
  for (int b = 0; b < 4; ++b) {
    const u32 byte = big_endian ? (v >> (24 - 8 * b)) & 0xffu : (v >> (8 * b)) & 0xffu;
    const u32 hi = byte >> 4, lo = byte & 15u;
    scr[at++] = (u8)(hi < 10u ? (u32)'0' + hi : (u32)'a' + hi - 10u);
    scr[at++] = (u8)(lo < 10u ? (u32)'0' + lo : (u32)'a' + lo - 10u);
  }
  return at;
}
__device__ const u32 gdv_sha256_k[64] = {
    0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u,
    0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u,
    0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau,
    0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u,
    0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u,
    0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u,
    0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u,
    0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u};
GDV_DEV u32 gdv_rotr32(u32 v, int d) { return (v >> d) | (v << (32 - d)); }
GDV_DEV_BIG gdv_str gdv_sha256_hex(const gdv_str& s, u8* scr) {
  u32 h[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
  const i64 padded = (((i64)s.len + 8) / 64 + 1) * 64;
  for (i64 blk = 0; blk < padded; blk += 64) {
    u32 w[16];
    for (int t = 0; t < 16; ++t) {
      u32 x = 0u;
      for (int b = 0; b < 4; ++b) x = (x << 8) | gdv_md_byte(s, blk + 4 * t + b, padded, true);
      w[t] = x;
    }
    u32 a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
    for (int t = 0; t < 64; ++t) {
      if (t >= 16) {
        const u32 w15 = w[(t + 1) & 15], w2 = w[(t + 14) & 15];
        const u32 s0 = gdv_rotr32(w15, 7) ^ gdv_rotr32(w15, 18) ^ (w15 >> 3);
        const u32 s1 = gdv_rotr32(w2, 17) ^ gdv_rotr32(w2, 19) ^ (w2 >> 10);
        w[t & 15] = w[t & 15] + s0 + w[(t + 9) & 15] + s1;
      }
      const u32 S1 = gdv_rotr32(e, 6) ^ gdv_rotr32(e, 11) ^ gdv_rotr32(e, 25);
      const u32 ch = (e & f) ^ (~e & g);
      const u32 t1 = hh + S1 + ch + gdv_sha256_k[t] + w[t & 15];
      const u32 S0 = gdv_rotr32(a, 2) ^ gdv_rotr32(a, 13) ^ gdv_rotr32(a, 22);
      const u32 mj = (a & b) ^ (a & c) ^ (b & c);
      const u32 t2 = S0 + mj;
      hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
  }
  i32 at = 0;
  for (int k = 0; k < 8; ++k) at = gdv_put_hex32(scr, at, h[k], true);
  return gdv_scratch_str(scr, at, 64);
}
GDV_DEV_BIG gdv_str gdv_sha1_hex(const gdv_str& s, u8* scr) {
  u32 h[5] = {0x67452301u, 0xefcdab89u, 0x98badcfeu, 0x10325476u, 0xc3d2e1f0u};
  const i64 padded = (((i64)s.len + 8) / 64 + 1) * 64;
  for (i64 blk = 0; blk < padded; blk += 64) {
    u32 w[16];
    for (int t = 0; t < 16; ++t) {
      u32 x = 0u;
      for (int b = 0; b < 4; ++b) x = (x << 8) | gdv_md_byte(s, blk + 4 * t + b, padded, true);
      w[t] = x;
    }
    u32 a = h[0], b = h[1], c = h[2], d = h[3], e = h[4];
    for (int t = 0; t < 80; ++t) {
      if (t >= 16) {
        const u32 x = w[(t + 13) & 15] ^ w[(t + 8) & 15] ^ w[(t + 2) & 15] ^ w[t & 15];
        w[t & 15] = (x << 1) | (x >> 31);
      }
      u32 f, k;
      if (t < 20) { f = (b & c) | (~b & d); k = 0x5a827999u; }
      else if (t < 40) { f = b ^ c ^ d; k = 0x6ed9eba1u; }
      else if (t < 60) { f = (b & c) | (b & d) | (c & d); k = 0x8f1bbcdcu; }
      else { f = b ^ c ^ d; k = 0xca62c1d6u; }
      const u32 tmp = ((a << 5) | (a >> 27)) + f + e + k + w[t & 15];
      e = d; d = c; c = (b << 30) | (b >> 2); b = a; a = tmp;
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e;
  }
  i32 at = 0;
  for (int k = 0; k < 5; ++k) at = gdv_put_hex32(scr, at, h[k], true);
  return gdv_scratch_str(scr, at, 64);
}
__device__ const u8 gdv_md5_s[64] = {7, 12, 17, 22, 7, 12, 17, 22, 7, 12, 17, 22, 7, 12, 17, 22, 5, 9, 14, 20, 5, 9,
                                     14, 20, 5, 9, 14, 20, 5, 9, 14, 20, 4, 11, 16, 23, 4, 11, 16, 23, 4, 11, 16, 23,
                                     4, 11, 16, 23, 6, 10, 15, 21, 6, 10, 15, 21, 6, 10, 15, 21, 6, 10, 15, 21};
__device__ const u32 gdv_md5_k[64] = {
    0xd76aa478u, 0xe8c7b756u, 0x242070dbu, 0xc1bdceeeu, 0xf57c0fafu, 0x4787c62au, 0xa8304613u, 0xfd469501u,
    0x698098d8u, 0x8b44f7afu, 0xffff5bb1u, 0x895cd7beu, 0x6b901122u, 0xfd987193u, 0xa679438eu, 0x49b40821u,
    0xf61e2562u, 0xc040b340u, 0x265e5a51u, 0xe9b6c7aau, 0xd62f105du, 0x02441453u, 0xd8a1e681u, 0xe7d3fbc8u,
    0x21e1cde6u, 0xc33707d6u, 0xf4d50d87u, 0x455a14edu, 0xa9e3e905u, 0xfcefa3f8u, 0x676f02d9u, 0x8d2a4c8au,
    0xfffa3942u, 0x8771f681u, 0x6d9d6122u, 0xfde5380cu, 0xa4beea44u, 0x4bdecfa9u, 0xf6bb4b60u, 0xbebfbc70u,
    0x289b7ec6u, 0xeaa127fau, 0xd4ef3085u, 0x04881d05u, 0xd9d4d039u, 0xe6db99e5u, 0x1fa27cf8u, 0xc4ac5665u,
    0xf4292244u, 0x432aff97u, 0xab9423a7u, 0xfc93a039u, 0x655b59c3u, 0x8f0ccc92u, 0xffeff47du, 0x85845dd1u,
    0x6fa87e4fu, 0xfe2ce6e0u, 0xa3014314u, 0x4e0811a1u, 0xf7537e82u, 0xbd3af235u, 0x2ad7d2bbu, 0xeb86d391u};
GDV_DEV_BIG gdv_str gdv_md5_hex(const gdv_str& s, u8* scr) {
  u32 h[4] = {0x67452301u, 0xefcdab89u, 0x98badcfeu, 0x10325476u};
  const i64 padded = (((i64)s.len + 8) / 64 + 1) * 64;
  for (i64 blk = 0; blk < padded; blk += 64) {
    u32 m[16];
    for (int t = 0; t < 16; ++t) {
      u32 x = 0u;
      for (int b = 3; b >= 0; --b) x = (x << 8) | gdv_md_byte(s, blk + 4 * t + b, padded, false);
      m[t] = x;
    }
    u32 a = h[0], b = h[1], c = h[2], d = h[3];
    for (int t = 0; t < 64; ++t) {
      u32 f;
      int g;
      if (t < 16) { f = (b & c) | (~b & d); g = t; }
      else if (t < 32) { f = (d & b) | (~d & c); g = (5 * t + 1) & 15; }
      else if (t < 48) { f = b ^ c ^ d; g = (3 * t + 5) & 15; }
      else { f = c ^ (b | ~d); g = (7 * t) & 15; }
      const u32 x = a + f + gdv_md5_k[t] + m[g];
      const int r = (int)gdv_md5_s[t];
      a = d; d = c; c = b; b = b + ((x << r) | (x >> (32 - r)));
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d;
  }
  i32 at = 0;
  for (int k = 0; k < 4; ++k) at = gdv_put_hex32(scr, at, h[k], false);
  return gdv_scratch_str(scr, at, 64);
}
GDV_DEV gdv_str hashSHA256_utf8(gdv_str s, u8* scr) { return gdv_sha256_hex(s, scr); }
GDV_DEV gdv_str hashSHA256_binary(gdv_str s, u8* scr) { return gdv_sha256_hex(s, scr); }
GDV_DEV gdv_str hashSHA1_utf8(gdv_str s, u8* scr) { return gdv_sha1_hex(s, scr); }
GDV_DEV gdv_str hashSHA1_binary(gdv_str s, u8* scr) { return gdv_sha1_hex(s, scr); }
GDV_DEV gdv_str hashMD5_utf8(gdv_str s, u8* scr) { return gdv_md5_hex(s, scr); }
GDV_DEV gdv_str hashMD5_binary(gdv_str s, u8* scr) { return gdv_md5_hex(s, scr); }

// SQL LIKE over a pattern tokenised at Make(): each token is (kind << 8) | byte with
// kind 0 = literal byte, 1 = '_' (exactly one glyph), 2 = '%' (any run of glyphs).
// Iterative matcher with single-level backtracking to the last '%'.
GDV_DEV bool gdv_like_match(const gdv_str& s, const u16* pat, i32 m) {
  i32 i = 0, j = 0, star_j = -1, star_i = 0;
  const i32 n = s.len;
  while (i < n) {
    if (j < m) {
      const u32 tok = pat[j];
      const u32 kind = tok >> 8;
      if (kind == 2u) {
        star_j = j++;
        star_i = i;
        continue;
      }
      if (kind == 1u) {
        i += gdv_glyph_len(s.p[i]);
        if (i > n) i = n;
        ++j;
        continue;
      }
      if (gdv_ch(s, i) == (u8)(tok & 0xffu)) {
        ++i;
        ++j;
        continue;
      }
    }
    if (star_j < 0) return false;
    star_i += gdv_glyph_len(s.p[star_i]);
    if (star_i > n) return false;
    i = star_i;
    j = star_j + 1;
  }
  while (j < m && (pat[j] >> 8) == 2u) ++j;
  return j == m;
}

// regexp_matches: the position automaton built at Make() (gdv_regex.h), run bit-parallel.  `live` holds
// the positions whose byte was just read; the next set is the union of their follow sets (plus the
// start positions wherever a match may begin) restricted to the positions that accept the next byte.
// prog: [0] first, [1] last, [2] flags (1 matches "", 2 '^', 4 '$'), [3..66] follow, [67..322] classes.
GDV_DEV_BIG bool gdv_regex_match(const gdv_str& s, const u64* prog) {
  const u64 first = prog[0], last = prog[1], flags = prog[2];
  const bool at_start = (flags & 2ull) != 0ull, at_end = (flags & 4ull) != 0ull;
  if ((flags & 1ull) != 0ull && (!at_start || !at_end || s.len == 0)) return true;
  u64 live = 0ull;
  for (i32 i = 0; i < s.len; ++i) {
    u64 next = (i == 0 || !at_start) ? first : 0ull;
    for (u64 t = live; t != 0ull; t &= t - 1ull) next |= prog[3 + (__ffsll((long long)t) - 1)];
    live = next & prog[67 + (u32)gdv_ch(s, i)];
    if (!at_end && (live & last) != 0ull) return true;
    if (at_start && live == 0ull) return false;
  }
  return (live & last) != 0ull;
}

// The same automaton with up to 128 positions (two words per set).
// prog: [0..1] first, [2..3] last, [4] flags, [5..260] follow (128 x 2), [261..772] classes (256 x 2).
GDV_DEV_BIG bool gdv_regex_match2(const gdv_str& s, const u64* prog) {
  const u64 flags = prog[4];
  const bool at_start = (flags & 2ull) != 0ull, at_end = (flags & 4ull) != 0ull;
  if ((flags & 1ull) != 0ull && (!at_start || !at_end || s.len == 0)) return true;
  u64 l0 = 0ull, l1 = 0ull;
  for (i32 i = 0; i < s.len; ++i) {
    const bool start = i == 0 || !at_start;
    u64 n0 = start ? prog[0] : 0ull, n1 = start ? prog[1] : 0ull;
    for (u64 t = l0; t != 0ull; t &= t - 1ull) {
      const i32 k = __ffsll((long long)t) - 1;
      n0 |= prog[5 + 2 * k];
      n1 |= prog[6 + 2 * k];
    }
    for (u64 t = l1; t != 0ull; t &= t - 1ull) {
      const i32 k = 64 + __ffsll((long long)t) - 1;
      n0 |= prog[5 + 2 * k];
      n1 |= prog[6 + 2 * k];
    }
    const u32 c = (u32)gdv_ch(s, i);
    l0 = n0 & prog[261 + 2 * c];
    l1 = n1 & prog[262 + 2 * c];
    if (!at_end && ((l0 & prog[2]) | (l1 & prog[3])) != 0ull) return true;
    if (at_start && (l0 | l1) == 0ull) return false;
  }
  return ((l0 & prog[2]) | (l1 & prog[3])) != 0ull;
}

// Largest row r in [lo, n) with offs[r] <= pos, given offs[lo] <= pos < offs[n] (Arrow int32
// offsets are non-decreasing): gallop from `lo`, then bisect.  Used by the key-scan string filter
// to map a byte position of the data buffer back to its row.
GDV_DEV i64 gdv_row_of_byte(const i32* offs, i64 lo, i64 n, i64 pos) {
  i64 step = 32, hi = lo + step;
  while (hi < n && (i64)__ldg(offs + hi) <= pos) {
    lo = hi;
    step <<= 1;
    hi = lo + step;
  }
  if (hi > n) hi = n;
  while (hi - lo > 1) {
    const i64 mid = (lo + hi) >> 1;
    if ((i64)__ldg(offs + mid) <= pos) lo = mid;
    else hi = mid;
  }
  return lo;
}

// ---- ordered stream compaction: decoupled look-back over CTA tiles ------------------------
// One 64-bit descriptor per tile: flag (2 bits) | count (62 bits).  A tile publishes its own
// count (AGGREGATE), looks back over its predecessors until it finds an INCLUSIVE prefix,
// then publishes its own inclusive prefix.  Tiles are handed out by a global ticket so every
// predecessor of a running tile has already started (no dependence on CTA scheduling order).
#define GDV_TILE_INVALID 0ull
#define GDV_TILE_AGGREGATE 1ull
#define GDV_TILE_INCLUSIVE 2ull
#define GDV_TILE_VALUE_MASK 0x3fffffffffffffffull
#ifndef GDV_HOST_EMU
GDV_DEV u64 gdv_ld_relaxed(const u64* p) {
  u64 v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
GDV_DEV void gdv_st_relaxed(u64* p, u64 v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
#endif
// Called by all 32 lanes of one warp.  Returns the exclusive prefix of `tile` (sum of the
// counts of tiles 0..tile-1) in every lane and publishes this tile's inclusive prefix.
GDV_DEV u64 gdv_tile_exclusive_prefix(u64* state, i64 tile, u64 count, u32 lane) {
  if (tile == 0) {
    if (lane == 0) gdv_st_relaxed(&state[0], (GDV_TILE_INCLUSIVE << 62) | count);
    return 0ull;
  }
  if (lane == 0) gdv_st_relaxed(&state[tile], (GDV_TILE_AGGREGATE << 62) | count);
  u64 excl = 0ull;
  i64 look = tile - 1;
  while (true) {
    const i64 idx = look - (i64)lane;
    u64 d = (GDV_TILE_INCLUSIVE << 62);  // tiles before 0 contribute an inclusive prefix of 0
    if (idx >= 0) d = gdv_ld_relaxed(&state[idx]);
    // Lane 0 holds the nearest predecessor.  Only the descriptors up to the nearest INCLUSIVE one
    // are needed: wait while one of THOSE is still unpublished, not for the whole window.
    u32 incl, first;
    while (true) {
      const u32 inv = __ballot_sync(GDV_FULL, (d >> 62) == GDV_TILE_INVALID);
      incl = __ballot_sync(GDV_FULL, (d >> 62) == GDV_TILE_INCLUSIVE);
      first = incl != 0u ? (u32)(__ffs((int)incl) - 1) : 32u;
      const u32 need = first >= 32u ? inv : (inv & ((1u << first) - 1u));
      if (need == 0u) break;
      if (idx >= 0 && (d >> 62) == GDV_TILE_INVALID) d = gdv_ld_relaxed(&state[idx]);
    }
    u64 contrib = (lane <= first) ? (d & GDV_TILE_VALUE_MASK) : 0ull;
    for (int o = 16; o > 0; o >>= 1) contrib += __shfl_xor_sync(GDV_FULL, contrib, o);
    excl += contrib;
    if (incl != 0u) break;
    look -= 32;
  }
  if (lane == 0) gdv_st_relaxed(&state[tile], (GDV_TILE_INCLUSIVE << 62) | (excl + count));
  return excl;
}
