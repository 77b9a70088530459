// Element types and reduction functors shared by the CPU shared-memory backend
// (g++) and the sm_90a kernels (nvcc).  Everything is header-only and
// host/device clean.
//
// Covers the reference's 12-op table (csrc/extension.cpp:204-252) over the
// reference's 7 dtypes (csrc/extension.cpp:106-129) plus bf16/f16/bool.
// 16-bit floats accumulate in fp32 (the NVLS path uses .acc::f32 to match).
#pragma once
#include <cstdint>
#include <cstring>
#include "common.h"

#if defined(__CUDACC__)
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#define M4T_HD __host__ __device__ __forceinline__
#else
#define M4T_HD inline
#endif

namespace m4t {

// ---- 16-bit float <-> fp32 (bit exact, RNE, NaN preserving) ---------------
M4T_HD float bf16_bits_to_float(uint16_t b) {
  uint32_t u = static_cast<uint32_t>(b) << 16;
  float f;
#if defined(__CUDA_ARCH__)
  f = __uint_as_float(u);
#else
  std::memcpy(&f, &u, 4);
#endif
  return f;
}

M4T_HD uint16_t float_to_bf16_bits(float f) {
  uint32_t u;
#if defined(__CUDA_ARCH__)
  u = __float_as_uint(f);
#else
  std::memcpy(&u, &f, 4);
#endif
  if ((u & 0x7fffffffu) > 0x7f800000u) return static_cast<uint16_t>((u >> 16) | 0x0040u);  // NaN
  uint32_t lsb = (u >> 16) & 1u;
  u += 0x7fffu + lsb;
  return static_cast<uint16_t>(u >> 16);
}

M4T_HD float f16_bits_to_float(uint16_t h) {
#if defined(__CUDA_ARCH__)
  return __half2float(__ushort_as_half(h));
#else
  uint32_t sign = (static_cast<uint32_t>(h) & 0x8000u) << 16;
  uint32_t exp = (h >> 10) & 0x1fu;
  uint32_t man = h & 0x3ffu;
  uint32_t u;
  if (exp == 0) {
    if (man == 0) {
      u = sign;
    } else {  // subnormal: renormalise
      int e = -1;
      do { man <<= 1; ++e; } while ((man & 0x400u) == 0);
      man &= 0x3ffu;
      u = sign | (static_cast<uint32_t>(127 - 15 - e) << 23) | (man << 13);
    }
  } else if (exp == 31) {
    u = sign | 0x7f800000u | (man << 13);
  } else {
    u = sign | ((exp + 112u) << 23) | (man << 13);
  }
  float f;
  std::memcpy(&f, &u, 4);
  return f;
#endif
}

M4T_HD uint16_t float_to_f16_bits(float f) {
#if defined(__CUDA_ARCH__)
  return __half_as_ushort(__float2half_rn(f));
#else
  uint32_t u;
  std::memcpy(&u, &f, 4);
  uint32_t sign = (u >> 16) & 0x8000u;
  uint32_t absu = u & 0x7fffffffu;
  if (absu > 0x7f800000u) return static_cast<uint16_t>(sign | 0x7e00u);          // NaN
  if (absu >= 0x477ff000u) return static_cast<uint16_t>(sign | 0x7c00u);         // overflow -> inf
  if (absu < 0x33000001u) return static_cast<uint16_t>(sign);                    // underflow -> 0
  int32_t exp = static_cast<int32_t>(absu >> 23) - 127;
  uint32_t man = (absu & 0x7fffffu) | 0x800000u;
  uint32_t shift, out;
  if (exp < -14) {  // subnormal half
    shift = static_cast<uint32_t>(13 + (-14 - exp));
    out = 0;
  } else {
    shift = 13;
    out = static_cast<uint32_t>(exp + 15 - 1) << 10;  // implicit bit adds the final +1
  }
  uint32_t q = man >> shift;
  uint32_t rem = man & ((1u << shift) - 1u);
  uint32_t half = 1u << (shift - 1);
  if (rem > half || (rem == half && (q & 1u))) ++q;
  return static_cast<uint16_t>(sign | (out + q));
#endif
}

// ---- Element traits --------------------------------------------------------
template <DType D> struct Elem;

#define M4T_NATIVE_ELEM(DT, T, A)                                   \
  template <> struct Elem<DT> {                                     \
    using storage = T;                                              \
    using acc = A;                                                  \
    static constexpr bool is_float = false;                         \
    static M4T_HD acc load(storage v) { return static_cast<acc>(v); } \
    static M4T_HD storage store(acc v) { return static_cast<storage>(v); } \
  };
M4T_NATIVE_ELEM(DType::U8, uint8_t, uint32_t)
M4T_NATIVE_ELEM(DType::I8, int8_t, int32_t)
M4T_NATIVE_ELEM(DType::I16, int16_t, int32_t)
M4T_NATIVE_ELEM(DType::I32, int32_t, int32_t)
M4T_NATIVE_ELEM(DType::I64, int64_t, int64_t)
#undef M4T_NATIVE_ELEM

template <> struct Elem<DType::BOOL> {
  using storage = uint8_t;
  using acc = uint32_t;
  static constexpr bool is_float = false;
  static M4T_HD acc load(storage v) { return v ? 1u : 0u; }
  static M4T_HD storage store(acc v) { return v ? 1 : 0; }
};
template <> struct Elem<DType::F32> {
  using storage = float;
  using acc = float;
  static constexpr bool is_float = true;
  static M4T_HD acc load(storage v) { return v; }
  static M4T_HD storage store(acc v) { return v; }
};
template <> struct Elem<DType::F64> {
  using storage = double;
  using acc = double;
  static constexpr bool is_float = true;
  static M4T_HD acc load(storage v) { return v; }
  static M4T_HD storage store(acc v) { return v; }
};
template <> struct Elem<DType::BF16> {
  using storage = uint16_t;
  using acc = float;
  static constexpr bool is_float = true;
  static M4T_HD acc load(storage v) { return bf16_bits_to_float(v); }
  static M4T_HD storage store(acc v) { return float_to_bf16_bits(v); }
};
template <> struct Elem<DType::F16> {
  using storage = uint16_t;
  using acc = float;
  static constexpr bool is_float = true;
  static M4T_HD acc load(storage v) { return f16_bits_to_float(v); }
  static M4T_HD storage store(acc v) { return float_to_f16_bits(v); }
};

// ---- Reduction functors over the accumulation type --------------------------
template <ReduceOp OP, typename A, bool IS_FLOAT> struct Combine;

template <typename A, bool F> struct Combine<ReduceOp::MAX, A, F> {
  static M4T_HD A apply(A a, A b) { return (b > a || b != b) ? b : a; }  // NaN propagates
};
template <typename A, bool F> struct Combine<ReduceOp::MIN, A, F> {
  static M4T_HD A apply(A a, A b) { return (b < a || b != b) ? b : a; }
};
template <typename A, bool F> struct Combine<ReduceOp::SUM, A, F> {
  static M4T_HD A apply(A a, A b) { return a + b; }
};
template <typename A, bool F> struct Combine<ReduceOp::PROD, A, F> {
  static M4T_HD A apply(A a, A b) { return a * b; }
};
template <typename A, bool F> struct Combine<ReduceOp::LAND, A, F> {
  static M4T_HD A apply(A a, A b) { return static_cast<A>((a != A(0)) && (b != A(0))); }
};
template <typename A, bool F> struct Combine<ReduceOp::LOR, A, F> {
  static M4T_HD A apply(A a, A b) { return static_cast<A>((a != A(0)) || (b != A(0))); }
};
template <typename A, bool F> struct Combine<ReduceOp::LXOR, A, F> {
  static M4T_HD A apply(A a, A b) { return static_cast<A>((a != A(0)) != (b != A(0))); }
};
template <typename A> struct Combine<ReduceOp::BAND, A, false> {
  static M4T_HD A apply(A a, A b) { return a & b; }
};
template <typename A> struct Combine<ReduceOp::BOR, A, false> {
  static M4T_HD A apply(A a, A b) { return a | b; }
};
template <typename A> struct Combine<ReduceOp::BXOR, A, false> {
  static M4T_HD A apply(A a, A b) { return a ^ b; }
};
// Bitwise ops on floats are rejected by check_op_dtype(); these keep the
// dispatch tables total without instantiating invalid expressions.
template <typename A> struct Combine<ReduceOp::BAND, A, true> {
  static M4T_HD A apply(A a, A) { return a; }
};
template <typename A> struct Combine<ReduceOp::BOR, A, true> {
  static M4T_HD A apply(A a, A) { return a; }
};
template <typename A> struct Combine<ReduceOp::BXOR, A, true> {
  static M4T_HD A apply(A a, A) { return a; }
};

// Single-operand normalisation so that P == 1 reductions agree with P > 1
// (logical ops map any non-zero value to 1).
template <ReduceOp OP, typename A> M4T_HD A normalise_single(A a) {
  if (OP == ReduceOp::LAND || OP == ReduceOp::LOR || OP == ReduceOp::LXOR)
    return static_cast<A>(a != A(0));
  return a;
}

// Run `F<DT, OP>::run(args...)` for runtime (dt, op).
#define M4T_DISPATCH_OP(OPV, DT, FUNCTOR, ...)                                         \
  switch (OPV) {                                                                       \
    case ReduceOp::MAX: FUNCTOR<DT, ReduceOp::MAX>::run(__VA_ARGS__); break;           \
    case ReduceOp::MIN: FUNCTOR<DT, ReduceOp::MIN>::run(__VA_ARGS__); break;           \
    case ReduceOp::SUM: FUNCTOR<DT, ReduceOp::SUM>::run(__VA_ARGS__); break;           \
    case ReduceOp::PROD: FUNCTOR<DT, ReduceOp::PROD>::run(__VA_ARGS__); break;         \
    case ReduceOp::LAND: FUNCTOR<DT, ReduceOp::LAND>::run(__VA_ARGS__); break;         \
    case ReduceOp::BAND: FUNCTOR<DT, ReduceOp::BAND>::run(__VA_ARGS__); break;         \
    case ReduceOp::LOR: FUNCTOR<DT, ReduceOp::LOR>::run(__VA_ARGS__); break;           \
    case ReduceOp::BOR: FUNCTOR<DT, ReduceOp::BOR>::run(__VA_ARGS__); break;           \
    case ReduceOp::LXOR: FUNCTOR<DT, ReduceOp::LXOR>::run(__VA_ARGS__); break;         \
    case ReduceOp::BXOR: FUNCTOR<DT, ReduceOp::BXOR>::run(__VA_ARGS__); break;         \
    default: throw std::invalid_argument("mpi4torch_b200: Collective operation not supported!"); \
  }

#define M4T_DISPATCH_DTYPE_OP(DTV, OPV, FUNCTOR, ...)                                   \
  switch (DTV) {                                                                        \
    case DType::U8: M4T_DISPATCH_OP(OPV, DType::U8, FUNCTOR, __VA_ARGS__) break;        \
    case DType::I8: M4T_DISPATCH_OP(OPV, DType::I8, FUNCTOR, __VA_ARGS__) break;        \
    case DType::I16: M4T_DISPATCH_OP(OPV, DType::I16, FUNCTOR, __VA_ARGS__) break;      \
    case DType::I32: M4T_DISPATCH_OP(OPV, DType::I32, FUNCTOR, __VA_ARGS__) break;      \
    case DType::I64: M4T_DISPATCH_OP(OPV, DType::I64, FUNCTOR, __VA_ARGS__) break;      \
    case DType::F32: M4T_DISPATCH_OP(OPV, DType::F32, FUNCTOR, __VA_ARGS__) break;      \
    case DType::F64: M4T_DISPATCH_OP(OPV, DType::F64, FUNCTOR, __VA_ARGS__) break;      \
    case DType::BF16: M4T_DISPATCH_OP(OPV, DType::BF16, FUNCTOR, __VA_ARGS__) break;    \
    case DType::F16: M4T_DISPATCH_OP(OPV, DType::F16, FUNCTOR, __VA_ARGS__) break;      \
    case DType::BOOL: M4T_DISPATCH_OP(OPV, DType::BOOL, FUNCTOR, __VA_ARGS__) break;    \
    default: throw std::invalid_argument("mpi4torch_b200: unsupported dtype");          \
  }

}  // namespace m4t
