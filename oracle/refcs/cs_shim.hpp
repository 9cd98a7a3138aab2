// cs_shim.hpp -- just enough of C#, Unity.Mathematics, Unity.Collections and UnityEngine, in C++, for the REFERENCE
// IMPORTER'S OWN packing code (package/Editor/GaussianSplatAssetCreator.cs and the helpers it calls, read where it lies
// under /root/reference and rewritten by build_ref_cs.py) to compile with g++ and run on the CPU.  TEST INFRASTRUCTURE
// ONLY: the result, oracle/_ref/libref_cs.so, exists to pin the asset packers (csrc/asset_creator.cpp, csrc/gs_pack.cu)
// against the reference's code itself.  Nothing here includes or restates code of csrc/.
//
// What is the reference's and what is this file's: every expression, constant, operation order and branch of the packing
// comes from the reference source.  This file supplies the third-party semantics that source relies on, each stated once:
//   - Unity.Mathematics 1.2.6 (the version package.json pins): math.min / max / clamp / saturate / sign / abs / rcp /
//     rsqrt / normalize / dot, math.f32tof16, math.pow / exp / sqrt, math.SQRT2, half / half3 / half4 from float;
//   - Unity.Collections 2.1.4: NativeArray<T> as a pointer and a length, Sort(comparer);
//   - C#'s unchecked float -> uint / ulong / ushort conversion (ECMA-334 §10.3.2: truncation toward zero when the result
//     fits; otherwise the result is unspecified).  `conv` counts every out-of-range operand in `g_conv_events`, so that
//     the harness can mark the bytes it produced as convention, not reference truth; the value it returns then (NaN -> 0,
//     otherwise saturated to the target range) is the convention the packers follow, not something the reference fixes.
//   - Burst compiles the jobs: integer and IEEE float32 arithmetic are the IL's (compile with -ffp-contract=off); the
//     transcendental calls below are the managed implementations, which Burst may replace with its own (see DESIGN.md §6).
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <stdexcept>
#include <type_traits>
#include <utility>

namespace cs {

typedef uint8_t byte;
typedef uint16_t ushort;
typedef uint32_t uint;
typedef uint64_t ulong;

constexpr float float_PositiveInfinity = std::numeric_limits<float>::infinity();
constexpr float float_NegativeInfinity = -std::numeric_limits<float>::infinity();

struct ArgumentOutOfRangeException : std::out_of_range {
  template <class... A> ArgumentOutOfRangeException(const char *what, A...) : std::out_of_range(what) {}
};
#define nameof(x) #x

inline uint asuint(float f) { uint u; std::memcpy(&u, &f, 4); return u; }
inline float asfloat(uint u) { float f; std::memcpy(&f, &u, 4); return f; }

// ---- C# unchecked float -> unsigned integer conversion ----
extern thread_local long g_conv_events;
template <class T, class S> T conv(S x) {
  if constexpr (std::is_floating_point<S>::value) {
    const double lim = std::ldexp(1.0, 8 * (int)sizeof(T));
    if (x > -1.0 && x < lim) return (T)x;   // in range: truncation toward zero
    ++g_conv_events;                         // unspecified in C#: a convention, counted
    if (x != x || x < 0) return 0;
    return std::numeric_limits<T>::max();
  } else {
    return (T)x;                             // integer -> integer: two's complement truncation, as in C#
  }
}

// ---- Unity.Mathematics vectors (component order and size as in memory: float3 is 12 bytes) ----
struct float2 { float x, y; float2() : x(0), y(0) {} float2(float a, float b) : x(a), y(b) {} };
struct float3;
struct float4;
struct float3 {
  float x, y, z;
  float3() : x(0), y(0), z(0) {}
  float3(float s) : x(s), y(s), z(s) {}
  float3(float a, float b, float c) : x(a), y(b), z(c) {}
  float &operator[](int i) { return (&x)[i]; }
  float operator[](int i) const { return (&x)[i]; }
};
struct float4 {
  float x, y, z, w;
  float4() : x(0), y(0), z(0), w(0) {}
  float4(float s) : x(s), y(s), z(s), w(s) {}
  float4(float a, float b, float c, float d) : x(a), y(b), z(c), w(d) {}
  float4(const float3 &a, float d) : x(a.x), y(a.y), z(a.z), w(d) {}
  float &operator[](int i) { return (&x)[i]; }
  float operator[](int i) const { return (&x)[i]; }
  float3 xyz() const { return float3(x, y, z); }
  float4 yzwx() const { return float4(y, z, w, x); }
  float4 xzwy() const { return float4(x, z, w, y); }
  float4 xywz() const { return float4(x, y, w, z); }
};
struct uint2 { uint x, y; uint2(uint a, uint b) : x(a), y(b) {} };
struct uint3 {
  uint x, y, z;
  uint3(uint a, uint b, uint c) : x(a), y(b), z(c) {}
  explicit uint3(const float3 &v) : x(conv<uint>(v.x)), y(conv<uint>(v.y)), z(conv<uint>(v.z)) {}   // (uint3) float3
};
static_assert(sizeof(float3) == 12 && sizeof(float4) == 16 && sizeof(float2) == 8, "Unity.Mathematics layouts");

#define CS_VEC_OPS(V, N)                                                                                              \
  inline V operator+(const V &a, const V &b) { V r; for (int i = 0; i < N; ++i) r[i] = a[i] + b[i]; return r; }     \
  inline V operator-(const V &a, const V &b) { V r; for (int i = 0; i < N; ++i) r[i] = a[i] - b[i]; return r; }     \
  inline V operator*(const V &a, const V &b) { V r; for (int i = 0; i < N; ++i) r[i] = a[i] * b[i]; return r; }     \
  inline V operator/(const V &a, const V &b) { V r; for (int i = 0; i < N; ++i) r[i] = a[i] / b[i]; return r; }     \
  inline V operator+(const V &a, float s) { V r; for (int i = 0; i < N; ++i) r[i] = a[i] + s; return r; }           \
  inline V operator-(const V &a, float s) { V r; for (int i = 0; i < N; ++i) r[i] = a[i] - s; return r; }           \
  inline V operator*(const V &a, float s) { V r; for (int i = 0; i < N; ++i) r[i] = a[i] * s; return r; }           \
  inline V operator*(float s, const V &a) { V r; for (int i = 0; i < N; ++i) r[i] = s * a[i]; return r; }           \
  inline V operator/(float s, const V &a) { V r; for (int i = 0; i < N; ++i) r[i] = s / a[i]; return r; }
CS_VEC_OPS(float3, 3)
CS_VEC_OPS(float4, 4)

// ---- UnityEngine: Vector3 converts to and from float3 implicitly (same three floats); Quaternion is (x, y, z, w) ----
typedef float3 Vector3;
struct Quaternion { float x, y, z, w; Quaternion() : x(0), y(0), z(0), w(0) {} Quaternion(float a, float b, float c, float d) : x(a), y(b), z(c), w(d) {} };

namespace math {
constexpr float SQRT2 = 1.41421356237309504880f;   // (float)SQRT2_DBL
// min / max: `float.IsNaN(y) || x < y ? x : y` -- a NaN second operand is ignored, and of two equal values (+0 / -0)
// the SECOND is returned
inline float min(float x, float y) { return (std::isnan(y) || x < y) ? x : y; }
inline float max(float x, float y) { return (std::isnan(y) || x > y) ? x : y; }
inline int min(int x, int y) { return x < y ? x : y; }
inline int max(int x, int y) { return x > y ? x : y; }
inline float clamp(float v, float lo, float hi) { return max(lo, min(hi, v)); }
inline float saturate(float x) { return clamp(x, 0.0f, 1.0f); }   // hence saturate(NaN) = 1
inline float abs(float x) { return asfloat(asuint(x) & 0x7FFFFFFFu); }
inline float sign(float x) { return (x > 0.0f ? 1.0f : 0.0f) - (x < 0.0f ? 1.0f : 0.0f); }
inline float rcp(float x) { return 1.0f / x; }
// the managed bodies: double-precision System.Math narrowed to float
inline float sqrt(float x) { return (float)std::sqrt((double)x); }
inline float rsqrt(float x) { return 1.0f / sqrt(x); }
inline float exp(float x) { return (float)std::exp((double)x); }
inline float pow(float x, float y) { return (float)std::pow((double)x, (double)y); }
inline float dot(const float4 &a, const float4 &b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }
inline float4 normalize(const float4 &x) { return rsqrt(dot(x, x)) * x; }
#define CS_MATH_VEC(V, N)                                                                                            \
  inline V min(const V &a, const V &b) { V r; for (int i = 0; i < N; ++i) r[i] = min(a[i], b[i]); return r; }      \
  inline V max(const V &a, const V &b) { V r; for (int i = 0; i < N; ++i) r[i] = max(a[i], b[i]); return r; }      \
  inline V saturate(const V &a) { V r; for (int i = 0; i < N; ++i) r[i] = saturate(a[i]); return r; }              \
  inline V abs(const V &a) { V r; for (int i = 0; i < N; ++i) r[i] = abs(a[i]); return r; }                        \
  inline V exp(const V &a) { V r; for (int i = 0; i < N; ++i) r[i] = exp(a[i]); return r; }                        \
  inline V pow(const V &a, const V &b) { V r; for (int i = 0; i < N; ++i) r[i] = pow(a[i], b[i]); return r; }
CS_MATH_VEC(float3, 3)
CS_MATH_VEC(float4, 4)
// f32tof16: keep the top 10 mantissa bits after adding half of bit 12's weight -- round half UP on the dropped bits,
// not to nearest even; overflow -> inf, NaN -> quiet NaN 0x7e00, sign copied
inline uint f32tof16(float x) {
  const int infinity_32 = 255 << 23;
  const uint msk = 0x7FFFF000u;
  uint ux = asuint(x);
  uint uux = ux & msk;
  uint h = (uint)(asuint(min(asfloat(uux) * 1.92592994e-34f, 260042752.0f)) + 0x1000) >> 13;
  if ((int)uux >= infinity_32) h = ((int)uux > infinity_32) ? 0x7e00u : 0x7c00u;
  return h | (ux & ~msk) >> 16;
}
}  // namespace math

// half(float): `value = (ushort)math.f32tof16(v)`; half3 / half4 from float3 / float4 convert each component so
struct half { ushort value; half() : value(0) {} explicit half(float v) : value((ushort)math::f32tof16(v)) {} };
struct half3 { half x, y, z; half3() {} explicit half3(const float3 &v) : x(v.x), y(v.y), z(v.z) {} };
struct half4 { half x, y, z, w; half4() {} explicit half4(const float4 &v) : x(v.x), y(v.y), z(v.z), w(v.w) {} };
static_assert(sizeof(half3) == 6 && sizeof(half4) == 8, "half layouts");

// ---- Unity.Collections ----
enum class Allocator { Temp, TempJob, Persistent };
struct UnsafeUtility { template <class T> static int SizeOf() { return (int)sizeof(T); } };
template <class T> struct NativeArray {
  T *m_Ptr = nullptr;
  int Length = 0;
  bool IsCreated = false;
  bool m_Owned = false;
  NativeArray() {}
  NativeArray(T *p, int n) : m_Ptr(p), Length(n), IsCreated(true) {}                                  // a view of caller memory
  NativeArray(int n, Allocator) : m_Ptr(new T[n]()), Length(n), IsCreated(true), m_Owned(true) {}     // zero-cleared, as by default
  NativeArray(const NativeArray &src, Allocator) : NativeArray(src.Length, Allocator::TempJob) { std::copy(src.m_Ptr, src.m_Ptr + src.Length, m_Ptr); }
  NativeArray(const NativeArray &) = default;
  NativeArray &operator=(const NativeArray &) = default;
  T &operator[](int i) const { return m_Ptr[i]; }
  void *GetUnsafePtr() const { return m_Ptr; }
  void Dispose() { if (m_Owned) delete[] m_Ptr; m_Ptr = nullptr; IsCreated = false; }
  // NativeSortExtension.Sort: an unstable sort; the comparers it is given here order every pair strictly
  template <class C> void Sort(C c) { std::sort(m_Ptr, m_Ptr + Length, [&](const T &a, const T &b) { return c.Compare(a, b) < 0; }); }
};

// Unity.Jobs: IJobParallelFor.Schedule(n, batch).Complete() runs Execute(0 .. n-1); every job here writes disjoint outputs
template <class J> void RunParallelFor(J &job, int n) { for (int i = 0; i < n; ++i) job.Execute(i); }

}  // namespace cs
