// Host stand-in for <cuda_runtime.h>, used ONLY to compile pytorch_volumetric_b200/csrc/pvb_device.cuh with g++ for
// the CPU-tier tests (tests/test_hostsim.py).  It supplies the few vector types and intrinsics the device header
// uses, each with the IEEE semantics of the CUDA intrinsic it replaces, so that the DEVICE SOURCE ITSELF -- not a
// re-implementation -- can be checked against the reference's golden vectors without a GPU.  Test infrastructure:
// nothing in the product includes this file.
//
// Differences from the GPU that remain (and why the CPU tests keep the GPU tests' tolerances rather than asking for
// bit equality of floating-point results): nvcc contracts a*b+c into FMA where g++ (-ffp-contract=off) does not,
// and rsqrtf is MUFU.RSQ (<= 2 ulp) on the device but correctly rounded here.  Integer results (voxel keys, in-range
// masks, face ids, crossing parity) do not depend on either.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

#define __device__
#define __host__
#define __global__
// Every translation unit of tests/hostsim is linked into one library: the header's functions get internal linkage, so
// each unit keeps its own copy (hostsim.cpp's PVB_STAT hook included) instead of the linker picking one of them.
#define __forceinline__ static inline
#define __noinline__ static __attribute__((noinline))

struct float2 { float x, y; };
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(16) int4 { int x, y, z, w; };
struct uchar4 { unsigned char x, y, z, w; };
struct alignas(16) longlong2 { long long x, y; };
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
static inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }

template <class T> static inline T __ldg(const T *p) { return *p; }

// round-to-nearest single operations that the compiler must not fuse or re-associate
static inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
static inline float __fsub_rn(float a, float b) { volatile float r = a - b; return r; }
static inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
static inline float __fdiv_rn(float a, float b) { volatile float r = a / b; return r; }
static inline double __ddiv_rn(double a, double b) { volatile double r = a / b; return r; }
static inline int __float_as_int(float f) { int i; std::memcpy(&i, &f, 4); return i; }
static inline float __int_as_float(int i) { float f; std::memcpy(&f, &i, 4); return f; }
static inline float rsqrtf(float x) { return 1.0f / std::sqrt(x); }

static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
static inline long long min(long long a, long long b) { return a < b ? a : b; }
static inline long long max(long long a, long long b) { return a > b ? a : b; }
