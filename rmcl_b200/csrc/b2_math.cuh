// b2_math.cuh -- device-side rmagine-compatible math with EXPLICIT rounding (no compiler FMA contraction on parity paths).
//
// Two families, mirroring the oracle's conventions (oracle/oracle.c header):
//  * "rmagine-level" math (quaternion products, Transform algebra, P2L, PF error): individually rounded mul/add in the
//    reference's left-to-right expression order  -> __fmul_rn / __fadd_rn / __fsub_rn, which nvcc never fuses.
//  * ray/triangle math (our stand-in for Embree's closest hit): explicit __fmaf_rn chains.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/rmcl_b200.h"

// B2_DEV functions are host+device so that tests/emul can run the SAME traversal/math code on the CPU (test harness only;
// the product library instantiates them in __global__ kernels, and on the host only in b2_pf_sample_cloud's loop over a host cloud,
// which api.cu compiles with -ffp-contract=off like the harness).
#define B2_DEV __host__ __device__ __forceinline__
#if defined(__CUDA_ARCH__)
#define B2_ON_DEVICE 1
#else
#define B2_ON_DEVICE 0
#include <cmath>
#include <cstring>
#endif

struct V3 { float x, y, z; };
struct Q4 { float x, y, z, w; };
struct Tf { Q4 R; V3 t; };

#if B2_ON_DEVICE
B2_DEV float mul(float a, float b) { return __fmul_rn(a, b); }
B2_DEV float add(float a, float b) { return __fadd_rn(a, b); }
B2_DEV float sub(float a, float b) { return __fsub_rn(a, b); }
B2_DEV float dvd(float a, float b) { return __fdiv_rn(a, b); }
B2_DEV float fma_rn(float a, float b, float c) { return __fmaf_rn(a, b, c); }
B2_DEV float sqrt_rn(float a) { return __fsqrt_rn(a); }
B2_DEV uint32_t f2u(float a) { return __float_as_uint(a); }
B2_DEV float u2f(uint32_t a) { return __uint_as_float(a); }
B2_DEV int clz32(uint32_t a) { return __clz((int)a); }
B2_DEV int popc32(uint32_t a) { return __popc(a); }
template <typename T> B2_DEV T ldg(const T* p) { return __ldg(p); }
B2_DEV void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
B2_DEV uint32_t byte_perm(uint32_t x, uint32_t y, uint32_t s) { return __byte_perm(x, y, s); }
// PRMT with an IMMEDIATE selector and the second operand in a register (nvcc otherwise folds the constant operand into the
// immediate slot and materialises every selector with a MOV)
template <int SEL> __device__ __forceinline__ uint32_t prmt_imm(uint32_t x, uint32_t y)
{
    uint32_t d; asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(x), "r"(y), "n"(SEL)); return d;
}
__device__ __forceinline__ uint32_t opaque_const(uint32_t v) { uint32_t d; asm("mov.b32 %0, %1;" : "=r"(d) : "r"(v)); return d; }
#else   // host emulation: compiled with -ffp-contract=off, so plain ops are individually rounded
B2_DEV float mul(float a, float b) { return a * b; }
B2_DEV float add(float a, float b) { return a + b; }
B2_DEV float sub(float a, float b) { return a - b; }
B2_DEV float dvd(float a, float b) { return a / b; }
B2_DEV float fma_rn(float a, float b, float c) { return std::fmaf(a, b, c); }
B2_DEV float sqrt_rn(float a) { return std::sqrt(a); }
B2_DEV uint32_t f2u(float a) { uint32_t u; memcpy(&u, &a, 4); return u; }
B2_DEV float u2f(uint32_t a) { float f; memcpy(&f, &a, 4); return f; }
B2_DEV int clz32(uint32_t a) { return a ? __builtin_clz(a) : 32; }
B2_DEV int popc32(uint32_t a) { return __builtin_popcount(a); }
template <typename T> B2_DEV T ldg(const T* p) { return *p; }
B2_DEV void prefetch_l1(const void*) {}
template <int SEL> inline uint32_t prmt_imm(uint32_t x, uint32_t y);
inline uint32_t opaque_const(uint32_t v) { return v; }
B2_DEV uint32_t byte_perm(uint32_t x, uint32_t y, uint32_t s)
{
    const uint64_t v = ((uint64_t)y << 32) | x; uint32_t r = 0;
    for (int i = 0; i < 4; i++) r |= (uint32_t)((v >> (8 * ((s >> (4 * i)) & 7))) & 0xff) << (8 * i);
    return r;
}
template <int SEL> inline uint32_t prmt_imm(uint32_t x, uint32_t y) { return byte_perm(x, y, (uint32_t)SEL); }
#endif

// FP64, individually rounded on both sides (atan2: CUDA's double atan2 on the device, libm's on the host)
#if B2_ON_DEVICE
B2_DEV double mul_d(double a, double b) { return __dmul_rn(a, b); }
B2_DEV double add_d(double a, double b) { return __dadd_rn(a, b); }
B2_DEV double sqrt_d(double a) { return __dsqrt_rn(a); }
B2_DEV double atan2_d(double y, double x) { return ::atan2(y, x); }
#else
B2_DEV double mul_d(double a, double b) { return a * b; }
B2_DEV double add_d(double a, double b) { return a + b; }
B2_DEV double sqrt_d(double a) { return std::sqrt(a); }
B2_DEV double atan2_d(double y, double x) { return std::atan2(y, x); }
#endif
// FP64 library sine and cosine (CUDA's on the device, libm's on the host), for the Stein step's half-angle
#if B2_ON_DEVICE
B2_DEV double sin_d(double a) { return ::sin(a); }
B2_DEV double cos_d(double a) { return ::cos(a); }
#else
B2_DEV double sin_d(double a) { return std::sin(a); }
B2_DEV double cos_d(double a) { return std::cos(a); }
#endif
B2_DEV float rint_f(float a)
{
#if B2_ON_DEVICE
    return rintf(a);
#else
    return std::nearbyint(a);                // round half to even, like rintf on the device
#endif
}

// exp in FP32, every operation individually rounded and the FMAs explicit, so the device and the host compute the same bits.  Cody-Waite
// reduction x = j ln2 + r (j = rint(x log2 e), ln2 split in a 16-bit-mantissa head and a tail, |r| <= 0.3466), Taylor polynomial of degree 7
// in Horner form (truncation below 6e-9 relative), then two exact power-of-two scalings 2^(j/2) 2^(j - j/2), the second one rounding into the
// subnormal range where the result lies there.  Within 2 ulp of exp(x) in float64 for x < 88.72 (tests/test_pf_stein.py); NaN gives NaN, x >=
// 88.7228394 gives +inf, x < -103.972084 gives 0.
B2_DEV float exp_f(float x)
{
    if (!(x < 88.7228394f)) return x != x ? x : u2f(0x7f800000u);
    if (x < -103.972084f) return 0.0f;
    const float j = rint_f(mul(x, 1.44269502f));
    float r = fma_rn(j, -0.693145752f, x);                 // j * head is exact for |j| <= 151
    r = fma_rn(j, -1.42860677e-06f, r);
    float p = 1.98412701e-04f;                             // 1 / 7!
    p = fma_rn(p, r, 1.38888892e-03f);
    p = fma_rn(p, r, 8.33333377e-03f);
    p = fma_rn(p, r, 4.16666679e-02f);
    p = fma_rn(p, r, 1.66666672e-01f);
    p = fma_rn(p, r, 0.5f);
    p = fma_rn(p, r, 1.0f);
    p = fma_rn(p, r, 1.0f);
    const int e = (int)j, e1 = e / 2, e2 = e - e1;         // |e1|, |e2| <= 76: both powers are normal floats
    return mul(mul(p, u2f((uint32_t)(e1 + 127) << 23)), u2f((uint32_t)(e2 + 127) << 23));
}

B2_DEV V3 mk3(float x, float y, float z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
B2_DEV V3 v_add(V3 a, V3 b) { return mk3(add(a.x, b.x), add(a.y, b.y), add(a.z, b.z)); }
B2_DEV V3 v_sub(V3 a, V3 b) { return mk3(sub(a.x, b.x), sub(a.y, b.y), sub(a.z, b.z)); }
B2_DEV V3 v_scale(V3 a, float s) { return mk3(mul(a.x, s), mul(a.y, s), mul(a.z, s)); }
B2_DEV V3 v_neg(V3 a) { return mk3(-a.x, -a.y, -a.z); }
// rm::Vector3::dot: x*o.x + y*o.y + z*o.z (left to right)
B2_DEV float v_dot(V3 a, V3 b) { return add(add(mul(a.x, b.x), mul(a.y, b.y)), mul(a.z, b.z)); }
B2_DEV float v_l2norm(V3 a) { return sqrt_rn(add(add(mul(a.x, a.x), mul(a.y, a.y)), mul(a.z, a.z))); }
B2_DEV V3 v_normalize(V3 a) { const float n = v_l2norm(a); return mk3(dvd(a.x, n), dvd(a.y, n), dvd(a.z, n)); }

// Hamilton product (SURVEY.md A.1), each component ((a*b op c*d) op e*f) op g*h
B2_DEV Q4 q_mul(Q4 a, Q4 b)
{
    Q4 r;
    r.w = sub(sub(sub(mul(a.w, b.w), mul(a.x, b.x)), mul(a.y, b.y)), mul(a.z, b.z));
    r.x = sub(add(add(mul(a.w, b.x), mul(a.x, b.w)), mul(a.y, b.z)), mul(a.z, b.y));
    r.y = add(add(sub(mul(a.w, b.y), mul(a.x, b.z)), mul(a.y, b.w)), mul(a.z, b.x));
    r.z = add(sub(add(mul(a.w, b.z), mul(a.x, b.y)), mul(a.y, b.x)), mul(a.z, b.w));
    return r;
}
B2_DEV Q4 q_conj(Q4 a) { Q4 r; r.x = -a.x; r.y = -a.y; r.z = -a.z; r.w = a.w; return r; }
B2_DEV V3 q_rot(Q4 q, V3 v)
{
    Q4 p; p.x = v.x; p.y = v.y; p.z = v.z; p.w = 0.0f;
    const Q4 r = q_mul(q_mul(q, p), q_conj(q));
    return mk3(r.x, r.y, r.z);
}
B2_DEV Q4 q_normalize(Q4 q)
{
    const float n = sqrt_rn(add(add(add(mul(q.x, q.x), mul(q.y, q.y)), mul(q.z, q.z)), mul(q.w, q.w)));
    Q4 r; r.x = dvd(q.x, n); r.y = dvd(q.y, n); r.z = dvd(q.z, n); r.w = dvd(q.w, n); return r;
}
B2_DEV Tf tf_identity() { Tf T; T.R.x = T.R.y = T.R.z = 0.f; T.R.w = 1.f; T.t = mk3(0.f, 0.f, 0.f); return T; }
B2_DEV Tf tf_mul(Tf a, Tf b) { Tf r; r.R = q_mul(a.R, b.R); r.t = v_add(q_rot(a.R, b.t), a.t); return r; }
B2_DEV Tf tf_inv(Tf a) { Tf r; r.R = q_conj(a.R); r.t = v_neg(q_rot(r.R, a.t)); return r; }
B2_DEV V3 tf_apply(Tf T, V3 p) { return v_add(q_rot(T.R, p), T.t); }

B2_DEV Tf tf_load(const b2_transform* p)
{
#if B2_ON_DEVICE
    const float4 a = *reinterpret_cast<const float4*>(p);             // device buffers of b2_transform are 32-byte aligned
    const float4 b = *(reinterpret_cast<const float4*>(p) + 1);
    Tf T; T.R.x = a.x; T.R.y = a.y; T.R.z = a.z; T.R.w = a.w; T.t = mk3(b.x, b.y, b.z); return T;
#else
    Tf T; T.R.x = p->R.x; T.R.y = p->R.y; T.R.z = p->R.z; T.R.w = p->R.w; T.t = mk3(p->t.x, p->t.y, p->t.z); return T;
#endif
}
B2_DEV void tf_store(b2_transform* p, Tf T)
{
#if B2_ON_DEVICE
    *reinterpret_cast<float4*>(p) = make_float4(T.R.x, T.R.y, T.R.z, T.R.w);
    *(reinterpret_cast<float4*>(p) + 1) = make_float4(T.t.x, T.t.y, T.t.z, 0.0f);
#else
    p->R.x = T.R.x; p->R.y = T.R.y; p->R.z = T.R.z; p->R.w = T.R.w; p->t.x = T.t.x; p->t.y = T.t.y; p->t.z = T.t.z; p->stamp = 0;
#endif
}
__host__ __device__ inline Tf tf_from_pod(const b2_transform& s)
{
    Tf T; T.R.x = s.R.x; T.R.y = s.R.y; T.R.z = s.R.z; T.R.w = s.R.w; T.t.x = s.t.x; T.t.y = s.t.y; T.t.z = s.t.z; return T;
}

// ---- explicit-FMA helpers for the ray/triangle kernel ----
B2_DEV float dot_fma(V3 a, V3 b) { return fma_rn(a.z, b.z, fma_rn(a.y, b.y, mul(a.x, b.x))); }
B2_DEV V3 cross_fma(V3 a, V3 b)
{
    return mk3(fma_rn(a.y, b.z, -mul(a.z, b.y)), fma_rn(a.z, b.x, -mul(a.x, b.z)), fma_rn(a.x, b.y, -mul(a.y, b.x)));
}

// ---- warp reductions ----
#if defined(__CUDACC__)
__device__ __forceinline__ double warp_sum(double v)
{
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ uint32_t warp_sum_u32(uint32_t v) { return __reduce_add_sync(0xffffffffu, v); }
__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v)
{
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
#endif
