// trace.cuh -- software closest-hit traversal of the 8-wide quantised BVH (bvh8.h) for sm_90a.
//
// Stands in for Embree's rtcIntersect1 behind rm::*SimulatorEmbree::simulate (called at
// rmcl/src/rmcl/registration/RCCEmbree.cpp:35,67,98,130) and for the direct call at
// rmcl_ros/src/rmcl/PCDSensorUpdaterEmbree.cpp:44.  The H100 has no RT cores: this is the whole ray tracer.
//
// HIT DEFINITION (identical to oracle/oracle.c, independent of the acceleration structure):
//   slab formula F for a box: idir_k = 1/(|d_k| < 1e-18 ? copysign(1e-18,d_k) : d_k); t = fl(fl(plane - o) * idir)
//   candidate t (Moeller-Trumbore, scaled form, explicit FMA chains) is a HIT iff t > 0 and, for the triangle's own AABB,
//       tn <= fl(t*C1)  and  tf >= fl(t*C2)                       C1 = 1+2^-14, C2 = 1-2^-14
//   result = argmin (t, face id) over HITs with t <= tfar.
// CULLING: a child box (exact float AABB of the triangles below it) is skipped only if NOT
//       max(tn'_x, tn'_y, tn'_z, 0) <= min(tf'_x, tf'_y, tf'_z, fl(tbest*C1))
//   with  tf'_k = fma(far_plane_k,  idir_k,      -cf_k),  cf_k = oi_k - dl_k            (two children per step on the device)                 oi_k = fl(o_k * idir_k)
//         tn'_k = fma(near_plane_k, idir_k*C3',  -cn_k),  cn_k = (oi_k + dl_k) * C3'         C3' = 1 - 2^-11
//         dl_k  = 2^-20 * (|oi_k| + B_k * |idir_k|)        B_k = max |vertex coordinate| on axis k
//   All constants are per RAY (RaySetup); a node visit is 48 FMAs + min/max, no per-node setup.  dl_k bounds the FMA-path error
//   (<= 2^-23 (|plane*idir| + |oi|)) plus F's own error, so tn' <= C3' * tn_F and tf' >= tf_F for the same float box; with the C3' scale
//   this test is at least as permissive as the oracle's visit rule V (tn <= tbest*C1 && tf >= max(0, tn*C3), C3 = 1-2^-12): if tn_F > 0,
//   tn' <= tn_F*C3' <= fl(tn_F*C3) <= tf_F <= tf'; if tn_F <= 0, tn' <= 0 <= tf_F.  Hence every HIT's leaf is visited and the result
//   equals the brute-force answer.
// INTEGER BOX TEST: the same predicate, tn = max(tn'_x, tn'_y, tn'_z, 0) <= tf = min(tf'_x, tf'_y, tf'_z, tlim), reduced on the float BIT
//   PATTERNS as signed ints: tn_i = __vimax3_s32_relu(near planes), tf_i = __vimin3_s32(far planes, tlim_i) (VIMNMX3 on sm_90), hit iff
//   tn_i <= tf_i.  Signed-int order equals float order on non-negative non-NaN floats (+0 .. +inf); every float with the sign bit set is a
//   negative int, -0 the smallest.  fmaxf / fminf drop a NaN operand.  The bits are the float test's exactly when (a) no near plane is NaN
//   and (b) no far plane is NaN or -0, and tlim_i maps tlim = -0 to 0 and NaN to INT_MAX:
//     tn: a negative or -0 near plane counts as 0 both ways (relu / fmaxf(., 0)); otherwise order is preserved, so tn_i = bits(tn) with
//         tn = +-0 -> 0.
//     tf: if some far plane or tlim is negative (< -0), tf_i < 0 <= tn_i and tf < 0 <= tn: miss both ways.  Otherwise every operand is
//         +0 .. +inf (or tlim NaN, dropped by fminf, INT_MAX here) and tf_i = bits(tf), so tn_i <= tf_i iff tn <= tf.
//   (a) and (b) hold for every node plane (finite, or +-inf in empty slots: the builders refuse non-finite vertices) when, per axis,
//   idir, idn, ncn, ncf are finite, idn != 0, and ncf is +0 with |idir| >= 1 or |ncf| >= 2^-100 (ray_setup flags such rays B2_RAY_INTBOX):
//     NaN needs a NaN operand, inf * 0 or inf - inf: none with finite nonzero slopes and finite addends.
//     -0: ncf is computed as dl - oi, never -0 (dl >= +0).  With ncf = +0 the FMA is +-0 + +0 = +0 for a zero plane and |plane * idir|
//     >= 2^-149 (not rounding to 0) for any other.  With |ncf| >= 2^-100: if |plane * idir| < 2^-101 the sum is nonzero and above 2^-101;
//     otherwise plane * idir is an integer multiple of 2^-148 (a product of two floats m1 2^e1 * m2 2^e2, m < 2^24, at least 2^-101 in
//     magnitude has e1 + e2 >= -148) and ncf one of 2^-149, so the exact sum is 0 (rounded to +0) or at least 2^-149 in magnitude.
//   Any other ray (NaN or inf components, denormal-scale addends; never a unit direction from a finite origin in practice) runs the
//   float reduction: trace_closest picks the instantiation once per ray.
#pragma once
#include "b2_math.cuh"
#include "bvh8.h"

#define B2_C1 1.00006103515625f
#define B2_C2 0.99993896484375f
#define B2_C3 0.999755859375f
#define B2_NOFACE 0xFFFFFFFFu

struct BvhView {
    const float4* nodes;    // B2_NODE_QUADS (14) x 16 B per node
    const float4* tris;     // 3 x float4 per triangle record
    float bx, by, bz;       // max |vertex coordinate| per axis
};

struct HitRec {
    float    t;             // closest t (== tfar on a miss)
    uint32_t face;          // original face id, B2_NOFACE on a miss
    uint32_t tri;           // leaf-record index of the hit triangle
};

struct RaySetup {
    V3 o, d, idir;
    V3 idn, ncn, ncf;       // near-plane slope (idir*C3'), NEGATED near / far constants of the box test (see header): the FMA addends
    uint32_t oct;           // bit k set iff idir_k >= 0
    uint32_t noff;          // byte offsets of the near planes inside a node, bits 0..23 one byte per axis (lo arrays for positive directions,
                            // hi arrays otherwise; the far planes sit at 96 - bnx, 160 - bny, 224 - bnz); bit 31 = B2_RAY_INTBOX
};

#define B2_RAY_INTBOX 0x80000000u    // noff flag: the box test of this ray may reduce on integer bit patterns (see header)

#define B2_C3P 0.99951171875f          // 1 - 2^-11

B2_DEV RaySetup ray_setup(V3 o, V3 d, const struct BvhView& bvh);

// formula F on an exact float box
B2_DEV void slab_F(const RaySetup& r, V3 lo, V3 hi, float& tn, float& tf)
{
    const float x0 = mul(sub(lo.x, r.o.x), r.idir.x), x1 = mul(sub(hi.x, r.o.x), r.idir.x);
    const float y0 = mul(sub(lo.y, r.o.y), r.idir.y), y1 = mul(sub(hi.y, r.o.y), r.idir.y);
    const float z0 = mul(sub(lo.z, r.o.z), r.idir.z), z1 = mul(sub(hi.z, r.o.z), r.idir.z);
    tn = fmaxf(fmaxf(fminf(x0, x1), fminf(y0, y1)), fminf(z0, z1));
    tf = fminf(fminf(fmaxf(x0, x1), fmaxf(y0, y1)), fmaxf(z0, z1));
}

// Moeller-Trumbore + validation; updates (tbest, face, tri) under the (t, face) lexicographic rule
B2_DEV void tri_test(const BvhView& bvh, const RaySetup& r, uint32_t tri_idx, HitRec& best)
{
    const float4 a = ldg(bvh.tris + 3 * (size_t)tri_idx + 0);
    const float4 b = ldg(bvh.tris + 3 * (size_t)tri_idx + 1);
    const float4 c = ldg(bvh.tris + 3 * (size_t)tri_idx + 2);
    const V3 v0 = mk3(a.x, a.y, a.z), v1 = mk3(b.x, b.y, b.z), v2 = mk3(c.x, c.y, c.z);
    const V3 e1 = v_sub(v1, v0), e2 = v_sub(v2, v0);
    const V3 pv = cross_fma(r.d, e2);
    const float det = dot_fma(e1, pv);
    if (!(det != 0.0f)) return;                 // zero or NaN
    const V3 tv = v_sub(r.o, v0);
    const float U = dot_fma(tv, pv);
    const V3 qv = cross_fma(tv, e1);
    const float V = dot_fma(r.d, qv);
    const float T = dot_fma(e2, qv);
    const float UV = add(U, V);
    bool ok;
    if (det > 0.0f) ok = (U >= 0.0f) && (V >= 0.0f) && (UV <= det) && (T > 0.0f);
    else            ok = (U <= 0.0f) && (V <= 0.0f) && (UV >= det) && (T < 0.0f);
    if (!ok) return;
    const float t = dvd(T, det);
    const uint32_t face = f2u(a.w);
    if (!(t < best.t || (t == best.t && face < best.face))) return;
    const V3 lo = mk3(fminf(fminf(v0.x, v1.x), v2.x), fminf(fminf(v0.y, v1.y), v2.y), fminf(fminf(v0.z, v1.z), v2.z));
    const V3 hi = mk3(fmaxf(fmaxf(v0.x, v1.x), v2.x), fmaxf(fmaxf(v0.y, v1.y), v2.y), fmaxf(fmaxf(v0.z, v1.z), v2.z));
    float tn, tf; slab_F(r, lo, hi, tn, tf);
    if (!(tn <= mul(t, B2_C1) && tf >= mul(t, B2_C2))) return;
    best.t = t; best.face = face; best.tri = tri_idx;
}

// raw geometric normal (v1-v0) x (v2-v0) of a leaf record (Embree's Ng, |Ng| = 2*area)
B2_DEV V3 tri_ng(const BvhView& bvh, uint32_t tri_idx)
{
    const float4 a = ldg(bvh.tris + 3 * (size_t)tri_idx + 0);
    const float4 b = ldg(bvh.tris + 3 * (size_t)tri_idx + 1);
    const float4 c = ldg(bvh.tris + 3 * (size_t)tri_idx + 2);
    const V3 v0 = mk3(a.x, a.y, a.z);
    return cross_fma(v_sub(mk3(b.x, b.y, b.z), v0), v_sub(mk3(c.x, c.y, c.z), v0));
}

// One axis of a ray admits the integer box test (header): slopes and addends finite, slopes nonzero, and the far addend either at least 2^-100
// in magnitude or +0 with |idir| >= 1 -- then no near plane is NaN and no far plane is NaN or -0.
B2_DEV bool intbox_axis(float idir, float idn, float ncn, float ncf)
{
    const float inf = u2f(0x7f800000u), afar = fabsf(ncf);
    return fabsf(idn) < inf && idn != 0.0f && fabsf(ncn) < inf && afar < inf && (afar >= u2f(0x0d800000u) || (ncf == 0.0f && fabsf(idir) >= 1.0f));
}

B2_DEV RaySetup ray_setup(V3 o, V3 d, const BvhView& bvh)
{
    RaySetup r; r.o = o; r.d = d;
    float dx = d.x, dy = d.y, dz = d.z;
    if (fabsf(dx) < 1e-18f) dx = copysignf(1e-18f, dx);
    if (fabsf(dy) < 1e-18f) dy = copysignf(1e-18f, dy);
    if (fabsf(dz) < 1e-18f) dz = copysignf(1e-18f, dz);
    r.idir = mk3(dvd(1.0f, dx), dvd(1.0f, dy), dvd(1.0f, dz));
    r.oct = (r.idir.x >= 0.f ? 1u : 0u) | (r.idir.y >= 0.f ? 2u : 0u) | (r.idir.z >= 0.f ? 4u : 0u);
    const float k20 = 9.5367431640625e-07f;   // 2^-20
    const float oix = o.x * r.idir.x, oiy = o.y * r.idir.y, oiz = o.z * r.idir.z;
    const float dlx = (fabsf(oix) + bvh.bx * fabsf(r.idir.x)) * k20, dly = (fabsf(oiy) + bvh.by * fabsf(r.idir.y)) * k20, dlz = (fabsf(oiz) + bvh.bz * fabsf(r.idir.z)) * k20;
    r.idn = mk3(r.idir.x * B2_C3P, r.idir.y * B2_C3P, r.idir.z * B2_C3P);
    r.ncn = mk3(-((oix + dlx) * B2_C3P), -((oiy + dly) * B2_C3P), -((oiz + dlz) * B2_C3P));
    r.ncf = mk3(dlx - oix, dly - oiy, dlz - oiz);   // = -(oi - dl), but +0 rather than -0 when oi == dl (INTEGER BOX TEST in the header)
    // node layout in bytes: lo_x 0, lo_y 32, lo_z 64, hi_x 96, hi_y 128, hi_z 160 (two quads each), header 192
    r.noff = ((r.oct & 1u) ? 0u : 96u) | (((r.oct & 2u) ? 32u : 128u) << 8) | (((r.oct & 4u) ? 64u : 160u) << 16);
    if (intbox_axis(r.idir.x, r.idn.x, r.ncn.x, r.ncf.x) && intbox_axis(r.idir.y, r.idn.y, r.ncn.y, r.ncf.y) && intbox_axis(r.idir.z, r.idn.z, r.ncn.z, r.ncf.z))
        r.noff |= B2_RAY_INTBOX;
#if B2_ON_DEVICE
    // Per-ray constants of the box test are made opaque to the optimiser: under the 72-register cap of the traversal kernels it otherwise
    // RE-DERIVES them from o / d in every node visit (octant, plane offsets, slack constants: ~45 of ~190 instructions per visit in the round-1
    // SASS).  Kept small on purpose -- 3 + 3 + 3 slopes / addends, the octant and ONE word of plane offsets; what is cheap to derive (the
    // near-plane slope idir * C3', the six plane offsets) is derived inside node_test from these.
    asm volatile("" : "+f"(r.ncn.x), "+f"(r.ncn.y), "+f"(r.ncn.z));
    asm volatile("" : "+r"(r.oct), "+r"(r.noff));
#endif
    return r;
}

// XOR-permutation of an 8-bit child mask: bit s moves to bit s ^ oct (three conditional swaps: nibbles, bit pairs, bits).  A ray visits the
// inner children of a node in descending order of (slot ^ octant); with the hit bits permuted like this that order is "highest set bit first".
B2_DEV uint32_t xor_permute8(uint32_t x, uint32_t oct)
{
    if (oct & 4u) x = ((x << 4) | (x >> 4)) & 0xffu;
    if (oct & 2u) x = ((x & 0x33u) << 2) | ((x >> 2) & 0x33u);
    if (oct & 1u) x = ((x & 0x55u) << 1) | ((x >> 1) & 0x55u);
    return x;
}
// 8 child bits -> 24 slot-space triangle bits: bit s becomes bits 3s..3s+2
B2_DEV uint32_t spread3x(uint32_t x)
{
    x = (x | (x << 8)) & 0x00f00fu;
    x = (x | (x << 4)) & 0x0c30c3u;
    x = (x | (x << 2)) & 0x249249u;
    return x * 7u;
}

// Intersect the 8 children of one node.  Outputs: `inner` = (hit inner children in priority positions 31..24) | imask 7..0 -- the stack-entry
// format; `tris` = pending leaf triangles in slot space (bit 3s+j = triangle j of leaf child s), `trimask` = the node's existing triangles in the
// same space (record index of bit b = tri_base + popc(trimask & ((1 << b) - 1))).
// 13 quads per visit (12 plane quads + one header quad); the masks come from the eight box-test bits with ~30 bit operations -- the first
// version decoded one meta byte per child (~60 instructions, a third of the visit in its SASS).
// Load order: the header and quad a (children 0..3) of all six plane arrays first -- one 16-byte load in each of the node's seven 32-byte
// sectors, so a node that misses L1 costs one round trip to L2 / DRAM -- then quad b (children 4..7), which the first loads brought into L1.
// INTBOX: reduce each child's six planes on their bit patterns (header, INTEGER BOX TEST); only for rays flagged B2_RAY_INTBOX.
B2_DEV int imin(int a, int b) { return a < b ? a : b; }

// Read-only 16-byte load that the compiler keeps in source order with the other ordered loads (volatile asm): the node visit issues the
// loads that touch all seven sectors of a node before any that does not.
B2_DEV float4 ldg_ordered(const float4* p)
{
#if B2_ON_DEVICE
    float4 v;
    asm volatile("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
#else
    return *p;
#endif
}

template <bool INTBOX>
B2_DEV void node_test(const float4* __restrict__ nodes, uint32_t node_idx, const RaySetup& r, float tbest, uint32_t& child_base, uint32_t& tri_base,
                      uint32_t& inner, uint32_t& tris, uint32_t& trimask)
{
    // one 64-bit node base; the plane arrays are reached by per-ray byte offsets, quad b (+16) and the header (+192) by immediates.  Near planes:
    // the "lo" arrays for positive directions, the "hi" arrays otherwise; far planes: the other one (96 bytes apart).  The offsets are
    // extracted HERE, per visit, not hoisted out of the traversal loop into six more live registers (or spill slots).
    const char* const nb = reinterpret_cast<const char*>(nodes) + (size_t)node_idx * (16u * B2_NODE_QUADS);
    uint32_t bnx, bny, bnz;
#if B2_ON_DEVICE
    asm volatile("bfe.u32 %0, %3, 0, 8;\n\tbfe.u32 %1, %3, 8, 8;\n\tbfe.u32 %2, %3, 16, 8;" : "=r"(bnx), "=r"(bny), "=r"(bnz) : "r"(r.noff));
#else
    bnx = r.noff & 0xffu; bny = (r.noff >> 8) & 0xffu; bnz = (r.noff >> 16) & 0xffu;
#endif
    const char* const pnx = nb + bnx; const char* const pfx = nb + (96u - bnx);
    const char* const pny = nb + bny; const char* const pfy = nb + (160u - bny);
    const char* const pnz = nb + bnz; const char* const pfz = nb + (224u - bnz);
#define B2_Q(P, OFF) ldg_ordered(reinterpret_cast<const float4*>((P) + (OFF)))
    const float4 h = B2_Q(nb, 192);
    const float4 nxa = B2_Q(pnx, 0), nya = B2_Q(pny, 0), nza = B2_Q(pnz, 0), fxa = B2_Q(pfx, 0), fya = B2_Q(pfy, 0), fza = B2_Q(pfz, 0);
    child_base = f2u(h.x); tri_base = f2u(h.y);
    const uint32_t masks = f2u(h.z), imask = masks & 0xffu;
    trimask = masks >> 8;
    const float tlim = tbest * B2_C1;
    int tl = (int)f2u(tlim);                   // integer reduction: tlim = -0 (a tfar of -0) compares as +0, NaN (ignored by fminf) as the maximum
    if (INTBOX) { if (tlim == 0.0f) tl = 0; if (tlim != tlim) tl = 0x7fffffff; }
    // every box test waits for the header: bits 24..30 of noff are zero but opaque to the compiler, so the header load is issued with the
    // quad-a loads instead of being sunk to the end of the visit, where its miss would be a second round trip
    tl |= (int)(masks & r.noff & 0x7f000000u);
    uint32_t hit8 = 0;
    // Two children per step, one plane of two neighbouring slots from the .xy / .zw halves of a 128-bit node load; slope and addend are
    // per-ray scalars.  Every plane is one round-to-nearest FMA, the same bits as the CPU emulation.
#define B2_HIT(BIT, NX, NY, NZ, FX, FY, FZ)                                                                            \
    if (INTBOX) {                                                                                                      \
        const int tn = __vimax3_s32_relu((int)f2u(NX), (int)f2u(NY), (int)f2u(NZ));                                    \
        const int tf = __vimin3_s32((int)f2u(FX), (int)f2u(FY), imin((int)f2u(FZ), tl));                                \
        hit8 |= (tn <= tf) ? (BIT) : 0u;                                                                               \
    } else {                                                                                                           \
        hit8 |= (fmaxf(fmaxf(NX, NY), fmaxf(NZ, 0.0f)) <= fminf(fminf(FX, FY), fminf(FZ, tlim))) ? (BIT) : 0u;         \
    }
#define B2_PAIR(S, NX0, NX1, NY0, NY1, NZ0, NZ1, FX0, FX1, FY0, FY1, FZ0, FZ1)                                        \
    {                                                                                                                  \
        const float nx0 = fma_rn(NX0, r.idn.x, r.ncn.x), nx1 = fma_rn(NX1, r.idn.x, r.ncn.x);                          \
        const float ny0 = fma_rn(NY0, r.idn.y, r.ncn.y), ny1 = fma_rn(NY1, r.idn.y, r.ncn.y);                          \
        const float nz0 = fma_rn(NZ0, r.idn.z, r.ncn.z), nz1 = fma_rn(NZ1, r.idn.z, r.ncn.z);                          \
        const float fx0 = fma_rn(FX0, r.idir.x, r.ncf.x), fx1 = fma_rn(FX1, r.idir.x, r.ncf.x);                        \
        const float fy0 = fma_rn(FY0, r.idir.y, r.ncf.y), fy1 = fma_rn(FY1, r.idir.y, r.ncf.y);                        \
        const float fz0 = fma_rn(FZ0, r.idir.z, r.ncf.z), fz1 = fma_rn(FZ1, r.idir.z, r.ncf.z);                        \
        B2_HIT(1u << (S), nx0, ny0, nz0, fx0, fy0, fz0)                                                                \
        B2_HIT(2u << (S), nx1, ny1, nz1, fx1, fy1, fz1)                                                                \
    }
    B2_PAIR(0, nxa.x, nxa.y, nya.x, nya.y, nza.x, nza.y, fxa.x, fxa.y, fya.x, fya.y, fza.x, fza.y)
    B2_PAIR(2, nxa.z, nxa.w, nya.z, nya.w, nza.z, nza.w, fxa.z, fxa.w, fya.z, fya.w, fza.z, fza.w)
    const float4 nxb = B2_Q(pnx, 16), nyb = B2_Q(pny, 16), nzb = B2_Q(pnz, 16), fxb = B2_Q(pfx, 16), fyb = B2_Q(pfy, 16), fzb = B2_Q(pfz, 16);
    B2_PAIR(4, nxb.x, nxb.y, nyb.x, nyb.y, nzb.x, nzb.y, fxb.x, fxb.y, fyb.x, fyb.y, fzb.x, fzb.y)
    B2_PAIR(6, nxb.z, nxb.w, nyb.z, nyb.w, nzb.z, nzb.w, fxb.z, fxb.w, fyb.z, fyb.w, fzb.z, fzb.w)
#undef B2_PAIR
#undef B2_HIT
#undef B2_Q
    inner = (xor_permute8(hit8 & imask, r.oct) << 24) | imask;
    tris = spread3x(hit8 & ~imask) & trimask;           // empty slots never pass the box test (lo = +inf, hi = -inf) and have no trimask bits
}

template <bool STATS, bool INTBOX>
B2_DEV void trace_closest_box(const BvhView& bvh, const RaySetup& r, HitRec& best, uint32_t& n_nodes, uint32_t& n_tris)
{
    uint2 stack[B2_TRAVERSAL_STACK];
    int sp = 0;
    // root group: slot 0 of a virtual parent -> priority bit 24 + (0 ^ oct), imask bit 0
    uint2 G = make_uint2(0u, (1u << (24 + r.oct)) | 1u);      // pending inner children: (child_base, hit bits 31..24 | imask 7..0)
    uint2 Gt = make_uint2(0u, 0u);                             // pending leaf triangles of the last visited node: (tri_base, slot-space bits 23..0)
    uint32_t Gm = 0u;                                          //   and that node's trimask (slot-space bit -> record index)
    // Each trip does ONE unit of work per lane -- a triangle test if one is pending, otherwise a node visit -- instead of a node visit
    // followed by an inner loop over that node's triangles: a warp then never waits for the lane with the most triangles in a node
    // (the max-over-lanes triangle loop dominated the slowest warps' instruction streams).  The closest hit under the
    // (t, face) rule does not depend on the order of the tests.
    while (true) {
        if (Gt.y) {
            const uint32_t i = 31u - (uint32_t)clz32(Gt.y);
            Gt.y &= ~(1u << i);
            tri_test(bvh, r, Gt.x + (uint32_t)popc32(Gm & ((1u << i) - 1u)), best);
            if (STATS) n_tris++;
        }
        if (!Gt.y) {                                           // last pending triangle done (or none): visit a node in the same trip
            if (!(G.y & 0xff000000u)) {
                if (sp == 0) break;
                G = stack[--sp];
            }
            const uint32_t bitpos = 31u - (uint32_t)clz32(G.y);
            G.y &= ~(1u << bitpos);
            const uint32_t slot = (bitpos - 24u) ^ r.oct;
            const uint32_t rel = popc32(G.y & 0xffu & ((1u << slot) - 1u));
            const uint32_t node_idx = G.x + rel;
            if (G.y & 0xff000000u) stack[sp++] = G;
            uint32_t child_base, tri_base, inner, tris;
            node_test<INTBOX>(bvh.nodes, node_idx, r, best.t, child_base, tri_base, inner, tris, Gm);
            if (STATS) n_nodes++;
            G = make_uint2(child_base, inner);
            Gt = make_uint2(tri_base, tris);
        }
    }
}

// Closest hit. best.t must be initialised to tfar, best.face to B2_NOFACE by the caller (see trace_init).  A ray whose box-test constants
// are outside the integer test's domain (non-finite or denormal-scale; never a unit direction from a finite origin in practice) walks the
// same tree with the float reduction.
template <bool STATS>
B2_DEV void trace_closest(const BvhView& bvh, const RaySetup& r, HitRec& best, uint32_t& n_nodes, uint32_t& n_tris)
{
    if (r.noff & B2_RAY_INTBOX) trace_closest_box<STATS, true>(bvh, r, best, n_nodes, n_tris);
    else                        trace_closest_box<STATS, false>(bvh, r, best, n_nodes, n_tris);
}

B2_DEV HitRec trace_init(float tfar) { HitRec h; h.t = tfar; h.face = B2_NOFACE; h.tri = 0u; return h; }

// =====================================================================================================================
// Closest point on the map (stand-in for rm::EmbreeMap::closestPoint / Embree point queries behind CPCEmbree::find,
// rmcl/src/rmcl/registration/CPCEmbree.cpp:33-42).  Same BVH8F nodes, distance test instead of slab test.
//
// RESULT DEFINITION (identical to oracle/oracle.c:orc_closest_point, independent of the acceleration structure):
//   candidate(tri) = closest point on the triangle (Ericson's region tests, individually rounded ops), d2 = |p - q|^2
//   b2(box)        = |max(lo - q, q - hi, 0)|^2                      monotone: a larger box never has a larger b2
//   lim(d2)        = (sqrt(d2) + DELTA)^2,  DELTA = 2^-16 (1 + max_k |q_k|)
//   a candidate COUNTS iff b2(triangle AABB) <= lim(d2);   result = argmin (d2, face id) over counting candidates.
// CULLING: a child is skipped only if b2(child box) > lim(best d2).  Child boxes are exact float AABBs of the triangles below, so
//   b2(child) <= b2(triangle AABB) <= lim(d2_tri) <= lim(best) for every triangle that could still win or tie: its leaf is visited.
// Stack: one entry per level as for rays -- (child_base, pending inner children | imask) with the spare 16 bits holding a bf16 LOWER
//   bound of the group's smallest b2 (float truncated toward zero), so a whole group is dropped at pop time once lim has shrunk.
// =====================================================================================================================
struct CpBest {
    float d2, lim;
    uint32_t face, tri;
    V3 p;
};

B2_DEV float cp_lim(float d2, float delta) { const float s = add(sqrtf(d2), delta); return mul(s, s); }
B2_DEV float cp_axis(float lo, float hi, float q) { return fmaxf(fmaxf(sub(lo, q), sub(q, hi)), 0.0f); }
B2_DEV float cp_b2(float ax, float ay, float az) { return add(add(mul(ax, ax), mul(ay, ay)), mul(az, az)); }
B2_DEV float dot_plain(V3 a, V3 b) { return add(add(mul(a.x, b.x), mul(a.y, b.y)), mul(a.z, b.z)); }

B2_DEV V3 cp_triangle(V3 a, V3 b, V3 c, V3 p)
{
    const V3 ab = v_sub(b, a), ac = v_sub(c, a), ap = v_sub(p, a);
    const float d1 = dot_plain(ab, ap), d2 = dot_plain(ac, ap);
    if (d1 <= 0.0f && d2 <= 0.0f) return a;
    const V3 bp = v_sub(p, b);
    const float d3 = dot_plain(ab, bp), d4 = dot_plain(ac, bp);
    if (d3 >= 0.0f && d4 <= d3) return b;
    const float vc = sub(mul(d1, d4), mul(d3, d2));
    if (vc <= 0.0f && d1 >= 0.0f && d3 <= 0.0f) { const float v = dvd(d1, sub(d1, d3)); return mk3(add(a.x, mul(ab.x, v)), add(a.y, mul(ab.y, v)), add(a.z, mul(ab.z, v))); }
    const V3 cp = v_sub(p, c);
    const float d5 = dot_plain(ab, cp), d6 = dot_plain(ac, cp);
    if (d6 >= 0.0f && d5 <= d6) return c;
    const float vb = sub(mul(d5, d2), mul(d1, d6));
    if (vb <= 0.0f && d2 >= 0.0f && d6 <= 0.0f) { const float w = dvd(d2, sub(d2, d6)); return mk3(add(a.x, mul(ac.x, w)), add(a.y, mul(ac.y, w)), add(a.z, mul(ac.z, w))); }
    const float va = sub(mul(d3, d6), mul(d5, d4));
    const float e43 = sub(d4, d3), e56 = sub(d5, d6);
    if (va <= 0.0f && e43 >= 0.0f && e56 >= 0.0f) {
        const float w = dvd(e43, add(e43, e56));
        return mk3(add(b.x, mul(sub(c.x, b.x), w)), add(b.y, mul(sub(c.y, b.y), w)), add(b.z, mul(sub(c.z, b.z), w)));
    }
    const float denom = dvd(1.0f, add(add(va, vb), vc));
    const float v = mul(vb, denom), w = mul(vc, denom);
    return mk3(add(add(a.x, mul(ab.x, v)), mul(ac.x, w)), add(add(a.y, mul(ab.y, v)), mul(ac.y, w)), add(add(a.z, mul(ab.z, v)), mul(ac.z, w)));
}

B2_DEV void cp_tri_test(const BvhView& bvh, V3 q, float delta, uint32_t tri_idx, CpBest& best)
{
    const float4 a = ldg(bvh.tris + 3 * (size_t)tri_idx + 0);
    const float4 b = ldg(bvh.tris + 3 * (size_t)tri_idx + 1);
    const float4 c = ldg(bvh.tris + 3 * (size_t)tri_idx + 2);
    const V3 v0 = mk3(a.x, a.y, a.z), v1 = mk3(b.x, b.y, b.z), v2 = mk3(c.x, c.y, c.z);
    const V3 p = cp_triangle(v0, v1, v2, q);
    const float dx = sub(p.x, q.x), dy = sub(p.y, q.y), dz = sub(p.z, q.z);
    const float d2 = add(add(mul(dx, dx), mul(dy, dy)), mul(dz, dz));
    const uint32_t face = f2u(a.w);
    if (!(d2 < best.d2 || (d2 == best.d2 && face < best.face))) return;
    const float ax = cp_axis(fminf(fminf(v0.x, v1.x), v2.x), fmaxf(fmaxf(v0.x, v1.x), v2.x), q.x);
    const float ay = cp_axis(fminf(fminf(v0.y, v1.y), v2.y), fmaxf(fmaxf(v0.y, v1.y), v2.y), q.y);
    const float az = cp_axis(fminf(fminf(v0.z, v1.z), v2.z), fmaxf(fmaxf(v0.z, v1.z), v2.z), q.z);
    const float lim = cp_lim(d2, delta);
    if (!(cp_b2(ax, ay, az) <= lim)) return;
    best.d2 = d2; best.lim = lim; best.face = face; best.tri = tri_idx; best.p = p;
}

B2_DEV float cp_delta(V3 q) { return mul(1.52587890625e-05f, add(1.0f, fmaxf(fmaxf(fabsf(q.x), fabsf(q.y)), fabsf(q.z)))); }

// BOUNDED QUERY (BOUNDED = true, trunc2 = fl(trunc * trunc) with trunc > 0): the walk starts with best.lim = lim(trunc2) instead of +inf;
//   best.d2 still starts at +inf and the candidate rule is unchanged.  Let (d2*, f*) be the unbounded result.
//   (a) d2* < trunc2: the winner and every candidate tying with it have b2(triangle AABB) <= lim(d2*) <= lim(trunc2) (lim is monotone), and
//       lim(best d2) >= lim(d2*) at every later point of the walk, so each such candidate's leaf is visited as in the unbounded walk and
//       tested against the same rule: the bounded result is (d2*, f*), bit for bit.
//   (b) d2* >= trunc2 (or no candidate): the bounded result is a counting candidate or none, so its d2 >= d2* >= trunc2 or +inf, and
//       sqrtf(d2) >= sqrtf(fl(trunc^2)) = trunc (a correctly rounded square root of a correctly rounded square returns |trunc|).
//   Hence min(sqrtf(d2), trunc) is the same for both forms of the query.  The unbounded form (BOUNDED = false, the default) compiles to the
//   code it always had.
template <bool STATS, bool BOUNDED = false>
B2_DEV void closest_point(const BvhView& bvh, V3 q, CpBest& best, uint32_t& n_nodes, uint32_t& n_tris, float trunc2 = 0.0f)
{
    best.d2 = u2f(0x7f800000u); best.lim = u2f(0x7f800000u); best.face = B2_NOFACE; best.tri = 0u; best.p = mk3(0.f, 0.f, 0.f);
    // a non-finite query has no counting candidate (every comparison fails); do not walk the tree for it
    if (!(fabsf(q.x) < u2f(0x7f800000u) && fabsf(q.y) < u2f(0x7f800000u) && fabsf(q.z) < u2f(0x7f800000u))) return;
    const float delta = cp_delta(q);
    if (BOUNDED) best.lim = cp_lim(trunc2, delta);
    uint2 stack[B2_TRAVERSAL_STACK];
    int sp = 0;
    uint32_t next = 0u; float next_b2 = 0.0f; bool have_next = true;        // node to visit once the pending leaves are done (root first)
    uint32_t tbits = 0u, tri_base = 0u;                                       // pending triangles of the leaf child being tested
    uint32_t lmask = 0u, m0 = 0u, m1 = 0u;                                    // pending leaf children (slots) of the last visited node, its meta bytes
    float b2[8];                                                              // child bounds of the last visited node (registers: static indexing only)
    #pragma unroll
    for (int s = 0; s < 8; s++) b2[s] = 0.0f;
    // One unit of work per trip and lane -- a triangle test if one is pending, else a node visit -- as in trace_closest: a warp never
    // waits for the lane with the most triangles in a node.  Leaf children are taken NEAREST FIRST and judged against the bound as it
    // stands then, so once a close triangle is found the remaining leaves of the node are dropped untested.  The order of the tests
    // does not change the result (argmin over counting candidates); it only changes how early the bound shrinks.
    while (true) {
        if (!tbits && lmask) {
            uint32_t sel = 0u; float bsel = u2f(0x7f800000u);
            #pragma unroll
            for (int s = 0; s < 8; s++) if (((lmask >> s) & 1u) && b2[s] < bsel) { bsel = b2[s]; sel = (uint32_t)s; }
            if (bsel <= best.lim) {
                lmask &= ~(1u << sel);
                const uint32_t meta = ((sel < 4u ? m0 : m1) >> (8u * (sel & 3u))) & 0xffu;
                tbits = (meta >> 5) << (meta & 0x1fu);
            } else lmask = 0u;                                                // every other pending leaf is at least as far
        }
        if (tbits) {
            const uint32_t i = 31u - (uint32_t)clz32(tbits);
            tbits &= ~(1u << i);
            cp_tri_test(bvh, q, delta, tri_base + i, best);
            if (STATS) n_tris++;
        }
        if (!tbits && !lmask) {
            // the node chosen at the previous visit was judged before that node's triangles were tested: judge it again
            if (have_next && !(next_b2 <= best.lim)) have_next = false;
            while (!have_next && sp > 0) {
                // next child of the youngest group whose lower bound is still within lim
                uint2 G = stack[sp - 1];
                const float lb = u2f(((G.y >> 8) & 0xffffu) << 16);
                if (!(lb <= best.lim)) { sp--; continue; }
                const uint32_t bitpos = 31u - (uint32_t)clz32(G.y);
                const uint32_t slot = bitpos - 24u;
                G.y &= ~(1u << bitpos);
                if (G.y & 0xff000000u) stack[sp - 1] = G; else sp--;
                next = G.x + popc32(G.y & 0xffu & ((1u << slot) - 1u));
                next_b2 = 0.0f; have_next = true;
            }
            if (!have_next) break;
            const float4* __restrict__ np = bvh.nodes + B2_NODE_QUADS * (size_t)next;
            const float4 lxa = ldg(np + 0), lxb = ldg(np + 1), lya = ldg(np + 2), lyb = ldg(np + 3), lza = ldg(np + 4), lzb = ldg(np + 5);
            const float4 hxa = ldg(np + 6), hxb = ldg(np + 7), hya = ldg(np + 8), hyb = ldg(np + 9), hza = ldg(np + 10), hzb = ldg(np + 11);
            const float4 h0 = ldg(np + 12), h1 = ldg(np + 13);
            const uint32_t child_base = f2u(h0.x), imask = f2u(h0.z) & 0xffu;
            tri_base = f2u(h0.y); m0 = f2u(h1.x); m1 = f2u(h1.y);
            if (STATS) n_nodes++;
            b2[0] = cp_b2(cp_axis(lxa.x, hxa.x, q.x), cp_axis(lya.x, hya.x, q.y), cp_axis(lza.x, hza.x, q.z));
            b2[1] = cp_b2(cp_axis(lxa.y, hxa.y, q.x), cp_axis(lya.y, hya.y, q.y), cp_axis(lza.y, hza.y, q.z));
            b2[2] = cp_b2(cp_axis(lxa.z, hxa.z, q.x), cp_axis(lya.z, hya.z, q.y), cp_axis(lza.z, hza.z, q.z));
            b2[3] = cp_b2(cp_axis(lxa.w, hxa.w, q.x), cp_axis(lya.w, hya.w, q.y), cp_axis(lza.w, hza.w, q.z));
            b2[4] = cp_b2(cp_axis(lxb.x, hxb.x, q.x), cp_axis(lyb.x, hyb.x, q.y), cp_axis(lzb.x, hzb.x, q.z));
            b2[5] = cp_b2(cp_axis(lxb.y, hxb.y, q.x), cp_axis(lyb.y, hyb.y, q.y), cp_axis(lzb.y, hzb.y, q.z));
            b2[6] = cp_b2(cp_axis(lxb.z, hxb.z, q.x), cp_axis(lyb.z, hyb.z, q.y), cp_axis(lzb.z, hzb.z, q.z));
            b2[7] = cp_b2(cp_axis(lxb.w, hxb.w, q.x), cp_axis(lyb.w, hyb.w, q.y), cp_axis(lzb.w, hzb.w, q.z));
            // children within lim: leaf children become pending; descend into the nearest inner child next, park the other inner children
            // as one group (judged again when popped)
            uint32_t hit = 0, near_slot = 0; float near_b2 = u2f(0x7f800000u), rest_b2 = u2f(0x7f800000u);
            #pragma unroll
            for (int s = 0; s < 8; s++) {
                const uint32_t meta = ((s < 4 ? m0 : m1) >> (8 * (s & 3))) & 0xffu;
                const bool within = b2[s] <= best.lim;
                const bool inner = (imask >> s) & 1u;
                if (within && !inner && meta != 0u) lmask |= 1u << s;                      // empty slots have meta 0
                if (within && inner) {
                    hit |= 1u << s;
                    if (b2[s] < near_b2) { rest_b2 = near_b2; near_b2 = b2[s]; near_slot = (uint32_t)s; }
                    else rest_b2 = fminf(rest_b2, b2[s]);
                }
            }
            have_next = hit != 0u;
            if (hit) {
                hit &= ~(1u << near_slot);
                if (hit) stack[sp++] = make_uint2(child_base, (hit << 24) | (f2u(rest_b2) >> 16 << 8) | imask);
                next = child_base + popc32(imask & ((1u << near_slot) - 1u));
                next_b2 = near_b2;
            }
        }
    }
}
