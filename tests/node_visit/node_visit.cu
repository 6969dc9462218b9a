// node_visit.cu -- TEST HARNESS ONLY (tests/test_node_visit.py): the box test of trace.cuh:node_test on the CPU, integer reduction against
// the float reduction.  Host-only compile through nvcc; the product's node_test / ray_setup are instantiated on the host as in tests/emul.
//
//   node_visit corner          special origins, directions and tbest values against nodes of special planes
//   node_visit random N SEED   N random rays x nodes, planes and tbest drawn from finite values with special values mixed in
//
// For every (ray, node, tbest) it compares the eight hit bits of
//   * the float reduction as it stood before the integer one: addends -(oi - dl), fmaxf / fminf over the six planes, 0 and tlim;
//   * node_test<false> (the float path the traversal takes for rays outside the integer domain);
//   * node_test<true> when ray_setup flagged the ray B2_RAY_INTBOX;
// and, for flagged rays, that no near plane value is NaN and no far plane value is NaN or -0 (the premise of the integer test).
// Prints "cases <n> intbox <n flagged> mismatch <n> premise <n>".
//
//   node_visit flags BX BY BZ  reads rays "ox oy oz dx dy dz" (strtof syntax, hex floats exact) from stdin, one per line, and prints
//                              ray_setup's B2_RAY_INTBOX flag (0 / 1) for each against a map whose max |vertex coordinate| per axis is BX BY BZ
#include "../../rmcl_b200/csrc/trace.cuh"

#include <cstdio>
#include <cstdlib>
#include <string_view>

static uint64_t g_state = 1;
static uint64_t next_u64()
{
    uint64_t z = (g_state += 0x9e3779b97f4a7c15ull);
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}
static float uni(float a, float b) { return a + (b - a) * (float)((next_u64() >> 40) * (1.0 / 16777216.0)); }

static const float kInf = u2f(0x7f800000u), kNaN = u2f(0x7fc00000u), kNegNaN = u2f(0xffc00000u);
static const float kSpecial[] = {0.0f, -0.0f, 1.0f, -1.0f, 1e-18f, -1e-18f, 1e-30f, -1e-30f, 1.4e-45f, -1.4e-45f, 1.2e-38f, 3e-39f, -3e-39f,
                                 1e30f, -1e30f, 3.4e38f, -3.4e38f, kInf, -kInf, kNaN, kNegNaN, 0.5f, -2.0f, 7.25f};
static const int kNSpecial = sizeof(kSpecial) / sizeof(kSpecial[0]);
// node planes are finite or +-inf (empty slots): the map builders refuse non-finite vertices
static float plane_special() { float v; do v = kSpecial[next_u64() % kNSpecial]; while (v != v); return v; }

// the float reduction before the integer one (trace.cuh header, CULLING), from o, d and the map bound
static uint32_t hits_reference(V3 o, V3 d, const BvhView& bvh, const float* node, float tbest)
{
    float dd[3] = {d.x, d.y, d.z}, oo[3] = {o.x, o.y, o.z}, bb[3] = {bvh.bx, bvh.by, bvh.bz};
    float idir[3], idn[3], ncn[3], ncf[3];
    for (int k = 0; k < 3; k++) {
        float dk = dd[k];
        if (fabsf(dk) < 1e-18f) dk = copysignf(1e-18f, dk);
        idir[k] = 1.0f / dk;
        const float oi = oo[k] * idir[k], dl = (fabsf(oi) + bb[k] * fabsf(idir[k])) * 9.5367431640625e-07f;
        idn[k] = idir[k] * B2_C3P;
        ncn[k] = -((oi + dl) * B2_C3P);
        ncf[k] = -(oi - dl);
    }
    const float tlim = tbest * B2_C1;
    uint32_t hit8 = 0;
    for (int s = 0; s < 8; s++) {
        float tn = 0.0f, tf = tlim;
        float n[3], f[3];
        for (int k = 0; k < 3; k++) {
            const float lo = node[8 * k + s], hi = node[24 + 8 * k + s];
            const bool pos = idir[k] >= 0.0f;
            n[k] = fmaf(pos ? lo : hi, idn[k], ncn[k]);
            f[k] = fmaf(pos ? hi : lo, idir[k], ncf[k]);
        }
        tn = fmaxf(fmaxf(n[0], n[1]), fmaxf(n[2], 0.0f));
        tf = fminf(fminf(f[0], f[1]), fminf(f[2], tlim));
        if (tn <= tf) hit8 |= 1u << s;
    }
    return hit8;
}

// premise of the integer test for a flagged ray: near planes never NaN, far planes never NaN or -0
static bool premise_holds(const RaySetup& r, const float* node)
{
    const float idir[3] = {r.idir.x, r.idir.y, r.idir.z}, idn[3] = {r.idn.x, r.idn.y, r.idn.z};
    const float ncn[3] = {r.ncn.x, r.ncn.y, r.ncn.z}, ncf[3] = {r.ncf.x, r.ncf.y, r.ncf.z};
    for (int s = 0; s < 8; s++)
        for (int k = 0; k < 3; k++) {
            const bool pos = (r.oct >> k) & 1u;
            const float n = fmaf(node[(pos ? 0 : 24) + 8 * k + s], idn[k], ncn[k]), f = fmaf(node[(pos ? 24 : 0) + 8 * k + s], idir[k], ncf[k]);
            if (n != n || f != f || f2u(f) == 0x80000000u) return false;
        }
    return true;
}

static uint32_t hits_of(uint32_t inner, uint32_t oct) { return xor_permute8(inner >> 24, oct); }

struct Counts { unsigned long long cases = 0, intbox = 0, mismatch = 0, premise = 0; };

static void check(V3 o, V3 d, const BvhView& bvh, float* node, float tbest, Counts& c)
{
    const RaySetup r = ray_setup(o, d, bvh);
    const uint32_t want = hits_reference(o, d, bvh, node, tbest);
    uint32_t cb, tb, inner, tris, trimask;
    node_test<false>(bvh.nodes, 0, r, tbest, cb, tb, inner, tris, trimask);
    bool bad = hits_of(inner, r.oct) != want;
    c.cases++;
    if (r.noff & B2_RAY_INTBOX) {
        c.intbox++;
        node_test<true>(bvh.nodes, 0, r, tbest, cb, tb, inner, tris, trimask);
        bad = bad || hits_of(inner, r.oct) != want;
        if (!premise_holds(r, node)) c.premise++;
    }
    if (bad && c.mismatch++ < 5)
        fprintf(stderr, "mismatch: o %a %a %a d %a %a %a tbest %a want %02x\n", o.x, o.y, o.z, d.x, d.y, d.z, tbest, want);
}

int main(int argc, char** argv)
{
    alignas(16) static float node[56];
    BvhView bvh; bvh.nodes = reinterpret_cast<const float4*>(node); bvh.tris = nullptr;
    uint32_t* hdr = reinterpret_cast<uint32_t*>(node + 48);
    hdr[0] = 0; hdr[1] = 0; hdr[2] = 0xffu; hdr[3] = 0;              // every slot inner: the hit bits come back in `inner`
    if (argc >= 5 && std::string_view(argv[1]) == "flags") {
        bvh.bx = strtof(argv[2], nullptr); bvh.by = strtof(argv[3], nullptr); bvh.bz = strtof(argv[4], nullptr);
        char line[512];
        while (fgets(line, sizeof line, stdin)) {
            float v[6];
            char* p = line;
            for (int k = 0; k < 6; k++) { char* e; v[k] = strtof(p, &e); if (e == p) return 2; p = e; }
            const RaySetup r = ray_setup(mk3(v[0], v[1], v[2]), mk3(v[3], v[4], v[5]), bvh);
            printf("%d\n", (r.noff & B2_RAY_INTBOX) ? 1 : 0);
        }
        return 0;
    }
    Counts c;
    const bool corner = argc >= 2 && std::string_view(argv[1]) == "corner";
    if (corner) {
        // planes: each slot a box from two special values per axis (lo, hi in either order, so empty and inverted boxes occur too)
        const float tb[] = {kInf, 0.0f, -0.0f, kNaN, kNegNaN, -1.0f, 1.0f, 1e-30f, 1e30f};
        for (int it = 0; it < 400; it++) {
            for (int i = 0; i < 48; i++) node[i] = plane_special();
            bvh.bx = kSpecial[next_u64() % kNSpecial]; bvh.bx = fabsf(bvh.bx); bvh.by = fabsf(kSpecial[next_u64() % kNSpecial]); bvh.bz = it & 1 ? 0.0f : 4.0f;
            for (int ia = 0; ia < kNSpecial; ia++)
                for (int ib = 0; ib < kNSpecial; ib += 3) {
                    const V3 o = mk3(kSpecial[ia], kSpecial[(ia + it) % kNSpecial], kSpecial[(ib + it) % kNSpecial]);
                    const V3 d = mk3(kSpecial[ib], kSpecial[(ib * 7 + it) % kNSpecial], kSpecial[(ia * 5 + ib + it) % kNSpecial]);
                    check(o, d, bvh, node, tb[(ia + ib + it) % 9], c);
                }
        }
    } else {
        const long n = argc >= 3 ? atol(argv[2]) : 100000;
        g_state = argc >= 4 ? strtoull(argv[3], nullptr, 10) : 1;
        for (long it = 0; it < n; it++) {
            bvh.bx = uni(0.0f, 50.0f); bvh.by = uni(0.0f, 50.0f); bvh.bz = (it % 7 == 0) ? 0.0f : uni(0.0f, 10.0f);
            // a node around the ray's neighbourhood: random boxes, some empty (lo = +inf, hi = -inf), some flat, special values mixed in
            for (int s = 0; s < 8; s++)
                for (int k = 0; k < 3; k++) {
                    float a = uni(-20.0f, 20.0f), b = a + uni(0.0f, 5.0f);
                    if (next_u64() % 8 == 0) b = a;
                    if (next_u64() % 16 == 0) { a = kInf; b = -kInf; }
                    if (next_u64() % 32 == 0) a = plane_special();
                    if (next_u64() % 32 == 0) b = plane_special();
                    node[8 * k + s] = a; node[24 + 8 * k + s] = b;
                }
            V3 o = mk3(uni(-20.0f, 20.0f), uni(-20.0f, 20.0f), it % 5 == 0 ? 0.0f : uni(-5.0f, 5.0f));
            V3 d = mk3(uni(-1.0f, 1.0f), uni(-1.0f, 1.0f), uni(-1.0f, 1.0f));
            if (it % 11 == 0) d.x = 0.0f;
            if (it % 13 == 0) d.z = -0.0f;
            if (it % 17 == 0) o.y = kSpecial[next_u64() % kNSpecial];
            if (it % 19 == 0) d.y = kSpecial[next_u64() % kNSpecial];
            float tbest = next_u64() % 4 ? uni(0.0f, 60.0f) : kSpecial[next_u64() % kNSpecial];
            check(o, d, bvh, node, tbest, c);
        }
    }
    printf("cases %llu intbox %llu mismatch %llu premise %llu\n", c.cases, c.intbox, c.mismatch, c.premise);
    return 0;
}
