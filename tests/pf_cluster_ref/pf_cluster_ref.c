/* pf_cluster_ref.c -- TEST INFRASTRUCTURE ONLY: a sequential restatement of the clustering of b2_pf_cluster_stats (SURVEY appendix H), written
 * from the rule in include/rmcl_b200.h and sharing nothing with the device code: the members' bin keys are sorted, touching bins are found
 * by binary search and joined in a union-find forest over the sorted order, and the clusters are ranked by (weight descending, key
 * ascending).  The keys and the integer weights themselves are those of the KLD restatement (pf_kld_ref).  Built by tests/pf_cluster_ref.py. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_CLUSTER_NONE_KEY 0xFFFFFFFFFFFFFFFFull
#define ORC_CLUSTER_NONE 0xFFFFFFFFu

/* the bin at (dx, dy, dz, ds) from `key` = (ix + 2^19) << 44 | (iy + 2^19) << 24 | (iz + 2^7) << 16 | sector, or NONE_KEY: no bin lies beyond a
 * clamp, none above or below when z is not binned; the sector wraps modulo K */
uint64_t orc_cluster_neighbour(uint64_t key, int dx, int dy, int dz, int ds, uint32_t K, int has_z)
{
    long long ix = (long long)(key >> 44) - 524288, iy = (long long)((key >> 24) & 0xFFFFF) - 524288, iz = (long long)((key >> 16) & 0xFF) - 128;
    long long s = (long long)(key & 0xFFFF);
    ix += dx; iy += dy; iz += dz;
    if (ix < -524288 || ix >= 524288 || iy < -524288 || iy >= 524288) return ORC_CLUSTER_NONE_KEY;
    if (has_z ? (iz < -128 || iz >= 128) : dz != 0) return ORC_CLUSTER_NONE_KEY;
    s += ds;
    if (s < 0) s += K;
    if (s >= (long long)K) s -= K;
    return (uint64_t)(ix + 524288) << 44 | (uint64_t)(iy + 524288) << 24 | (uint64_t)(iz + 128) << 16 | (uint64_t)s;
}
void orc_cluster_neighbours(const uint64_t* keys, uint64_t count, int dx, int dy, int dz, int ds, uint32_t K, int has_z, uint64_t* out)
{
    for (uint64_t i = 0; i < count; i++) out[i] = orc_cluster_neighbour(keys[i], dx, dy, dz, ds, K, has_z);
}

static int cmp_u64(const void* a, const void* b)
{
    const uint64_t x = *(const uint64_t*)a, y = *(const uint64_t*)b;
    return x < y ? -1 : x > y;
}
static long long find_key(const uint64_t* u, long long m, uint64_t key)
{
    long long lo = 0, hi = m - 1;
    while (lo <= hi) {
        const long long mid = lo + (hi - lo) / 2;
        if (u[mid] == key) return mid;
        if (u[mid] < key) lo = mid + 1; else hi = mid - 1;
    }
    return -1;
}
static long long root_of(long long* parent, long long x)
{
    while (parent[x] != x) { parent[x] = parent[parent[x]]; x = parent[x]; }
    return x;
}
typedef struct { uint64_t weight, key, bins, members; } cluster;
static int cmp_cluster(const void* a, const void* b)
{
    const cluster* x = (const cluster*)a; const cluster* y = (const cluster*)b;
    if (x->weight != y->weight) return x->weight > y->weight ? -1 : 1;
    return x->key < y->key ? -1 : x->key > y->key;
}

/* keys[i] = NONE_KEY or w[i] = 0: particle i is in no cluster.  labels[n]; c_weight / c_key / c_bins / c_members hold up to n clusters in rank
 * order; res = n_clusters, bins, n_clustered, weight_total */
void orc_pf_cluster(uint32_t n, const uint64_t* keys, const uint64_t* w, uint32_t K, int has_z, uint32_t* labels, uint64_t* c_weight, uint64_t* c_key,
                    uint64_t* c_bins, uint64_t* c_members, uint64_t* res)
{
    uint64_t* u = (uint64_t*)malloc(sizeof(uint64_t) * (n + 1));
    long long m = 0;
    uint64_t n_clustered = 0, total = 0;
    for (uint32_t i = 0; i < n; i++)
        if (w[i] > 0 && keys[i] != ORC_CLUSTER_NONE_KEY) { u[m++] = keys[i]; n_clustered++; total += w[i]; }
    qsort(u, (size_t)m, sizeof(uint64_t), cmp_u64);
    long long bins = 0;
    for (long long i = 0; i < m; i++) if (i == 0 || u[i] != u[i - 1]) u[bins++] = u[i];
    long long* parent = (long long*)malloc(sizeof(long long) * (bins + 1));
    for (long long b = 0; b < bins; b++) parent[b] = b;
    for (long long b = 0; b < bins; b++)
        for (int dx = -1; dx <= 1; dx++) for (int dy = -1; dy <= 1; dy++) for (int dz = -1; dz <= 1; dz++) for (int ds = -1; ds <= 1; ds++) {
            const uint64_t nk = orc_cluster_neighbour(u[b], dx, dy, dz, ds, K, has_z);
            if (nk == ORC_CLUSTER_NONE_KEY) continue;
            const long long t = find_key(u, bins, nk);
            if (t < 0) continue;
            const long long ra = root_of(parent, b), rb = root_of(parent, t);
            if (ra < rb) parent[rb] = ra; else parent[ra] = rb;      /* the smaller index is the smaller key */
        }
    cluster* cl = (cluster*)calloc((size_t)bins + 1, sizeof(cluster));
    long long* cluster_of = (long long*)malloc(sizeof(long long) * (bins + 1));
    long long n_clusters = 0;
    for (long long b = 0; b < bins; b++)
        if (root_of(parent, b) == b) { cluster_of[b] = n_clusters; cl[n_clusters].key = u[b]; n_clusters++; }
    for (long long b = 0; b < bins; b++) cl[cluster_of[root_of(parent, b)]].bins++;
    for (uint32_t i = 0; i < n; i++)
        if (w[i] > 0 && keys[i] != ORC_CLUSTER_NONE_KEY) {
            cluster* c = cl + cluster_of[root_of(parent, find_key(u, bins, keys[i]))];
            c->weight += w[i]; c->members++;
        }
    qsort(cl, (size_t)n_clusters, sizeof(cluster), cmp_cluster);
    /* rank of a cluster: its place in the sorted list, found again through its key (the smallest of its bins) */
    uint64_t* rank_keys = (uint64_t*)malloc(sizeof(uint64_t) * (n_clusters + 1));
    uint32_t* rank_of = (uint32_t*)malloc(sizeof(uint32_t) * (n_clusters + 1));
    for (long long r = 0; r < n_clusters; r++) {
        c_weight[r] = cl[r].weight; c_key[r] = cl[r].key; c_bins[r] = cl[r].bins; c_members[r] = cl[r].members;
        rank_keys[r] = cl[r].key;
    }
    qsort(rank_keys, (size_t)n_clusters, sizeof(uint64_t), cmp_u64);
    for (long long r = 0; r < n_clusters; r++) rank_of[find_key(rank_keys, n_clusters, cl[r].key)] = (uint32_t)r;
    for (uint32_t i = 0; i < n; i++) {
        labels[i] = ORC_CLUSTER_NONE;
        if (w[i] > 0 && keys[i] != ORC_CLUSTER_NONE_KEY) {
            const uint64_t root_key = u[root_of(parent, find_key(u, bins, keys[i]))];
            labels[i] = rank_of[find_key(rank_keys, n_clusters, root_key)];
        }
    }
    res[0] = (uint64_t)n_clusters; res[1] = (uint64_t)bins; res[2] = n_clustered; res[3] = total;
    free(u); free(parent); free(cl); free(cluster_of); free(rank_keys); free(rank_of);
}
