// K2: level-synchronous hydration of the hash-consed store DAG.
//
// Replaces StoreCore::hydrate_z_cache / hash_ptr_val_unsafe (reference src/lem/store_core.rs:199-269), which walks
// the DAG recursively on the CPU (rayon only inside chunks of 256), with: (host) one pass over the topologically
// ordered node list to assign each node its height, a counting sort by (height, arity); (device) per height and
// arity one gather of the children's digests into flat preimages -- layouts of `impl StoreHasher for PoseidonCache`,
// src/lem/store.rs:29-78 -- one batch Poseidon launch, one scatter of the digests into the digest table.  All
// nodes of one height are independent.  Digest table and preimages stay in Montgomery form on the device.
#include "poseidon_api.h"

#include <algorithm>
#include <cstring>

namespace lurk {

// node -> preimage row; tag -> field element is F::from(u16) (src/tag.rs:99-101)
template <class F>
__global__ void __launch_bounds__(128) dag_gather_kernel(const lurk_dag_node *__restrict__ nodes, const uint32_t *__restrict__ batch,
                                                         uint32_t count, int arity, const F *__restrict__ table, F *__restrict__ pre) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const lurk_dag_node nd = nodes[batch[i]];
    F *o = pre + (size_t)i * arity;
    if (nd.kind <= LURK_DAG_TUPLE4) {
        const int nch = nd.kind;
        for (int c = 0; c < nch; c++) {
            store_fe(o + 2 * c, F::from_u64(nd.tag[c]));
            store_fe(o + 2 * c + 1, load_fe<F>(table + nd.child[c]));
        }
    } else if (nd.kind == LURK_DAG_COMPACT) {
        store_fe(o + 0, load_fe<F>(table + nd.child[0]));
        store_fe(o + 1, F::from_u64(nd.tag[1]));
        store_fe(o + 2, load_fe<F>(table + nd.child[1]));
        store_fe(o + 3, load_fe<F>(table + nd.child[2]));
    } else {   // commitment
        store_fe(o + 0, load_fe<F>(table + nd.child[0]));
        store_fe(o + 1, F::from_u64(nd.tag[1]));
        store_fe(o + 2, load_fe<F>(table + nd.child[1]));
    }
}
template <class F>
__global__ void __launch_bounds__(128) dag_scatter_kernel(const F *__restrict__ digests, const uint32_t *__restrict__ batch, uint32_t count,
                                                          uint32_t n_atoms, F *__restrict__ table) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    store_fe(table + n_atoms + batch[i], load_fe<F>(digests + i));
}

static int kind_arity(int kind) {
    switch (kind) {
        case LURK_DAG_TUPLE2: return 4;
        case LURK_DAG_TUPLE3: return 6;
        case LURK_DAG_TUPLE4: return 8;
        case LURK_DAG_COMPACT: return 4;
        case LURK_DAG_COMMITMENT: return 3;
    }
    return 0;
}
static int kind_children(int kind) {
    switch (kind) {
        case LURK_DAG_TUPLE2: return 2;
        case LURK_DAG_TUPLE3: return 3;
        case LURK_DAG_TUPLE4: return 4;
        case LURK_DAG_COMPACT: return 3;
        case LURK_DAG_COMMITMENT: return 2;
    }
    return 0;
}

// host pass shared by the hash and the plan: height of every node (children first), LURK_ERR_* on malformed input
static int dag_heights(const lurk_dag_node *nodes, size_t n, size_t n_atoms, std::vector<uint32_t> &height, uint32_t *max_h) {
    if (n + n_atoms >= 0xffffffffull) { set_error("DAG too large"); return LURK_ERR_ARG; }
    height.resize(n);
    uint32_t mh = 0;
    for (size_t i = 0; i < n; i++) {
        const int nch = kind_children(nodes[i].kind);
        if (!nch) { set_error("node %zu: unknown kind %d", i, (int)nodes[i].kind); return LURK_ERR_ARG; }
        uint32_t h = 0;
        for (int c = 0; c < nch; c++) {
            uint64_t ix = nodes[i].child[c];
            if (ix < n_atoms) continue;
            ix -= n_atoms;
            if (ix >= i) { set_error("node %zu refers to node %llu which does not precede it", i, (unsigned long long)ix); return LURK_ERR_ORDER; }
            h = std::max(h, height[ix] + 1);
        }
        height[i] = h;
        mh = std::max(mh, h);
    }
    *max_h = mh;
    return LURK_OK;
}

// per-thread stream + stream-ordered scratch: concurrent hydrations from rayon workers neither serialise on the legacy
// default stream nor synchronise the device with cudaMalloc / cudaFree
struct DagStream {
    cudaStream_t s = nullptr;
    int device = -1;
    ~DagStream() { if (s) cudaStreamDestroy(s); }
    int get(cudaStream_t *out) {
        int dev = 0;
        LURK_CUDA_TRY(cudaGetDevice(&dev));
        if (s && dev != device) { cudaStreamDestroy(s); s = nullptr; }
        if (!s) { LURK_CUDA_TRY(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking)); device = dev; }
        *out = s;
        return LURK_OK;
    }
};
struct AsyncBuf {
    void *p = nullptr;
    cudaStream_t s = nullptr;
    ~AsyncBuf() { if (p) cudaFreeAsync(p, s); }
    int alloc(size_t bytes, cudaStream_t st) { s = st; LURK_CUDA_TRY(cudaMallocAsync(&p, bytes ? bytes : 16, st)); return LURK_OK; }
    template <class T> T *as() const { return reinterpret_cast<T *>(p); }
};

template <class F>
static int dag_hash(const lurk_dag_node *nodes, size_t n, const uint8_t *atoms, size_t n_atoms, uint8_t *out) {
    // ---- host: heights and (height, arity) batches
    std::vector<uint32_t> height;
    uint32_t max_h = 0;
    LURK_TRY(dag_heights(nodes, n, n_atoms, height, &max_h));
    static const int ARITIES[4] = {3, 4, 6, 8};
    auto slot = [&](size_t i) { int a = kind_arity(nodes[i].kind); return (size_t)height[i] * 4 + (a == 3 ? 0 : a == 4 ? 1 : a == 6 ? 2 : 3); };
    std::vector<uint32_t> start(((size_t)max_h + 1) * 4 + 1, 0);
    for (size_t i = 0; i < n; i++) start[slot(i) + 1]++;
    for (size_t k = 1; k < start.size(); k++) start[k] += start[k - 1];
    std::vector<uint32_t> order(n), fill(start.begin(), start.end() - 1);
    size_t max_batch = 0;
    for (size_t i = 0; i < n; i++) order[fill[slot(i)]++] = (uint32_t)i;
    for (size_t k = 0; k + 1 < start.size(); k++) max_batch = std::max<size_t>(max_batch, start[k + 1] - start[k]);

    // ---- device
    static thread_local DagStream tls;
    cudaStream_t st = nullptr;
    LURK_TRY(tls.get(&st));
    AsyncBuf d_nodes, d_order, d_table, d_pre, d_dig;
    LURK_TRY(d_nodes.alloc(n * sizeof(lurk_dag_node), st));
    LURK_TRY(d_order.alloc(n * sizeof(uint32_t), st));
    LURK_TRY(d_table.alloc((n_atoms + n) * sizeof(F), st));
    LURK_TRY(d_pre.alloc(max_batch * 8 * sizeof(F), st));
    LURK_TRY(d_dig.alloc(max_batch * sizeof(F), st));
    LURK_CUDA_TRY(cudaMemcpyAsync(d_nodes.p, nodes, n * sizeof(lurk_dag_node), cudaMemcpyHostToDevice, st));
    LURK_CUDA_TRY(cudaMemcpyAsync(d_order.p, order.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    if (n_atoms) {
        LURK_CUDA_TRY(cudaMemcpyAsync(d_table.p, atoms, n_atoms * sizeof(F), cudaMemcpyHostToDevice, st));
        int bad = 0;
        LURK_TRY(check_reduced_dev<F>(d_table.p, n_atoms, st, &bad));
        if (bad) { set_error("%d atom digest(s) are not reduced below the field modulus", bad); return LURK_ERR_RANGE; }
        LURK_TRY(convert_dev<F>(d_table.p, n_atoms, LURK_FMT_MONTGOMERY, d_table.p, st));
    }
    for (uint32_t h = 0; h <= max_h; h++) {
        for (int a = 0; a < 4; a++) {
            const uint32_t b0 = start[(size_t)h * 4 + a], cnt = start[(size_t)h * 4 + a + 1] - b0;
            if (!cnt) continue;
            const uint32_t *batch = d_order.as<uint32_t>() + b0;
            dag_gather_kernel<F><<<(cnt + 127) / 128, 128, 0, st>>>(d_nodes.as<lurk_dag_node>(), batch, cnt, ARITIES[a], d_table.as<F>(), d_pre.as<F>());
            LURK_CUDA_TRY(cudaGetLastError());
            LURK_TRY((launch_poseidon<F, false>(ARITIES[a], d_pre.p, cnt, d_dig.p, LURK_FMT_MONTGOMERY, LURK_FMT_MONTGOMERY, st)));
            dag_scatter_kernel<F><<<(cnt + 127) / 128, 128, 0, st>>>(d_dig.as<F>(), batch, cnt, (uint32_t)n_atoms, d_table.as<F>());
            LURK_CUDA_TRY(cudaGetLastError());
        }
    }
    F *node_table = d_table.as<F>() + n_atoms;
    LURK_TRY(convert_dev<F>(node_table, n, LURK_FMT_CANONICAL, node_table, st));
    LURK_CUDA_TRY(cudaMemcpyAsync(out, node_table, n * sizeof(F), cudaMemcpyDeviceToHost, st));
    LURK_CUDA_TRY(cudaStreamSynchronize(st));
    return LURK_OK;
}

}  // namespace lurk

using namespace lurk;

extern "C" int lurk_dag_hash(int field_id, const lurk_dag_node *nodes, size_t n, const uint8_t *atom_digests, size_t n_atoms,
                             uint8_t *out_digests) {
    LURK_TRY(require_gpu());
    if (n == 0) return LURK_OK;
    if (!nodes || !out_digests || (n_atoms && !atom_digests)) { set_error("null argument"); return LURK_ERR_ARG; }
    return dispatch_field(field_id, [&](auto f) { return dag_hash<decltype(f)>(nodes, n, atom_digests, n_atoms, out_digests); });
}

// Routing aid for the caller (StoreCore::hydrate_z_cache, src/lem/store_core.rs:256-269): a level of the DAG costs one
// dependent Poseidon latency on the GPU (~170 us: three launches + one warp-per-sponge hash) whatever its width, a CPU core
// hashes ~20 k nodes/s, and the wide-DAG GPU rate is ~23 M nodes/s (constants of an earlier GPU generation, not re-measured on
// the H100).  The library never hashes on the CPU itself; it tells the caller when its own CPU path is the better choice (deep,
// narrow stores).
extern "C" int lurk_dag_hash_plan(const lurk_dag_node *nodes, size_t n, size_t n_atoms, lurk_dag_plan *plan) {
    if (!plan || (n && !nodes)) { set_error("null argument"); return LURK_ERR_ARG; }
    memset(plan, 0, sizeof *plan);
    if (n == 0) return LURK_OK;
    std::vector<uint32_t> height;
    uint32_t max_h = 0;
    LURK_TRY(dag_heights(nodes, n, n_atoms, height, &max_h));
    std::vector<uint32_t> width((size_t)max_h + 1, 0);
    for (size_t i = 0; i < n; i++) width[height[i]]++;
    plan->nodes = n;
    plan->levels = (uint64_t)max_h + 1;
    plan->max_width = *std::max_element(width.begin(), width.end());
    const double gpu_us = 150.0 + plan->levels * 170.0 + (double)n / 23.0 + (double)(n * 60) / 25000.0;   // launch chain + throughput + PCIe
    const double cpu_core_us = (double)n * 50.0;
    plan->est_gpu_us = (uint64_t)gpu_us;
    plan->est_cpu_core_us = (uint64_t)cpu_core_us;
    // the CPU side parallelises over a level too (rayon): assume 8 cores on levels wider than 8 nodes
    double cpu_us = 0;
    for (uint32_t w : width) cpu_us += 50.0 * ((w + 7) / 8);
    plan->use_gpu = gpu_us < cpu_us ? 1 : 0;
    return LURK_OK;
}
