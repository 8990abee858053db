// Batched point combination: out[g] = sum_j s[g][j] P[g][j] for independent groups of 1 .. PC_MAX_TERMS terms, one CTA per group, in one
// launch (include/lurk_b200.h, lurk_point_combination_batch).  The verifiers' point arithmetic -- the joint commitment, HyperKZG's P and Q,
// the inner-product argument's Q -- has 2 to about 130 terms, too few for a Pippenger over buckets and too many for the host Straus of
// ipa.cu to be cheap.  Straus with 4-bit windows, laid out so that little but the doublings is serial:
//   1. tables     thread j: d P_j for d = 1 .. 15 (14 mixed additions), to global scratch;
//   2. windows    thread (w, c), w < 64, c < 4: the sum over terms j = c (mod 4) of table[j][digit_w(s_j)], then a tree over c in shared
//                 memory, so W_w = sum_j digit_w(s_j) P_j;
//   3. shifts     thread w: 16^w W_w (4w doublings), then a tree over w -- window 63's 252 doublings are the critical path no layout of
//                 the windows shortens; the 63 additions a Horner pass would chain after them are 6 levels of a tree instead.
// The group law is curve.cuh's XYZZ, the arithmetic of the host Straus and of the MSM; every branch of add (an identity operand, P + P,
// P + (-P)) is taken where the sums make it so.  The host converts the result to affine, so each group's bytes are those point_combination
// writes for it.
#include "pcs.cuh"

#include <vector>

namespace lurk {

namespace {

constexpr int PC_THREADS = 256;
constexpr int PC_WINDOWS = 64;                          // 4-bit digits of a scalar < 2^256
constexpr int PC_CHUNKS = PC_THREADS / PC_WINDOWS;      // threads sharing a window's terms
constexpr int PC_TABLE = 15;                            // d P for d = 1 .. 15
// A group of fewer terms is combined on the host by point_combination_groups (unless the caller asks for the device): below it the
// kernel's fixed critical path -- 252 doublings on one GPU thread, plus the copies and the launch -- costs more than the host Straus of
// the whole group.  On an H100 (700 W) a call costs about 1.2 ms whatever its size up to ~50 terms, the host 0.5 ms for 2 terms and
// 1.1-1.2 ms (best of 20) for 10 to 16 (tools/point_combination_bench.py, profiles/h100_point_combination.jsonl).
constexpr int PC_DEVICE_MIN_TERMS = 12;

template <class Fb>
LURK_D XYZZ<Fb> load_xyzz(const XYZZ<Fb> *p) {
    XYZZ<Fb> r;
    r.x = load_fe<Fb>(&p->x); r.y = load_fe<Fb>(&p->y); r.zz = load_fe<Fb>(&p->zz); r.zzz = load_fe<Fb>(&p->zzz);
    return r;
}
template <class Fb>
LURK_D void store_xyzz(XYZZ<Fb> *p, const XYZZ<Fb> &v) {
    store_fe(&p->x, v.x); store_fe(&p->y, v.y); store_fe(&p->zz, v.zz); store_fe(&p->zzz, v.zzz);
}

template <class Fb, class Fs>
struct PcArgs {
    const Affine<Fb> *pts;        // Montgomery; the identity (0, 0)
    const Fs *k;                  // canonical
    const uint32_t *first;        // group g: terms first[g] .. first[g + 1] - 1
    XYZZ<Fb> *tab;                // PC_TABLE per term
    XYZZ<Fb> *out;                // one per group
};

template <class Fb, class Fs>
__global__ void __launch_bounds__(PC_THREADS) point_comb_kernel(const __grid_constant__ PcArgs<Fb, Fs> a) {
    __shared__ uint4 part_raw[PC_CHUNKS * PC_WINDOWS * sizeof(XYZZ<Fb>) / sizeof(uint4)];
    XYZZ<Fb> *part = reinterpret_cast<XYZZ<Fb> *>(part_raw);      // part[c * PC_WINDOWS + w]
    const uint32_t lo = a.first[blockIdx.x], n = a.first[blockIdx.x + 1] - lo;
    const Affine<Fb> *P = a.pts + lo;
    const Fs *K = a.k + lo;
    XYZZ<Fb> *T = a.tab + (size_t)PC_TABLE * lo;
    for (uint32_t j = threadIdx.x; j < n; j += PC_THREADS) {
        Affine<Fb> p;
        p.x = load_fe<Fb>(&P[j].x);
        p.y = load_fe<Fb>(&P[j].y);
        XYZZ<Fb> acc = XYZZ<Fb>::from_affine(p);
        store_xyzz(T + PC_TABLE * j, acc);
        for (int d = 1; d < PC_TABLE; d++) {
            acc.add_affine(p);
            store_xyzz(T + PC_TABLE * j + d, acc);
        }
    }
    __syncthreads();
    // a warp is 32 windows of one chunk: every lane walks the same terms
    const int w = threadIdx.x % PC_WINDOWS, c = threadIdx.x / PC_WINDOWS;
    XYZZ<Fb> acc = XYZZ<Fb>::identity();
    for (uint32_t j = c; j < n; j += PC_CHUNKS) {
        const uint32_t d = (K[j].v[w >> 3] >> (4 * (w & 7))) & 15u;
        if (d) acc.add(load_xyzz(T + PC_TABLE * j + d - 1));
    }
    part[c * PC_WINDOWS + w] = acc;
    for (int h = PC_CHUNKS / 2; h >= 1; h /= 2) {
        __syncthreads();
        if (c < h) {
            acc.add(part[(c + h) * PC_WINDOWS + w]);
            part[c * PC_WINDOWS + w] = acc;
        }
    }
    // thread w (c = 0) holds W_w: 16^w W_w by 4w doublings, then a tree over the windows -- the 63 additions of a Horner pass leave the
    // serial chain, which is window 63's 252 doublings and 6 additions
    if (c == 0) {
        for (int t = 0; t < 4 * w; t++) acc = acc.dbl();
        part[w] = acc;
    }
    for (int h = PC_WINDOWS / 2; h >= 1; h /= 2) {
        __syncthreads();
        if ((int)threadIdx.x < h) {
            acc.add(part[threadIdx.x + h]);
            part[threadIdx.x] = acc;
        }
    }
    if (threadIdx.x == 0) store_xyzz(a.out + blockIdx.x, acc);
}

// The calling thread's device and pinned scratch, grown on demand and kept for the life of the thread (as sc_scratch.cuh's pool): an
// allocation per call would cost more than the kernel.  A call synchronises its stream before it returns, so the next call of the thread
// finds the scratch free, whatever its stream.
struct PcPool {
    void *dev = nullptr, *pinned = nullptr;
    size_t dev_bytes = 0, pinned_bytes = 0;
    int device = -1;
    ~PcPool() { release(); }
    void release() {
        if (dev) cudaFree(dev);
        if (pinned) cudaFreeHost(pinned);
        dev = pinned = nullptr;
        dev_bytes = pinned_bytes = 0;
    }
    int reserve(size_t d_bytes, size_t h_bytes) {
        int cur = -1;
        LURK_CUDA_TRY(cudaGetDevice(&cur));
        if (cur != device) { release(); device = cur; }
        if (dev_bytes < d_bytes) {
            if (dev) cudaFree(dev);
            dev = nullptr;
            dev_bytes = 0;
            LURK_CUDA_TRY(cudaMalloc(&dev, d_bytes));
            dev_bytes = d_bytes;
        }
        if (pinned_bytes < h_bytes) {
            if (pinned) cudaFreeHost(pinned);
            pinned = nullptr;
            pinned_bytes = 0;
            LURK_CUDA_TRY(cudaHostAlloc(&pinned, h_bytes, cudaHostAllocDefault));
            pinned_bytes = h_bytes;
        }
        return LURK_OK;
    }
};
PcPool &pc_pool() {
    static thread_local PcPool pool;
    return pool;
}

// the parsed terms of one call and the device half of it
template <class C>
struct Batch {
    using Fb = typename C::Base;
    using Fs = typename C::Scalar;
    std::vector<Affine<Fb>> pts;      // the device groups' terms, in order
    std::vector<Fs> k;                // canonical
    std::vector<uint32_t> first{0};
    std::vector<int> dev_groups;      // indices into the caller's groups
    XYZZ<Fb> *d_out = nullptr, *h_out = nullptr;

    int launch(cudaStream_t s) {
        const size_t n = pts.size(), g = dev_groups.size();
        const size_t o_k = n * sizeof(Affine<Fb>), o_first = o_k + n * sizeof(Fs), in_bytes = o_first + 4 * (g + 1);
        const size_t o_tab = (in_bytes + 127) / 128 * 128, o_out = o_tab + PC_TABLE * n * sizeof(XYZZ<Fb>), out_bytes = g * sizeof(XYZZ<Fb>);
        const size_t o_hout = (in_bytes + 127) / 128 * 128;
        PcPool &pool = pc_pool();
        LURK_TRY(pool.reserve(o_out + out_bytes, o_hout + out_bytes));
        uint8_t *host = static_cast<uint8_t *>(pool.pinned), *d = static_cast<uint8_t *>(pool.dev);
        memcpy(host, pts.data(), o_k);
        memcpy(host + o_k, k.data(), n * sizeof(Fs));
        memcpy(host + o_first, first.data(), 4 * (g + 1));
        h_out = reinterpret_cast<XYZZ<Fb> *>(host + o_hout);
        LURK_CUDA_TRY(cudaMemcpyAsync(d, host, in_bytes, cudaMemcpyHostToDevice, s));
        PcArgs<Fb, Fs> a;
        a.pts = reinterpret_cast<const Affine<Fb> *>(d);
        a.k = reinterpret_cast<const Fs *>(d + o_k);
        a.first = reinterpret_cast<const uint32_t *>(d + o_first);
        a.tab = reinterpret_cast<XYZZ<Fb> *>(d + o_tab);
        a.out = d_out = reinterpret_cast<XYZZ<Fb> *>(d + o_out);
        point_comb_kernel<Fb, Fs><<<(unsigned)g, PC_THREADS, 0, s>>>(a);
        LURK_CUDA_TRY(cudaGetLastError());
        LURK_CUDA_TRY(cudaMemcpyAsync(h_out, d_out, out_bytes, cudaMemcpyDeviceToHost, s));
        return LURK_OK;
    }
    // waits for the stream even when the launch failed half-way, so that the scratch is free when the call returns
    int finish(const PointGroup *groups, int fmt, cudaStream_t s) {
        LURK_CUDA_TRY(cudaStreamSynchronize(s));
        for (size_t i = 0; i < dev_groups.size(); i++) point_to_bytes_fmt(h_out[i], fmt, groups[dev_groups[i]].out);
        return LURK_OK;
    }
};

}  // namespace

int point_combination_groups(int curve_id, const PointGroup *groups, int n_groups, int fmt, bool all_device, cudaStream_t s) {
    return dispatch_curve(curve_id, [&](auto cv) {
        using C = decltype(cv);
        using Fb = typename C::Base;
        using Fs = typename C::Scalar;
        const Fb b = curve_b<C>();
        Batch<C> batch;
        std::vector<char> on_device(n_groups);
        for (int g = 0; g < n_groups; g++) {
            const PointGroup &G = groups[g];
            on_device[g] = all_device || G.count >= PC_DEVICE_MIN_TERMS;
            for (int j = 0; j < G.count; j++) {
                XYZZ<Fb> p;
                Fs k;
                if (!point_in(G.points[j], fmt, b, p)) {
                    set_error("group %d: point %d is not a point of the header's form on the curve", g, j);
                    return LURK_ERR_RANGE;
                }
                if (!fe_in(G.scalars + 32 * (size_t)j, fmt, k)) { set_error("group %d: scalar %d is not reduced", g, j); return LURK_ERR_RANGE; }
                if (!on_device[g]) continue;
                Affine<Fb> a;
                a.x = p.x;          // (0, 0) for the identity, whose XYZZ form is all zeros
                a.y = p.y;
                batch.pts.push_back(a);
                batch.k.push_back(k.to_canonical());
            }
            if (on_device[g]) {
                batch.dev_groups.push_back(g);
                batch.first.push_back((uint32_t)batch.pts.size());
            }
        }
        if (!batch.dev_groups.empty()) {
            const int rc = batch.launch(s);
            if (rc != LURK_OK) {
                cudaStreamSynchronize(s);               // nothing of this call stays queued on the thread's scratch
                return rc;
            }
        }
        for (int g = 0; g < n_groups; g++)              // the host's groups while the kernel runs (checked above: they cannot fail)
            if (!on_device[g]) point_combination(curve_id, groups[g].points, groups[g].scalars, groups[g].count, fmt, groups[g].out);
        return batch.dev_groups.empty() ? LURK_OK : batch.finish(groups, fmt, s);
    });
}

}  // namespace lurk

using namespace lurk;

extern "C" {

int lurk_point_combination_batch(int curve_id, int n_groups, const uint32_t *counts, const uint8_t *points_xyz, const uint8_t *scalars, int fmt,
                                 uint8_t *out_xyz, void *stream) {
    if (!counts || !points_xyz || !scalars || !out_xyz) { set_error("null argument"); return LURK_ERR_ARG; }
    if (n_groups < 1) { set_error("at least one group, got %d", n_groups); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    if (curve_id < LURK_CURVE_BN254_G1 || curve_id > LURK_CURVE_VESTA) { set_error("unknown curve id %d", curve_id); return LURK_ERR_ARG; }
    for (int g = 0; g < n_groups; g++)
        if (counts[g] < 1 || counts[g] > (uint32_t)PC_MAX_TERMS) { set_error("group %d has %u terms, not 1 .. %d", g, counts[g], PC_MAX_TERMS); return LURK_ERR_ARG; }
    LURK_TRY(require_gpu());
    std::vector<PointGroup> groups(n_groups);
    size_t total = 0;
    for (int g = 0; g < n_groups; g++) total += counts[g];
    std::vector<const uint8_t *> pts(total);
    for (size_t k = 0; k < total; k++) pts[k] = points_xyz + 96 * k;
    size_t at = 0;
    for (int g = 0; g < n_groups; g++) {
        groups[g] = PointGroup{pts.data() + at, scalars + 32 * at, (int)counts[g], out_xyz + 96 * (size_t)g};
        at += counts[g];
    }
    return point_combination_groups(curve_id, groups.data(), n_groups, fmt, true, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
