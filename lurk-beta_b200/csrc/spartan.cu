// N4 -- the Spartan prover context (include/lurk_b200.h, "Spartan prover context"): RelaxedR1CSSNARK::prove and
// BatchedRelaxedR1CSSNARK::prove (Nova's / SuperNova's `compress`, reference src/proof/nova.rs:341-356, supernova.rs:293-317) as one
// C-ABI call each.  The host side is the chain of lurk-beta_b200/spartan.py's RelaxedR1CSProver / BatchedRelaxedR1CSProver step for step,
// but it calls the N4 templates (sumcheck_impl.cuh) directly and keeps every vector on one stream.
//
// Kernels:
//   sp_hist_kernel / sp_scan_kernel / sp_scatter_kernel   context creation: the merged transpose of A, B, C by counting sort (column
//                              histogram over the padded z, exclusive scan, scatter matrix after matrix so that a row's entries stay
//                              grouped A | B | C; the matrix rides in the top two bits of the entry's row index).
//   sp_prep_kernel             the padded z (twice: the inner sum-check binds one copy in place), the padded E and u Cz + E straight
//                              from d_z = (W, u, X) and d_E, with u read on the device; zeroes the padding rows of A z, B z, C z.
//   sp_eval_table_kernel       compute_eval_table_sparse: abc[j] = sum_e eq_rx[row_e] v_e accumulated per matrix and combined as
//                              acc_A + r acc_B + r^2 acc_C, one product per non-zero and two per row run, in one launch.  Work is split
//                              by non-zeros (SP_CHUNK per thread), so the columns of u and X (10^4 - 10^5 entries) cost what any other
//                              16 entries cost: a row cut by a chunk boundary leaves one partial per chunk it touches, the last chunk
//                              to arrive (a per-row ticket) sums them with its whole warp.  Empty rows are written in a separate
//                              row-indexed sweep of the same threads.
//   sp_matrix_eval_kernel      the verifier's (A, B, C)(r_x, r_y) in one launch: the row-major CSRs streamed once, eq(r_x) and eq(r_y)
//                              looked up in product-tensor tables in shared memory (tensor.cuh).
#include "sumcheck_impl.cuh"
#include "spmv3.cuh"
#include "tensor.cuh"

namespace lurk {

constexpr int SP_MAX_INSTANCES = SC_MAX_INSTANCES / 2;    // the reduction takes two claims (W_i, E_i) per instance
constexpr uint32_t SP_TAG_SHIFT = 30;                      // matrix of a transpose entry: top two bits of its row index
constexpr uint32_t SP_ROW_MASK = (1u << SP_TAG_SHIFT) - 1;
constexpr int SP_CHUNK = 16;                               // non-zeros per thread of the eval-table kernel

__device__ __forceinline__ uint64_t sp_col(uint32_t c, uint64_t n_w, uint64_t num_vars) { return c < n_w ? c : num_vars + (c - n_w); }

// ------------------------------------------------------------------------------------------------ context creation
__global__ void __launch_bounds__(256) sp_hist_kernel(const uint32_t *__restrict__ col, size_t nnz, uint64_t n_w, uint64_t num_vars,
                                                      unsigned long long *count) {
    for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < nnz; k += (size_t)gridDim.x * blockDim.x)
        atomicAdd(&count[sp_col(col[k], n_w, num_vars)], 1ull);
}

// exclusive scan of n counts into rp[0..n]: one CTA, every thread a contiguous segment (runs once per context)
__global__ void __launch_bounds__(1024) sp_scan_kernel(const unsigned long long *__restrict__ count, size_t n, uint64_t *__restrict__ rp) {
    __shared__ unsigned long long part[1024];
    const size_t seg = (n + blockDim.x - 1) / blockDim.x;
    const size_t lo = min(n, threadIdx.x * seg), hi = min(n, lo + seg);
    unsigned long long s = 0;
    for (size_t j = lo; j < hi; j++) s += count[j];
    part[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long run = 0;
        for (unsigned t = 0; t < blockDim.x; t++) { const unsigned long long v = part[t]; part[t] = run; run += v; }
        rp[n] = run;
    }
    __syncthreads();
    s = part[threadIdx.x];
    for (size_t j = lo; j < hi; j++) { rp[j] = s; s += count[j]; }
}

// one thread per row of matrix `tag`: every non-zero to the next free slot of its padded-z column
template <class F>
__global__ void __launch_bounds__(256) sp_scatter_kernel(const uint64_t *__restrict__ rp, const uint32_t *__restrict__ col, const F *__restrict__ val,
                                                         size_t rows, uint64_t n_w, uint64_t num_vars, uint32_t tag, unsigned long long *cursor,
                                                         uint32_t *__restrict__ trow, F *__restrict__ tval) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < rows; i += (size_t)gridDim.x * blockDim.x)
        for (uint64_t k = rp[i]; k < rp[i + 1]; k++) {
            const unsigned long long pos = atomicAdd(&cursor[sp_col(col[k], n_w, num_vars)], 1ull);
            trow[pos] = (uint32_t)i | (tag << SP_TAG_SHIFT);
            store_fe(tval + pos, load_fe<F>(val + k));
        }
}

// ------------------------------------------------------------------------------------------------ prove-time kernels
template <class F>
struct SpPrepArgs {
    const F *z, *E;
    F *zpad, *zwork, *ep, *ucze, *az, *bz, *cz;
    uint64_t n_w, n_x, rows, num_vars, rows_pad;
};

template <class F>
__global__ void __launch_bounds__(256) sp_prep_kernel(const __grid_constant__ SpPrepArgs<F> a) {
    const F u = load_fe<F>(a.z + a.n_w);
    const uint64_t nz = 2 * a.num_vars, total = nz > a.rows_pad ? nz : a.rows_pad;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        if (i < nz) {
            F v = F::zero();
            if (i < a.n_w) v = load_fe<F>(a.z + i);
            else if (i >= a.num_vars && i - a.num_vars <= a.n_x) v = load_fe<F>(a.z + a.n_w + (i - a.num_vars));
            store_fe(a.zpad + i, v);
            store_fe(a.zwork + i, v);
        }
        if (i < a.rows) {
            const F e = load_fe<F>(a.E + i);
            store_fe(a.ep + i, e);
            store_fe(a.ucze + i, u * load_fe<F>(a.cz + i) + e);
        } else if (i < a.rows_pad) {
            const F zero = F::zero();
            store_fe(a.ep + i, zero);
            store_fe(a.ucze + i, zero);
            store_fe(a.az + i, zero);
            store_fe(a.bz + i, zero);
            store_fe(a.cz + i, zero);
        }
    }
}

template <class F>
struct SpTableArgs {
    const uint64_t *rp;          // merged transpose: rows + 1 offsets
    const uint32_t *trow;        // row of the original matrix | matrix << SP_TAG_SHIFT
    const F *tval;
    size_t rows, nnz;            // rows = 2 num_vars
    size_t threads;              // ceil(nnz / SP_CHUNK), 0 without non-zeros
    size_t rows_per_thread;      // of the empty-row sweep
    const F *eq;
    F r, r2;
    F *out;
    F *slot_own, *slot_first;    // per thread: the partial of a row that starts in its chunk and runs past it / of the row it starts inside
    unsigned *ticket;            // per owner thread; reset by the finishing warp
};

// the non-empty row holding entry e: rp[j] <= e < rp[j + 1]
__device__ __forceinline__ size_t sp_row_of(const uint64_t *rp, size_t rows, uint64_t e) {
    size_t lo = 0, hi = rows;
    while (hi - lo > 1) {
        const size_t mid = (lo + hi) >> 1;
        if (rp[mid] <= e) lo = mid;
        else hi = mid;
    }
    return lo;
}

template <class F>
__device__ __forceinline__ F ldcg_fe(const F *p) {
    const uint4 *q = reinterpret_cast<const uint4 *>(p);
    const uint4 lo = __ldcg(q), hi = __ldcg(q + 1);
    F t;
    t.v[0] = lo.x; t.v[1] = lo.y; t.v[2] = lo.z; t.v[3] = lo.w; t.v[4] = hi.x; t.v[5] = hi.y; t.v[6] = hi.z; t.v[7] = hi.w;
    return t;
}

// No early exit: every lane of a warp reaches the ballots at the end.
template <class F>
__global__ void __launch_bounds__(256) sp_eval_table_kernel(const __grid_constant__ SpTableArgs<F> a) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    for (size_t j = t * a.rows_per_thread, je = min(a.rows, j + a.rows_per_thread); j < je; j++)
        if (a.rp[j] == a.rp[j + 1]) store_fe(a.out + j, F::zero());

    bool has_first = false, has_own = false;
    size_t row_first = 0, row_own = 0;
    if (t < a.threads) {
        const uint64_t c0 = (uint64_t)t * SP_CHUNK, c1 = min((uint64_t)a.nnz, c0 + SP_CHUNK);
        uint64_t e = c0;
        size_t j = sp_row_of(a.rp, a.rows, e);
        while (true) {
            const uint64_t r0 = a.rp[j], r1 = a.rp[j + 1], stop = min(r1, c1);
            F acc0 = F::zero(), acc1 = F::zero(), acc2 = F::zero();
            for (; e < stop; e++) {
                const uint32_t w = a.trow[e];
                const F p = load_fe<F>(a.tval + e) * load_fe<F>(a.eq + (w & SP_ROW_MASK));
                const uint32_t m = w >> SP_TAG_SHIFT;
                if (m == 0) acc0 += p;
                else if (m == 1) acc1 += p;
                else acc2 += p;
            }
            const F v = acc0 + a.r * acc1 + a.r2 * acc2;
            const bool starts = r0 >= c0, ends = r1 <= c1;
            if (starts && ends) store_fe(a.out + j, v);
            else if (starts) { store_fe(a.slot_own + t, v); row_own = j; has_own = true; }
            else { store_fe(a.slot_first + t, v); row_first = j; has_first = true; }
            if (e >= c1) break;
            j++;
            if (a.rp[j + 1] == e) j = sp_row_of(a.rp, a.rows, e);      // skip a run of empty rows
        }
    }
    // a row cut by chunk boundaries: owner t0 = rp[j] / SP_CHUNK contributes slot_own, chunks t0 + 1 .. t1 slot_first
    bool fin_first = false, fin_own = false;
    if (has_first || has_own) __threadfence();
    if (has_first) {
        const uint64_t t0 = a.rp[row_first] / SP_CHUNK, t1 = (a.rp[row_first + 1] - 1) / SP_CHUNK;
        fin_first = atomicAdd(&a.ticket[t0], 1u) == (unsigned)(t1 - t0);
    }
    if (has_own) {
        const uint64_t t0 = a.rp[row_own] / SP_CHUNK, t1 = (a.rp[row_own + 1] - 1) / SP_CHUNK;
        fin_own = atomicAdd(&a.ticket[t0], 1u) == (unsigned)(t1 - t0);
    }
#pragma unroll 1
    for (int pass = 0; pass < 2; pass++) {
        unsigned mask = __ballot_sync(0xffffffffu, pass ? fin_own : fin_first);
        while (mask) {
            const int src = __ffs(mask) - 1;
            mask &= mask - 1;
            const size_t j = (size_t)__shfl_sync(0xffffffffu, (unsigned long long)(pass ? row_own : row_first), src);
            __threadfence();
            const uint64_t t0 = a.rp[j] / SP_CHUNK, t1 = (a.rp[j + 1] - 1) / SP_CHUNK;
            F s = F::zero();
            for (uint64_t q = t0 + lane; q <= t1; q += 32) s += ldcg_fe(q == t0 ? a.slot_own + q : a.slot_first + q);
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) s = s + shfl_down_fe(s, off);
            if (lane == 0) {
                store_fe(a.out + j, s);
                a.ticket[t0] = 0;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ verify-time kernel
// (A(rx, ry), B(rx, ry), C(rx, ry)) = sum over the non-zeros of M of eq(rx, row) M[row][col] eq(ry, col') with col' the column in the
// padded z.  The three row-major CSRs are one range of non-zeros (A | B | C) cut into SP_CHUNK-element chunks, so a row of 2000 entries
// is spread over many threads; a cut row needs no fix-up because the partial sums only add.  eq(rx) and eq(ry) come from product-tensor
// tables built per CTA in shared memory (tensor.cuh): nothing of O(rows) or O(columns) is read or written besides the CSR itself.
template <class F>
struct SpMatArgs {
    const uint64_t *rp[3];
    const uint32_t *col[3];
    const F *val[3];
    uint64_t off[4];             // first non-zero of A, B, C in the joint range; off[3] = total
    uint64_t chunks;             // ceil(off[3] / SP_CHUNK)
    size_t rows;
    uint64_t n_w, num_vars;
    TensorSpec<F> x, y;          // eq(rx) over the log_rows row bits, eq(ry) over the log_vars + 1 bits of the padded z
    F *partial;
    unsigned *counter;
    F *result;                   // 3 elements
};

template <class F>
__global__ void __launch_bounds__(256, 2) sp_matrix_eval_kernel(const __grid_constant__ SpMatArgs<F> a) {
    extern __shared__ uint4 sp_tensor_smem[];
    F *tx = reinterpret_cast<F *>(sp_tensor_smem);
    const int gx = tensor_groups(a.x.l), gy = tensor_groups(a.y.l);
    F *ty = tx + gx * TENSOR_GROUP;
    tensor_build(a.x, tx);
    tensor_build(a.y, ty);
    __syncthreads();
    F acc[3] = {F::zero(), F::zero(), F::zero()};
    for (uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; c < a.chunks; c += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t c1 = min(a.off[3], (c + 1) * SP_CHUNK);
        uint64_t e = c * SP_CHUNK;
        while (e < c1) {
            const int m = (e >= a.off[1]) + (e >= a.off[2]);        // empty matrices have off[m] = off[m + 1] and are skipped
            const uint64_t base = a.off[m], stop = min(c1, a.off[m + 1]) - base;
            const uint64_t *rp = m == 0 ? a.rp[0] : m == 1 ? a.rp[1] : a.rp[2];
            const uint32_t *col = m == 0 ? a.col[0] : m == 1 ? a.col[1] : a.col[2];
            const F *val = m == 0 ? a.val[0] : m == 1 ? a.val[1] : a.val[2];
            uint64_t k = e - base;
            size_t j = sp_row_of(rp, a.rows, k);
            F sum = F::zero();
            while (true) {
                const uint64_t end = min(rp[j + 1], stop);
                F row = F::zero();
                for (; k < end; k++) row += load_fe<F>(val + k) * tensor_at(ty, gy, sp_col(col[k], a.n_w, a.num_vars));
                sum += tensor_at(tx, gx, j) * row;
                if (k >= stop) break;
                j++;
                if (rp[j + 1] == k) j = sp_row_of(rp, a.rows, k);      // skip a run of empty rows
            }
            if (m == 0) acc[0] += sum;
            else if (m == 1) acc[1] += sum;
            else acc[2] += sum;
            e = base + stop;
        }
    }
    grid_sum<F, 3>(acc, a.partial, a.counter, a.result);
}

}  // namespace lurk

using namespace lurk;

// ------------------------------------------------------------------------------------------------ the context
struct lurk_spartan_ctx {
    int field_id = 0;
    uint64_t n_w = 0, n_x = 0, rows = 0, num_vars = 0;
    int log_rows = 0, log_vars = 0;
    bool verifier_only = false;  // the three CSRs only: no merged transpose, eval-table slots or tickets
    virtual ~lurk_spartan_ctx() {}
    size_t z_len() const { return n_w + 1 + n_x; }
};

namespace lurk {

template <class F>
struct SpartanCtx : lurk_spartan_ctx {
    DevBuf rp[3], col[3], val[3];
    CsrDev csr[3];
    DevBuf trp, trow, tval, slots, ticket;
    DevBuf work;                 // the prover's vectors, allocated by the first proof and kept: a fresh 0.6 GB per call at fib rc = 100
                                 // would cost more than the eval table saves
    size_t tnnz = 0, threads = 0;
    uint64_t nnz[3] = {0, 0, 0};

    // Az, Bz, Cz, u Cz + E, eq, E padded (2^log_rows each) | z padded, its working copy, abc (2 num_vars each)
    int work_area(F **out) {
        const size_t want = (6 * ((size_t)1 << log_rows) + 3 * 2 * (size_t)num_vars) * sizeof(F);
        if (work.bytes < want) LURK_TRY(work.alloc(want));
        *out = work.as<F>();
        return LURK_OK;
    }

    int init(const uint64_t *const row_ptr[3], const uint32_t *const cols[3], const uint8_t *const vals[3], int fmt) {
        cudaStream_t s = 0;
        for (int m = 0; m < 3; m++) {
            const size_t nnz = (size_t)row_ptr[m][rows];
            LURK_TRY(rp[m].alloc((rows + 1) * sizeof(uint64_t)));
            LURK_TRY(col[m].alloc(std::max<size_t>(1, nnz) * sizeof(uint32_t)));
            LURK_TRY(val[m].alloc(std::max<size_t>(1, nnz) * sizeof(F)));
            LURK_CUDA_TRY(cudaMemcpy(rp[m].p, row_ptr[m], (rows + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice));
            if (nnz) {
                LURK_CUDA_TRY(cudaMemcpy(col[m].p, cols[m], nnz * sizeof(uint32_t), cudaMemcpyHostToDevice));
                LURK_CUDA_TRY(cudaMemcpy(val[m].p, vals[m], nnz * sizeof(F), cudaMemcpyHostToDevice));
                int bad = 0;
                LURK_TRY(check_reduced_dev<F>(val[m].p, nnz, s, &bad));
                if (bad) { set_error("matrix %d: %d coefficient(s) not reduced", m, bad); return LURK_ERR_RANGE; }
                if (fmt == LURK_FMT_CANONICAL) LURK_TRY(convert_dev<F>(val[m].p, nnz, LURK_FMT_MONTGOMERY, val[m].p, s));
            }
            csr[m].row_ptr = rp[m].as<uint64_t>();
            csr[m].col = col[m].as<uint32_t>();
            csr[m].val = val[m].p;
            this->nnz[m] = nnz;
            tnnz += nnz;
        }
        if (verifier_only) {
            LURK_CUDA_TRY(cudaStreamSynchronize(s));     // the conversions above
            return LURK_OK;
        }
        // merged transpose over the padded z's 2 num_vars columns
        const size_t trows = 2 * num_vars;
        DevBuf count;
        LURK_TRY(count.alloc(trows * sizeof(unsigned long long)));
        LURK_TRY(trp.alloc((trows + 1) * sizeof(uint64_t)));
        LURK_TRY(trow.alloc(std::max<size_t>(1, tnnz) * sizeof(uint32_t)));
        LURK_TRY(tval.alloc(std::max<size_t>(1, tnnz) * sizeof(F)));
        LURK_CUDA_TRY(cudaMemsetAsync(count.p, 0, trows * sizeof(unsigned long long), s));
        for (int m = 0; m < 3; m++) {
            const size_t nnz = (size_t)row_ptr[m][rows];
            if (nnz) sp_hist_kernel<<<sc_grid(nnz, 256), 256, 0, s>>>(col[m].as<uint32_t>(), nnz, n_w, num_vars, count.as<unsigned long long>());
        }
        sp_scan_kernel<<<1, 1024, 0, s>>>(count.as<unsigned long long>(), trows, trp.as<uint64_t>());
        LURK_CUDA_TRY(cudaMemcpyAsync(count.p, trp.p, trows * sizeof(uint64_t), cudaMemcpyDeviceToDevice, s));     // the cursors
        for (int m = 0; m < 3; m++)
            sp_scatter_kernel<F><<<sc_grid(rows, 256), 256, 0, s>>>(rp[m].as<uint64_t>(), col[m].as<uint32_t>(), val[m].as<F>(), rows, n_w, num_vars,
                                                                     (uint32_t)m, count.as<unsigned long long>(), trow.as<uint32_t>(), tval.as<F>());
        LURK_CUDA_TRY(cudaGetLastError());
        threads = (tnnz + SP_CHUNK - 1) / SP_CHUNK;
        LURK_TRY(slots.alloc(2 * std::max<size_t>(1, threads) * sizeof(F)));
        LURK_TRY(ticket.alloc(std::max<size_t>(1, threads) * sizeof(unsigned)));
        LURK_CUDA_TRY(cudaMemsetAsync(ticket.p, 0, std::max<size_t>(1, threads) * sizeof(unsigned), s));
        LURK_CUDA_TRY(cudaStreamSynchronize(s));
        return LURK_OK;
    }

    int eval_table(const F *eq, const F &r, F *out, cudaStream_t s) {
        SpTableArgs<F> a;
        memset(&a, 0, sizeof a);
        a.rp = trp.as<uint64_t>();
        a.trow = trow.as<uint32_t>();
        a.tval = tval.as<F>();
        a.rows = 2 * num_vars;
        a.nnz = tnnz;
        a.threads = threads;
        const size_t grid = std::max<size_t>(1, (threads + 255) / 256);
        a.rows_per_thread = (a.rows + grid * 256 - 1) / (grid * 256);
        a.eq = eq;
        a.r = r;
        a.r2 = r * r;
        a.out = out;
        a.slot_own = slots.as<F>();
        a.slot_first = slots.as<F>() + threads;
        a.ticket = ticket.as<unsigned>();
        sp_eval_table_kernel<F><<<(unsigned)grid, 256, 0, s>>>(a);
        LURK_CUDA_TRY(cudaGetLastError());
        return LURK_OK;
    }

    // (A, B, C)(rx, ry) into res[0..3) of the scratch's pinned result slots, Montgomery; asynchronous on s.  rx: log_rows elements,
    // ry: log_vars + 1.
    int matrix_evals(const F *rx, const F *ry, ScScratch<F> &sc, F *res, cudaStream_t s) {
        SpMatArgs<F> a;
        memset(&a, 0, sizeof a);
        for (int m = 0; m < 3; m++) {
            a.rp[m] = csr[m].row_ptr;
            a.col[m] = csr[m].col;
            a.val[m] = static_cast<const F *>(csr[m].val);
            a.off[m + 1] = a.off[m] + nnz[m];
        }
        a.chunks = (a.off[3] + SP_CHUNK - 1) / SP_CHUNK;
        a.rows = rows;
        a.n_w = n_w;
        a.num_vars = num_vars;
        a.x.l = log_rows;
        a.y.l = log_vars + 1;
        for (int j = 0; j < a.x.l; j++) { a.x.hi[j] = rx[j]; a.x.lo[j] = F::one() - rx[j]; }
        for (int j = 0; j < a.y.l; j++) { a.y.hi[j] = ry[j]; a.y.lo[j] = F::one() - ry[j]; }
        a.partial = sc.partial;
        a.counter = sc.counter;
        a.result = res;
        const size_t smem = (size_t)(tensor_groups(a.x.l) + tensor_groups(a.y.l)) * TENSOR_GROUP * sizeof(F);
        LURK_CUDA_TRY(cudaFuncSetAttribute(sp_matrix_eval_kernel<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const uint64_t want = (a.chunks + 255) / 256;
        const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(want, 2 * (uint64_t)sm_count()));
        sp_matrix_eval_kernel<F><<<grid, 256, smem, s>>>(a);
        LURK_CUDA_TRY(cudaGetLastError());
        return LURK_OK;
    }
};

// the phase-tagged transcript behind the templates' plain callbacks
struct PhaseChallenge { lurk_spartan_challenge_fn fn; void *user; int phase; };
static int phase_challenge(void *user, int round, const uint8_t *message, size_t message_len, uint8_t challenge_out[32]) {
    const PhaseChallenge *c = static_cast<const PhaseChallenge *>(user);
    return c->fn(c->user, c->phase, round, message, message_len, challenge_out);
}

template <class F>
static int ask(lurk_spartan_challenge_fn fn, void *user, int phase, int round, const uint8_t *msg, size_t len, int fmt, F &out) {
    uint8_t b[32];
    const int rc = fn(user, phase, round, msg, len, b);
    if (rc != 0) { set_error("challenge callback failed in phase %d, round %d (%d)", phase, round, rc); return LURK_ERR_ARG; }
    if (!fe_in(b, fmt, out)) { set_error("challenge of phase %d, round %d is not reduced", phase, round); return LURK_ERR_RANGE; }
    return LURK_OK;
}

template <class F>
static EqArgs<F> eq_args(const F *tau, int l) {
    EqArgs<F> a;
    memset(&a, 0, sizeof a);
    a.l = l;
    for (int j = 0; j < l; j++) { a.tau[j] = tau[j]; a.one_minus[j] = F::one() - tau[j]; }
    return a;
}

// RelaxedR1CSSNARK::prove (batched = false, n = 1) or BatchedRelaxedR1CSSNARK::prove, then batch_eval_reduce over [W_i .., E_i ..]
template <class F>
static int spartan_prove(int n, lurk_spartan_ctx *const *ctxs, const void *const *d_z, const void *const *d_E, lurk_spartan_challenge_fn fn,
                         void *user, lurk_spartan_proof *out, void *d_joint, int fmt, cudaStream_t s, bool batched) {
    struct Inst { F *az, *bz, *cz, *ucze, *eq, *ep, *zpad, *zwork, *abc; };
    std::vector<SpartanCtx<F> *> C(n);
    std::vector<int> S(n), T(n), V(n);
    std::vector<Inst> I(n);
    int maxS = 0, maxT = 0;
    for (int i = 0; i < n; i++) {
        C[i] = static_cast<SpartanCtx<F> *>(ctxs[i]);
        S[i] = C[i]->log_rows;
        V[i] = C[i]->log_vars;
        T[i] = V[i] + 1;
        maxS = std::max(maxS, S[i]);
        maxT = std::max(maxT, T[i]);
    }
    for (int i = 0; i < n; i++)
        for (int k = 0; k < i; k++)
            if (C[k] == C[i]) { set_error("instances %d and %d share a context", k, i); return LURK_ERR_ARG; }
    for (int i = 0; i < n; i++) {
        const size_t rp = (size_t)1 << S[i], nz = 2 * (size_t)C[i]->num_vars;
        Inst &x = I[i];
        F *p = nullptr;
        LURK_TRY(C[i]->work_area(&p));
        x.az = p; x.bz = p + rp; x.cz = p + 2 * rp; x.ucze = p + 3 * rp; x.eq = p + 4 * rp; x.ep = p + 5 * rp;
        p += 6 * rp;
        x.zpad = p; x.zwork = p + nz; x.abc = p + 2 * nz;
        SpartanCtx<F> &c = *C[i];
        spmv3_kernel<F><<<dim3(sc_grid(c.rows, 256), 3), 256, 0, s>>>(c.csr[0], c.csr[1], c.csr[2], c.rows, static_cast<const F *>(d_z[i]), x.az, x.bz, x.cz);
        SpPrepArgs<F> pa;
        pa.z = static_cast<const F *>(d_z[i]);
        pa.E = static_cast<const F *>(d_E[i]);
        pa.zpad = x.zpad; pa.zwork = x.zwork; pa.ep = x.ep; pa.ucze = x.ucze; pa.az = x.az; pa.bz = x.bz; pa.cz = x.cz;
        pa.n_w = c.n_w; pa.n_x = c.n_x; pa.rows = c.rows; pa.num_vars = c.num_vars; pa.rows_pad = rp;
        sp_prep_kernel<F><<<sc_grid(std::max(nz, rp), 256), 256, 0, s>>>(pa);
    }
    LURK_CUDA_TRY(cudaGetLastError());

    // tau -> eq tables of the outer sum-check
    if (!batched) {
        std::vector<F> tau(S[0]);
        for (int j = 0; j < S[0]; j++) LURK_TRY(ask(fn, user, LURK_SPARTAN_TAU, j, nullptr, 0, fmt, tau[j]));
        LURK_TRY(eq_launch<F>(eq_args(tau.data(), S[0]), I[0].eq, 0, s));
    } else {
        F tau;
        LURK_TRY(ask(fn, user, LURK_SPARTAN_TAU, 0, nullptr, 0, fmt, tau));
        for (int i = 0; i < n; i++) {
            std::vector<F> pw(S[i]);
            pw[0] = tau;
            for (int j = 1; j < S[i]; j++) pw[j] = pw[j - 1] * pw[j - 1];
            LURK_TRY(eq_launch<F>(eq_args(pw.data(), S[i]), I[i].eq, 0, s));
        }
    }
    // outer sum-check: sum_i coeff_i eq_i (Az_i Bz_i - (u_i Cz_i + E_i)) = 0
    std::vector<uint8_t> zeros(32 * (size_t)n, 0), coeffs(32 * (size_t)n);
    if (batched) {
        F outer_r, c = F::one();
        LURK_TRY(ask(fn, user, LURK_SPARTAN_OUTER_R, 0, nullptr, 0, fmt, outer_r));
        for (int i = 0; i < n; i++, c = c * outer_r) fe_out(c, fmt, coeffs.data() + 32 * i);
    }
    std::vector<void *> polys(4 * (size_t)n);
    for (int i = 0; i < n; i++) { polys[4 * i] = I[i].eq; polys[4 * i + 1] = I[i].az; polys[4 * i + 2] = I[i].bz; polys[4 * i + 3] = I[i].ucze; }
    std::vector<uint8_t> o_rounds(32 * 4 * (size_t)maxS), rx(32 * (size_t)maxS), fin(32 * 4 * (size_t)n);
    PhaseChallenge pc{fn, user, LURK_SPARTAN_OUTER};
    LURK_TRY((sumcheck_prove_batch<F, SC_CUBIC>(n, polys.data(), S.data(), zeros.data(), batched ? coeffs.data() : nullptr, phase_challenge, &pc,
                                                o_rounds.data(), rx.data(), fin.data(), fmt, s)));

    // claims at rx_i: Az, Bz from the sum-check, Cz and E as <., eq(rx_i)>
    ScScratch<F> sc;
    LURK_TRY(sc.init(s));
    std::vector<uint8_t> claims(32 * 4 * (size_t)n);
    std::vector<F> cl(4 * (size_t)n);
    for (int i = 0; i < n; i++) {
        std::vector<F> x(S[i]);
        for (int j = 0; j < S[i]; j++) fe_in(rx.data() + 32 * (size_t)(maxS - S[i] + j), fmt, x[j]);
        LURK_TRY(eq_launch<F>(eq_args(x.data(), S[i]), I[i].eq, 0, s));      // the outer sum-check has consumed eq(tau)
        fe_in(fin.data() + 32 * (4 * i + 1), fmt, cl[4 * i]);
        fe_in(fin.data() + 32 * (4 * i + 2), fmt, cl[4 * i + 1]);
        LURK_TRY(dot_dev<F>(I[i].cz, I[i].eq, (size_t)1 << S[i], &cl[4 * i + 2], sc, s));
        LURK_TRY(dot_dev<F>(I[i].ep, I[i].eq, (size_t)1 << S[i], &cl[4 * i + 3], sc, s));
        for (int k = 0; k < 4; k++) fe_out(cl[4 * i + k], fmt, claims.data() + 32 * (4 * i + k));
    }
    F r;
    LURK_TRY(ask(fn, user, LURK_SPARTAN_CLAIMS, 0, claims.data(), claims.size(), fmt, r));
    const F r2 = r * r, r3 = r2 * r;

    // eval tables, then the inner sum-check: sum_i coeff_i <abc_i, z_i> = sum_i coeff_i joint_i
    std::vector<uint8_t> joint(32 * (size_t)n);
    F c = F::one();
    for (int i = 0; i < n; i++, c = c * r3) {
        LURK_TRY(C[i]->eval_table(I[i].eq, r, I[i].abc, s));
        fe_out(cl[4 * i] + r * cl[4 * i + 1] + r2 * cl[4 * i + 2], fmt, joint.data() + 32 * i);
        fe_out(c, fmt, coeffs.data() + 32 * i);
        polys[2 * i] = I[i].abc;
        polys[2 * i + 1] = I[i].zwork;
    }
    std::vector<uint8_t> i_rounds(32 * 3 * (size_t)maxT), ry(32 * (size_t)maxT);
    pc.phase = LURK_SPARTAN_INNER;
    LURK_TRY((sumcheck_prove_batch<F, SC_QUAD>(n, polys.data(), T.data(), joint.data(), batched ? coeffs.data() : nullptr, phase_challenge, &pc,
                                               i_rounds.data(), ry.data(), nullptr, fmt, s)));

    // eval_W = <W padded, eq(ry_i[1:])>; the eq table goes where abc was (consumed)
    std::vector<uint8_t> eval_w(32 * (size_t)n);
    std::vector<uint8_t> points, evals(32 * 2 * (size_t)n);
    std::vector<const void *> rpolys(2 * (size_t)n);
    std::vector<int> rnv(2 * (size_t)n);
    for (int i = 0; i < n; i++) {
        const uint8_t *y = ry.data() + 32 * (size_t)(maxT - T[i] + 1);
        std::vector<F> x(V[i]);
        for (int j = 0; j < V[i]; j++) fe_in(y + 32 * j, fmt, x[j]);
        LURK_TRY(eq_launch<F>(eq_args(x.data(), V[i]), I[i].abc, 0, s));
        F ew;
        LURK_TRY(dot_dev<F>(I[i].zpad, I[i].abc, C[i]->num_vars, &ew, sc, s));
        fe_out(ew, fmt, eval_w.data() + 32 * i);
        points.insert(points.end(), y, y + 32 * (size_t)V[i]);
        memcpy(evals.data() + 32 * i, eval_w.data() + 32 * i, 32);
        memcpy(evals.data() + 32 * (n + i), claims.data() + 32 * (4 * i + 3), 32);
        rpolys[i] = I[i].zpad;
        rnv[i] = V[i];
        rpolys[n + i] = I[i].ep;
        rnv[n + i] = S[i];
    }
    for (int i = 0; i < n; i++) points.insert(points.end(), rx.data() + 32 * (size_t)(maxS - S[i]), rx.data() + 32 * (size_t)maxS);
    pc.phase = LURK_SPARTAN_BATCH_EVAL;
    LURK_TRY(batch_eval_reduce<F>(2 * n, rpolys.data(), rnv.data(), points.data(), evals.data(), phase_challenge, &pc, out->reduce_rounds, out->r,
                                  out->claims_left, out->weights, out->joint_eval, d_joint, fmt, s));
    LURK_CUDA_TRY(cudaStreamSynchronize(s));
    if (out->outer_rounds) memcpy(out->outer_rounds, o_rounds.data(), o_rounds.size());
    if (out->r_x) memcpy(out->r_x, rx.data(), rx.size());
    if (out->claims) memcpy(out->claims, claims.data(), claims.size());
    if (out->inner_rounds) memcpy(out->inner_rounds, i_rounds.data(), i_rounds.size());
    if (out->r_y) memcpy(out->r_y, ry.data(), ry.size());
    if (out->eval_W) memcpy(out->eval_W, eval_w.data(), eval_w.size());
    return LURK_OK;
}

// the prover behind lurk_spartan_prove_dev / _batch_dev for compress.cu, whose arguments its own checks have covered
int spartan_prove_checked(int n, lurk_spartan_ctx *const *ctxs, const void *const *d_z, const void *const *d_E, lurk_spartan_challenge_fn fn, void *user,
                          lurk_spartan_proof *out, void *d_joint, int fmt, cudaStream_t s, bool batched) {
    return dispatch_field(ctxs[0]->field_id, [&](auto f) { return spartan_prove<decltype(f)>(n, ctxs, d_z, d_E, fn, user, out, d_joint, fmt, s, batched); });
}

// ------------------------------------------------------------------------------------------------ the verifier
template <class F>
static F pow2(int k) { F r = F::one(); const F two = F::from_u64(2); for (int j = 0; j < k; j++) r = r * two; return r; }

// eq(a, b) = prod_j (a_j b_j + (1 - a_j)(1 - b_j))
template <class F>
static F eq_at(const F *a, const F *b, int l) {
    F r = F::one();
    for (int j = 0; j < l; j++) r = r * (a[j] * b[j] + (F::one() - a[j]) * (F::one() - b[j]));
    return r;
}

// The MLE of (tail | 0 ..) of 2^l elements at y[0 .. l): with 2^q >= |tail| the top l - q variables only select the zero-padded prefix.
template <class F>
static F tail_eval(std::vector<F> v, const F *y, int l) {
    int q = 0;
    while (((size_t)1 << q) < v.size()) q++;
    F scale = F::one();
    for (int j = 0; j < l - q; j++) scale = scale * (F::one() - y[j]);
    v.resize((size_t)1 << q, F::zero());
    for (int j = l - q; j < l; j++) {
        const size_t half = v.size() / 2;
        for (size_t i = 0; i < half; i++) v[i] = v[i] + y[j] * (v[i + half] - v[i]);
        v.resize(half);
    }
    return scale * v[0];
}

static bool all_reduced(const uint8_t *in, size_t count, int fmt, int field_id) {
    return dispatch_field(field_id, [&](auto f) {
        using F = decltype(f);
        F x;
        for (size_t i = 0; i < count; i++)
            if (!fe_in(in + 32 * i, fmt, x)) return 0;
        return 1;
    }) == 1;
}

// Round j of a sum-check of degree `deg` as the proof holds it: s(0) | .. | s(deg) (LURK_SPARTAN_ROUNDS_EVALS; the round must sum to the
// running claim) or Arecibo's CompressedUniPoly, every coefficient but the linear one, constant first (LURK_SPARTAN_ROUNDS_COMPRESSED;
// decompress(hint): the linear coefficient is what makes s(0) + s(1) the claim).  Each round hands s(0) | .. | s(deg) to the transcript
// (phase, round first_round + j) and continues from s(r_j).  Returns LURK_OK with ok = false when a round does not sum to its claim.
template <class F>
static int sumcheck_verify(const uint8_t *rounds_in, int rounds, int deg, int rounds_fmt, lurk_spartan_challenge_fn fn, void *user, int phase,
                           int first_round, int fmt, F &claim, std::vector<F> &r, bool &ok) {
    const ScLagrange<F> lagrange(deg + 1);
    const int per = rounds_fmt == LURK_SPARTAN_ROUNDS_EVALS ? deg + 1 : deg;
    r.assign(rounds, F::zero());
    ok = true;
    for (int j = 0; j < rounds; j++) {
        const uint8_t *in = rounds_in + (size_t)32 * per * j;
        F ev[4];
        if (rounds_fmt == LURK_SPARTAN_ROUNDS_EVALS) {
            for (int t = 0; t <= deg; t++) fe_in(in + 32 * t, fmt, ev[t]);
            if (ev[0] + ev[1] != claim) { ok = false; return LURK_OK; }
        } else {
            F c[4];
            fe_in(in, fmt, c[0]);
            c[1] = claim - c[0] - c[0];
            for (int t = 2; t <= deg; t++) { fe_in(in + 32 * (t - 1), fmt, c[t]); c[1] = c[1] - c[t]; }
            for (int x = 0; x <= deg; x++) {
                const F xv = F::from_u64((uint64_t)x);
                F v = c[deg];
                for (int t = deg - 1; t >= 0; t--) v = v * xv + c[t];
                ev[x] = v;
            }
        }
        uint8_t msg[4 * 32];
        for (int t = 0; t <= deg; t++) fe_out(ev[t], fmt, msg + 32 * t);
        LURK_TRY(ask(fn, user, phase, first_round + j, msg, (size_t)32 * (deg + 1), fmt, r[j]));
        claim = lagrange.eval(ev, r[j]);
    }
    return LURK_OK;
}

// The verifier's inputs read and range-checked: u, X of every instance and the proof's fields.  A value >= p is an error, not a rejection.
template <class F>
static int verify_inputs(int n, lurk_spartan_ctx *const *ctxs, const uint8_t *u_in, const uint8_t *const *X_in, const lurk_spartan_proof *proof,
                         int rounds_fmt, int fmt, std::vector<F> &u, std::vector<std::vector<F>> &X, std::vector<F> &cl, std::vector<F> &ew,
                         std::vector<F> &left) {
    int maxS = 0, maxT = 0;
    for (int i = 0; i < n; i++) {
        maxS = std::max(maxS, ctxs[i]->log_rows);
        maxT = std::max(maxT, ctxs[i]->log_vars + 1);
    }
    const int m = std::max(maxS, maxT - 1);
    const bool evals = rounds_fmt == LURK_SPARTAN_ROUNDS_EVALS;
    const int fid = ctxs[0]->field_id;
    u.assign(n, F::zero());
    cl.assign(4 * (size_t)n, F::zero());
    ew.assign(n, F::zero());
    left.assign(2 * (size_t)n, F::zero());
    X.assign(n, {});
    for (int i = 0; i < n; i++) {
        if (!fe_in(u_in + 32 * i, fmt, u[i])) { set_error("u of instance %d is not reduced", i); return LURK_ERR_RANGE; }
        X[i].resize(ctxs[i]->n_x);
        for (uint64_t k = 0; k < ctxs[i]->n_x; k++)
            if (!fe_in(X_in[i] + 32 * k, fmt, X[i][k])) { set_error("X[%llu] of instance %d is not reduced", (unsigned long long)k, i); return LURK_ERR_RANGE; }
    }
    struct Field { const uint8_t *p; size_t count; const char *name; F *out; };
    const Field fields[] = {{proof->outer_rounds, (size_t)maxS * (evals ? 4 : 3), "outer_rounds", nullptr},
                            {proof->inner_rounds, (size_t)maxT * (evals ? 3 : 2), "inner_rounds", nullptr},
                            {proof->reduce_rounds, (size_t)m * (evals ? 3 : 2), "reduce_rounds", nullptr},
                            {proof->claims, 4 * (size_t)n, "claims", cl.data()},
                            {proof->eval_W, (size_t)n, "eval_W", ew.data()},
                            {proof->claims_left, 2 * (size_t)n, "claims_left", left.data()}};
    for (const Field &f : fields) {
        if (!all_reduced(f.p, f.count, fmt, fid)) { set_error("proof field %s holds a value that is not reduced", f.name); return LURK_ERR_RANGE; }
        for (size_t k = 0; f.out && k < f.count; k++) fe_in(f.p + 32 * k, fmt, f.out[k]);
    }
    return LURK_OK;
}

// RelaxedR1CSSNARK::verify (batched = false, n = 1) or BatchedRelaxedR1CSSNARK::verify up to the opening, then the verifier of
// batch_eval_reduce over [W_i .., E_i ..]: the same transcript calls as spartan_prove, in the same order.  The matrices' evaluations at
// (rx_i, ry_i) are one sp_matrix_eval_kernel launch per instance and one synchronisation; everything else is O(log) host arithmetic (and
// O(n_x) for eval_X).  A failed check returns LURK_OK with *accepted = 0.
template <class F>
static int spartan_verify(int n, lurk_spartan_ctx *const *ctxs, const uint8_t *u_in, const uint8_t *const *X_in, lurk_spartan_proof *proof,
                          int rounds_fmt, lurk_spartan_challenge_fn fn, void *user, int *accepted, int fmt, cudaStream_t s, bool batched) {
    *accepted = 0;
    std::vector<SpartanCtx<F> *> C(n);
    std::vector<int> S(n), T(n);
    int maxS = 0, maxT = 0;
    for (int i = 0; i < n; i++) {
        C[i] = static_cast<SpartanCtx<F> *>(ctxs[i]);
        S[i] = C[i]->log_rows;
        T[i] = C[i]->log_vars + 1;
        maxS = std::max(maxS, S[i]);
        maxT = std::max(maxT, T[i]);
    }
    const int m = std::max(maxS, maxT - 1);
    // every input is checked before the first transcript call
    std::vector<F> u, cl, ew, left;
    std::vector<std::vector<F>> X;
    LURK_TRY(verify_inputs<F>(n, ctxs, u_in, X_in, proof, rounds_fmt, fmt, u, X, cl, ew, left));

    // tau, outer_r
    std::vector<std::vector<F>> tau(n);
    F outer_r = F::one();
    if (!batched) {
        tau[0].resize(S[0]);
        for (int j = 0; j < S[0]; j++) LURK_TRY(ask(fn, user, LURK_SPARTAN_TAU, j, nullptr, 0, fmt, tau[0][j]));
    } else {
        F t;
        LURK_TRY(ask(fn, user, LURK_SPARTAN_TAU, 0, nullptr, 0, fmt, t));
        for (int i = 0; i < n; i++) {
            tau[i].resize(S[i]);
            tau[i][0] = t;
            for (int j = 1; j < S[i]; j++) tau[i][j] = tau[i][j - 1] * tau[i][j - 1];
        }
        LURK_TRY(ask(fn, user, LURK_SPARTAN_OUTER_R, 0, nullptr, 0, fmt, outer_r));
    }
    // outer sum-check: claim 0, final value sum_i outer_r^i eq(tau_i, rx_i) (Az Bz - u Cz - E)_i
    bool ok = true;
    F e = F::zero();
    std::vector<F> rx, ry, rr;
    LURK_TRY(sumcheck_verify<F>(proof->outer_rounds, maxS, 3, rounds_fmt, fn, user, LURK_SPARTAN_OUTER, 0, fmt, e, rx, ok));
    if (!ok) return LURK_OK;
    F want = F::zero(), c = F::one();
    for (int i = 0; i < n; i++, c = c * outer_r) {
        const F *k = &cl[4 * i];
        want += c * eq_at(tau[i].data(), rx.data() + (maxS - S[i]), S[i]) * (k[0] * k[1] - u[i] * k[2] - k[3]);
    }
    if (e != want) return LURK_OK;
    // r, the inner sum-check: claim sum_i (r^3)^i 2^(maxT - T_i) joint_i
    F r;
    LURK_TRY(ask(fn, user, LURK_SPARTAN_CLAIMS, 0, proof->claims, 4 * 32 * (size_t)n, fmt, r));
    const F r2 = r * r, r3 = r2 * r;
    e = F::zero();
    c = F::one();
    for (int i = 0; i < n; i++, c = c * r3) e += c * (cl[4 * i] + r * cl[4 * i + 1] + r2 * cl[4 * i + 2]) * pow2<F>(maxT - T[i]);
    LURK_TRY(sumcheck_verify<F>(proof->inner_rounds, maxT, 2, rounds_fmt, fn, user, LURK_SPARTAN_INNER, 0, fmt, e, ry, ok));
    if (!ok) return LURK_OK;
    ScScratch<F> sc;
    LURK_TRY(sc.init(s));
    for (int i = 0; i < n; i++) LURK_TRY(C[i]->matrix_evals(rx.data() + (maxS - S[i]), ry.data() + (maxT - T[i]), sc, sc.result + 3 * i, s));
    LURK_CUDA_TRY(cudaStreamSynchronize(s));
    const F *abc = static_cast<const F *>(sc.pinned);
    want = F::zero();
    c = F::one();
    for (int i = 0; i < n; i++, c = c * r3) {
        const F *y = ry.data() + (maxT - T[i]);
        std::vector<F> tail(1 + X[i].size());
        tail[0] = u[i];
        std::copy(X[i].begin(), X[i].end(), tail.begin() + 1);
        const F eval_z = (F::one() - y[0]) * ew[i] + y[0] * tail_eval(std::move(tail), y + 1, T[i] - 1);
        want += c * (abc[3 * i] + r * abc[3 * i + 1] + r2 * abc[3 * i + 2]) * eval_z;
    }
    if (e != want) return LURK_OK;

    // batch_eval_reduce's verifier over [W_0 .. W_{n-1}, E_0 .. E_{n-1}] at [ry_i[1:] .., rx_i ..]
    const int nc = 2 * n;
    std::vector<int> nv(nc);
    std::vector<const F *> pts(nc);
    std::vector<F> ev(nc);
    std::vector<uint8_t> msg(32 * (size_t)nc);
    for (int i = 0; i < n; i++) {
        nv[i] = T[i] - 1;
        pts[i] = ry.data() + (maxT - T[i]) + 1;
        ev[i] = ew[i];
        nv[n + i] = S[i];
        pts[n + i] = rx.data() + (maxS - S[i]);
        ev[n + i] = cl[4 * i + 3];
    }
    for (int k = 0; k < nc; k++) fe_out(ev[k], fmt, msg.data() + 32 * k);
    F rho;
    LURK_TRY(ask(fn, user, LURK_SPARTAN_BATCH_EVAL, 0, msg.data(), msg.size(), fmt, rho));
    e = F::zero();
    c = F::one();
    for (int k = 0; k < nc; k++, c = c * rho) e += c * ev[k] * pow2<F>(m - nv[k]);
    LURK_TRY(sumcheck_verify<F>(proof->reduce_rounds, m, 2, rounds_fmt, fn, user, LURK_SPARTAN_BATCH_EVAL, 1, fmt, e, rr, ok));
    if (!ok) return LURK_OK;
    want = F::zero();
    c = F::one();
    for (int k = 0; k < nc; k++, c = c * rho) want += c * eq_at(pts[k], rr.data() + (m - nv[k]), nv[k]) * left[k];
    if (e != want) return LURK_OK;
    F gamma;
    LURK_TRY(ask(fn, user, LURK_SPARTAN_BATCH_EVAL, m + 1, proof->claims_left, 32 * (size_t)nc, fmt, gamma));
    std::vector<F> w(nc);
    F joint = F::zero();
    for (int k = 0; k < nc; k++) {
        w[k] = k ? w[k - 1] * gamma : F::one();
        F scale = w[k];
        for (int j = 0; j < m - nv[k]; j++) scale = scale * (F::one() - rr[j]);
        joint += scale * left[k];
    }
    *accepted = 1;
    for (int j = 0; proof->r_x && j < maxS; j++) fe_out(rx[j], fmt, proof->r_x + 32 * j);
    for (int j = 0; proof->r_y && j < maxT; j++) fe_out(ry[j], fmt, proof->r_y + 32 * j);
    for (int j = 0; proof->r && j < m; j++) fe_out(rr[j], fmt, proof->r + 32 * j);
    for (int k = 0; proof->weights && k < nc; k++) fe_out(w[k], fmt, proof->weights + 32 * k);
    if (proof->joint_eval) fe_out(joint, fmt, proof->joint_eval);
    return LURK_OK;
}

}  // namespace lurk

static int ceil_log2(uint64_t x) { int l = 0; while (((uint64_t)1 << l) < x) l++; return l; }

namespace lurk {

// the prover's calls need the merged transpose a verifier-only context does not build
int refuse_verifier_only(const lurk_spartan_ctx *ctx, const char *who) {
    if (!ctx->verifier_only) return LURK_OK;
    set_error("%s needs a full Spartan context; this one was made by lurk_spartan_ctx_create_verifier, which keeps no transpose", who);
    return LURK_ERR_ARG;
}

// what the recursive verifier (recursive.cu) reads of a shape: sizes, field and the three device CSRs
void spartan_ctx_shape(const lurk_spartan_ctx *ctx, int *field_id, uint64_t *n_w, uint64_t *n_x, uint64_t *rows, CsrDev csr[3]) {
    *field_id = ctx->field_id;
    *n_w = ctx->n_w;
    *n_x = ctx->n_x;
    *rows = ctx->rows;
    dispatch_field(ctx->field_id, [&](auto f) {
        const SpartanCtx<decltype(f)> *c = static_cast<const SpartanCtx<decltype(f)> *>(ctx);
        for (int m = 0; m < 3; m++) csr[m] = c->csr[m];
        return LURK_OK;
    });
}

}  // namespace lurk

static bool overlaps(const void *a, size_t a_bytes, const void *b, size_t b_bytes) {
    const uintptr_t a0 = reinterpret_cast<uintptr_t>(a), b0 = reinterpret_cast<uintptr_t>(b);
    return a0 < b0 + b_bytes && b0 < a0 + a_bytes;
}

// argument checks of both provers, before any device work
static int check_prove_args(int n, lurk_spartan_ctx *const *ctxs, const void *const *d_z, const void *const *d_E, lurk_spartan_challenge_fn fn,
                            lurk_spartan_proof *out, void *d_joint, int fmt) {
    if (n < 1 || n > SP_MAX_INSTANCES) { set_error("1..%d instances, got %d", SP_MAX_INSTANCES, n); return LURK_ERR_ARG; }
    if (!ctxs || !d_z || !d_E) { set_error("null instance array"); return LURK_ERR_ARG; }
    if (!fn) { set_error("null challenge callback"); return LURK_ERR_ARG; }
    if (!out) { set_error("null proof record"); return LURK_ERR_ARG; }
    if (!d_joint) { set_error("null d_joint"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    int m = 0;
    for (int i = 0; i < n; i++) {
        if (!ctxs[i]) { set_error("null context %d", i); return LURK_ERR_ARG; }
        LURK_TRY(refuse_verifier_only(ctxs[i], "the prover"));
        if (!d_z[i] || !d_E[i]) { set_error("null d_z / d_E of instance %d", i); return LURK_ERR_ARG; }
        if (ctxs[i]->field_id != ctxs[0]->field_id) {
            set_error("context %d is over field %d, context 0 over field %d", i, ctxs[i]->field_id, ctxs[0]->field_id);
            return LURK_ERR_ARG;
        }
        m = std::max(m, std::max(ctxs[i]->log_rows, ctxs[i]->log_vars));
    }
    const size_t joint_bytes = (size_t)32 << m;
    for (int i = 0; i < n; i++) {
        if (overlaps(d_joint, joint_bytes, d_z[i], 32 * ctxs[i]->z_len())) { set_error("d_joint overlaps d_z of instance %d", i); return LURK_ERR_ARG; }
        if (overlaps(d_joint, joint_bytes, d_E[i], 32 * ctxs[i]->rows)) { set_error("d_joint overlaps d_E of instance %d", i); return LURK_ERR_ARG; }
    }
    return LURK_OK;
}

// argument checks of both verifiers, before any device work (the contexts are only read for their sizes and field)
static int check_verify_args(int n, lurk_spartan_ctx *const *ctxs, const uint8_t *u, const uint8_t *const *X, const lurk_spartan_proof *proof,
                             int rounds_fmt, lurk_spartan_challenge_fn fn, const int *accepted, int fmt) {
    if (n < 1 || n > SP_MAX_INSTANCES) { set_error("1..%d instances, got %d", SP_MAX_INSTANCES, n); return LURK_ERR_ARG; }
    if (!ctxs || !X) { set_error("null instance array"); return LURK_ERR_ARG; }
    if (!u) { set_error("null u"); return LURK_ERR_ARG; }
    if (!fn) { set_error("null challenge callback"); return LURK_ERR_ARG; }
    if (!accepted) { set_error("null accepted"); return LURK_ERR_ARG; }
    if (!proof) { set_error("null proof record"); return LURK_ERR_ARG; }
    if (!proof->outer_rounds || !proof->claims || !proof->inner_rounds || !proof->eval_W || !proof->reduce_rounds || !proof->claims_left) {
        set_error("null proof field (outer_rounds, claims, inner_rounds, eval_W, reduce_rounds and claims_left are read)");
        return LURK_ERR_ARG;
    }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    if (rounds_fmt != LURK_SPARTAN_ROUNDS_EVALS && rounds_fmt != LURK_SPARTAN_ROUNDS_COMPRESSED) { set_error("unknown rounds_fmt %d", rounds_fmt); return LURK_ERR_ARG; }
    for (int i = 0; i < n; i++) {
        if (!ctxs[i]) { set_error("null context %d", i); return LURK_ERR_ARG; }
        for (int k = 0; k < i; k++)
            if (ctxs[k] == ctxs[i]) { set_error("instances %d and %d share a context", k, i); return LURK_ERR_ARG; }
    }
    for (int i = 0; i < n; i++) {
        if (ctxs[i]->field_id != ctxs[0]->field_id) {
            set_error("context %d is over field %d, context 0 over field %d", i, ctxs[i]->field_id, ctxs[0]->field_id);
            return LURK_ERR_ARG;
        }
        if (ctxs[i]->n_x && !X[i]) { set_error("null X of instance %d", i); return LURK_ERR_ARG; }
    }
    return LURK_OK;
}

namespace lurk {

// every check lurk_spartan_verify / _batch make before their first transcript call -- the arguments, then the values of u, X and the proof
// -- for compress_verify.cu, which makes them for both circuits before either circuit's transcript starts
int spartan_verify_precheck(int n, lurk_spartan_ctx *const *ctxs, const uint8_t *u, const uint8_t *const *X, const lurk_spartan_proof *proof,
                            int rounds_fmt, lurk_spartan_challenge_fn fn, const int *accepted, int fmt) {
    LURK_TRY(check_verify_args(n, ctxs, u, X, proof, rounds_fmt, fn, accepted, fmt));
    return dispatch_field(ctxs[0]->field_id, [&](auto f) {
        using F = decltype(f);
        std::vector<F> uv, cl, ew, left;
        std::vector<std::vector<F>> Xv;
        return verify_inputs<F>(n, ctxs, u, X, proof, rounds_fmt, fmt, uv, Xv, cl, ew, left);
    });
}

// the verifier behind lurk_spartan_verify / _batch for compress_verify.cu, after spartan_verify_precheck
int spartan_verify_checked(int n, lurk_spartan_ctx *const *ctxs, const uint8_t *u, const uint8_t *const *X, lurk_spartan_proof *proof, int rounds_fmt,
                           lurk_spartan_challenge_fn fn, void *user, int *accepted, int fmt, cudaStream_t s, bool batched) {
    return dispatch_field(ctxs[0]->field_id, [&](auto f) {
        return spartan_verify<decltype(f)>(n, ctxs, u, X, proof, rounds_fmt, fn, user, accepted, fmt, s, batched);
    });
}

}  // namespace lurk

static int spartan_ctx_create(int field_id, uint64_t n_w, uint64_t n_x, uint64_t n_rows, const uint64_t *const row_ptr[3], const uint32_t *const col[3],
                              const uint8_t *const val[3], int fmt, bool verifier_only, lurk_spartan_ctx **out) {
    if (!out) { set_error("null out"); return LURK_ERR_ARG; }
    *out = nullptr;
    if (!row_ptr || !col || !val) { set_error("null matrix arrays"); return LURK_ERR_ARG; }
    if (field_id < LURK_FIELD_BN254_FR || field_id > LURK_FIELD_PALLAS_FP) { set_error("unknown field id %d", field_id); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    if (n_rows < 1 || n_rows >= (1ull << SP_TAG_SHIFT)) { set_error("n_rows must be in 1..2^30 - 1, got %llu", (unsigned long long)n_rows); return LURK_ERR_ARG; }
    if (n_w + 1 + n_x >= (1ull << 31)) { set_error("instance too large"); return LURK_ERR_ARG; }
    const uint64_t nz = n_w + 1 + n_x;
    for (int m = 0; m < 3; m++) {
        if (!row_ptr[m]) { set_error("null row_ptr of matrix %d", m); return LURK_ERR_ARG; }
        if (row_ptr[m][0] != 0) { set_error("matrix %d: row_ptr[0] != 0", m); return LURK_ERR_ARG; }
        for (uint64_t i = 0; i < n_rows; i++)
            if (row_ptr[m][i + 1] < row_ptr[m][i]) { set_error("matrix %d: row_ptr decreases at row %llu", m, (unsigned long long)i); return LURK_ERR_ARG; }
        const uint64_t nnz = row_ptr[m][n_rows];
        if (nnz && (!col[m] || !val[m])) { set_error("null col / val of matrix %d", m); return LURK_ERR_ARG; }
        for (uint64_t k = 0; k < nnz; k++)
            if (col[m][k] >= nz) { set_error("matrix %d: column %u out of range", m, col[m][k]); return LURK_ERR_ARG; }
    }
    LURK_TRY(require_gpu());
    lurk_spartan_ctx *ctx = nullptr;
    const int rc = dispatch_field(field_id, [&](auto f) {
        using F = decltype(f);
        SpartanCtx<F> *c = new SpartanCtx<F>();
        c->field_id = field_id;
        c->n_w = n_w; c->n_x = n_x; c->rows = n_rows;
        c->log_rows = std::max(1, ceil_log2(n_rows));
        c->log_vars = std::max(1, ceil_log2(std::max(n_w, n_x + 1)));
        c->num_vars = (uint64_t)1 << c->log_vars;
        c->verifier_only = verifier_only;
        const int r = c->init(row_ptr, col, val, fmt);
        if (r != LURK_OK) { delete c; return r; }
        ctx = c;
        return LURK_OK;
    });
    if (rc != LURK_OK) return rc;
    *out = ctx;
    return LURK_OK;
}

extern "C" {

int lurk_spartan_ctx_create(int field_id, uint64_t n_w, uint64_t n_x, uint64_t n_rows, const uint64_t *const row_ptr[3], const uint32_t *const col[3],
                            const uint8_t *const val[3], int fmt, lurk_spartan_ctx **out) {
    return spartan_ctx_create(field_id, n_w, n_x, n_rows, row_ptr, col, val, fmt, false, out);
}

int lurk_spartan_ctx_create_verifier(int field_id, uint64_t n_w, uint64_t n_x, uint64_t n_rows, const uint64_t *const row_ptr[3],
                                     const uint32_t *const col[3], const uint8_t *const val[3], int fmt, lurk_spartan_ctx **out) {
    return spartan_ctx_create(field_id, n_w, n_x, n_rows, row_ptr, col, val, fmt, true, out);
}

void lurk_spartan_ctx_destroy(lurk_spartan_ctx *ctx) { delete ctx; }

int lurk_spartan_ctx_info(lurk_spartan_ctx *ctx, int *field_id, int *log_rows, int *log_vars, size_t *joint_len) {
    if (!ctx) { set_error("null context"); return LURK_ERR_ARG; }
    if (field_id) *field_id = ctx->field_id;
    if (log_rows) *log_rows = ctx->log_rows;
    if (log_vars) *log_vars = ctx->log_vars;
    if (joint_len) *joint_len = (size_t)1 << std::max(ctx->log_rows, ctx->log_vars);
    return LURK_OK;
}

int lurk_spartan_prove_batch_dev(int n, lurk_spartan_ctx *const *ctxs, const void *const *d_z, const void *const *d_E, lurk_spartan_challenge_fn challenge,
                                 void *user, lurk_spartan_proof *out, void *d_joint, int fmt, void *stream) {
    LURK_TRY(check_prove_args(n, ctxs, d_z, d_E, challenge, out, d_joint, fmt));
    LURK_TRY(require_gpu());
    return dispatch_field(ctxs[0]->field_id, [&](auto f) {
        return spartan_prove<decltype(f)>(n, ctxs, d_z, d_E, challenge, user, out, d_joint, fmt, static_cast<cudaStream_t>(stream), true);
    });
}

int lurk_spartan_prove_dev(lurk_spartan_ctx *ctx, const void *d_z, const void *d_E, lurk_spartan_challenge_fn challenge, void *user,
                           lurk_spartan_proof *out, void *d_joint, int fmt, void *stream) {
    if (!ctx) { set_error("null context"); return LURK_ERR_ARG; }
    if (!d_z || !d_E) { set_error("null d_z / d_E"); return LURK_ERR_ARG; }
    LURK_TRY(check_prove_args(1, &ctx, &d_z, &d_E, challenge, out, d_joint, fmt));
    LURK_TRY(require_gpu());
    return dispatch_field(ctx->field_id, [&](auto f) {
        return spartan_prove<decltype(f)>(1, &ctx, &d_z, &d_E, challenge, user, out, d_joint, fmt, static_cast<cudaStream_t>(stream), false);
    });
}

int lurk_spartan_eval_table_dev(lurk_spartan_ctx *ctx, const void *d_eq_rx, const uint8_t r[32], void *d_out, int fmt, void *stream) {
    if (!ctx || !d_eq_rx || !r || !d_out) { set_error("null argument"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    LURK_TRY(refuse_verifier_only(ctx, "lurk_spartan_eval_table_dev"));
    LURK_TRY(require_gpu());
    return dispatch_field(ctx->field_id, [&](auto f) {
        using F = decltype(f);
        F rv;
        if (!fe_in(r, fmt, rv)) { set_error("r is not reduced"); return LURK_ERR_RANGE; }
        return static_cast<SpartanCtx<F> *>(ctx)->eval_table(static_cast<const F *>(d_eq_rx), rv, static_cast<F *>(d_out), static_cast<cudaStream_t>(stream));
    });
}

int lurk_spartan_matrix_evals_dev(lurk_spartan_ctx *ctx, const uint8_t *r_x, const uint8_t *r_y, uint8_t out[96], int fmt, void *stream) {
    if (!ctx || !r_x || !r_y || !out) { set_error("null argument"); return LURK_ERR_ARG; }
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    LURK_TRY(require_gpu());
    return dispatch_field(ctx->field_id, [&](auto f) {
        using F = decltype(f);
        SpartanCtx<F> *c = static_cast<SpartanCtx<F> *>(ctx);
        std::vector<F> x(c->log_rows), y(c->log_vars + 1);
        for (int j = 0; j < c->log_rows; j++)
            if (!fe_in(r_x + 32 * j, fmt, x[j])) { set_error("r_x[%d] is not reduced", j); return LURK_ERR_RANGE; }
        for (int j = 0; j <= c->log_vars; j++)
            if (!fe_in(r_y + 32 * j, fmt, y[j])) { set_error("r_y[%d] is not reduced", j); return LURK_ERR_RANGE; }
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        ScScratch<F> sc;
        LURK_TRY(sc.init(s));
        LURK_TRY(c->matrix_evals(x.data(), y.data(), sc, sc.result, s));
        F res[3];
        LURK_TRY(sc.fetch(3, res, s));
        for (int k = 0; k < 3; k++) fe_out(res[k], fmt, out + 32 * k);
        return LURK_OK;
    });
}

int lurk_spartan_verify(lurk_spartan_ctx *ctx, const uint8_t u[32], const uint8_t *X, lurk_spartan_proof *proof, int rounds_fmt,
                        lurk_spartan_challenge_fn challenge, void *user, int *accepted, int fmt, void *stream) {
    if (!ctx) { set_error("null context"); return LURK_ERR_ARG; }
    const uint8_t *const xs[1] = {X};
    LURK_TRY(check_verify_args(1, &ctx, u, xs, proof, rounds_fmt, challenge, accepted, fmt));
    LURK_TRY(require_gpu());
    return dispatch_field(ctx->field_id, [&](auto f) {
        return spartan_verify<decltype(f)>(1, &ctx, u, xs, proof, rounds_fmt, challenge, user, accepted, fmt, static_cast<cudaStream_t>(stream), false);
    });
}

int lurk_spartan_verify_batch(int n, lurk_spartan_ctx *const *ctxs, const uint8_t *u, const uint8_t *const *X, lurk_spartan_proof *proof,
                              int rounds_fmt, lurk_spartan_challenge_fn challenge, void *user, int *accepted, int fmt, void *stream) {
    LURK_TRY(check_verify_args(n, ctxs, u, X, proof, rounds_fmt, challenge, accepted, fmt));
    LURK_TRY(require_gpu());
    return dispatch_field(ctxs[0]->field_id, [&](auto f) {
        return spartan_verify<decltype(f)>(n, ctxs, u, X, proof, rounds_fmt, challenge, user, accepted, fmt, static_cast<cudaStream_t>(stream), true);
    });
}

}  // extern "C"
