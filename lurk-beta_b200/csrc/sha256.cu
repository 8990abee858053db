// Witness of the SHA-256 coprocessor's circuit (synthesize_sha256, reference src/coprocessor/sha256.rs:27-64) on the GPU.
//
// Which aux bellpepper's gadget allocates, and from which bit, depends only on (field, n): the host replays the gadget's
// constant propagation once per (field, n) and records, for every aux bit, the native SHA-256 word and bit it holds
// (negated where bellpepper stores the underlying bit of a Not).  The kernel evaluates SHA-256 natively into shared
// memory, one CTA per call (or per slice of a call when there are few calls), and streams the block from that table
// with coalesced 32-byte stores: it is bound by HBM writes (32 B per aux).  The restatement of the gadget's rules that
// this replays is tests/sha256_gadget_oracle.py.
#include "sha256.cuh"

#include <map>
#include <memory>

namespace lurk {

namespace {

// ---------------------------------------------------------------------------------------------- native word layout
// Per call in shared memory: per input element j, 8 words of its canonical value and 4 words of the AND-chain aux of its
// to_bits_le_strict; then per compression the words below; then the 8 words of the packed digest.
constexpr int IN_WORDS = 12;
constexpr int OFF_W = 0, OFF_WH = 64, OFF_SCHED = 128, OFF_ROUND = 384, ROUND_WORDS = 11, OFF_FINAL = 384 + 64 * ROUND_WORDS;
constexpr int WPC = OFF_FINAL + 16;   // words per compression
enum { R_E_LO, R_E_HI, R_S1A, R_S1, R_CH, R_A_LO, R_A_HI, R_S0A, R_S0, R_MAJ, R_BC };
constexpr int MAX_CHAIN = 128;        // AND-chain aux of one to_bits_le_strict (99 on BN254, 42 on Pasta)

__host__ __device__ inline int n_compressions(int n) { return n + 1; }   // 512n message bits + a padding block
__host__ __device__ inline int words_per_call(int n) { return 2 * n * IN_WORDS + n_compressions(n) * WPC + 8; }

#define SHA256_K { \
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01, 0x243185be, \
    0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, \
    0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967, 0x27b70a85, \
    0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85, 0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, \
    0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, \
    0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2}
__constant__ uint32_t K_DEV[64] = SHA256_K;
const uint32_t K_HOST[64] = SHA256_K;
#define SHA256_IV {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19}
__constant__ uint32_t IV_DEV[8] = SHA256_IV;
const uint32_t IV[8] = SHA256_IV;

template <class P>
__host__ __device__ inline uint32_t pm1_bit(int i) {   // bit i of p - 1 (p is odd: no borrow)
    uint32_t w = P::MOD(i >> 5);
    if ((i >> 5) == 0) w -= 1;
    return (w >> (i & 31)) & 1;
}
template <class P>
__host__ __device__ inline int num_bits() {
    for (int i = 255; i >= 0; i--)
        if ((P::MOD(i >> 5) >> (i & 31)) & 1) return i + 1;
    return 0;
}

// ---------------------------------------------------------------------------------------------- host: the schedule
// Symbolic replay of the gadget: only whether each Boolean is Constant(false/true), Is or Not matters; every allocated
// aux is recorded as (word << 6 | bit << 1 | negate).
enum : uint8_t { B0 = 0, B1 = 1, IS = 2, NOT = 3 };
struct U32 { uint8_t b[32]; };

struct Builder {
    std::vector<uint32_t> out;
    void push(int word, int bit, int neg) { out.push_back((uint32_t)word << 6 | (uint32_t)bit << 1 | (uint32_t)neg); }
    static uint8_t bnot(uint8_t x) { return x ^ 1; }   // B0 <-> B1, IS <-> NOT
    static bool konst(uint8_t x) { return x <= B1; }
    static U32 constant(uint32_t v) { U32 u; for (int i = 0; i < 32; i++) u.b[i] = (v >> i) & 1; return u; }
    static U32 rotr(const U32 &u, int by) { U32 r; for (int i = 0; i < 32; i++) r.b[i] = u.b[(i + by) % 32]; return r; }
    static U32 shr(const U32 &u, int by) { U32 r; for (int i = 0; i < 32; i++) r.b[i] = i + by < 32 ? u.b[i + by] : B0; return r; }

    U32 xor32(const U32 &a, const U32 &c, int word) {
        U32 r;
        for (int i = 0; i < 32; i++) {
            uint8_t x = a.b[i], y = c.b[i];
            if (x == B0) r.b[i] = y;
            else if (y == B0) r.b[i] = x;
            else if (x == B1) r.b[i] = bnot(y);
            else if (y == B1) r.b[i] = bnot(x);
            else {
                const int neg = (x == NOT) != (y == NOT);   // AllocatedBit::xor of the underlying bits
                push(word, i, neg);
                r.b[i] = neg ? NOT : IS;
            }
        }
        return r;
    }
    // Boolean::and; `neg` says how the allocated bit relates to the word bit it is recorded from
    uint8_t band(uint8_t x, uint8_t y, int word, int bit, int neg) {
        if (x == B0 || y == B0) return B0;
        if (x == B1) return y;
        if (y == B1) return x;
        push(word, bit, neg);
        return IS;
    }
    // sha256_ch: every allocation holds ch (or, under the negated reductions, its complement)
    uint8_t ch(uint8_t a, uint8_t b, uint8_t c, int word, int i) {
        if (konst(a) && konst(b) && konst(c)) return (a & b) ^ ((a ^ 1) & c);
        if (a == B0) return c;
        if (b == B0) return band(bnot(a), c, word, i, 0);
        if (c == B0) return band(a, b, word, i, 0);
        if (c == B1) return bnot(band(a, bnot(b), word, i, 1));
        if (b == B1) return bnot(band(bnot(a), bnot(c), word, i, 1));
        push(word, i, 0);
        return IS;
    }
    uint8_t maj(uint8_t a, uint8_t b, uint8_t c, int word, int bc_word, int i) {
        if (konst(a) && konst(b) && konst(c)) return (a & b) ^ (a & c) ^ (b & c);
        if (a == B0) return band(b, c, word, i, 0);
        if (b == B0) return band(a, c, word, i, 0);
        if (c == B0) return band(a, b, word, i, 0);
        if (c == B1) return bnot(band(bnot(a), bnot(b), word, i, 1));
        if (b == B1) return bnot(band(bnot(a), bnot(c), word, i, 1));
        if (a == B1) return bnot(band(bnot(b), bnot(c), word, i, 1));
        band(b, c, bc_word, i, 0);
        push(word, i, 0);
        return IS;
    }
    U32 addmany(const std::vector<U32> &ops, int lo, int hi) {
        bool all_const = true;
        uint64_t sum = 0;
        for (const U32 &u : ops)
            for (int i = 0; i < 32; i++) {
                all_const &= konst(u.b[i]);
                if (konst(u.b[i])) sum += (uint64_t)u.b[i] << i;
            }
        if (all_const) return constant((uint32_t)sum);
        uint64_t max_value = (uint64_t)ops.size() * 0xFFFFFFFFull;
        for (int i = 0; max_value; i++, max_value >>= 1) push(i < 32 ? lo : hi, i & 31, 0);
        U32 r;
        for (int i = 0; i < 32; i++) r.b[i] = IS;
        return r;
    }

    // sha256_compression_function; `base` = first word of this compression
    void compression(const uint8_t *block_bits, U32 cur[8], int base) {
        U32 w[64];
        for (int i = 0; i < 16; i++)
            for (int k = 0; k < 32; k++) w[i].b[k] = block_bits[32 * i + 31 - k];   // UInt32::from_bits_be
        for (int i = 16; i < 64; i++) {
            const int s = base + OFF_SCHED + 4 * i;
            U32 s0 = xor32(xor32(rotr(w[i - 15], 7), rotr(w[i - 15], 18), s), shr(w[i - 15], 3), s + 1);
            U32 s1 = xor32(xor32(rotr(w[i - 2], 17), rotr(w[i - 2], 19), s + 2), shr(w[i - 2], 10), s + 3);
            w[i] = addmany({w[i - 16], s0, w[i - 7], s1}, base + OFF_W + i, base + OFF_WH + i);
        }
        // Maybe::Concrete when `ea` / `aa` is empty
        std::vector<U32> ea, aa;
        U32 a = cur[0], b = cur[1], c = cur[2], d = cur[3], e = cur[4], f = cur[5], g = cur[6], h = cur[7];
        for (int r = 0; r < 64; r++) {
            const int R = base + OFF_ROUND + ROUND_WORDS * r;
            U32 new_e = ea.empty() ? e : addmany(ea, R + R_E_LO, R + R_E_HI);
            U32 s1 = xor32(xor32(rotr(new_e, 6), rotr(new_e, 11), R + R_S1A), rotr(new_e, 25), R + R_S1);
            U32 chw;
            for (int i = 0; i < 32; i++) chw.b[i] = ch(new_e.b[i], f.b[i], g.b[i], R + R_CH, i);
            std::vector<U32> temp1 = {h, s1, chw, constant(K_HOST[r]), w[r]};
            U32 new_a = aa.empty() ? a : addmany(aa, R + R_A_LO, R + R_A_HI);
            U32 s0 = xor32(xor32(rotr(new_a, 2), rotr(new_a, 13), R + R_S0A), rotr(new_a, 22), R + R_S0);
            U32 mj;
            for (int i = 0; i < 32; i++) mj.b[i] = maj(new_a.b[i], b.b[i], c.b[i], R + R_MAJ, R + R_BC, i);
            h = g; g = f; f = new_e;
            ea = temp1; ea.push_back(d);
            d = c; c = b; b = new_a;
            aa = temp1; aa.push_back(s0); aa.push_back(mj);
        }
        const int F0 = base + OFF_FINAL;
        U32 out[8];
        std::vector<U32> l0 = aa; l0.push_back(cur[0]);
        std::vector<U32> l4 = ea; l4.push_back(cur[4]);
        out[0] = addmany(l0, F0 + 0, F0 + 1);
        out[1] = addmany({cur[1], b}, F0 + 2, F0 + 3);
        out[2] = addmany({cur[2], c}, F0 + 4, F0 + 5);
        out[3] = addmany({cur[3], d}, F0 + 6, F0 + 7);
        out[4] = addmany(l4, F0 + 8, F0 + 9);
        out[5] = addmany({cur[5], f}, F0 + 10, F0 + 11);
        out[6] = addmany({cur[6], g}, F0 + 12, F0 + 13);
        out[7] = addmany({cur[7], h}, F0 + 14, F0 + 15);
        for (int i = 0; i < 8; i++) cur[i] = out[i];
    }
};

template <class P>
std::vector<uint32_t> build_schedule(int n) {
    Builder B;
    const int nb = num_bits<P>();
    // to_bits_le_strict of every element: its run bits / conditional bits are input bits, its AND results the chain words
    for (int j = 0; j < 2 * n; j++) {
        const int in = j * IN_WORDS;
        int q = 0, run = 0;
        bool found = false, have_last = false;
        for (int i = 255; i >= 0; i--) {
            const uint32_t bb = pm1_bit<P>(i);
            found |= bb != 0;
            if (!found) continue;
            if (bb) { B.push(in + (i >> 5), i & 31, 0); run++; continue; }
            if (run) {
                for (int k = 0; k < run - 1 + (have_last ? 1 : 0); k++, q++) B.push(in + 8 + (q >> 5), q & 31, 0);
                have_last = true;
                run = 0;
            }
            B.push(in + (i >> 5), i & 31, 0);
        }
        if (q > MAX_CHAIN) return {};
    }
    // the gadget's bits: per element its num_bits bits (Is) padded to 256 with Constant(false); the vector reversed; then
    // sha256's padding (1, zeros, 64-bit length)
    const size_t len = (size_t)512 * n, total = (size_t)512 * n_compressions(n);
    std::vector<uint8_t> bits(total, B0);
    for (int j = 0; j < 2 * n; j++)
        for (int i = 0; i < nb; i++) bits[len - 1 - (256 * j + i)] = IS;
    bits[len] = B1;
    for (int i = 0; i < 64; i++) bits[total - 1 - i] = ((uint64_t)len >> i) & 1;
    U32 cur[8];
    for (int i = 0; i < 8; i++) cur[i] = Builder::constant(IV[i]);
    for (int c = 0; c < n_compressions(n); c++) B.compression(bits.data() + 512 * c, cur, 2 * n * IN_WORDS + c * WPC);
    return std::move(B.out);
}

// ---------------------------------------------------------------------------------------------- device
__device__ __forceinline__ uint32_t rotr32(uint32_t x, int by) { return __funnelshift_r(x, x, by); }

template <class F>
__global__ void __launch_bounds__(256) sha256_witness_kernel(const F *__restrict__ in, size_t count, int n, const uint32_t *__restrict__ sched,
                                                             int nsched, int slices, F *__restrict__ out, const uint64_t *__restrict__ offs,
                                                             int in_fmt, int out_fmt) {
    using P = typename F::Params;
    extern __shared__ uint32_t sw[];
    const size_t blk = (size_t)nsched + 2;
    const size_t per_slice = (blk + slices - 1) / slices;
    const int base0 = 2 * n * IN_WORDS, ncomp = n_compressions(n), dig = base0 + ncomp * WPC;
    const F one = out_fmt == LURK_FMT_MONTGOMERY ? F::one() : F::from_u64(1).to_canonical();
    const F zero = F::zero();
    for (size_t item = blockIdx.x; item < count * (size_t)slices; item += gridDim.x) {
        const size_t call = item / slices;
        const size_t lo = (item % slices) * per_slice, hi = lo + per_slice < blk ? lo + per_slice : blk;
        __syncthreads();   // the previous item's stream has read the words
        // input elements in canonical form, and the AND chains of their to_bits_le_strict
        for (int j = threadIdx.x; j < 2 * n; j += blockDim.x) {
            F x = load_fe<F>(in + call * 2 * n + j);
            if (in_fmt == LURK_FMT_MONTGOMERY) x = x.to_canonical();
            uint32_t *wj = sw + j * IN_WORDS;
            for (int k = 0; k < 8; k++) wj[k] = x.v[k];
            uint32_t chain[4] = {0, 0, 0, 0};
            int q = 0, run = 0;
            bool found = false, have_last = false;
            uint32_t last = 0;
            for (int i = 255; i >= 0; i--) {
                const uint32_t bb = pm1_bit<P>(i);
                found |= bb != 0;
                if (!found) continue;
                if (bb) { run++; continue; }
                if (run) {
                    uint32_t cur = (x.v[(i + run) >> 5] >> ((i + run) & 31)) & 1;   // top bit of the run first
                    for (int k = 1; k < run; k++, q++) {
                        const int pos = i + run - k;
                        cur &= (x.v[pos >> 5] >> (pos & 31)) & 1;
                        chain[q >> 5] |= cur << (q & 31);
                    }
                    if (have_last) { cur &= last; chain[q >> 5] |= cur << (q & 31); q++; }
                    last = cur;
                    have_last = true;
                    run = 0;
                }
            }
            for (int k = 0; k < 4; k++) wj[8 + k] = chain[k];
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            // message = the input elements' little-endian bytes, reversed as a whole, then SHA-256's padding
            const int mlen = 64 * n;
            auto msg_byte = [&](int t) -> uint32_t {
                const int s = mlen - 1 - t;                               // byte s of the little-endian concatenation
                return (sw[(s >> 5) * IN_WORDS + ((s & 31) >> 2)] >> (8 * (s & 3))) & 0xff;
            };
            uint32_t cur[8];
            for (int i = 0; i < 8; i++) cur[i] = IV_DEV[i];
            for (int c = 0; c < ncomp; c++) {
                uint32_t *B = sw + base0 + c * WPC;
                for (int i = 0; i < 16; i++) {
                    if (c < n) {
                        const int t = 64 * c + 4 * i;
                        B[OFF_W + i] = msg_byte(t) << 24 | msg_byte(t + 1) << 16 | msg_byte(t + 2) << 8 | msg_byte(t + 3);
                    } else {
                        const uint64_t len = (uint64_t)512 * n;
                        B[OFF_W + i] = i == 0 ? 0x80000000u : (i == 14 ? (uint32_t)(len >> 32) : (i == 15 ? (uint32_t)len : 0u));
                    }
                }
                for (int i = 16; i < 64; i++) {
                    const uint32_t *w = B + OFF_W, x = w[i - 15], y = w[i - 2];
                    const uint32_t s0a = rotr32(x, 7) ^ rotr32(x, 18), s0 = s0a ^ (x >> 3);
                    const uint32_t s1a = rotr32(y, 17) ^ rotr32(y, 19), s1 = s1a ^ (y >> 10);
                    const uint64_t sum = (uint64_t)w[i - 16] + s0 + w[i - 7] + s1;
                    B[OFF_W + i] = (uint32_t)sum;
                    B[OFF_WH + i] = (uint32_t)(sum >> 32);
                    uint32_t *S = B + OFF_SCHED + 4 * i;
                    S[0] = s0a; S[1] = s0; S[2] = s1a; S[3] = s1;
                }
                uint32_t b = cur[1], cc = cur[2], d = cur[3], f = cur[5], g = cur[6], h = cur[7];
                uint64_t esum = cur[4], asum = cur[0];   // the deferred sums (round 0: the concrete state words)
                for (int r = 0; r < 64; r++) {
                    uint32_t *R = B + OFF_ROUND + ROUND_WORDS * r;
                    const uint32_t e = (uint32_t)esum;
                    R[R_E_LO] = e; R[R_E_HI] = (uint32_t)(esum >> 32);
                    const uint32_t S1a = rotr32(e, 6) ^ rotr32(e, 11), S1 = S1a ^ rotr32(e, 25);
                    const uint32_t ch = (e & f) ^ (~e & g);
                    const uint64_t temp1 = (uint64_t)h + S1 + ch + K_DEV[r] + B[OFF_W + r];
                    const uint32_t a = (uint32_t)asum;
                    R[R_A_LO] = a; R[R_A_HI] = (uint32_t)(asum >> 32);
                    const uint32_t S0a = rotr32(a, 2) ^ rotr32(a, 13), S0 = S0a ^ rotr32(a, 22);
                    const uint32_t mj = (a & b) ^ (a & cc) ^ (b & cc);
                    R[R_S1A] = S1a; R[R_S1] = S1; R[R_CH] = ch; R[R_S0A] = S0a; R[R_S0] = S0; R[R_MAJ] = mj; R[R_BC] = b & cc;
                    h = g; g = f; f = e;
                    esum = temp1 + d;
                    d = cc; cc = b; b = a;
                    asum = temp1 + S0 + mj;
                }
                const uint64_t sums[8] = {asum + cur[0], (uint64_t)cur[1] + b, (uint64_t)cur[2] + cc, (uint64_t)cur[3] + d,
                                          esum + cur[4], (uint64_t)cur[5] + f, (uint64_t)cur[6] + g, (uint64_t)cur[7] + h};
                for (int i = 0; i < 8; i++) {
                    B[OFF_FINAL + 2 * i] = cur[i] = (uint32_t)sums[i];
                    B[OFF_FINAL + 2 * i + 1] = (uint32_t)(sums[i] >> 32);
                }
            }
            // pack_bits: the digest as a big-endian integer, low CAPACITY = num_bits - 1 bits
            for (int q = 0; q < 8; q++) sw[dig + q] = cur[7 - q];
            const int cap = num_bits<P>() - 1;
            sw[dig + 7] &= (1u << (cap - 224)) - 1;
        }
        __syncthreads();
        F *o = out + (offs ? offs[call] : call * blk);
        for (size_t k = lo + threadIdx.x; k < hi; k += blockDim.x) {
            F v;
            if (k < (size_t)nsched) {
                const uint32_t e = __ldg(sched + k);
                v = ((sw[e >> 6] >> ((e >> 1) & 31)) ^ e) & 1 ? one : zero;
            } else if (k == (size_t)nsched) {
                for (int q = 0; q < 8; q++) v.v[q] = sw[dig + q];
                if (out_fmt == LURK_FMT_MONTGOMERY) v = F::from_canonical(v);
            } else {
                v = F::from_u64(4);                   // allocate_constant(ExprTag::Num)
                if (out_fmt != LURK_FMT_MONTGOMERY) v = v.to_canonical();
            }
            store_fe(o + k, v);
        }
    }
}

// ---------------------------------------------------------------------------------------------- schedule cache
struct Schedule {
    std::vector<uint32_t> host;
    std::map<int, uint32_t *> dev;   // per device
};

template <class F>
Schedule *schedule(int n) {
    static std::mutex mu;
    static std::map<int, std::unique_ptr<Schedule>> cache;
    if (n < 1 || n > LURK_SHA256_MAX_N) return nullptr;
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(n);
    if (it == cache.end()) {
        auto s = std::make_unique<Schedule>();
        s->host = build_schedule<typename F::Params>(n);
        it = cache.emplace(n, std::move(s)).first;
    }
    return it->second->host.empty() ? nullptr : it->second.get();
}

template <class F>
int device_schedule(Schedule *s, const uint32_t **out) {
    static std::mutex mu;
    std::lock_guard<std::mutex> g(mu);
    int dev = 0;
    LURK_CUDA_TRY(cudaGetDevice(&dev));
    auto it = s->dev.find(dev);
    if (it == s->dev.end()) {
        uint32_t *d = nullptr;
        LURK_CUDA_TRY(cudaMalloc(&d, s->host.size() * sizeof(uint32_t)));
        LURK_CUDA_TRY(cudaMemcpy(d, s->host.data(), s->host.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
        it = s->dev.emplace(dev, d).first;
    }
    *out = it->second;
    return LURK_OK;
}

}  // namespace

template <class F>
size_t sha256_block_len(int n) {
    Schedule *s = schedule<F>(n);
    return s ? s->host.size() + 2 : 0;
}

constexpr int SHA_THREADS = 256, SHA_CTAS_PER_SM = 8, SHA_SLICE_MIN = 4096;

template <class F>
int launch_sha256_witness(const void *d_in, size_t count, int n, void *d_out, const uint64_t *d_offs, int in_fmt, int out_fmt,
                          cudaStream_t st) {
    Schedule *s = schedule<F>(n);
    if (!s) { set_error("SHA-256 coprocessor arity %d: 1..%d", n, LURK_SHA256_MAX_N); return LURK_ERR_ARG; }
    if (!count) return LURK_OK;
    const uint32_t *d_sched = nullptr;
    LURK_TRY(device_schedule<F>(s, &d_sched));
    const size_t smem = (size_t)words_per_call(n) * sizeof(uint32_t);
    // opt in, once per device, to the shared memory of the largest n: the attribute is a per-kernel ceiling, so setting
    // it for the first n launched would refuse every larger n later in the process
    static std::mutex mu;
    static std::vector<int> opted;
    if (smem > 48 * 1024) {
        int dev = 0;
        LURK_CUDA_TRY(cudaGetDevice(&dev));
        std::lock_guard<std::mutex> g(mu);
        bool done = false;
        for (int d : opted) done |= d == dev;
        if (!done) {
            const int most = words_per_call(LURK_SHA256_MAX_N) * (int)sizeof(uint32_t);
            LURK_CUDA_TRY(cudaFuncSetAttribute(sha256_witness_kernel<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, most));
            opted.push_back(dev);
        }
    }
    // few calls: split each call's block into slices so that every SM has work; each slice recomputes the call's hash
    const size_t blk = s->host.size() + 2, cap = (size_t)sm_count() * SHA_CTAS_PER_SM;
    size_t slices = (cap + count - 1) / count, most = (blk + SHA_SLICE_MIN - 1) / SHA_SLICE_MIN;
    if (slices > most) slices = most;
    if (slices < 1) slices = 1;
    const size_t items = count * slices, grid = items < cap ? items : cap;
    sha256_witness_kernel<F><<<(unsigned)grid, SHA_THREADS, smem, st>>>((const F *)d_in, count, n, d_sched, (int)s->host.size(), (int)slices,
                                                                        (F *)d_out, d_offs, in_fmt, out_fmt);
    LURK_CUDA_TRY(cudaGetLastError());
    return LURK_OK;
}

#define LURK_SHA256_INSTANTIATE(F)                   \
    template size_t sha256_block_len<F>(int);        \
    template int launch_sha256_witness<F>(const void *, size_t, int, void *, const uint64_t *, int, int, cudaStream_t);
LURK_SHA256_INSTANTIATE(Fe<Bn254Fr>)
LURK_SHA256_INSTANTIATE(Fe<Bn254Fq>)
LURK_SHA256_INSTANTIATE(Fe<PallasFq>)
LURK_SHA256_INSTANTIATE(Fe<PallasFp>)

}  // namespace lurk

using namespace lurk;

extern "C" {

size_t lurk_sha256_witness_block(int field_id, int n) {
    size_t out = 0;
    dispatch_field(field_id, [&](auto f) {
        out = sha256_block_len<decltype(f)>(n);
        return LURK_OK;
    });
    return out;
}

static int sha256_args(int field_id, int n, int fmt, size_t count, const void *a, const void *b) {
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    if (!lurk_sha256_witness_block(field_id, n)) { set_error("unsupported field %d / SHA-256 arity %d", field_id, n); return LURK_ERR_ARG; }
    if (count && (!a || !b)) { set_error("null buffer"); return LURK_ERR_ARG; }
    return LURK_OK;
}

int lurk_sha256_witness_scatter_dev(int field_id, int n, const void *d_inputs, size_t count, const uint64_t *d_offsets, void *d_W, int fmt,
                                    void *stream) {
    LURK_TRY(sha256_args(field_id, n, fmt, count, d_inputs, d_W));
    if (count && !d_offsets) { set_error("null offsets"); return LURK_ERR_ARG; }
    LURK_TRY(require_gpu());
    return dispatch_field(field_id, [&](auto f) {
        return launch_sha256_witness<decltype(f)>(d_inputs, count, n, d_W, d_offsets, fmt, fmt, (cudaStream_t)stream);
    });
}

int lurk_sha256_witness_batch_dev(int field_id, int n, const void *d_inputs, size_t count, void *d_aux, int fmt, void *stream) {
    LURK_TRY(sha256_args(field_id, n, fmt, count, d_inputs, d_aux));
    LURK_TRY(require_gpu());
    return dispatch_field(field_id, [&](auto f) {
        return launch_sha256_witness<decltype(f)>(d_inputs, count, n, d_aux, nullptr, fmt, fmt, (cudaStream_t)stream);
    });
}

int lurk_sha256_witness_batch(int field_id, int n, const uint8_t *inputs, size_t count, uint8_t *aux_out, int fmt) {
    LURK_TRY(sha256_args(field_id, n, fmt, count, inputs, aux_out));
    LURK_TRY(require_gpu());
    if (!count) return LURK_OK;
    const size_t blk = lurk_sha256_witness_block(field_id, n), in_per = (size_t)2 * n * 32, out_per = blk * 32;
    // calls per chunk: bounded device staging for any count
    size_t chunk = ((size_t)256 << 20) / out_per;
    if (chunk < 1) chunk = 1;
    if (chunk > count) chunk = count;
    return dispatch_field(field_id, [&](auto f) {
        using F = decltype(f);
        DevBuf din, dout;
        LURK_TRY(din.alloc(count * in_per));
        LURK_TRY(dout.alloc(chunk * out_per));
        LURK_CUDA_TRY(cudaMemcpy(din.p, inputs, din.bytes, cudaMemcpyHostToDevice));
        int bad = 0;
        LURK_TRY(check_reduced_dev<F>(din.p, count * 2 * n, 0, &bad));
        if (bad) { set_error("%d input element(s) are not reduced below the field modulus", bad); return LURK_ERR_RANGE; }
        for (size_t first = 0; first < count; first += chunk) {
            const size_t m = count - first < chunk ? count - first : chunk;
            LURK_TRY(launch_sha256_witness<F>((const uint8_t *)din.p + first * in_per, m, n, dout.p, nullptr, fmt, fmt, 0));
            LURK_CUDA_TRY(cudaMemcpy(aux_out + first * out_per, dout.p, m * out_per, cudaMemcpyDeviceToHost));
        }
        return LURK_OK;
    });
}

}  // extern "C"
