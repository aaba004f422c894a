// b2k_pfk.cu -- higher-order partial derivatives of forward kinematics, reference ETS.partial_fkine0 (Haviland & Corke,
// "Manipulator Differential Kinematics Part II"): D_k (N, n^(k-1), 6, n) from jacob0 J (N, 6, n), k = 3..5.
//
// D_k[a_1, ..., a_{k-1}, :, j] = d^(k-1) J[:, j] / dq_{a_1} ... dq_{a_{k-1}}.  With J's column j = (v_j, w_j) in chain
// order, d_i v_j = w_lo x v_hi (lo = min(i, j), hi = max(i, j)) and d_i w_j = [i < j] w_i x w_j hold as identities in q;
// for a sorted index tuple S = (i, rest) the product rule gives
//     d^S zeta_j = sum over the 2^|rest| splits of rest into (A, B) of  d^A w_lo x d^B (v or w)_hi
// (rotational rows: zero unless i < j).  The value only depends on the multiset S, so it is computed once per sorted
// tuple and stored at every permutation of it.
//
// A block owns a group of R rows at a time (R > 1 only where a row is small).  Per group it builds, in shared memory,
// the table of d^S zeta for every sorted S of size 0..k-2 (size 0 is J itself), one size after the other, then a thread
// per (row, sorted tuple of size k-1, element of the 6 x n block) forms its value with one product-rule step from the
// table and writes it to each distinct permutation of the tuple.  The 6 x n block of a permutation is contiguous in the
// output, so consecutive threads store to consecutive addresses.  The sorted tuples of every size are listed once per
// block (a persistent grid), packed 4 bits per index.
#include "b2k_common.cuh"

namespace {

constexpr int PFK_THREADS = 256;

__host__ __device__ constexpr int cbinom(int x, int p)
{
    long long r = 1;
    for (int i = 0; i < p; i++) r = r * (x - i) / (i + 1);
    return x < p ? 0 : (int)r;
}

template <typename real, int N, int K> struct Pfk {
    static constexpr int M = K - 1; // length of the derivative index tuple of D_k
    static constexpr int E = 6 * N;
    // sorted tuples of size l: C(N + l - 1, l); those of sizes < l come first, so size l starts at C(N + l - 1, l - 1)
    __host__ __device__ static constexpr int count(int l) { return cbinom(N + l - 1, l); }
    __host__ __device__ static constexpr int start(int l) { return l == 0 ? 0 : cbinom(N + l - 1, l - 1); }
    static constexpr int TAB = start(M);       // tuples in the table (sizes 0..M-1)
    static constexpr int NF = count(M);        // tuples of the output
    static constexpr int NTUP = start(M + 1);  // TAB + NF
    static constexpr int OUT = E * N * N * (M >= 3 ? N : 1) * (M >= 4 ? N : 1); // 6 n^k values per row
    // rows per group: about 2048 output values to form per group, at most 128 rows
    static constexpr int RW = (2048 + NF * E - 1) / (NF * E);
    static constexpr int R = RW < 1 ? 1 : (RW > 128 ? 128 : RW);
    static constexpr int TUPB = (NTUP * 4 + 15) / 16 * 16;
    static constexpr int SMEM = TUPB + R * TAB * E * (int)sizeof(real);
    static_assert(N >= 1 && N <= 15 && M >= 2 && M <= 4, "4-bit packed tuples of 2..4 indices");
};

__host__ __device__ constexpr int cfact(int m) { return m <= 1 ? 1 : m * cfact(m - 1); }

// the P-th permutation of 0..M-1 in lexicographic order, packed: pi(m) in bits 4m.., its inverse in bits 16 + 4s..
__host__ __device__ constexpr unsigned perm_code(int M, int P)
{
    int avail[4] = {0, 1, 2, 3};
    unsigned code = 0;
    int f = cfact(M - 1);
    for (int m = 0; m < M; m++) {
        const int k = P / f;
        P -= k * f;
        const int s = avail[k];
        for (int t = k; t + 1 < M - m; t++) avail[t] = avail[t + 1];
        code |= (unsigned)s << (4 * m);
        code |= (unsigned)m << (16 + 4 * s);
        if (M - 1 - m > 0) f /= (M - 1 - m);
    }
    return code;
}

// C(x, p), p <= 4 and known after unrolling
__device__ __forceinline__ unsigned binom(unsigned x, int p)
{
    if (p == 0) return 1u;
    if (p == 1) return x;
    if (p == 2) return x * (x - 1) / 2;
    if (p == 3) return x * (x - 1) * (x - 2) / 6;
    return x * (x - 1) * (x - 2) * (x - 3) / 24;
}

// d^S zeta_j, component r, for the sorted tuple S of L indices (packed), from the table of sizes < L of one row
template <typename real, int N, int K, int L>
__device__ __forceinline__ real pfk_value(const real *__restrict__ tab, unsigned S, int r, int j)
{
    typedef Pfk<real, N, K> P;
    const int i = S & 15;
    const bool rot = r >= 3;
    if (rot && i >= j) return (real)0;
    const int lo = i <= j ? i : j, hi = i <= j ? j : i;
    const int c = rot ? r - 3 : r, c1 = c == 2 ? 0 : c + 1, c2 = c == 0 ? 2 : c - 1;
    const int xrow = rot ? 3 : 0;
    unsigned rest[L > 1 ? L - 1 : 1];
#pragma unroll
    for (int p = 0; p < L - 1; p++) rest[p] = (S >> (4 * (p + 1))) & 15u;
    real acc = 0;
#pragma unroll
    for (int mask = 0; mask < (1 << (L - 1)); mask++) {
        // A: the indices of rest at the set bits, B: the others; each stays sorted, ranked in colex order
        unsigned ra = 0, rb = 0;
        int na = 0, nb = 0;
#pragma unroll
        for (int p = 0; p < L - 1; p++) {
            if ((mask >> p) & 1) { ra += binom(rest[p] + na, na + 1); na++; }
            else { rb += binom(rest[p] + nb, nb + 1); nb++; }
        }
        const real *u = tab + (P::start(na) + (int)ra) * P::E + 3 * N + lo;
        const real *x = tab + (P::start(nb) + (int)rb) * P::E + xrow * N + hi;
        acc += u[c1 * N] * x[c2 * N] - u[c2 * N] * x[c1 * N];
    }
    return acc;
}

// store v at element e of the 6 x n block of every distinct permutation of the sorted tuple a (permutations P.. of M!)
template <int N, int M, int E, int P = 0, typename real>
__device__ __forceinline__ void pfk_scatter(real *__restrict__ o, const unsigned (&a)[M], real v)
{
    constexpr unsigned code = perm_code(M, P);
    // a permutation that puts two equal neighbours of the sorted tuple out of order repeats another one
    bool dup = false;
#pragma unroll
    for (int s = 0; s + 1 < M; s++)
        if (((code >> (16 + 4 * s)) & 15u) > ((code >> (16 + 4 * (s + 1))) & 15u)) dup |= a[s] == a[s + 1];
    if (!dup) {
        unsigned t = 0;
#pragma unroll
        for (int m = 0; m < M; m++) t = t * N + a[(code >> (4 * m)) & 15u];
        o[t * E] = v;
    }
    if constexpr (P + 1 < cfact(M)) pfk_scatter<N, M, E, P + 1>(o, a, v);
}

template <typename real, int N, int K, int L>
__device__ __forceinline__ void pfk_build(real *__restrict__ tabs, const unsigned *__restrict__ tup, int nr)
{
    typedef Pfk<real, N, K> P;
    constexpr int CNT = P::count(L) * P::E;
    for (int x = threadIdx.x; x < nr * CNT; x += PFK_THREADS) {
        const int rho = x / CNT, rem = x - rho * CNT, t = rem / P::E, e = rem - t * P::E;
        real *tab = tabs + rho * (P::TAB * P::E);
        tab[(P::start(L) + t) * P::E + e] = pfk_value<real, N, K, L>(tab, tup[P::start(L) + t], e / N, e % N);
    }
    __syncthreads();
    if constexpr (L + 1 < P::M) pfk_build<real, N, K, L + 1>(tabs, tup, nr);
}

template <typename real, int N, int K>
__global__ void __launch_bounds__(PFK_THREADS) k_partial_fkine(const real *__restrict__ J, long long nrows, real *__restrict__ D)
{
    typedef Pfk<real, N, K> P;
    extern __shared__ __align__(16) unsigned char pfk_smem[];
    unsigned *tup = reinterpret_cast<unsigned *>(pfk_smem);
    real *tabs = reinterpret_cast<real *>(pfk_smem + P::TUPB);

    // every sorted tuple of sizes 0..M by unranking its colex rank: b_p = a_p + p is strictly increasing and the rank
    // is sum_p C(b_p, p + 1)
    for (int t = threadIdx.x; t < P::NTUP; t += PFK_THREADS) {
        int l = 0;
        while (t >= P::start(l + 1)) l++;
        int rem = t - P::start(l);
        unsigned packed = 0;
        for (int p = l - 1; p >= 0; p--) {
            int b = p;
            while (cbinom(b + 1, p + 1) <= rem) b++;
            rem -= cbinom(b, p + 1);
            packed |= (unsigned)(b - p) << (4 * p);
        }
        tup[t] = packed;
    }

    const long long ngroups = (nrows + P::R - 1) / P::R;
    for (long long g = blockIdx.x; g < ngroups; g += gridDim.x) {
        const long long row0 = g * P::R;
        const int nr = (int)(nrows - row0 < P::R ? nrows - row0 : P::R);
        __syncthreads(); // the tuple list is written / the previous group's table is no longer read
        const real *src = J + row0 * P::E;
        for (int x = threadIdx.x; x < nr * P::E; x += PFK_THREADS) {
            const int rho = x / P::E;
            tabs[rho * (P::TAB * P::E) + (x - rho * P::E)] = src[x];
        }
        __syncthreads();
        pfk_build<real, N, K, 1>(tabs, tup, nr);

        constexpr int CNT = P::NF * P::E;
        for (int x = threadIdx.x; x < nr * CNT; x += PFK_THREADS) {
            const int rho = x / CNT, rem = x - rho * CNT, f = rem / P::E, e = rem - f * P::E;
            const unsigned S = tup[P::TAB + f];
            const real v = pfk_value<real, N, K, P::M>(tabs + rho * (P::TAB * P::E), S, e / N, e % N);
            unsigned a[P::M];
#pragma unroll
            for (int m = 0; m < P::M; m++) a[m] = (S >> (4 * m)) & 15u;
            pfk_scatter<N, P::M, P::E>(D + (row0 + rho) * (long long)P::OUT + e, a, v);
        }
    }
}

template <typename real, int N, int K>
int pfk_launch(const void *J, long long nrows, void *D, cudaStream_t st)
{
    typedef Pfk<real, N, K> P;
    const void *fn = (const void *)k_partial_fkine<real, N, K>;
    const int per_sm = b2k_blocks_per_sm(fn, PFK_THREADS, P::SMEM);
    if (per_sm < 0) return per_sm;
    if (per_sm == 0) { b2k_set_error("b2k_partial_fkine: n = %d, order %d does not fit on this device", N, K); return B2K_ERR_INVALID; }
    const long long groups = (nrows + P::R - 1) / P::R, cap = (long long)b2k_num_sms() * per_sm;
    k_partial_fkine<real, N, K><<<(unsigned)(groups < cap ? groups : cap), PFK_THREADS, P::SMEM, st>>>((const real *)J, nrows, (real *)D);
    b2k_count_launch();
    B2K_CUDA(cudaGetLastError());
    return B2K_OK;
}

template <typename real, int N>
int pfk_order(int order, const void *J, long long nrows, void *D, cudaStream_t st)
{
    switch (order) {
    case 3: return pfk_launch<real, N, 3>(J, nrows, D, st);
    case 4: return pfk_launch<real, N, 4>(J, nrows, D, st);
    default: return pfk_launch<real, N, 5>(J, nrows, D, st);
    }
}

} // namespace

// The launcher of b2k_partial_fkine; jacfun_dispatch (b2k_extra.cu) has checked its arguments
template <typename real>
int b2k_pfk_launch(int n, int order, const void *J, long long nrows, void *D, cudaStream_t st)
{
    switch (n) {
    case 1: return pfk_order<real, 1>(order, J, nrows, D, st);
    case 2: return pfk_order<real, 2>(order, J, nrows, D, st);
    case 3: return pfk_order<real, 3>(order, J, nrows, D, st);
    case 4: return pfk_order<real, 4>(order, J, nrows, D, st);
    case 5: return pfk_order<real, 5>(order, J, nrows, D, st);
    case 6: return pfk_order<real, 6>(order, J, nrows, D, st);
    case 7: return pfk_order<real, 7>(order, J, nrows, D, st);
    case 8: return pfk_order<real, 8>(order, J, nrows, D, st);
    case 9: return pfk_order<real, 9>(order, J, nrows, D, st);
    case 10: return pfk_order<real, 10>(order, J, nrows, D, st);
    }
    b2k_set_error("b2k_partial_fkine: unsupported joint count %d", n);
    return B2K_ERR_INVALID;
}
template int b2k_pfk_launch<float>(int, int, const void *, long long, void *, cudaStream_t);
template int b2k_pfk_launch<double>(int, int, const void *, long long, void *, cudaStream_t);
