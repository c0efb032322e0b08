// Next-token sampling on the GPU: repetition / presence penalties, temperature, top-k and top-p, in ONE launch for
// every row of a batch, greedy and sampled rows alike.
//
// Stands in for SearcherImplV1::random_sample (reference src/generator/batch_generator.cpp:1854-1883), i.e.
// functions::softmax with temperature + beam_utility::random_sampler_gpu (src/generator/random_util.cu:81-198: cub radix
// sort of the vocabulary, inclusive scan, one-thread binary search, once per task) and for the penalty scatter
// beam_repetition_penalty (src/generator/beam_util.cu:198-281).  No sort: the position where the descending cumulative
// mass crosses a target is found by radix selection, once for the top-k mass C_{k-1} and once for the sampled token.
//
// One thread-block cluster of kCluster CTAs per row.  CTA r keeps its contiguous slice of the row, penalised and divided
// by the temperature, in shared memory; every later pass runs over shared memory.  Per-CTA histograms are merged through
// distributed shared memory in rank order, so every CTA of the cluster takes the same decisions.
//
// Masses are fixed point: w = round(exp(x - max x) * 2^44) as uint64, so sums are exact integers and do not depend on
// the summation order (a launch is reproducible bit for bit, whatever the atomics' order).  A token whose weight is below
// ~2^-45 of the maximum gets mass 0 and is never picked (probability < 3e-14 under the exact contract).
//
// Logits processors (zl_sample_processed): the n-gram repetition penalty (calc_repetition_ngram +
// apply_beam_repetition_penalty, src/generator/beam_util.cu:318-375) and logit_bias (SearcherImplV1::add_logit_bias,
// batch_generator.cpp:1709-1728).  k_ngram_levels gives each distinct token of a task's generated sequence its largest
// n-gram level, in a per-row hash table; k_sample then stages a processed copy of its slice in shared memory.
//
// Token automata (zl_sample_masked, zl_llama_set_constraint): a constrained row reads NaN for every token outside the
// allowed set of its task's state (in the staging pass, or in pass 1 when no other processor stages the row) -- NaN is
// never the greedy pick and has probability 0, exactly as a NaN logit -- and an allowed NaN logit as -inf, so that a row
// whose allowed tokens all end at -inf picks the smallest allowed token.  The CTA that writes the pick moves the task's state along the automaton's edge of that token.
#include "common.cuh"
#include "sample.cuh"

#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace zl {

constexpr int kSampleCluster = 8;
constexpr int kSampleThreads = 1024;
constexpr int kSampleMaxVocab = 262144;
constexpr int kSampleMaxSlice = kSampleMaxVocab / kSampleCluster;
constexpr float kMassScale = 17592186044416.0f;   // 2^44: V * 2^44 < 2^63 for V <= 2^18

// Philox4x32-10 (Salmon et al., SC'11; the round function and constants of CUDA's curand_philox4x32_x.h), first output
// word for key = (seed lo, seed hi), counter = (counter, 0, 0, 0).
__host__ __device__ inline uint32_t philox_first(uint64_t seed, uint32_t counter) {
    uint32_t c0 = counter, c1 = 0, c2 = 0, c3 = 0;
    uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    for (int i = 0; i < 10; ++i) {
        if (i) {
            k0 += 0x9E3779B9u;
            k1 += 0xBB67AE85u;
        }
        const uint64_t p0 = (uint64_t)0xD2511F53u * c0;
        const uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
        const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
        const uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
        c1 = (uint32_t)p1;
        c3 = (uint32_t)p0;
        c0 = n0;
        c2 = n2;
    }
    return c0;
}

// ascending key == descending x; -0 and +0 share one key (they compare equal, so they tie by index)
__device__ __forceinline__ uint32_t desc_key(float x) {
    const uint32_t u = __float_as_uint(x);
    const uint32_t k = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return ~k;
}
// first radix digit: a monotone (non-increasing in x) bucket of width 1/4 below the row maximum.  Logit rows crowd into a
// few float exponents, so the float's own top bits would send nearly every element to one shared-memory counter.
__device__ __forceinline__ int bucket0(float x, float xmax) {
    const float d = (xmax - x) * 4.0f;
    return d < 255.0f ? (int)d : 255;
}
__device__ __forceinline__ unsigned long long mass_of(float x, float xmax) {
    return __float2ull_rn(expf(x - xmax) * kMassScale);
}

struct SampleShared {
    uint32_t cnt[2][256];   // this CTA's histogram of the current round (double-buffered across rounds)
    unsigned long long mass[2][256];
    uint32_t mcnt[256];     // cluster-merged histogram of the current round
    unsigned long long mmass[256];
    uint32_t cnt0[256];     // cluster-merged histogram of round 0 (shared by both selections)
    unsigned long long mass0[256];
    float wv[32], wx[32];
    int wi[32];
    float cta_best, cta_xmax;   // read by the other CTAs of the cluster
    int cta_bi;
    unsigned long long scan[32];
    int sel_digit;
    unsigned long long sel_cnt_before, sel_mass_before, sel_bin_cnt, sel_bin_mass, total_mass;
    int tok;
};

// Warp 0: over 256 merged bins, find the first bin whose inclusive cumulative metric (mass or count) reaches `need`
// (>= 1); write the digit, the count / mass of the bins before it and of the bin itself.
__device__ void scan_select(SampleShared& s, const uint32_t* cnt, const unsigned long long* mass, bool by_mass,
                            unsigned long long need) {
    const int lane = threadIdx.x & 31;
    unsigned long long tc = 0, tm = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        tc += cnt[lane * 8 + j];
        tm += mass[lane * 8 + j];
    }
    unsigned long long ic = tc, im = tm;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long a = __shfl_up_sync(0xffffffffu, ic, o);
        const unsigned long long b = __shfl_up_sync(0xffffffffu, im, o);
        if (lane >= o) {
            ic += a;
            im += b;
        }
    }
    const unsigned long long total = __shfl_sync(0xffffffffu, by_mass ? im : ic, 31);
    const unsigned long long total_m = __shfl_sync(0xffffffffu, im, 31);
    if (need > total) need = total;   // exact integers make this a no-op; kept so a pick always exists
    if (need < 1) need = 1;
    const unsigned long long inc = by_mass ? im : ic, exc = inc - (by_mass ? tm : tc);
    const unsigned hit = __ballot_sync(0xffffffffu, exc < need && inc >= need);
    const int owner = hit ? __ffs(hit) - 1 : 0;
    if (lane == 0) s.total_mass = total_m;
    if (lane == owner) {
        unsigned long long bc = ic - tc, bm = im - tm;
        int d = lane * 8;
        for (int j = 0; j < 8; ++j) {
            const unsigned long long c = cnt[lane * 8 + j], m = mass[lane * 8 + j];
            d = lane * 8 + j;
            if ((by_mass ? bm + m : bc + c) >= need || j == 7 || !hit) {
                s.sel_digit = d;
                s.sel_cnt_before = bc;
                s.sel_mass_before = bm;
                s.sel_bin_cnt = c;
                s.sel_bin_mass = m;
                break;
            }
            bc += c;
            bm += m;
        }
    }
}

struct SelResult {
    int b0;
    uint32_t key;   // full descending key of the selected tie group
    unsigned long long cnt_before, mass_before, grp_cnt, grp_mass;
};

// Radix selection over the order (descending x, ascending index): the tie group of elements with equal x that contains
// the `target`-th unit of the metric (count or mass) counted from the top.  Round 0 uses the merged bucket histogram,
// rounds 1..4 the bytes of the descending key inside the selected bucket.  `rc` numbers the rounds for the histogram
// double buffer.
__device__ SelResult cluster_select(SampleShared& s, cg::cluster_group& cl, const float* xs, int n, float xmax,
                                    bool by_mass, unsigned long long target, int& rc) {
    SelResult r{};
    if (threadIdx.x < 32) scan_select(s, s.cnt0, s.mass0, by_mass, target);
    __syncthreads();
    r.b0 = s.sel_digit;
    r.cnt_before = s.sel_cnt_before;
    r.mass_before = s.sel_mass_before;
    r.grp_cnt = s.sel_bin_cnt;
    r.grp_mass = s.sel_bin_mass;
    uint32_t prefix = 0;
    for (int round = 1; round <= 4; ++round, ++rc) {
        const int buf = rc & 1;
        if (threadIdx.x < 256) {
            s.cnt[buf][threadIdx.x] = 0;
            s.mass[buf][threadIdx.x] = 0;
        }
        __syncthreads();
        const int shift = 32 - 8 * round;
        for (int i = threadIdx.x; i < n; i += kSampleThreads) {
            const float x = xs[i];
            if (bucket0(x, xmax) != r.b0) continue;
            const uint32_t k = desc_key(x);
            if (round > 1 && (k >> (shift + 8)) != prefix) continue;
            const int dg = (k >> shift) & 255;
            atomicAdd(&s.cnt[buf][dg], 1u);
            atomicAdd(&s.mass[buf][dg], mass_of(x, xmax));   // the count selection needs C_{k-1} too
        }
        cl.sync();
        if (threadIdx.x < 256) {
            uint32_t c = 0;
            unsigned long long m = 0;
            for (int q = 0; q < kSampleCluster; ++q) {
                c += cl.map_shared_rank(&s.cnt[buf][0], q)[threadIdx.x];
                m += cl.map_shared_rank(&s.mass[buf][0], q)[threadIdx.x];
            }
            s.mcnt[threadIdx.x] = c;
            s.mmass[threadIdx.x] = m;
        }
        __syncthreads();
        if (threadIdx.x < 32)
            scan_select(s, s.mcnt, s.mmass, by_mass, target - (by_mass ? r.mass_before : r.cnt_before));
        __syncthreads();
        prefix = (prefix << 8) | (uint32_t)s.sel_digit;
        r.cnt_before += s.sel_cnt_before;
        r.mass_before += s.sel_mass_before;
        r.grp_cnt = s.sel_bin_cnt;
        r.grp_mass = s.sel_bin_mass;
        __syncthreads();   // s.sel_* is rewritten by the next round's scan
    }
    r.key = prefix;
    return r;
}

constexpr int kNgramThreads = 1024;
constexpr int kNgramSmem = 12032;   // sequence elements staged in shared memory; the rest is read from global memory

// Fibonacci hashing: the top log2(h) bits of tok * 2^32 / phi (h is a power of two >= 2)
__device__ __forceinline__ int ngram_slot(int tok, int h) {
    return (int)(((uint32_t)tok * 2654435761u) >> (32 - (__ffs(h) - 1)));
}

// open addressing: the slot of `tok` keeps the largest level inserted for it
__device__ void ngram_insert(int2* tab, int h, int tok, int lev) {
    if (tok < 0) return;   // -1 marks an empty slot; a negative id never matches a vocabulary slice
    for (int i = ngram_slot(tok, h);; i = (i + 1) & (h - 1)) {
        const int prev = atomicCAS(&tab[i].x, -1, tok);
        if (prev == -1 || prev == tok) {
            if (lev > 0) atomicMax(&tab[i].y, lev);
            return;
        }
    }
}

// One CTA per row whose task has ngram > 1.  r = the task's sequence, most recent first (r[k] = seq[n-1-k]).  The
// reference's levels (KMP next[] over r, then ngrams[i - L] = max(ngrams[i - L], L) with L = next[i] + 1) equal, with
// z the Z-function of r and R(s) = max(0, max over s' < s of s' + z[s'] - 1):
//   lev[s-1] = z[s] where z[s] > 0 and s + z[s] - 1 > R(s), and 0 everywhere else.
// One thread per start s extends z[s] by direct comparison (work = sum of z: ~n / alphabet on text, n^2 / 2 for one
// repeated token); a block max-scan over tiles of 1024 starts carries R.  Writes, for every distinct token of r, its
// largest level into the row's table of ngram_table_size(n) slots.
__global__ void __launch_bounds__(kNgramThreads) k_ngram_levels(int T, const int32_t* __restrict__ row_task, SampleProc pr) {
    __shared__ int rs[kNgramSmem];
    __shared__ int wmax[kNgramThreads / 32];
    __shared__ int carry;
    const int row = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    pdl_trigger();
    pdl_wait();
    if (row >= T) return;
    const int task = row_task ? row_task[row] : row;
    if (!(pr.ngram[task] > 1.f)) return;
    const int n = min(max(pr.seq_len[task], 0), pr.seq_stride);
    const int32_t* sq = pr.seq + (size_t)task * pr.seq_stride;
    int2* tab = pr.table + (size_t)row * pr.table_stride;
    const int h = ngram_table_size(n);
    for (int k = tid; k < min(n, kNgramSmem); k += kNgramThreads) rs[k] = sq[n - 1 - k];
    for (int i = tid; i < h; i += kNgramThreads) tab[i] = make_int2(-1, 0);
    if (tid == 0) carry = 0;
    __syncthreads();
    auto at = [&](int k) { return k < kNgramSmem ? rs[k] : sq[n - 1 - k]; };
    for (int base = 1; base < n; base += kNgramThreads) {
        const int s = base + tid;
        int z = 0;
        if (s < n)
            while (s + z < n && at(s + z) == at(z)) ++z;
        const int e = s < n ? s + z - 1 : 0;
        int inc = e;   // inclusive max-scan within the warp
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc = max(inc, v);
        }
        const int exc = __shfl_up_sync(0xffffffffu, inc, 1);
        if (lane == 31) wmax[warp] = inc;
        __syncthreads();
        int R = carry;
        for (int w = 0; w < warp; ++w) R = max(R, wmax[w]);
        if (lane > 0) R = max(R, exc);
        if (s < n) ngram_insert(tab, h, at(s - 1), (z > 0 && e > R) ? z : 0);
        __syncthreads();   // every thread has read carry and wmax
        if (tid == 0) {
            int c = carry;
            for (int w = 0; w < kNgramThreads / 32; ++w) c = max(c, wmax[w]);
            carry = c;
        }
        __syncthreads();
    }
    if (tid == 0 && n > 0) ngram_insert(tab, h, at(n - 1), 0);   // the oldest token has level 0
}

__global__ void __cluster_dims__(kSampleCluster, 1, 1) __launch_bounds__(kSampleThreads, 1)
    k_sample(const float* __restrict__ logits, int T, int V, int S, const zl_sample_params_t* __restrict__ params,
             const int32_t* __restrict__ row_task, const int32_t* __restrict__ counter, uint32_t* __restrict__ history,
             int hwords, int32_t* __restrict__ out, SampleProc pr) {
    extern __shared__ float xs[];
    __shared__ SampleShared s;
    cg::cluster_group cl = cg::this_cluster();
    const int rank = (int)cl.block_rank();
    const int row = blockIdx.z * gridDim.y + blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    pdl_trigger();
    if (row >= T) return;   // the whole cluster shares the row
    pdl_wait();
    const int task = row_task ? row_task[row] : row;
    const zl_sample_params_t p = params[task];
    const bool greedy = !(p.temperature > 0.f) || p.top_k == 1;
    uint32_t* hist = history ? history + (size_t)task * hwords : nullptr;
    const bool pen = hist && (p.presence_penalty != 0.f || p.repetition_penalty != 1.f);
    const int lo = rank * S;
    const int n = max(0, min(V, lo + S) - lo);
    const float* src = logits + (size_t)row * V + lo;
    const int nbias = pr.bias_tok ? min(pr.bias_cnt[task], pr.bias_stride) : 0;
    const float ngram = pr.ngram ? pr.ngram[task] : 1.f;
    const int ast = pr.au.mask ? (pr.au.state ? pr.au.state[task] : task) : -1;
    const uint32_t* amask = ast >= 0 ? pr.au.mask + ((size_t)task * pr.au.states + ast) * pr.au.words : nullptr;
    const bool proc = nbias > 0 || ngram > 1.f;   // a row with only a mask applies it in pass 1, unstaged
    if (proc) {
        // this thread's first bias entry, loaded before the slice so that its latency overlaps the slice's
        const int32_t* bt = pr.bias_tok + (size_t)task * pr.bias_stride;
        const float* bv = pr.bias_val + (size_t)task * pr.bias_stride;
        const int g0 = tid < nbias ? bt[tid] : -1;
        const float b0 = tid < nbias ? bv[tid] : 0.f;
        // the processed slice in shared memory: the automaton's mask, penalties (the n-gram rule replaces the bitmap
        // rule), then the bias
        for (int i = tid; i < n; i += kSampleThreads) {
            float l = src[i];
            const int g = lo + i;
            if (amask) l = ((amask[g >> 5] >> (g & 31)) & 1u) ? (l == l ? l : -INFINITY) : NAN;
            if (!(ngram > 1.f) && pen && ((hist[g >> 5] >> (g & 31)) & 1u))
                l = p.presence_penalty != 0.f ? l - p.presence_penalty
                                              : (l < 0.f ? l * p.repetition_penalty : l / p.repetition_penalty);
            xs[i] = l;
        }
        __syncthreads();
        if (ngram > 1.f) {   // each table slot names a distinct token: no two threads touch one element
            const int2* tab = pr.table + (size_t)row * pr.table_stride;
            const int h = ngram_table_size(min(max(pr.seq_len[task], 0), pr.seq_stride));
            for (int i = tid; i < h; i += kSampleThreads) {
                const int2 e = tab[i];
                if (e.x < lo || e.x >= lo + n) continue;
                const float f = powf(ngram, (float)(e.y + 1)) * p.repetition_penalty;   // beam_util.cu:345, :368
                const float l = xs[e.x - lo];
                xs[e.x - lo] = l < 0.f ? l * f : l / f;
            }
            __syncthreads();
        }
        if (g0 >= lo && g0 < lo + n) xs[g0 - lo] += b0;   // distinct tokens (zl_llama_set_logits_processors checks)
        for (int j = tid + kSampleThreads; j < nbias; j += kSampleThreads) {
            const int g = bt[j];
            if (g >= lo && g < lo + n) xs[g - lo] += bv[j];
        }
        __syncthreads();
    }

    // pass 1: the mask and penalties of an unstaged row, the greedy pick of the penalised row (zl_argmax's rule: max,
    // ties -> lowest index), max of x
    float best = -INFINITY, xmax = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = tid; i < n; i += kSampleThreads) {
        float l = proc ? xs[i] : src[i];
        const int g = lo + i;
        if (!proc && amask) l = ((amask[g >> 5] >> (g & 31)) & 1u) ? (l == l ? l : -INFINITY) : NAN;
        if (!proc && pen && ((hist[g >> 5] >> (g & 31)) & 1u)) {   // beam_util.cu:212-219
            if (p.presence_penalty != 0.f)
                l = l - p.presence_penalty;
            else
                l = l < 0.f ? l * p.repetition_penalty : l / p.repetition_penalty;
        }
        if (l > best || (l == best && g < bi)) {
            best = l;
            bi = g;
        }
        if (!greedy) {
            float x = l / p.temperature;
            if (x != x) x = -INFINITY;   // NaN: probability 0
            if (x == 0.f) x = 0.f;       // one key for -0 / +0
            xs[i] = x;
            xmax = fmaxf(xmax, x);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) {
            best = ov;
            bi = oi;
        }
        xmax = fmaxf(xmax, __shfl_xor_sync(0xffffffffu, xmax, o));
    }
    if (lane == 0) {
        s.wv[warp] = best;
        s.wi[warp] = bi;
        s.wx[warp] = xmax;
    }
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < kSampleThreads / 32; ++w) {
            if (s.wv[w] > best || (s.wv[w] == best && s.wi[w] < bi)) {
                best = s.wv[w];
                bi = s.wi[w];
            }
            xmax = fmaxf(xmax, s.wx[w]);
        }
        s.cta_best = best;
        s.cta_bi = bi;
        s.cta_xmax = xmax;
    }
    cl.sync();
    // every CTA merges the cluster's candidates in rank order (= index order: ties keep the lower index)
    best = -INFINITY;
    bi = 0x7fffffff;
    xmax = -INFINITY;
    for (int q = 0; q < kSampleCluster; ++q) {
        SampleShared* o = cl.map_shared_rank(&s, q);
        const float ov = o->cta_best;
        const int oi = o->cta_bi;
        if (ov > best || (ov == best && oi < bi)) {
            best = ov;
            bi = oi;
        }
        xmax = fmaxf(xmax, o->cta_xmax);
    }
    const int greedy_tok = (bi >= 0 && bi < V) ? bi : 0;

    int tok = greedy_tok;
    bool owner = rank == 0;   // the CTA that writes the result
    // a row whose penalised maximum is not finite falls back to the greedy pick
    if (!greedy && xmax > -INFINITY && xmax < INFINITY) {
        // round 0: bucket histogram with masses, over the whole row
        if (tid < 256) {
            s.cnt[0][tid] = 0;
            s.mass[0][tid] = 0;
        }
        __syncthreads();
        for (int i = tid; i < n; i += kSampleThreads) {
            const float x = xs[i];
            const int b = bucket0(x, xmax);
            atomicAdd(&s.cnt[0][b], 1u);
            atomicAdd(&s.mass[0][b], mass_of(x, xmax));
        }
        cl.sync();
        if (tid < 256) {
            uint32_t c = 0;
            unsigned long long m = 0;
            for (int q = 0; q < kSampleCluster; ++q) {
                c += cl.map_shared_rank(&s.cnt[0][0], q)[tid];
                m += cl.map_shared_rank(&s.mass[0][0], q)[tid];
            }
            s.cnt0[tid] = c;
            s.mass0[tid] = m;
        }
        __syncthreads();
        int rc = 1;
        if (tid < 32) scan_select(s, s.cnt0, s.mass0, true, 1);
        __syncthreads();
        const unsigned long long Z = s.total_mass;
        __syncthreads();
        // P' = min(top_p * Z, C_{k-1})   (random_util.cu:89-94)
        unsigned long long P = Z;
        if (p.top_p < 1.f) {
            const double tp = (double)p.top_p * (double)Z;
            P = tp >= 1.0 ? (unsigned long long)tp : 1ull;
        }
        if (p.top_k > 1 && p.top_k < V) {
            const SelResult k = cluster_select(s, cl, xs, n, xmax, false, (unsigned long long)p.top_k, rc);
            const unsigned long long pos = (unsigned long long)p.top_k - 1 - k.cnt_before;   // position in its tie group
            const unsigned long long ck = k.mass_before + (k.grp_cnt ? (pos + 1) * (k.grp_mass / k.grp_cnt) : 0);
            if (ck < P) P = ck;
        }
        if (P < 1) P = 1;
        // target = u * P' with u = m / 2^24, m in [1, 2^24]; rounded up: C_j >= target <=> C_j >= ceil(m P' / 2^24)
        const uint32_t r = philox_first(p.seed, counter ? (uint32_t)counter[row] : 0u);
        const unsigned long long m = (unsigned long long)(r >> 8) + 1;
        const unsigned long long target = m * (P >> 24) + ((m * (P & 0xFFFFFFull) + 0xFFFFFFull) >> 24);
        const SelResult t = cluster_select(s, cl, xs, n, xmax, true, target, rc);
        // inside the tie group every element carries the same mass: the pick is its p-th element in index order
        unsigned long long pgrp = 0;
        if (t.grp_cnt > 0 && t.grp_mass > 0) {
            const unsigned long long wt = t.grp_mass / t.grp_cnt;
            const unsigned long long need = target > t.mass_before ? target - t.mass_before : 1;
            pgrp = (need + wt - 1) / wt - 1;
            if (pgrp >= t.grp_cnt) pgrp = t.grp_cnt - 1;
        }
        // which CTA holds it: the last round's per-CTA counts of the group's bin, in rank order
        const int lbuf = (rc - 1) & 1;
        unsigned long long before = 0;
        int q_own = kSampleCluster - 1;
        for (int q = 0; q < kSampleCluster; ++q) {
            const unsigned long long c = cl.map_shared_rank(&s.cnt[lbuf][0], q)[t.key & 255];
            if (pgrp < before + c) {
                q_own = q;
                break;
            }
            before += c;
        }
        owner = rank == q_own;
        tok = -1;
        if (owner) {
            const unsigned long long want = pgrp - before;
            // each thread counts the group's elements in its contiguous chunk; block scan; the owning thread walks
            const int per = (n + kSampleThreads - 1) / kSampleThreads;
            const int a = tid * per, e = min(n, a + per);
            uint32_t c = 0;
            for (int i = a; i < e; ++i) c += (bucket0(xs[i], xmax) == t.b0 && desc_key(xs[i]) == t.key);
            unsigned long long inc = c;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned long long v = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += v;
            }
            if (lane == 31) s.scan[warp] = inc;
            if (tid == 0) s.tok = -1;
            __syncthreads();
            unsigned long long wbase = 0;
            for (int w = 0; w < warp; ++w) wbase += s.scan[w];
            const unsigned long long exc = wbase + inc - c;
            if (c > 0 && want >= exc && want < exc + c) {
                unsigned long long k = exc;
                for (int i = a; i < e; ++i) {
                    if (bucket0(xs[i], xmax) == t.b0 && desc_key(xs[i]) == t.key) {
                        if (k == want) {
                            s.tok = lo + i;
                            break;
                        }
                        ++k;
                    }
                }
            }
            __syncthreads();
            tok = s.tok >= 0 ? s.tok : greedy_tok;
        }
    }
    if (owner && tid == 0) {
        out[row] = tok;
        const bool record = !pr.frozen || pr.frozen[task] == 0;
        if (hist && record) atomicOr(&hist[tok >> 5], 1u << (tok & 31));
        if (pr.seq && record) {   // appends past the capacity are dropped
            const int len = pr.seq_len[task];
            if (len >= 0 && len < pr.seq_stride) {
                pr.seq[(size_t)task * pr.seq_stride + len] = tok;
                pr.seq_len[task] = len + 1;
            }
        }
        // the automaton's move (every CTA of the cluster read the state before the first cluster barrier)
        const int cur = pr.au.next ? pr.au.state[task] : -1;
        if (cur >= 0 && record) {
            const int32_t* rp = pr.au.row_ptr + (size_t)task * (pr.au.states + 1);
            const int32_t* et = pr.au.edge_tok + (size_t)task * pr.au.max_edges;
            int a = rp[cur], b = rp[cur + 1], nx = pr.au.dflt[(size_t)task * pr.au.states + cur];
            while (a < b) {   // the state's edge tokens are sorted
                const int mid = (a + b) >> 1, et_mid = et[mid];
                if (et_mid == tok) {
                    nx = pr.au.next[(size_t)task * pr.au.max_edges + mid];
                    break;
                }
                if (et_mid < tok) a = mid + 1;
                else b = mid;
            }
            pr.au.state[task] = nx;
        }
    }
    cl.sync();   // no CTA leaves while another may still read its shared memory
}

}  // namespace zl

using namespace zl;

extern "C" unsigned zl_sample_uniform(uint64_t seed, unsigned counter) { return philox_first(seed, counter); }

extern "C" size_t zl_sample_workspace_bytes(int T, int V) {
    (void)T;
    (void)V;
    return 0;
}

extern "C" int zl_sample_check_params(const zl_sample_params_t* p, int n) {
    ZL_CHECK_ARG(p && n > 0);
    for (int i = 0; i < n; ++i) {
        const zl_sample_params_t& q = p[i];
        ZL_CHECK_ARG(q.temperature >= 0.f && q.temperature < INFINITY);
        ZL_CHECK_ARG(q.top_p > 0.f && q.top_p <= 1.f);
        ZL_CHECK_ARG(q.top_k >= 0);
        ZL_CHECK_ARG(q.repetition_penalty > 0.f && q.repetition_penalty < INFINITY);
        ZL_CHECK_ARG(q.presence_penalty > -INFINITY && q.presence_penalty < INFINITY);
    }
    return ZL_OK;
}

extern "C" int zl_token_automaton_check(int vocab, int n_states, const uint32_t* masks, const int32_t* row_ptr,
                                        int n_edges, const int32_t* edge_tok, const int32_t* edge_next,
                                        const int32_t* default_next, int start) {
    ZL_CHECK_ARG(vocab > 0 && n_states >= 1 && n_edges >= 0);
    ZL_CHECK_ARG(masks && row_ptr && default_next && (n_edges == 0 || (edge_tok && edge_next)));
    ZL_CHECK_ARG(start >= 0 && start < n_states && row_ptr[0] == 0 && row_ptr[n_states] == n_edges);
    for (int s = 0; s < n_states; ++s) ZL_CHECK_ARG(row_ptr[s] <= row_ptr[s + 1]);
    const int W = cdiv(vocab, 32);
    const uint32_t tail = vocab % 32 ? ~0u << (vocab % 32) : 0u;   // bits at or past vocab in the last word
    for (int s = 0; s < n_states; ++s) {
        const uint32_t* a = masks + (size_t)s * W;
        uint32_t any = 0;
        for (int i = 0; i < W; ++i) any |= a[i];
        ZL_CHECK_ARG(any != 0 && (a[W - 1] & tail) == 0);
        ZL_CHECK_ARG(default_next[s] >= 0 && default_next[s] < n_states);
        for (int e = row_ptr[s]; e < row_ptr[s + 1]; ++e) {
            const int x = edge_tok[e];
            ZL_CHECK_ARG(x >= 0 && x < vocab && ((a[x >> 5] >> (x & 31)) & 1u));
            ZL_CHECK_ARG(e == row_ptr[s] || edge_tok[e - 1] < x);
            ZL_CHECK_ARG(edge_next[e] >= 0 && edge_next[e] < n_states);
        }
    }
    return ZL_OK;
}

int prepare_sample() {
    static bool done[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 0 && dev < 64 && done[dev]) return ZL_OK;
    ZL_CHECK_CUDA(cudaFuncSetAttribute(k_sample, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       kSampleMaxSlice * (int)sizeof(float)));
    if (dev >= 0 && dev < 64) done[dev] = true;
    return ZL_OK;
}

int zl::sample_launch(const float* logits, int T, int V, const zl_sample_params_t* params, const int32_t* row_task,
                      const int32_t* counter, uint32_t* history, int history_words, const SampleProc& pr, int32_t* out,
                      int pdl, cudaStream_t stream) {
    ZL_CHECK_ARG(!pr.seq || (pr.seq_len && pr.seq_stride > 0));
    ZL_CHECK_ARG(!pr.ngram || (pr.seq && pr.table));
    ZL_CHECK_ARG(!pr.bias_tok || (pr.bias_val && pr.bias_cnt && pr.bias_stride > 0));
    ZL_CHECK_ARG(!pr.au.mask || (pr.au.words >= cdiv(V, 32) && pr.au.states >= 0));
    ZL_CHECK_ARG(!pr.au.next || (pr.au.mask && pr.au.state && pr.au.row_ptr && pr.au.edge_tok && pr.au.dflt &&
                                 pr.au.states > 0));
    ZL_CHECK_ARG(logits && params && out && T > 0 && V > 0);
    ZL_CHECK_SUPPORTED(V <= kSampleMaxVocab);
    ZL_CHECK_ARG(!history || history_words >= cdiv(V, 32));
    const int rc = prepare_sample();
    if (rc != ZL_OK) return rc;
    if (pr.ngram)
        ZL_CHECK_CUDA(launch(k_ngram_levels, dim3(T), dim3(kNgramThreads), 0, stream, pdl != 0, T, row_task, pr));
    const int S = cdiv(V, kSampleCluster);
    const int ty = T < 65535 ? T : 65535;   // rows: blockIdx.z * gridDim.y + blockIdx.y
    ZL_CHECK_CUDA(launch(k_sample, dim3(kSampleCluster, ty, cdiv(T, ty)), dim3(kSampleThreads), (size_t)S * sizeof(float),
                         stream, pdl != 0, logits, T, V, S, params, row_task, counter, history, history_words, out, pr));
    return ZL_OK;
}

extern "C" int zl_sample(const float* logits, int T, int V, const zl_sample_params_t* params, const int32_t* row_task,
                         const int32_t* counter, uint32_t* history, int history_words, int32_t* out, void* ws,
                         size_t ws_bytes, int pdl, zl_stream_t stream) {
    (void)ws;
    ZL_CHECK_ARG(ws_bytes >= zl_sample_workspace_bytes(T, V));
    return sample_launch(logits, T, V, params, row_task, counter, history, history_words, SampleProc{}, out, pdl, stream);
}

extern "C" size_t zl_sample_processed_workspace_bytes(int T, int seq_stride) {
    if (T <= 0 || seq_stride <= 0) return 0;
    return (size_t)T * ngram_table_size(seq_stride) * sizeof(int2);
}

extern "C" int zl_sample_processed(const float* logits, int T, int V, const zl_sample_params_t* params,
                                   const int32_t* row_task, const int32_t* counter, uint32_t* history, int history_words,
                                   const float* ngram_penalty, int32_t* seq, int32_t* seq_len, int seq_stride,
                                   const int32_t* bias_tokens, const float* bias_values, const int32_t* bias_count,
                                   int bias_stride, int32_t* out, void* ws, size_t ws_bytes, int pdl, zl_stream_t stream) {
    ZL_CHECK_ARG(!ngram_penalty || ws_bytes >= zl_sample_processed_workspace_bytes(T, seq_stride));
    const SampleProc pr{ngram_penalty, seq, seq_len, seq_stride, bias_tokens, bias_values, bias_count, bias_stride,
                        static_cast<int2*>(ws), seq_stride > 0 ? ngram_table_size(seq_stride) : 0};
    return sample_launch(logits, T, V, params, row_task, counter, history, history_words, pr, out, pdl,
                         static_cast<cudaStream_t>(stream));
}

extern "C" int zl_sample_masked(const float* logits, int T, int V, const zl_sample_params_t* params,
                                const int32_t* row_task, const int32_t* counter, uint32_t* history, int history_words,
                                const float* ngram_penalty, int32_t* seq, int32_t* seq_len, int seq_stride,
                                const int32_t* bias_tokens, const float* bias_values, const int32_t* bias_count,
                                int bias_stride, const uint32_t* masks, int mask_words, const int32_t* mask_row,
                                int32_t* out, void* ws, size_t ws_bytes, int pdl, zl_stream_t stream) {
    ZL_CHECK_ARG(!ngram_penalty || ws_bytes >= zl_sample_processed_workspace_bytes(T, seq_stride));
    ZL_CHECK_ARG(masks);
    SampleProc pr{ngram_penalty, seq, seq_len, seq_stride, bias_tokens, bias_values, bias_count, bias_stride,
                  static_cast<int2*>(ws), seq_stride > 0 ? ngram_table_size(seq_stride) : 0};
    // mask row of task t: (t * 0 + mask_row[t]), or t when mask_row is NULL; no automaton moves
    pr.au.mask = masks;
    pr.au.words = mask_words;
    pr.au.state = const_cast<int32_t*>(mask_row);   // read only: au.next is NULL
    return sample_launch(logits, T, V, params, row_task, counter, history, history_words, pr, out, pdl,
                         static_cast<cudaStream_t>(stream));
}
