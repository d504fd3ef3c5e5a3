// The Qwen3-TTS in-graph sampler kernel (qwen3_sampler.cuh), its launch and its test entry; the product caller is the talker loop
// in llama.cu.
#include "qwen3_sampler.cuh"

namespace b2a {
namespace q3s {

__device__ __forceinline__ float uniform01(unsigned long long seed, unsigned long long a, unsigned long long b) {
    unsigned long long z = seed + 0x9E3779B97F4A7C15ull * (a * 1000003ull + b * 131ull + 1ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    return (float)(z >> 40) * (1.0f / 16777216.0f);
}
__device__ __forceinline__ bool before(float ka, int ia, float kb, int ib) { return ka > kb || (ka == kb && ia < ib); }

// inclusive scan over the 4096 slots: thread t owns slots [4t, 4t + 4); `rev` scans from the top slot down (suffix sums).
// v[] in: the slot values, out: the inclusive (pre/suf)fix sums.  Returns the total.
static __device__ float block_scan(float v[PER], bool rev, float* wsum /*[32]*/) {
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    float loc = 0.f;
    if (!rev) { for (int i = 0; i < PER; ++i) { loc += v[i]; v[i] = loc; } }
    else { for (int i = PER - 1; i >= 0; --i) { loc += v[i]; v[i] = loc; } }
    // scan of the per-thread totals, in thread order (forward) or reverse thread order
    float inc = loc;
    for (int o = 1; o < 32; o <<= 1) {
        const float n = rev ? __shfl_down_sync(0xffffffffu, inc, o) : __shfl_up_sync(0xffffffffu, inc, o);
        if (rev ? (lane + o < 32) : (lane >= o)) inc += n;
    }
    __syncthreads();
    if (lane == (rev ? 0 : 31)) wsum[warp] = inc;          // the warp's total
    __syncthreads();
    float base = 0.f, total = 0.f;
    for (int w = 0; w < 32; ++w) {
        total += wsum[w];
        if (rev ? (w > warp) : (w < warp)) base += wsum[w];
    }
    const float excl = base + inc - loc;                     // sum of everything scanned before this thread
    for (int i = 0; i < PER; ++i) v[i] += excl;
    return total;
}


// ---- warp-local bitonic machinery: 128 elements per warp, element e = lane * 4 + r ------------------------------------------------
struct KV { float k; int i; };
__device__ __forceinline__ void cx_reg(KV& a, KV& b, bool first_low) {       // a at the lower position; first_low: `before` element goes low
    const bool a_before = before(a.k, a.i, b.k, b.i);
    if (a_before != first_low) { const KV t = a; a = b; b = t; }
}
// one compare-exchange stage (k, j) of the bitonic network over the warp's 128 elements
__device__ __forceinline__ void bitonic_stage(KV v[4], int k, int j, int lane) {
    if (j >= 4) {
        const int lm = j >> 2;
        const bool lower = (lane & lm) == 0;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int e = lane * 4 + r;
            const float ok = __shfl_xor_sync(0xffffffffu, v[r].k, lm);
            const int oi = __shfl_xor_sync(0xffffffffu, v[r].i, lm);
            const bool want_first = ((e & k) == 0) == lower;
            const bool mine_before = before(v[r].k, v[r].i, ok, oi);
            if (mine_before != want_first) { v[r].k = ok; v[r].i = oi; }
        }
    } else if (j == 2) {
        const bool fl = ((lane * 4) & k) == 0;
        cx_reg(v[0], v[2], fl);
        cx_reg(v[1], v[3], fl);
    } else {
        cx_reg(v[0], v[1], ((lane * 4) & k) == 0);
        cx_reg(v[2], v[3], ((lane * 4 + 2) & k) == 0);
    }
}

static __global__ void __launch_bounds__(THREADS)
sample_kernel(Args a) {
    __shared__ float key[SLOTS];
    __shared__ int idx[SLOTS];
    __shared__ float wsum[32];
    __shared__ float s_f[32];
    __shared__ int s_i[32];
    __shared__ float s_eos;
    __shared__ int s_tok;
    const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const float* lg = a.logits + (long long)b * a.V;
    const int words = (a.V + 31) / 32;
    const unsigned* seen = a.seen ? a.seen + (long long)b * words : nullptr;

    // 1. load with suppression and repetition penalty; pad with -inf
    for (int i = t; i < SLOTS; i += THREADS) {
        float v = -INFINITY;
        if (i < a.V) {
            v = lg[i];
            if (i >= a.suppress_lo && i < a.suppress_hi && i != a.eos) v = -INFINITY;
            if (seen && a.rep_penalty != 1.0f && ((seen[i >> 5] >> (i & 31)) & 1u)) v = v < 0.f ? v * a.rep_penalty : v / a.rep_penalty;
        }
        key[i] = v;
        idx[i] = i < a.V ? i : 0x7fffffff;
    }
    __syncthreads();

    if (a.temperature <= 0.f) {
        // 2. greedy: argmax, lowest index wins ties
        float best = -INFINITY;
        int bi = 0x7fffffff;
        for (int i = t; i < a.V; i += THREADS)
            if (before(key[i], i, best, bi)) { best = key[i]; bi = i; }
        for (int o = 16; o; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (before(ov, oi, best, bi)) { best = ov; bi = oi; }
        }
        if (lane == 0) { s_f[warp] = best; s_i[warp] = bi; }
        __syncthreads();
        if (t == 0) {
            for (int w = 1; w < 32; ++w)
                if (before(s_f[w], s_i[w], best, bi)) { best = s_f[w]; bi = s_i[w]; }
            s_tok = bi == 0x7fffffff ? 0 : bi;
        }
        __syncthreads();
        if (a.filtered)
            for (int i = t; i < a.V; i += THREADS) a.filtered[(long long)b * a.V + i] = key[i];
    } else if (a.top_k > 0 && a.top_k <= 64 && a.top_k < a.V) {
        // ---- fast path: the row's best 64 by a warp tournament, the tail in one warp ----
        float* Lk = reinterpret_cast<float*>(idx);               // [32 warps][64] keys   (idx[] is not needed here: a slot's index is its position)
        int* Li = idx + SLOTS / 2;                               // [32 warps][64] indices
        KV v[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int i = warp * 128 + lane * 4 + r;
            v[r].k = key[i];
            v[r].i = i < a.V ? i : 0x7fffffff;
        }
        __syncthreads();                                         // every warp has read idx-independent data; idx[] may now be overwritten
        for (int k = 2; k <= 128; k <<= 1)
            for (int j = k >> 1; j > 0; j >>= 1) bitonic_stage(v, k, j, lane);
        if (lane < 16) {
#pragma unroll
            for (int r = 0; r < 4; ++r) { Lk[warp * 64 + lane * 4 + r] = v[r].k; Li[warp * 64 + lane * 4 + r] = v[r].i; }
        }
        __syncthreads();
        for (int s = 1; s < 32; s <<= 1) {
            const bool active = (warp % (2 * s)) == 0;
            if (active) {
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    const int e = lane * 4 + r;
                    const int src = e < 64 ? warp * 64 + e : (warp + s) * 64 + (127 - e);     // the partner's list reversed: a bitonic sequence
                    v[r].k = Lk[src]; v[r].i = Li[src];
                }
                for (int j = 64; j > 0; j >>= 1) bitonic_stage(v, 128, j, lane);
            }
            __syncthreads();
            if (active && lane < 16) {
#pragma unroll
                for (int r = 0; r < 4; ++r) { Lk[warp * 64 + lane * 4 + r] = v[r].k; Li[warp * 64 + lane * 4 + r] = v[r].i; }
            }
            __syncthreads();
        }
        if (a.filtered)
            for (int i = t; i < a.V; i += THREADS) a.filtered[(long long)b * a.V + i] = -INFINITY;
        __syncthreads();
        if (warp == 0) {
            // lane owns sorted slots 2 * lane, 2 * lane + 1
            const bool has_eos = a.eos >= 0 && a.eos < a.V;
            const float eos_logit = has_eos ? key[a.eos] : -INFINITY;
            float kk[2];
            int ii[2];
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int sl = lane * 2 + r;
                kk[r] = sl < a.top_k ? Lk[sl] : -INFINITY;      // top-k: a prefix of the sorted row
                ii[r] = Li[sl];
            }
            const float top = __shfl_sync(0xffffffffu, kk[0], 0);
            if (a.top_p > 0.f && a.top_p < 1.0f) {               // keep where the ascending cumulative probability exceeds 1 - top_p
                const float e0 = __expf(kk[0] - top), e1 = __expf(kk[1] - top);
                float suf = e0 + e1;                             // suffix sums over lanes (this lane's two slots and everything after)
                for (int o = 1; o < 32; o <<= 1) {
                    const float n = __shfl_down_sync(0xffffffffu, suf, o);
                    if (lane + o < 32) suf += n;
                }
                const float Z = __shfl_sync(0xffffffffu, suf, 0);
                const float thr = (1.0f - a.top_p) * Z;
                const float v0 = suf, v1 = suf - e0;             // slot 2 * lane sees both of its lane's terms, slot 2 * lane + 1 only its own
                if (!(v0 > thr)) kk[0] = -INFINITY;
                if (!(v1 > thr)) kk[1] = -INFINITY;
            }
            if (a.min_p > 0.f) {
                const float cut = top + logf(a.min_p);
                if (kk[0] < cut) kk[0] = -INFINITY;
                if (kk[1] < cut) kk[1] = -INFINITY;
            }
            // the EOS logit goes back in: in place if it is one of the 64, as an extra candidate otherwise
            bool eos_here = false;
#pragma unroll
            for (int r = 0; r < 2; ++r)
                if (has_eos && ii[r] == a.eos) { kk[r] = eos_logit; eos_here = true; }
            const bool eos_listed = __any_sync(0xffffffffu, eos_here);
            if (a.filtered) {
#pragma unroll
                for (int r = 0; r < 2; ++r)
                    if (ii[r] < a.V && kk[r] > -INFINITY) a.filtered[(long long)b * a.V + ii[r]] = kk[r];
                if (has_eos && !eos_listed && lane == 0) a.filtered[(long long)b * a.V + a.eos] = eos_logit;
            }
            // categorical(filtered / temperature) by Gumbel-max: argmax of logit / T - log(-log u), one uniform per (row, draw, token)
            const unsigned long long draw = a.step_ptr ? (unsigned long long)a.step_ptr[b] * (unsigned long long)a.step_mul + (unsigned long long)a.step
                                                       : (unsigned long long)a.step;
            const float inv_t = 1.0f / a.temperature;
            auto score = [&](float logit, int tok) {
                if (!(logit > -INFINITY)) return -INFINITY;
                const float u = uniform01(a.seed + 0x632BE59BD9B4E019ull * (unsigned long long)(tok + 1), (unsigned long long)b, draw);
                return logit * inv_t - __logf(-__logf(fmaxf(u, 1e-12f)));
            };
            float best = score(kk[0], ii[0]);
            int bi = ii[0];
            { const float s1 = score(kk[1], ii[1]); if (before(s1, ii[1], best, bi)) { best = s1; bi = ii[1]; } }
            if (has_eos && !eos_listed && lane == 0) { const float se = score(eos_logit, a.eos); if (before(se, a.eos, best, bi)) { best = se; bi = a.eos; } }
            for (int o = 16; o; o >>= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, best, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (before(ov, oi, best, bi)) { best = ov; bi = oi; }
            }
            if (lane == 0) s_tok = (bi >= 0 && bi < a.V) ? bi : 0;
        }
        __syncthreads();
    } else {
        if (t == 0) s_eos = (a.eos >= 0 && a.eos < a.V) ? key[a.eos] : 0.f;
        __syncthreads();
        // 3. bitonic sort, `before` order
        for (int k = 2; k <= SLOTS; k <<= 1)
            for (int j = k >> 1; j > 0; j >>= 1) {
                for (int i = t; i < SLOTS; i += THREADS) {
                    const int p = i ^ j;
                    if (p > i) {
                        const float ka = key[i], kb = key[p];
                        const int ia = idx[i], ib = idx[p];
                        const bool asc = (i & k) == 0;
                        const bool sw = asc ? before(kb, ib, ka, ia) : before(ka, ia, kb, ib);
                        if (sw) { key[i] = kb; key[p] = ka; idx[i] = ib; idx[p] = ia; }
                    }
                }
                __syncthreads();
            }
        // 4. top-k: a prefix of the sorted row
        if (a.top_k > 0 && a.top_k < a.V)
            for (int i = t; i < SLOTS; i += THREADS)
                if (i >= a.top_k) key[i] = -INFINITY;
        __syncthreads();
        const float top = key[0];
        float v[PER];
        // 5. top-p: keep where the ascending cumulative probability exceeds 1 - top_p  (suffix sums of the descending row)
        if (a.top_p > 0.f && a.top_p < 1.0f) {
            float e[PER];
            for (int i = 0; i < PER; ++i) { e[i] = __expf(key[t * PER + i] - top); v[i] = e[i]; }
            const float Z = block_scan(v, true, wsum);
            const float thr = (1.0f - a.top_p) * Z;
            for (int i = 0; i < PER; ++i)
                if (!(v[i] > thr)) key[t * PER + i] = -INFINITY;
            __syncthreads();
        }
        // 6. min-p relative to the largest surviving logit (the top of the row always survives top-p)
        if (a.min_p > 0.f) {
            const float cut = top + logf(a.min_p);
            for (int i = t; i < SLOTS; i += THREADS)
                if (key[i] < cut) key[i] = -INFINITY;
            __syncthreads();
        }
        // 7. the EOS logit goes back in
        if (a.eos >= 0 && a.eos < a.V)
            for (int i = t; i < SLOTS; i += THREADS)
                if (idx[i] == a.eos) key[i] = s_eos;
        __syncthreads();
        if (a.filtered) {
            for (int i = t; i < SLOTS; i += THREADS)
                if (idx[i] < a.V) a.filtered[(long long)b * a.V + idx[i]] = key[i];
        }
        // 8. categorical(filtered / temperature): inverse CDF over the row
        const float m = fmaxf(top, (a.eos >= 0 && a.eos < a.V) ? s_eos : -INFINITY);
        const float inv_t = 1.0f / a.temperature;
        float p[PER];
        for (int i = 0; i < PER; ++i) { p[i] = __expf((key[t * PER + i] - m) * inv_t); v[i] = p[i]; }
        const float Z = block_scan(v, false, wsum);
        const unsigned long long draw = a.step_ptr ? (unsigned long long)a.step_ptr[b] * (unsigned long long)a.step_mul + (unsigned long long)a.step
                                                   : (unsigned long long)a.step;
        const float r = uniform01(a.seed, (unsigned long long)b, draw) * Z;
        // first slot whose inclusive prefix exceeds r (slots with p == 0 never qualify); fall back to the last slot with p > 0
        int cand = 0x7fffffff, lastpos = -1;
        for (int i = 0; i < PER; ++i) {
            if (p[i] > 0.f) {
                lastpos = t * PER + i;
                if (v[i] > r && cand == 0x7fffffff) cand = t * PER + i;
            }
        }
        for (int o = 16; o; o >>= 1) {
            cand = min(cand, __shfl_xor_sync(0xffffffffu, cand, o));
            lastpos = max(lastpos, __shfl_xor_sync(0xffffffffu, lastpos, o));
        }
        if (lane == 0) { s_i[warp] = cand; s_f[warp] = (float)lastpos; }
        __syncthreads();
        if (t == 0) {
            int c = 0x7fffffff, lp = -1;
            for (int w = 0; w < 32; ++w) { c = min(c, s_i[w]); lp = max(lp, (int)s_f[w]); }
            const int slot = c != 0x7fffffff ? c : max(lp, 0);
            s_tok = idx[slot] < a.V ? idx[slot] : 0;
        }
        __syncthreads();
    }
    if (t == 0) {
        const int tok = s_tok;
        a.tokens[(long long)b * (a.tokens_stride > 0 ? a.tokens_stride : 1)] = tok;
        if (a.seen && a.track) atomicOr(&a.seen[(long long)b * words + (tok >> 5)], 1u << (tok & 31));
    }
}

void launch(const Args& a, int B, cudaStream_t s) {
    sample_kernel<<<B, THREADS, 0, s>>>(a);
    count_launch();
}

}  // namespace q3s
}  // namespace b2a

using namespace b2a;

extern "C" {

// Test entry (tests/test_gpu_qwen3_sampler.py): HOST logits [B, V], HOST seen bitmap [B, ceil(V/32)] (nullable, in/out when
// track != 0), tokens_out [B], filtered_out [B, V] (nullable).  One launch of q3s::sample_kernel on device 0.
int32_t b2a_qwen3_sample_test(const float* logits, int32_t B, int32_t V, float temperature, float top_p, int32_t top_k, float min_p,
                              float repetition_penalty, int32_t eos, int32_t suppress_lo, int32_t suppress_hi, uint32_t* seen, int32_t track,
                              uint64_t seed, int32_t step, int32_t* tokens_out, float* filtered_out) {
    return guarded([&] {
        B2A_CHECK(logits && tokens_out && B >= 1 && V >= 1 && V <= q3s::SLOTS, B2A_ERR_INVALID_INPUT, "b2a_qwen3_sample_test: bad argument (vocabulary <= 4096)");
        require_device(0);
        const int words = (V + 31) / 32;
        DBuf<float> dl, df;
        DBuf<unsigned> ds;
        DBuf<int> dt;
        dl.upload(logits, (size_t)B * V);
        dt.alloc(B);
        q3s::Args a{};
        a.logits = dl.p; a.V = V; a.temperature = temperature; a.top_p = top_p; a.top_k = top_k; a.min_p = min_p; a.rep_penalty = repetition_penalty;
        a.eos = eos; a.suppress_lo = suppress_lo; a.suppress_hi = suppress_hi; a.track = track; a.seed = seed; a.step = step; a.tokens = dt.p;
        if (seen) { ds.upload(seen, (size_t)B * words); a.seen = ds.p; }
        if (filtered_out) { df.alloc((size_t)B * V); a.filtered = df.p; }
        B2A_CUDA(cudaDeviceSynchronize());
        q3s::launch(a, B, 0);
        B2A_CUDA(cudaGetLastError());
        B2A_CUDA(cudaDeviceSynchronize());
        B2A_CUDA(cudaMemcpy(tokens_out, dt.p, (size_t)B * sizeof(int), cudaMemcpyDeviceToHost));
        if (seen) B2A_CUDA(cudaMemcpy(seen, ds.p, (size_t)B * words * sizeof(unsigned), cudaMemcpyDeviceToHost));
        if (filtered_out) B2A_CUDA(cudaMemcpy(filtered_out, df.p, (size_t)B * V * sizeof(float), cudaMemcpyDeviceToHost));
    });
}

}  // extern "C"
