// sampling.cu -- the token sampler of the generate loop, on the device.
//
// The reference samples on the host from a copy of the logits (LLaMAGenerate.cu:112-166 builds a candidate array from n_vocab floats it
// has just memcpy'd out of the model output).  Here one 1024-thread block per sequence does the whole chain next to the logits, so that a
// generated token costs 4 bytes of PCIe traffic instead of n_vocab * 4:
//   repetition / frequency / presence penalties over the window of recent tokens      llm/src/Generate.cc:14-60
//   greedy arg-max when temp <= 0                                                      Generate.cc:62-70
//   otherwise top-k (partial sort, descending) -> [tail-free z = 1, typical p = 1: identity in the reference's defaults and not offered
//   here] -> top-p over the softmax of the survivors -> logits / temp -> softmax -> one draw             Generate.cc:72-136, 304-327
// The draw is an inverse-CDF lookup with a counter-based uniform (seed, draw index): reproducible without carrying generator state; the
// reference's std::discrete_distribution over std::mt19937 is not reproducible across standard libraries either.
//
// Selection of the k largest logits: three histogram passes (11 + 11 + 10 bits of the order-preserving key) find the key of the k-th
// largest, one ordered compaction pass gathers the candidates (ties at the threshold: lowest ids first), one bitonic sort orders them
// (logit descending, id ascending).  Everything after that is O(k) work on shared memory.
#include "../../include/tce_b200.h"
#include "common.cuh"
#include "kernels.h"
#include "kernels_attn.h"

namespace tce {

namespace {

constexpr int kSampleThreads = 1024;
constexpr int kMaxK = 1024;

TCE_DEVINL uint32_t order_key(float f) {  // larger float <=> larger key (NaN-free logits)
    const uint32_t b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

TCE_DEVINL float uniform01(unsigned long long seed, unsigned long long idx) {  // splitmix64 of (seed, idx) -> [0, 1)
    unsigned long long z = seed + 0x9E3779B97F4A7C15ull * (idx + 1ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z = z ^ (z >> 31);
    return (float)(z >> 40) * (1.0f / 16777216.0f);
}

struct SampleShared {
    unsigned hist[2048];
    unsigned long long cand[kMaxK];  // (order key << 32) | (0xFFFFFFFF - id): descending sort = logit descending, id ascending
    float p[kMaxK];
    unsigned warp_tot[2][32];
    unsigned prefix, need, base_gt, base_eq;
    int result, size;
    float q;  // probability of the excluded id (0: none, or not a candidate)
};

// block-wide exclusive scan of one flag per thread over a chunk; returns this thread's offset, `total` = chunk total
TCE_DEVINL unsigned block_flag_scan(bool flag, unsigned *warp_tot, unsigned &total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned bal = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) warp_tot[warp] = __popc(bal);
    __syncthreads();
    unsigned before = 0;
    total = 0;
#pragma unroll
    for (int w = 0; w < kSampleThreads / 32; w++) {
        const unsigned c = warp_tot[w];
        if (w < warp) before += c;
        total += c;
    }
    return before + __popc(bal & ((1u << lane) - 1u));
}

// penalties + selection of the chain for one sequence, on one kSampleThreads-thread block; returns the id on thread 0 (sh.result, sh.size
// and sh.p hold it for every thread after the call).  The window is the last W tokens of a sequence of `head` entries: entries below
// ring_head come from the history ring, entries from ring_head on from `tail` (the acceptance kernel's drafts; tail = nullptr: head ==
// ring_head).
// excl >= 0 (a draft): sh.q = its probability p[i*] when it is a candidate, else 0.  With q = 0 the id is the plain draw.  With q > 0 it
// is the replacement draw of speculative sampling: the same uniform u scaled to S = the sum of p[i] over i != i* (candidate order, fp32),
// and the first i != i* whose running sum over i != i* exceeds u * S (the last i != i* if none); -1 when S = 0 (nothing to replace with).
TCE_DEVINL int sample_chain(const SampleArgs &a, SampleShared &sh, int head, int ring_head, const int *tail, int excl = -1) {
    const int tid = threadIdx.x;
    float *logits = a.logits;
    const int V = a.n_vocab;

    // ---- window of recent tokens: the last `W` entries of the history ring (zeros before the first real token, as the reference's
    // last_n_tokens vector of n_ctx zeros, LLaMAGenerate.cu:43-44, 137-141) ----
    const int cap = a.hist_cap;
    int W = a.repeat_last_n < 0 ? cap : (a.repeat_last_n < cap ? a.repeat_last_n : cap);
    if (!a.hist) W = 0;
    auto window = [&](int j) -> int {  // j-th entry of the window, oldest first
        const int logical = head - W + j;  // index into the unbounded sequence; negative = initial zero
        return logical < 0 ? 0 : (logical >= ring_head ? tail[logical - ring_head] : a.hist[logical % cap]);
    };
    const bool pen = W > 0 && (a.repeat_penalty != 1.0f || a.frequency_penalty != 0.0f || a.presence_penalty != 0.0f);
    if (pen) {
        for (int j = tid; j < W; j += kSampleThreads) {
            const int tok = window(j);
            if (tok < 0 || tok >= V) continue;
            int count = 0;
            bool first = true;
            for (int i = 0; i < W; i++) {
                const bool same = window(i) == tok;
                count += same ? 1 : 0;
                if (same && i < j) first = false;
            }
            if (!first) continue;  // one update per distinct token, as the reference's per-candidate lookup does
            float l = logits[tok];
            // IEEE operations one by one, as the host code evaluates them (no fast-math division, no FMA contraction)
            if (a.repeat_penalty != 1.0f) l = (l <= 0.f) ? __fmul_rn(l, a.repeat_penalty) : __fdiv_rn(l, a.repeat_penalty);
            if (a.frequency_penalty != 0.0f || a.presence_penalty != 0.0f)
                l = __fsub_rn(l, __fadd_rn(__fmul_rn((float)count, a.frequency_penalty), a.presence_penalty));
            logits[tok] = l;
        }
        __syncthreads();
    }

    int K = a.top_k <= 0 ? V : (a.top_k < V ? a.top_k : V);
    if (K < 1) K = 1;
    const bool greedy = a.temp <= 0.f;
    if (greedy) K = 1;
    // (K > kMaxK with temp > 0 is rejected on the host)

    // ---- key of the K-th largest logit: radix select, most significant digit first ----
    if (tid == 0) {
        sh.prefix = 0u;
        sh.need = (unsigned)K;
    }
    const int shifts[3] = {21, 10, 0};
    const int bits[3] = {11, 11, 10};
    uint32_t known_mask = 0u;
#pragma unroll 1
    for (int pass = 0; pass < 3; pass++) {
        for (int i = tid; i < 2048; i += kSampleThreads) sh.hist[i] = 0u;
        __syncthreads();
        const uint32_t prefix = sh.prefix;
        const int sft = shifts[pass];
        const uint32_t dmask = (1u << bits[pass]) - 1u;
        for (int i = tid; i < V; i += kSampleThreads) {
            const uint32_t k = order_key(logits[i]);
            if ((k & known_mask) == prefix) atomicAdd(&sh.hist[(k >> sft) & dmask], 1u);
        }
        __syncthreads();
        if (tid == 0) {
            unsigned need = sh.need, acc = 0u;
            int d = (int)dmask;
            for (; d > 0; d--) {
                if (acc + sh.hist[d] >= need) break;
                acc += sh.hist[d];
            }
            sh.need = need - acc;  // how many of the elements that share the new prefix are still wanted
            sh.prefix = prefix | ((uint32_t)d << sft);
        }
        known_mask |= dmask << sft;
        __syncthreads();
    }
    const uint32_t T = sh.prefix;        // key of the K-th largest
    const unsigned need_eq = sh.need;    // how many elements with key == T belong to the top K (>= 1)
    const unsigned n_gt = (unsigned)K - need_eq;

    // ---- gather: everything above the threshold, then the `need_eq` lowest ids at the threshold ----
    if (tid == 0) {
        sh.base_gt = 0u;
        sh.base_eq = 0u;
    }
    __syncthreads();
#pragma unroll 1
    for (int c0 = 0; c0 < V; c0 += kSampleThreads) {
        const int i = c0 + tid;
        uint32_t k = 0u;
        bool gt = false, eq = false;
        if (i < V) {
            k = order_key(logits[i]);
            gt = k > T;
            eq = k == T;
        }
        unsigned tot_gt, tot_eq;
        const unsigned off_gt = block_flag_scan(gt, sh.warp_tot[0], tot_gt);
        const unsigned off_eq = block_flag_scan(eq, sh.warp_tot[1], tot_eq);
        const unsigned bg = sh.base_gt, be = sh.base_eq;
        const unsigned long long packed = ((unsigned long long)k << 32) | (unsigned long long)(0xFFFFFFFFu - (uint32_t)i);
        if (gt) sh.cand[bg + off_gt] = packed;
        if (eq && be + off_eq < need_eq) sh.cand[n_gt + be + off_eq] = packed;
        __syncthreads();
        if (tid == 0) {
            sh.base_gt = bg + tot_gt;
            sh.base_eq = be + tot_eq;
        }
        __syncthreads();
        if (sh.base_gt >= n_gt && sh.base_eq >= need_eq) break;  // uniform
    }

    // ---- order the K candidates: bitonic sort, descending, padded with zeros (below every real key) ----
    int n2 = 1;
    while (n2 < K) n2 <<= 1;
    for (int i = K + tid; i < n2; i += kSampleThreads) sh.cand[i] = 0ull;
    __syncthreads();
    for (int size = 2; size <= n2; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = tid; i < n2; i += kSampleThreads) {
                const int j = i ^ stride;
                if (j > i) {
                    const unsigned long long x = sh.cand[i], y = sh.cand[j];
                    const bool desc = (i & size) == 0;
                    if (desc ? (x < y) : (x > y)) {
                        sh.cand[i] = y;
                        sh.cand[j] = x;
                    }
                }
            }
            __syncthreads();
        }
    }
    auto cand_id = [&](int i) -> int { return (int)(0xFFFFFFFFu - (uint32_t)(sh.cand[i] & 0xFFFFFFFFull)); };

    if (tid == 0) {
        int size = K;
        int result;
        float u = 0.f;
        if (greedy) {
            result = cand_id(0);  // the largest logit, lowest id among equals (std::max_element keeps the first)
            size = 1;
            sh.p[0] = 1.f;
        } else {
            // sample_top_p (Generate.cc:304-327): softmax of the sorted survivors, keep the prefix before the running sum first exceeds p
            if (a.top_p < 1.0f) {
                const float max_l = logits[cand_id(0)];
                float cum = 0.f;
                for (int i = 0; i < size; i++) {
                    sh.p[i] = expf(__fsub_rn(logits[cand_id(i)], max_l));
                    cum = __fadd_rn(cum, sh.p[i]);
                }
                float run = 0.f;
                int last = size;
                for (int i = 0; i < size; i++) {
                    run = __fadd_rn(run, __fdiv_rn(sh.p[i], cum));
                    if (run > a.top_p && i >= 1) {  // min_keep = 1
                        last = i;
                        break;
                    }
                }
                size = last;
            }
            // sample_temperature + sample_token's softmax (Generate.cc:72-118)
            const float max_l = __fdiv_rn(logits[cand_id(0)], a.temp);
            float cum = 0.f;
            for (int i = 0; i < size; i++) {
                sh.p[i] = expf(__fsub_rn(__fdiv_rn(logits[cand_id(i)], a.temp), max_l));
                cum = __fadd_rn(cum, sh.p[i]);
            }
            for (int i = 0; i < size; i++) sh.p[i] = __fdiv_rn(sh.p[i], cum);
            u = uniform01(a.seed, a.draw_index + (a.hist_head ? (unsigned long long)head : 0ull));
            float run = 0.f;
            result = cand_id(size - 1);
            for (int i = 0; i < size; i++) {
                run += sh.p[i];
                if (u < run) {
                    result = cand_id(i);
                    break;
                }
            }
        }
        float q = 0.f;
        int ex = -1;
        if (excl >= 0) {
            for (int i = 0; i < size; i++) {
                if (cand_id(i) == excl) {
                    ex = i;
                    q = sh.p[i];
                    break;
                }
            }
        }
        if (q > 0.f) {  // greedy: the arg-max is the only candidate, so S = 0
            float S = 0.f;
            for (int i = 0; i < size; i++)
                if (i != ex) S = __fadd_rn(S, sh.p[i]);
            result = -1;
            if (S > 0.f) {
                const float t = __fmul_rn(u, S);
                float run = 0.f;
                for (int i = 0; i < size; i++) {
                    if (i == ex) continue;
                    run = __fadd_rn(run, sh.p[i]);
                    result = cand_id(i);
                    if (t < run) break;
                }
            }
        }
        sh.result = result;
        sh.size = size;
        sh.q = q;
    }
    __syncthreads();
    return sh.result;
}

// the whole chain for one sequence, then the publishing of its id
TCE_DEVINL void sample_one(const SampleArgs &a, SampleShared &sh) {
    const int tid = threadIdx.x;
    if (a.stop && *a.stop) return;  // the sequence has ended (EOS drawn earlier): leave every buffer as it is
    const int cap = a.hist_cap;
    const int head = a.hist_head ? *a.hist_head : 0;  // entries written so far
    const int result = sample_chain(a, sh, head, head, nullptr);
    auto cand_id = [&](int i) -> int { return (int)(0xFFFFFFFFu - (uint32_t)(sh.cand[i] & 0xFFFFFFFFull)); };
    if (tid == 0) {
        // ---- publish: the token, the next decode step's {token, position}, the history ring, the output list, the stop flag ----
        if (a.out_token) *a.out_token = result;
        if (a.tokpos) {
            a.tokpos[0] = result;
            a.tokpos[1] = a.tokpos[1] + 1;
        }
        if (a.hist && a.hist_head) {
            a.hist[head % cap] = result;
            *a.hist_head = head + 1;
        }
        if (a.out_list && a.out_count) {
            const int n = *a.out_count;
            if (n < a.out_cap) a.out_list[n] = result;
            *a.out_count = n + 1;
        }
        // stop at eos_id, at out_limit outputs, or when the next position would be pos_limit; a stopped batched row's request gets an
        // out-of-range position, so the batched step appends nothing more for it
        bool done = result == a.eos_id;
        if (a.out_limit > 0 && a.out_count && *a.out_count >= a.out_limit) done = true;
        if (a.pos_limit > 0 && a.tokpos && a.tokpos[1] >= a.pos_limit) done = true;
        if (a.stop && done) {
            *a.stop = 1;
            if (a.pos_limit > 0 && a.tokpos) a.tokpos[1] = a.pos_limit;
        }
    }
    __syncthreads();
    // optional: the candidate set and its final probabilities (tests)
    if (a.dbg_ids && a.dbg_probs && a.dbg_size) {
        const int size = sh.size;
        for (int i = tid; i < size; i += kSampleThreads) {
            a.dbg_ids[i] = cand_id(i);
            a.dbg_probs[i] = sh.p[i];
        }
        if (tid == 0) *a.dbg_size = size;
    }
}

// one row with its arguments as a kernel parameter (tce_sample, the single-sequence generate loop): the chain reads them from the constant
// bank, where sample_rows_kernel holds its row's in registers and runs the chain slower
__global__ void __launch_bounds__(kSampleThreads, 1) sample_kernel(SampleArgs a) {
    __shared__ SampleShared sh;
    sample_one(a, sh);
}

// one block per row of a batch, each with its own arguments (logits row, history ring, output list, control words, request triple)
__global__ void __launch_bounds__(kSampleThreads, 1) sample_rows_kernel(const SampleArgs *__restrict__ rows) {
    __shared__ SampleShared sh;
    sample_one(rows[blockIdx.x], sh);
}

// Acceptance of a speculative step (the rule stated at tce_spec_accept): block j runs the chain on logits row j with the window the
// one-token loop would have had after emitting drafts 0..j-1 (the ring, then drafts[<j]) and draft j (none for the last row) as the
// excluded id, and publishes {q_j, r_j}.  The last block to finish accepts drafts while a_j < q_j (or r_j = -1: no other candidate), emits
// them plus r_k of the first row k not accepted (of the last row when every draft was), cut at eos_id (inclusive) and at the budget, and
// appends the emitted ids to the history ring.  At temp <= 0, q_j is 1 when draft j is the arg-max and 0 otherwise: the greedy rule.
__global__ void __launch_bounds__(kSampleThreads, 1) accept_kernel(const __grid_constant__ AcceptArgs a) {
    __shared__ SampleShared sh;
    __shared__ int drafts[kMaxDrafts];
    __shared__ int is_last;
    const int tid = threadIdx.x, j = blockIdx.x;
    if (tid < kMaxDrafts) drafts[tid] = a.drafts[tid];
    const int ring_head = *a.chain.hist_head;
    __syncthreads();
    SampleArgs s = a.chain;
    s.logits += (size_t)j * a.ld;
    const int r = sample_chain(s, sh, ring_head + j, ring_head, drafts, j < a.rows - 1 ? drafts[j] : -1);
    if (tid == 0) {
        a.repl[j] = r;
        a.q[j] = sh.q;
        __threadfence();
        const unsigned prev = atomicAdd(a.arrive, 1u);
        is_last = prev == (unsigned)(a.rows - 1);
    }
    __syncthreads();
    if (!is_last || tid != 0) return;
    __threadfence();
    *a.arrive = 0u;  // re-armed for the next step
    const volatile int *repl = a.repl;
    const volatile float *q = a.q;
    // row j's acceptance uniform has the index of its draw uniform, u_j, in the second counter stream
    const unsigned long long idx0 = a.chain.draw_index + (unsigned long long)ring_head;
    int k = 0;
    while (k < a.rows - 1 && (repl[k] < 0 || uniform01(a.chain.seed ^ TCE_SPEC_ACCEPT_STREAM, idx0 + k) < q[k])) k++;
    int n = 0, stop = 0;
    const int cap = a.chain.hist_cap;
    for (int i = 0; i <= k && n < a.budget; i++) {
        const int t = i < k ? drafts[i] : repl[k];
        a.result[3 + n] = t;
        a.chain.hist[(ring_head + n) % cap] = t;
        n++;
        if (t == a.eos_id) {
            stop = 1;
            break;
        }
    }
    *a.chain.hist_head = ring_head + n;
    a.result[0] = n;
    a.result[1] = stop;
    a.result[2] = k < n ? k : n;  // emitted ids that were drafts
}

}  // namespace

cudaError_t launch_accept(const AcceptArgs &a, cudaStream_t stream) {
    if (a.rows < 1 || a.rows > kMaxDrafts + 1 || !a.chain.logits || !a.chain.hist || !a.chain.hist_head || a.chain.hist_cap < 1 || !a.repl || !a.q ||
        !a.arrive || !a.result)
        return cudaErrorInvalidValue;
    if (!sampling_supported(a.chain.temp, a.chain.top_k, a.chain.n_vocab)) return cudaErrorNotSupported;
    accept_kernel<<<a.rows, kSampleThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_sample(const SampleArgs &a, cudaStream_t stream) {
    sample_kernel<<<1, kSampleThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_sample_rows(const SampleArgs *rows_dev, int rows, cudaStream_t stream) {
    if (!rows_dev || rows < 1) return cudaErrorInvalidValue;
    sample_rows_kernel<<<rows, kSampleThreads, 0, stream>>>(rows_dev);
    return cudaGetLastError();
}

SampleArgs sample_args(const tce_sampling &sc, float *logits, int n_vocab) {
    SampleArgs a{};
    a.logits = logits;
    a.n_vocab = n_vocab;
    a.top_k = sc.top_k;
    a.top_p = sc.top_p;
    a.temp = sc.temp;
    a.repeat_penalty = sc.repeat_penalty;
    a.frequency_penalty = sc.frequency_penalty;
    a.presence_penalty = sc.presence_penalty;
    a.repeat_last_n = sc.repeat_last_n;
    a.seed = sc.seed;
    a.draw_index = 0;
    return a;
}

bool sampling_supported(float temp, int top_k, int n_vocab) { return !(temp > 0.f && (top_k <= 0 || top_k > kMaxK) && n_vocab > kMaxK); }

}  // namespace tce
