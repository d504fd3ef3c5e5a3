// Qwen3-TTS in-graph sampler for sm_90a (SURVEY.md section 8f row N1): `sampleToken`
// (Sources/MLXAudioTTS/Models/Qwen3TTS/Qwen3TTS.swift:1003-1118) as ONE kernel, one CTA per row, vocabulary <= 4096 (the talker's
// codec head has 3072 entries, the code predictor's heads 2048).
// Checked against oracle/qwen3_tts.py (filter_logits / sample_token): tests/test_gpu_qwen3_sampler.py.  The kernel is compiled in
// qwen3_sampler.cu only; q3s::launch runs it per frame for the talker / code-predictor loop (llama.cu, b2a_qwen3_talker) and for
// the test hook.
//
// Order of operations, as the reference: suppress (-inf) -> repetition penalty over the UNIQUE tokens generated so far (a per-row
// bitmap here, updated by the kernel itself) -> greedy argmax if temperature <= 0 -> remember the EOS logit -> top-k on the
// un-tempered logits -> top-p on softmax(filtered) with the ascending-cumulative rule `cum > 1 - top_p` -> min-p relative to the
// largest surviving logit -> EOS logit written back -> categorical(filtered / temperature).
// The row is sorted once (bitonic, (logit desc, index asc), 4096 slots in shared memory); top-k is a prefix of the sorted row,
// the ascending cumulative sum is a suffix sum of it, and the categorical draw is an inverse-CDF walk over it, so no second
// pass over the vocabulary is needed.  Ties at the top-k boundary go to the lower index (the reference's argPartition leaves
// them implementation-defined).
// Fast path (0 < top_k <= 64 < V, the shipped default top_k = 50): the full sort cost 70 us per launch, 16 launches per frame = a quarter
// of the frame.  Instead every warp sorts its 128 slots in registers (shuffle bitonic network, 4 elements per lane), keeps its best 64,
// and five pairwise merge rounds (bitonic merge of two sorted 64-lists, again warp-local) leave the row's best 64 in exact
// (logit desc, index asc) order; top-p / min-p / EOS / the draw then run in ONE warp over <= 65 candidates.  The draw is Gumbel-max
// (argmax of logit / T - log(-log u_token)), the same categorical distribution without a prefix sum.
#pragma once
#include "common.cuh"

#include <cmath>

namespace b2a {
namespace q3s {

constexpr int THREADS = 1024, SLOTS = 4096, PER = SLOTS / THREADS;

struct Args {
    const float* logits;      // [B, V]
    int V;
    float temperature, top_p, min_p, rep_penalty;
    int top_k;
    int eos;                  // < 0: none
    int suppress_lo, suppress_hi;   // [lo, hi) is set to -inf except eos; lo >= hi: nothing
    unsigned* seen;           // nullable [B, ceil(V / 32)]: tokens generated so far (repetition penalty); updated when track != 0
    int track;
    unsigned long long seed;
    int step;                 // draw index; with step_ptr != null the draw index of row b is step_ptr[b] * step_mul + step
    const int* step_ptr;      // nullable [B] (a device counter, so that one captured CUDA graph can be replayed every frame)
    int step_mul;
    int* tokens;              // out: token of row b at tokens[b * tokens_stride]
    int tokens_stride;        // 0 or 1: dense [B]
    float* filtered;          // nullable [B, V] out: the logits handed to categorical (parity hook); -inf = removed
};

// One launch of sample_kernel (qwen3_sampler.cu): one CTA per row of a.logits, B rows, on stream s
void launch(const Args& a, int B, cudaStream_t s);

}  // namespace q3s
}  // namespace b2a
