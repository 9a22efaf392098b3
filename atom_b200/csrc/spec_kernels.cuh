// spec_kernels.cuh -- speculative decoding's per-step bookkeeping on the device: commit the tokens a verify step accepted to each
// sequence's token history and propose the next step's drafts by prompt lookup (atom_spec_commit_propose, include/atom_b200.h;
// DESIGN section 5.8).
//
// One CTA per sequence.  Thread 0 commits (at most SPEC_MAX_DRAFT + 1 tokens, a short serial loop); then every thread scores
// the match ends e of its share of the history against the history's tail, and one 64-bit shared maximum of (match length,
// e) picks the longest n-gram and, among its matches, the latest.  Integers only: the result is reproducible on the host.
#pragma once
#include "ptx_sm90.cuh"

namespace atom {

constexpr int SPEC_THREADS = 256;
constexpr int SPEC_MAX_DRAFT = 7;                  // drafts per sequence: a verify step carries at most 8 tokens
constexpr int SPEC_MAX_NGRAM = 16;

struct SpecArgs {
  const int32_t* tok;                              // [rows]: the sampler's tokens
  const int32_t* cand;                             // [rows]: the candidate each row was given (-1: none)
  const int32_t* row_indptr;                       // [B + 1]
  const int32_t* slots;                            // [B]: history slot of each sequence
  int32_t* hist;                                   // [nslots][cap]
  int32_t* hist_len;                               // [nslots]
  int nslots, cap, k, nmin, nmax;
  int32_t* out;                                    // [B][2k + 3]: emitted, draft_len, tokens [k + 1], drafts [k]
};

__global__ void __launch_bounds__(SPEC_THREADS) spec_commit_propose_kernel(const SpecArgs a, int pdl) {
  __shared__ int32_t tail[SPEC_MAX_NGRAM];
  __shared__ int s_len;
  __shared__ unsigned long long s_best;
  const int i = blockIdx.x, tid = threadIdx.x, W = 2 * a.k + 3;
  if (pdl) { griddep_launch_dependents(); griddep_wait(); }
  int32_t* o = a.out + (long long)i * W;
  const int slot = a.slots[i];
  if (slot < 0 || slot >= a.nslots) {              // no history: nothing committed, nothing proposed
    for (int j = tid; j < W; j += SPEC_THREADS) o[j] = j < 2 ? 0 : -1;
    return;
  }
  int32_t* h = a.hist + (long long)slot * a.cap;
  if (tid == 0) {
    // commit: m = the first row whose candidate is missing or was not drawn; tokens 0 .. m are emitted
    const int r0 = a.row_indptr[i], last = min(a.row_indptr[i + 1] - r0, a.k + 1) - 1;
    int m = 0, L = a.hist_len[slot];
    while (m < last && a.cand[r0 + m] >= 0 && a.tok[r0 + m] == a.cand[r0 + m]) ++m;
    const int e = last < 0 ? 0 : m + 1;
    for (int j = 0; j <= a.k; ++j) {
      const int32_t t = j < e ? a.tok[r0 + j] : -1;
      o[2 + j] = t;
      if (j < e && L < a.cap) h[L++] = t;          // never past cap
    }
    o[0] = e;
    a.hist_len[slot] = L;
    s_len = L;
    s_best = 0;
  }
  __syncthreads();
  const int L = s_len;
  if (tid < a.nmax) tail[tid] = tid < L ? h[L - 1 - tid] : -1;
  __syncthreads();
  // propose: a match of length n ends at e (exclusive) when h[e - n, e) == h[L - n, L); e <= L - 1 leaves one token to draft
  // and keeps the tail itself out.  c(e) = the longest such n, capped at nmax.
  unsigned long long best = 0;
  for (int e = a.nmin + tid; e <= L - 1; e += SPEC_THREADS) {
    int c = 0;
    while (c < a.nmax && c < e && h[e - 1 - c] == tail[c]) ++c;
    if (c >= a.nmin) best = max(best, ((unsigned long long)c << 32) | (unsigned)e);
  }
#pragma unroll
  for (int off = 16; off; off >>= 1) best = max(best, __shfl_xor_sync(0xFFFFFFFFu, best, off));
  if ((tid & 31) == 0 && best) atomicMax(&s_best, best);
  __syncthreads();
  const unsigned long long b = s_best;
  const int e = (int)(b & 0xFFFFFFFFull), dl = b ? min(a.k, L - e) : 0;
  for (int j = tid; j < a.k; j += SPEC_THREADS) o[a.k + 3 + j] = j < dl ? h[e + j] : -1;
  if (tid == 0) o[1] = dl;
}

}  // namespace atom
