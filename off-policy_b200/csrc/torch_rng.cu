// torch's CPU generator (the mt19937 behind torch.manual_seed, uniform_ and normal_) continued on the device, so that the actor-critic
// learners' per-update noise draws need no host work: the draws of one torch call are one fill, written straight into the learner's
// noise layout.
//
// torch's engine: MT19937 seeded like NumPy's (state[0] = seed mod 2^32, init_genrand), a read of the next word first decrements `left`
// and twists all 624 words when it reaches 0 (`next` restarts at 0).  So the next word is key[625 - left], a twist coming first when
// that index is 624.  A float uniform_ reads one word per value: (word & 0xFFFFFF) * 2^-24.  normal_ of a contiguous float tensor of
// n >= 16 values fills n uniforms, turns each block of 16 into 16 normals with a Box-Muller pairing element j with j + 8, and, when
// 16 does not divide n, draws 16 fresh uniforms and recomputes the last 16 values from them.
//
// A fill is two launches: k_trng_twist (one CTA: the only serial part, copies the words the fill consumes into a scratch area,
// twisting as often as it needs and leaving key / left / next in device memory, so that graph replays advance the stream), then
// k_trng_fill (grid-wide: tempers, transforms, scatters every value).
#include <math.h>
#include <string.h>

#include "mx_internal.h"
#include "mx_mt19937.cuh"

#define TR_LEFT MT_N          // state words: key[624], left, next
#define TR_NEXT (MT_N + 1)

__global__ void __launch_bounds__(256) k_trng_twist(uint32_t* st, uint32_t* words, int n) {
  __shared__ uint32_t key[MT_N];
  const int tid = threadIdx.x;
  for (int i = tid; i < MT_N; i += blockDim.x) key[i] = st[i];
  int p = MT_N + 1 - (int)st[TR_LEFT];
  __syncthreads();
  int out = 0;
  bool twisted = false;
  while (true) {
    const int take = mx_imin(MT_N - p, n - out);
    for (int i = tid; i < take; i += blockDim.x) words[out + i] = key[p + i];
    out += take;
    p += take;
    if (out == n) break;
    mt_twist_cta(key);          // its first barrier orders the reads above before the words are rewritten
    twisted = true;
    p = 0;
  }
  if (twisted)
    for (int i = tid; i < MT_N; i += blockDim.x) st[i] = key[i];
  if (tid == 0) {
    st[TR_LEFT] = (uint32_t)(MT_N + 1 - p);
    st[TR_NEXT] = (uint32_t)p;
  }
}

struct TrngFillArgs {
  const uint32_t* words;      // the fill's words in stream order
  int n;                      // values (T * rows_n * rows_b * cols)
  int kind;
  float std;
  int rows_b, rows, cols;     // rows = rows_n * rows_b
  float* dst;
  long long ld_t, ld_n, ld_b;
};

MX_DEVINL float trng_uniform(uint32_t w) { return (float)(mt_temper(w) & 0xFFFFFFu) * 5.9604644775390625e-08f; }

__global__ void __launch_bounds__(256) k_trng_fill(TrngFillArgs a) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
    float v;
    if (a.kind == MX_TRNG_NORMAL) {
      int base = i & ~15, j = i & 15;
      if ((a.n & 15) && i >= a.n - 16) { base = a.n; j = i - (a.n - 16); }     // the tail block, recomputed from 16 fresh words
      const int k = j & 7;
      const float u1 = 1.0f - trng_uniform(a.words[base + k]);
      const float u2 = trng_uniform(a.words[base + k + 8]);
      const float r = sqrtf(-2.0f * logf(u1));
      const float th = 6.28318548f * u2;                                          // float(2 pi) * u2
      v = (j < 8 ? r * cosf(th) : r * sinf(th)) * a.std;
    } else {
      v = trng_uniform(a.words[i]);
      if (a.kind == MX_TRNG_GUMBEL) v = -logf(-logf(v + 1e-20f) + 1e-20f);      // sample_gumbel, utils/util.py:127-130
    }
    const int c = i % a.cols, r = (i / a.cols) % a.rows, t = i / (a.cols * a.rows);
    a.dst[t * a.ld_t + (r / a.rows_b) * a.ld_n + (r % a.rows_b) * a.ld_b + c] = v;
  }
}

extern "C" int64_t mx_trng_words(const mx_trng_draw* f) {
  if (!f) { mx_set_error("mx_trng_fill: null fill"); return -1; }
  if (f->kind < MX_TRNG_UNIFORM || f->kind > MX_TRNG_NORMAL) { mx_set_error("mx_trng_fill: unknown kind %d", f->kind); return -1; }
  if (f->T <= 0 || f->rows_n <= 0 || f->rows_b <= 0 || f->cols <= 0) {
    mx_set_error("mx_trng_fill: empty or negative source shape (%d, %d*%d, %d)", f->T, f->rows_n, f->rows_b, f->cols); return -1;
  }
  const int64_t n = (int64_t)f->T * f->rows_n * f->rows_b * f->cols;
  if (n >= (1ll << 30)) { mx_set_error("mx_trng_fill: %lld values exceed the fill's 2^30 limit", (long long)n); return -1; }
  if (f->kind == MX_TRNG_NORMAL && n < 16) {
    mx_set_error("mx_trng_fill: a normal draw of %lld < 16 values takes torch's scalar path (two words per value and a cached sample); "
                 "it is not reproduced on the device", (long long)n);
    return -1;
  }
  if (!f->dst) { mx_set_error("mx_trng_fill: null destination"); return -1; }
  return n + (f->kind == MX_TRNG_NORMAL && (n & 15) ? 16 : 0);
}

extern "C" int mx_trng_set_state(uint32_t* state_dev, const uint32_t key[624], int32_t left, int32_t next, void* stream) {
  if (!state_dev || !key) { mx_set_error("mx_trng_set_state: null argument"); return 1; }
  if (left < 1 || left > MT_N || next < 0 || next > MT_N) { mx_set_error("mx_trng_set_state: left %d / next %d outside torch's range", left, next); return 1; }
  uint32_t st[MX_TRNG_WORDS];
  memset(st, 0, sizeof(st));
  memcpy(st, key, MT_N * 4);
  st[TR_LEFT] = (uint32_t)left;
  st[TR_NEXT] = (uint32_t)next;
  cudaStream_t s = (cudaStream_t)stream;
  cudaMemcpyAsync(state_dev, st, sizeof(st), cudaMemcpyHostToDevice, s);
  cudaStreamSynchronize(s);     // `st` is stack memory
  return 0;
}

extern "C" int mx_trng_get_state(const uint32_t* state_dev, uint32_t key[624], int32_t* left, int32_t* next, void* stream) {
  if (!state_dev || !key || !left || !next) { mx_set_error("mx_trng_get_state: null argument"); return 1; }
  uint32_t st[MT_N + 2];
  cudaStream_t s = (cudaStream_t)stream;
  cudaMemcpyAsync(st, state_dev, sizeof(st), cudaMemcpyDeviceToHost, s);
  cudaStreamSynchronize(s);
  memcpy(key, st, MT_N * 4);
  *left = (int32_t)st[TR_LEFT];
  *next = (int32_t)st[TR_NEXT];
  return 0;
}

// torch.manual_seed(seed): mt19937(seed) keeps the low 32 bits, init_genrand, left = 1, next = 0
extern "C" int mx_trng_seed(uint32_t* state_dev, uint64_t seed, void* stream) {
  uint32_t key[MT_N];
  key[0] = (uint32_t)seed;
  for (int i = 1; i < MT_N; ++i) key[i] = 1812433253u * (key[i - 1] ^ (key[i - 1] >> 30)) + (uint32_t)i;
  return mx_trng_set_state(state_dev, key, 1, 0, stream);
}

extern "C" int mx_trng_fill(uint32_t* state_dev, const mx_trng_draw* f, uint32_t* scratch_dev, int64_t scratch_words, void* stream) {
  const int64_t words = mx_trng_words(f);
  if (words < 0) return 1;
  if (!state_dev || !scratch_dev) { mx_set_error("mx_trng_fill: null state or scratch"); return 1; }
  if (scratch_words < words) { mx_set_error("mx_trng_fill: scratch of %lld words, the fill consumes %lld", (long long)scratch_words, (long long)words); return 1; }
  cudaStream_t s = (cudaStream_t)stream;
  if (const int rc = mx_launch("k_trng_twist", k_trng_twist, dim3(1), dim3(256), 0, s, MX_PLAIN, state_dev, scratch_dev, (int)words)) return rc;
  TrngFillArgs a;
  a.words = scratch_dev;
  a.n = (int)((int64_t)f->T * f->rows_n * f->rows_b * f->cols);
  a.kind = f->kind;
  a.std = f->std;
  a.rows_b = f->rows_b;
  a.rows = f->rows_n * f->rows_b;
  a.cols = f->cols;
  a.dst = f->dst;
  a.ld_t = f->ld_t; a.ld_n = f->ld_n; a.ld_b = f->ld_b;
  int grid = (a.n + 255) / 256;
  if (grid > mx_num_sms() * 4) grid = mx_num_sms() * 4;
  return mx_launch("k_trng_fill", k_trng_fill, dim3(grid), dim3(256), 0, s, MX_PLAIN, a);
}
