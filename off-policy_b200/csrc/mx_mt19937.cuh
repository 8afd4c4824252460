// MT19937 core shared by the two device copies of host generators: NumPy's legacy stream behind the replay's index draws (k_draw,
// replay.cu) and torch's CPU generator behind the actor-critic noise draws (torch_rng.cu).  Both engines are the same MT19937; they differ
// only in how a word becomes a value and in how the position is recorded.
#pragma once
#include "mx_common.cuh"

#define MT_N 624
#define MT_M 397

MX_DEVINL uint32_t mt_temper(uint32_t y) {
  y ^= y >> 11;
  y ^= (y << 7) & 0x9D2C5680u;
  y ^= (y << 15) & 0xEFC60000u;
  y ^= y >> 18;
  return y;
}
MX_DEVINL uint32_t mt_mix(uint32_t cur, uint32_t nxt, uint32_t far) {
  uint32_t y = (cur & 0x80000000u) | (nxt & 0x7FFFFFFFu);
  return far ^ (y >> 1) ^ ((y & 1u) ? 0x9908B0DFu : 0u);
}
// In-place regeneration of all 624 words by the whole CTA (>= 256 threads): three dependency-free phases.
MX_DEVINL void mt_twist_cta(uint32_t* key) {
  const int tid = threadIdx.x;
  const int lo[3] = {0, 227, 454}, hi[3] = {227, 454, 624};
  for (int ph = 0; ph < 3; ++ph) {
    uint32_t v = 0;
    const int i = lo[ph] + tid;
    const bool act = i < hi[ph];
    if (act) {
      uint32_t nxt = key[(i + 1) % MT_N];
      uint32_t far = key[(i + MT_M) % MT_N];
      v = mt_mix(key[i], nxt, far);
    }
    __syncthreads();
    if (act) key[i] = v;   // i == 623 reads key[0], already regenerated in phase 0, exactly like the serial loop
    __syncthreads();
  }
}
