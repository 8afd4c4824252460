// Episode gather on the TMA unit (rec_buffer.py:192-240: RecPolicyBuffer.sample_inds -- B sampled episodes, every field).
//
// The replay is episode-major (DESIGN.md section 3): one episode's slice of a field is ONE contiguous 16-byte-aligned run, so sampling
// B episodes is B straight copies per field.  Each field is described to the TMA unit twice as a 2-D tensor [rows][episode words]:
// the store (`capacity` rows) and the batch region (`max_batch` rows) -- and again as a 3-D tensor [rows][full 1 KB lines][256 words].
// The bulk of an episode's field moves as 8 KB boxes of the 3-D view (8 lines x 256 words at (0, line, episode index)); the partial last
// line, which a multi-line box would run into the next episode, as one clipped 2-D box.  A copy is a tile load into shared memory,
// completion signalled on an mbarrier by byte count, followed by a tile store to the batch row.  One elected lane per warp runs a
// four-stage pipeline (two loads in flight ahead of the store being issued); no thread touches the data except for the reward normalisation ((r - mean) / std on the rewards field, rec_buffer.py:221-223),
// which the warp applies in shared memory between the load and the store.  The kernel issues UTMALDG / UTMASTG only: address
// generation, bounds handling and the 128-byte transactions are the copy engine's.
#include <string.h>

#include "mx_internal.h"
#include "mx_kernels.h"

#if !MX_EMU
#include <cuda.h>

#define GT_WARPS 2
#define GT_STAGES 4
#define GT_AHEAD 2            // loads in flight per pipeline
#define GT_BOX 256            // 32-bit words per box row (the TMA limit per dimension)
#define GT_ROWS 8             // rows of 256 words per big box: 8 KB per copy

struct GatherTmaMaps {
  CUtensorMap src[8], dst[8];        // 2-D [rows][episode words], box {256, 1}: the clipped tail of an episode's field
  CUtensorMap src3[8], dst3[8];      // 3-D [rows][full 1 KB lines of the episode][256], box {256, GT_ROWS, 1}: the bulk
};
struct GatherTmaArgs {
  int nf, B, rew_field;
  int cum[9];                  // copy slots per episode before field f (cum[nf] = slots per episode)
  int nbig[8];                 // big boxes per episode of field f (then one tail box if tail[f])
  int lines[8];                // full 256-word lines of field f
  int tail[8];                 // 1: the field has a partial last line
  const long long* idx;        // [B] sampled episode indices
  const MxReplayState* state;
};

__device__ __forceinline__ uint32_t gt_smem(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__global__ void __launch_bounds__(GT_WARPS * 32) k_gather_tma(const __grid_constant__ GatherTmaMaps maps, GatherTmaArgs a) {
  extern __shared__ __align__(128) unsigned char gt_dyn[];          // 64 KB of stages: above the static limit
  float (*stage)[GT_STAGES][GT_ROWS * GT_BOX] = reinterpret_cast<float (*)[GT_STAGES][GT_ROWS * GT_BOX]>(gt_dyn);
  __shared__ __align__(8) unsigned long long bars[GT_WARPS][GT_STAGES];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    for (int s = 0; s < GT_STAGES; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(gt_smem(&bars[warp][s])) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  MX_PDL_WAIT();
  const int per_ep = a.cum[a.nf];
  const long long total = (long long)per_ep * a.B;
  const long long first = (long long)blockIdx.x * GT_WARPS + warp, stride = (long long)gridDim.x * GT_WARPS;
  const int n_my = first < total ? (int)((total - first + stride - 1) / stride) : 0;
  float mean = 0.f, stdv = 1.f;
  if (a.rew_field >= 0) { mean = (float)a.state->reward_mean; stdv = (float)a.state->reward_std; }

  // slot -> (field, big box index or -1 for the tail, batch row)
  auto decode = [&](int k, int& f, int& box, int& b) {
    const long long item = first + (long long)k * stride;
    b = (int)(item / per_ep);
    const int rem = (int)(item - (long long)b * per_ep);
    f = 0;
    while (f + 1 < a.nf && rem >= a.cum[f + 1]) ++f;
    box = rem - a.cum[f];
    if (box >= a.nbig[f]) box = -1;
  };
  auto load = [&](int k) {          // lane 0 only
    int f, box, b;
    decode(k, f, box, b);
    const int e = (int)a.idx[b];
    const uint32_t bar = gt_smem(&bars[warp][k % GT_STAGES]), dst = gt_smem(&stage[warp][k % GT_STAGES][0]);
    if (box >= 0) {
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(GT_ROWS * GT_BOX * 4) : "memory");
      asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(dst),
                   "l"(&maps.src3[f]), "r"(0), "r"(box * GT_ROWS), "r"(e), "r"(bar)
                   : "memory");
    } else {
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(GT_BOX * 4) : "memory");
      asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
                   "l"(&maps.src[f]), "r"(a.lines[f] * GT_BOX), "r"(e), "r"(bar)
                   : "memory");
    }
  };
  if (lane == 0)
    for (int k = 0; k < GT_AHEAD && k < n_my; ++k) load(k);
  for (int k = 0; k < n_my; ++k) {
    if (lane == 0 && k + GT_AHEAD < n_my) {
      // the stage of item k + AHEAD was last used by item k + AHEAD - STAGES: its store must have finished READING shared memory.
      // Stores committed so far: items 0 .. k-1; allowing STAGES - AHEAD - 1 pending groups leaves exactly that one complete.
      asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(GT_STAGES - GT_AHEAD - 1) : "memory");
      load(k + GT_AHEAD);
    }
    int f, box, b;
    decode(k, f, box, b);
    const uint32_t bar = gt_smem(&bars[warp][k % GT_STAGES]);
    const uint32_t parity = (uint32_t)((k / GT_STAGES) & 1);
    const bool transform = f == a.rew_field;           // warp-uniform
    if (lane == 0 || transform) {
      uint32_t done = 0;
      while (!done)
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n" : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    }
    if (transform) {
      float* sbuf = &stage[warp][k % GT_STAGES][0];
      const int nw = box >= 0 ? GT_ROWS * GT_BOX : GT_BOX;
      for (int i = lane; i < nw; i += 32) sbuf[i] = (sbuf[i] - mean) / stdv;
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy writes before the async-proxy (TMA) read
      __syncwarp();
    }
    if (lane == 0) {
      const uint32_t src = gt_smem(&stage[warp][k % GT_STAGES][0]);
      if (box >= 0)
        asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(&maps.dst3[f]), "r"(src), "r"(0),
                     "r"(box * GT_ROWS), "r"(b)
                     : "memory");
      else
        asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(&maps.dst[f]), "r"(src),
                     "r"(a.lines[f] * GT_BOX), "r"(b)
                     : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    __syncwarp();        // the other lanes never run ahead of the elected one (a lane a full ring ahead would misread the barrier parity)
  }
  if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static int tried = 0;
  if (!tried) {
    tried = 1;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = (EncodeTiledFn)p;
    cudaGetLastError();
  }
  return fn;
}

struct MxGatherTma {
  GatherTmaMaps maps;
  GatherTmaArgs args;
  long long bytes_per_episode;
};

static bool encode_lines(EncodeTiledFn fn, CUtensorMap* m, void* base, long long rows, long long row_words, long long lines) {
  const cuuint64_t dims[3] = {GT_BOX, (cuuint64_t)lines, (cuuint64_t)rows};
  const cuuint64_t strides[2] = {GT_BOX * 4, (cuuint64_t)row_words * 4};
  const cuuint32_t box[3] = {GT_BOX, GT_ROWS, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  return fn(m, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
static bool encode_rows(EncodeTiledFn fn, CUtensorMap* m, void* base, long long rows, long long row_words) {
  const cuuint64_t dims[2] = {(cuuint64_t)row_words, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)row_words * 4};
  const cuuint32_t box[2] = {GT_BOX, 1};
  const cuuint32_t estr[2] = {1, 1};
  return fn(m, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Tensor maps of every field of a replay (built once at mx_replay_create).  Returns null when the driver entry point is missing or a
// field cannot be described (the vectorised k_gather is used then).
void* mx_gather_tma_create(mx_replay* r) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return nullptr;
  const mx_replay_layout& L = r->L;
  MxGatherTma* g = new MxGatherTma();
  memset(g, 0, sizeof(*g));
  int nf = 0, cum = 0;
  bool ok = true;
  auto add = [&](int64_t src_off, int64_t dst_off, int64_t ep_words) {
    if (ep_words == 0 || !ok) return;
    ok = ok && encode_rows(fn, &g->maps.src[nf], r->blob + src_off, r->cfg.capacity, ep_words) &&
         encode_rows(fn, &g->maps.dst[nf], r->blob + dst_off, r->cfg.max_batch, ep_words);
    const long long lines = ep_words / GT_BOX;
    if (lines > 0)
      ok = ok && encode_lines(fn, &g->maps.src3[nf], r->blob + src_off, r->cfg.capacity, ep_words, lines) &&
           encode_lines(fn, &g->maps.dst3[nf], r->blob + dst_off, r->cfg.max_batch, ep_words, lines);
    g->bytes_per_episode += ep_words * 4;
    g->args.lines[nf] = (int)lines;
    g->args.nbig[nf] = (int)((lines + GT_ROWS - 1) / GT_ROWS);
    g->args.tail[nf] = (ep_words % GT_BOX) ? 1 : 0;
    g->args.cum[nf] = cum;
    cum += g->args.nbig[nf] + g->args.tail[nf];
    ++nf;
  };
  add(L.off_obs, L.off_b_obs, L.ep_obs);
  add(L.off_share, L.off_b_share, L.ep_share);
  add(L.off_acts, L.off_b_acts, L.ep_acts);
  add(L.off_avail, L.off_b_avail, L.ep_avail);
  g->args.rew_field = r->cfg.reward_norm ? nf : -1;
  add(L.off_rew, L.off_b_rew, L.ep_rew);
  add(L.off_dones, L.off_b_dones, L.ep_dones);
  add(L.off_dones_env, L.off_b_dones_env, L.ep_dones_env);
  add(L.off_actidx, L.off_b_actidx, L.ep_actidx);
  g->args.cum[nf] = cum;
  g->args.nf = nf;
  g->args.state = reinterpret_cast<const MxReplayState*>(r->blob + L.off_state);
  if (!ok) { delete g; return nullptr; }
  return g;
}
void mx_gather_tma_destroy(void* p) { delete reinterpret_cast<MxGatherTma*>(p); }

int g_mx_gather_tma = 1;
// returns -1 when the TMA path is not available / switched off (the caller launches k_gather)
int mx_launch_gather_tma(void* p, const int64_t* idx_dev, int B, cudaStream_t s) {
  if (!p || !g_mx_gather_tma) return -1;
  MxGatherTma* g = reinterpret_cast<MxGatherTma*>(p);
  // The TMA copy is for small batches, the vectorised loads for large ones (tools/gather_sweep.py measures the crossover; the 96 MB
  // threshold is not yet measured on the H100).  gather_tma = 2 forces TMA at any size.
  if (g_mx_gather_tma == 1 && (long long)g->bytes_per_episode * B > (96ll << 20)) return -1;
  GatherTmaArgs a = g->args;
  a.B = B;
  a.idx = (const long long*)idx_dev;
  const long long total = (long long)a.cum[a.nf] * B;
  const int sms = mx_num_sms();
  long long want = (total + GT_WARPS - 1) / GT_WARPS;          // one box per warp at least
  int grid = (int)(want < 1 ? 1 : want);
  if (grid > sms * 3) grid = sms * 3;                          // three resident CTAs (64 KB of stages each) per SM
  else if (grid > sms) grid = grid / sms * sms;
  const size_t smem = (size_t)GT_WARPS * GT_STAGES * GT_ROWS * GT_BOX * 4;
  const int rc = mx_launch("k_gather", k_gather_tma, dim3(grid), dim3(GT_WARPS * 32), smem, s, MX_STEP, g->maps, a);
  return rc == MX_ERR_SMEM ? -1 : rc;      // no room for the stages: the vectorised gather instead
}
#else
void* mx_gather_tma_create(mx_replay*) { return nullptr; }
void mx_gather_tma_destroy(void*) {}
int g_mx_gather_tma = 0;
int mx_launch_gather_tma(void*, const int64_t*, int, cudaStream_t) { return -1; }
#endif
