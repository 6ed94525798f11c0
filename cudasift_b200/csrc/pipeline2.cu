// pipeline2.cu -- host side of the extraction pipeline: one stream-ordered sequence of
//   [ScaleUp] -> pyr_lowpass_sd (TMA) -> pyr_chain -> detect2 (TMA, all octaves, all images) -> cap32 fix-up
//   -> describe (all octaves, all images) [-> rescale] [-> rank (ranked extractors)]
// for 1..CS_MAX_BATCH images of one size.  Replaces the reference's per-image loop (mainSift.cpp:65-69 around
// cudaSiftH.cu:72-144); the drop-in ExtractSift is the batch-of-one case.  Over the same levels a batch of one also
// runs the round-1 per-image kernels (LowPass, ScaleDown chain, detect, describe): CUDASIFT_LEGACY, and images TMA
// cannot address.
#include "common.cuh"
#include "pipeline2.h"

#include <cstring>
#include <vector>

namespace cs {

// ------------------------------------------------------------------------------ tensor maps
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn()
{
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void *p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    // resolved through the runtime: the library has no link-time dependency on libcuda
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
    else
      cudaGetLastError();
  }
  return fn;
}

bool tensor_map_compatible(const float *base, int pitch)
{
  return encode_fn() != nullptr && (reinterpret_cast<uintptr_t>(base) & 15) == 0 && (pitch & 3) == 0;
}

int make_tensor_map_2d(CUtensorMap *out, const float *base, int w, int h, int pitch, int boxW, int boxH)
{
  EncodeTiledFn fn = encode_fn();
  if (!fn || !tensor_map_compatible(base, pitch)) {
    set_error("tensor map: image %p (pitch %d floats) does not meet the TMA alignment rules", (const void *)base, pitch);
    return CS_E_ARG;
  }
  cuuint64_t dims[2] = {(cuuint64_t)w, (cuuint64_t)h};
  cuuint64_t strides[1] = {(cuuint64_t)pitch * sizeof(float)};
  cuuint32_t box[2] = {(cuuint32_t)boxW, (cuuint32_t)boxH};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float *>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d) for %dx%d pitch %d", (int)r, w, h, pitch);
    return CS_E_CUDA;
  }
  return 0;
}

// ------------------------------------------------------------------------------ tuning
int g_d2_hs = 0;          // rows per detector stream (0 = choose by batch size)
int g_pa_rows = 0;        // level-0 rows per CTA of kernel A (0 = choose by batch size)
int g_cap32 = -1;         // reference cap of 32 extrema per 30x8 block and scale: 1 on (default), 0 off
int g_cap_limit = 32;     // tests only
int g_sd_split = 1;       // batches: level 1 -> 2 by the tiled ScaleDown kernel, the chain kernel for the small levels (0 = chain only)

static bool cap32_enabled()
{
  if (g_cap32 < 0) {
    const char *e = getenv("CUDASIFT_NO_CAP32");
    g_cap32 = (e && *e && *e != '0') ? 0 : 1;
  }
  return g_cap32 == 1;
}

// CUDASIFT_DEBUG_SYNC=1: synchronise after every stage and name the one that failed (not during graph capture)
static int debug_stage(cudaStream_t st, const char *name)
{
  static int on = -1;
  if (on < 0) { const char *e = getenv("CUDASIFT_DEBUG_SYNC"); on = (e && *e && *e != '0') ? 1 : 0; }
  if (!on) return 0;
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(st, &cap);
  if (cap != cudaStreamCaptureStatusNone) return 0;
  cudaError_t e = cudaStreamSynchronize(st);
  if (e == cudaSuccess) e = cudaGetLastError();
  fprintf(stderr, "cudasift_b200 debug: stage %s: %s\n", name, cudaGetErrorString(e));
  if (e != cudaSuccess) { set_error("stage %s failed: %s", name, cudaGetErrorString(e)); return CS_E_CUDA; }
  return 0;
}

// ------------------------------------------------------------------------------ Pipeline
int check_level0_size(const char *who, int w, int h, bool up)
{
  const long long W = (long long)w * (up ? 2 : 1), H = (long long)h * (up ? 2 : 1);
  if (W > CS_MAX_LEVEL0 || H > CS_MAX_LEVEL0) {
    set_error("%s: invalid argument (CS_E_ARG): level 0 of %lldx%lld exceeds the detector's size limit of %d pixels "
              "(CS_MAX_LEVEL0: 13-bit extremum positions)", who, W, H, CS_MAX_LEVEL0);
    return CS_E_ARG;
  }
  return 0;
}

int Pipeline::init(int w, int h, int octaves, bool up, int maxBatch, float *arenaPtr)
{
  { int r0 = check_level0_size("ExtractSift", w, h, up); if (r0 < 0) return r0; }
  if (w < 1 || h < 1 || octaves < 1 || octaves > 7) {   // quirk Q17: taps table holds octave <= 7
    set_error("ExtractSift: invalid size %dx%d or numOctaves %d (1..7)", w, h, octaves);
    return CS_E_ARG;
  }
  if (maxBatch < 1 || maxBatch > CS_MAX_BATCH || (arenaPtr && maxBatch != 1)) {
    set_error("batch size %d out of range (1..%d)", maxBatch, CS_MAX_BATCH);
    return CS_E_ARG;
  }
  { int r0 = detect2_init_device(); if (r0 < 0) return r0; }
  w0 = w; h0 = h; numOctaves = octaves; scaleUp = up; B = maxBatch;
  const int W = w * (up ? 2 : 1), H = h * (up ? 2 : 1);
  numLevels = octaves;
  lw[0] = W; lh[0] = H; lp[0] = ialignup(W, 128);
  size_t off = 0;
  for (int i = 0; i < octaves; i++) {
    if (i > 0) { lw[i] = lw[i - 1] / 2; lh[i] = lh[i - 1] / 2; lp[i] = ialignup(lw[i], 128); }
    if (lw[i] < 1 || lh[i] < 1) { numLevels = i; break; }
    levOff[i] = off;
    off += (size_t)lh[i] * lp[i];
  }
  if (up) { upOff = off; off += (size_t)lh[0] * lp[0]; }
  perImage = (off + 63) & ~(size_t)63;                    // 256-byte multiples: every level stays 16-byte aligned
  if (arenaPtr) { arena = arenaPtr; ownArena = false; }   // the reference's sizing rule (cudaSiftH.cu:39-57) is larger
  else {
    CS_CUDA(cudaMalloc((void **)&arena, perImage * B * sizeof(float)));
    ownArena = true;
  }
  // the batched kernels read the levels through tensor maps; on an arena TMA cannot address only enqueue_round1 runs
  tma = encode_fn() != nullptr && (reinterpret_cast<uintptr_t>(arena) & 15) == 0;

  // textures (+ tensor maps) of every level of every image slot
  std::vector<CUtensorMap> maps((size_t)B * CS_MAX_LEVELS);
  memset(maps.data(), 0, maps.size() * sizeof(CUtensorMap));
  h_tex.assign((size_t)B * CS_MAX_LEVELS, 0);
  upMaps.resize(B);
  for (int b = 0; b < B; b++) {
    for (int i = 0; i < numLevels; i++) {
      int r = make_texture(&h_tex[(size_t)b * CS_MAX_LEVELS + i], level(b, i), lw[i], lh[i], lp[i]);
      if (r < 0) return r;
      if (tma && (r = make_tensor_map_2d(&maps[(size_t)b * CS_MAX_LEVELS + i], level(b, i), lw[i], lh[i], lp[i], 256, 1)) < 0) return r;
    }
    if (tma && up) {
      int r = make_tensor_map_2d(&upMaps[b], arena + (size_t)b * perImage + upOff, lw[0], lh[0], lp[0], CS_PA_BOX, 1);
      if (r < 0) return r;
    }
  }
  CS_CUDA(cudaMalloc((void **)&d_tex, h_tex.size() * sizeof(cudaTextureObject_t)));
  CS_CUDA(cudaMemcpy(d_tex, h_tex.data(), h_tex.size() * sizeof(cudaTextureObject_t), cudaMemcpyHostToDevice));
  CS_CUDA(cudaMalloc((void **)&d_maps, maps.size() * sizeof(CUtensorMap)));
  CS_CUDA(cudaMemcpy(d_maps, maps.data(), maps.size() * sizeof(CUtensorMap), cudaMemcpyHostToDevice));

  // per-launch state, cleared by one memset: [B x 4 counters][scheduler, 4 words][B x cellWords]
  cellWords = 0;
  for (int i = 0; i < numLevels; i++) {
    cellsX[i] = idivup(lw[i], 30);
    cellBase[i] = cellWords * 4;
    cellWords += idivup(cellsX[i] * idivup(lh[i], 8) * CS_NUM_SCALES, 4);
  }
  stateWords = (size_t)B * CS_CNT_STRIDE + 4 + (size_t)B * cellWords;
  CS_CUDA(cudaMalloc((void **)&d_state, stateWords * sizeof(unsigned int)));

  if (B == 1) {
    // the round-1 detector's tiles, coarsest level first: its tiles carry the most extrema candidates, so the
    // persistent CTAs finish on the light tiles of the finest level
    std::vector<uint2> tl;
    int nl = 0, idx[CS_MAX_LEVELS];
    for (int i = 0; i < numLevels; i++) idx[i] = (lw[i] < 3 || lh[i] < 3) ? -1 : nl++;   // no interior pixel -> no extrema
    for (int i = numLevels - 1; i >= 0; i--) {
      if (idx[i] < 0) continue;
      const int tx = idivup(lw[i] - 2, CS_DETECT_TILE_W), ty = idivup(lh[i] - 2, CS_DETECT_TILE_H);
      for (int y = 0; y < ty; y++)
        for (int x = 0; x < tx; x++)
          tl.push_back(make_uint2((unsigned)idx[i] | ((unsigned)(x * CS_DETECT_TILE_W) << 8), (unsigned)(y * CS_DETECT_TILE_H)));
    }
    numTiles = (int)tl.size();
    if (numTiles > 0) {
      CS_CUDA(cudaMalloc((void **)&d_tiles, tl.size() * sizeof(uint2)));
      CS_CUDA(cudaMemcpy(d_tiles, tl.data(), tl.size() * sizeof(uint2), cudaMemcpyHostToDevice));
    }
  }
  memset(lapTaps, 0, sizeof(lapTaps));
  laplace_taps(octaves, 0.0f, lapTaps);           // cudaSiftH.cu:110
  scaledown_taps(0.5f, sdTaps.k);                 // cudaSiftH.cu:157
  int dev = 0;
  sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return 0;
}

void Pipeline::destroy()
{
  for (size_t i = 0; i < h_tex.size(); i++)
    if (h_tex[i]) cudaDestroyTextureObject(h_tex[i]);
  h_tex.clear();
  if (d_tex) { cudaFree(d_tex); d_tex = nullptr; }
  if (d_maps) { cudaFree(d_maps); d_maps = nullptr; }
  if (d_state) { cudaFree(d_state); d_state = nullptr; }
  if (d_tiles) { cudaFree(d_tiles); d_tiles = nullptr; }
  for (auto &it : items) if (it.second.d) cudaFree(it.second.d);
  items.clear();
  if (ownArena && arena) cudaFree(arena);
  arena = nullptr;
}

// Detector work items for a batch of n images: coarsest level first (its strips carry the most extrema
// candidates), so the persistent CTAs finish on the light strips of the finest level.  An item = one strip of
// CS_D2_STRIP tested columns x two row streams of `hs` tested rows each; every interior pixel of every level
// belongs to exactly one item (tests/test_host_cpu.py).
void build_detector_items(const int *lw, const int *lh, int numLevels, int n, int hs, std::vector<uint4> &v)
{
  for (int l = numLevels - 1; l >= 0; l--) {
    if (lw[l] < 3 || lh[l] < 3) continue;                    // no interior pixel -> no extrema possible
    const int strips = idivup(lw[l] - 2, CS_D2_STRIP);
    const int rows = lh[l] - 2;                              // tested rows 1 .. h-2
    const int nitems = idivup(rows, 2 * hs);
    for (int b = 0; b < n; b++)
      for (int r = 0; r < nitems; r++) {
        const int ry0 = 1 + r * 2 * hs;
        const int left = rows - r * 2 * hs;
        const int hsi = left >= 2 * hs ? hs : (left + 1) / 2;   // the last item splits what is left between its two streams
        for (int s = 0; s < strips; s++)
          v.push_back(make_uint4((unsigned)l | ((unsigned)b << 8), (unsigned)(s * CS_D2_STRIP), (unsigned)ry0, (unsigned)hsi));
      }
  }
}

int Pipeline::get_items(int n, int hs, const uint4 **d_items, int *count)
{
  const int key = n * 1024 + hs;
  auto it = items.find(key);
  if (it == items.end()) {
    std::vector<uint4> v;
    build_detector_items(lw, lh, numLevels, n, hs, v);
    ItemList il;
    il.n = (int)v.size();
    il.d = nullptr;
    if (il.n > 0) {
      CS_CUDA(cudaMalloc((void **)&il.d, v.size() * sizeof(uint4)));
      CS_CUDA(cudaMemcpy(il.d, v.data(), v.size() * sizeof(uint4), cudaMemcpyHostToDevice));
    }
    it = items.emplace(key, il).first;
  }
  *d_items = it->second.d;
  *count = it->second.n;
  return 0;
}

int Pipeline::fill_pyr_a(PyrAParams &pa, int n, const float *const *d_imgs, int pitch, double initBlur)
{
  memset(&pa, 0, sizeof(pa));
  for (int b = 0; b < n; b++) {
    if (scaleUp) pa.inMaps[b] = upMaps[b];
    else {
      int r = make_tensor_map_2d(&pa.inMaps[b], d_imgs[b], w0, h0, pitch, CS_PA_BOX, 1);
      if (r < 0) return r;
    }
  }
  pa.lev0 = arena + levOff[0]; pa.lev0Stride = (long long)perImage;
  pa.w = lw[0]; pa.h = lh[0]; pa.p0 = lp[0];
  if (numLevels > 1) {
    pa.lev1 = arena + levOff[1]; pa.lev1Stride = (long long)perImage;
    pa.w1 = lw[1]; pa.h1 = lh[1]; pa.p1 = lp[1];
  }
  float sigma = (float)(initBlur > (double)0.001f ? initBlur : (double)0.001f);   // cudaSiftH.cu:112
  lowpass_taps(sigma, pa.lp.k);
  pa.sd = sdTaps;
  int rows = g_pa_rows > 0 ? g_pa_rows : (n >= 8 ? 72 : (n >= 2 ? 48 : 16));   // rows per warp (+12 halo rows each); measured at batch 16 / 32: 64: 6.5 / 5.7 us, 72: 6.0 / 5.5, 90: 6.8 / 5.5, 108: 7.3 / 5.8
  rows = (rows + 1) & ~1;
  pa.rowsPerCta = rows;
  pa.stripsX = idivup(lw[0], CS_PA_OWN);
  pa.rowBlocks = idivup(lh[0], rows);
  return 0;
}

int Pipeline::enqueue(int n, const float *const *d_imgs, int pitch, double initBlur, float thresh, float lowestScale,
                       SiftPoint *d_pts, long long ptsStride, int maxPts, cudaStream_t st, cudaEvent_t *ev,
                       PyrAParams *paOut, const RankParams *rank)
{
  int r;
  if (n < 1 || n > B) { set_error("batch of %d images on a pipeline built for %d", n, B); return CS_E_ARG; }
  if (!tma) {
    set_error("the batched pipeline needs cuTensorMapEncodeTiled and a 16-byte aligned arena (arena %p)", (void *)arena);
    return CS_E_ARG;
  }
  CS_CUDA(cudaMemsetAsync(d_state, 0, stateWords * sizeof(unsigned int), st));   // cudaSiftH.cu:77
  if (ev) cudaEventRecord(ev[0], st);
  unsigned int *d_counters = d_state, *d_sched = d_state + (size_t)B * CS_CNT_STRIDE;
  unsigned int *d_cells = d_sched + 4;

  if (scaleUp) {                                                            // cudaSiftH.cu:119-123
    for (int b = 0; b < n; b++)
      if ((r = launch_scaleup(d_imgs[b], arena + (size_t)b * perImage + upOff, w0, h0, pitch, lp[0], st)) < 0) return r;
    lowestScale *= 2.0f;                                                    // cudaSiftH.cu:127
  }
  PyrAParams pa;
  if ((r = fill_pyr_a(pa, n, d_imgs, pitch, initBlur)) < 0) return r;
  if (paOut) *paOut = pa;
  if ((r = debug_stage(st, "memset/scaleup")) < 0) return r;
  if ((r = launch_pyr_a(pa, n, st)) < 0) return r;
  if ((r = debug_stage(st, "pyr_lowpass_sd")) < 0) return r;
  if (ev) cudaEventRecord(ev[1], st);
  int from0 = 1;
  if (g_sd_split && n >= 2 && numLevels >= 4) {
    // a whole batch keeps the 64x16-tile ScaleDown of round 1 busy (13 % halo); the chain kernel's 8x8 tiles recompute
    // 1.6x on the level it would produce first, which is the large one.  It keeps the small levels.
    if ((r = launch_scaledown(arena + levOff[1], arena + levOff[2], lw[1], lh[1], lp[1], lp[2], sdTaps, st, n,
                              (long long)perImage, (long long)perImage)) < 0) return r;
    if ((r = debug_stage(st, "scaledown 1->2")) < 0) return r;
    from0 = 2;
  }
  for (int from = from0; from + 1 < numLevels; from += 3) {                 // cudaSiftH.cu:153-157, three levels per launch
    PyrBParams pb;
    memset(&pb, 0, sizeof(pb));
    pb.steps = numLevels - 1 - from < 3 ? numLevels - 1 - from : 3;
    for (int k = 0; k <= pb.steps; k++) {
      pb.img[k] = arena + levOff[from + k]; pb.stride[k] = (long long)perImage;
      pb.w[k] = lw[from + k]; pb.h[k] = lh[from + k]; pb.pitch[k] = lp[from + k];
    }
    pb.sd = sdTaps;
    if ((r = launch_pyr_b(pb, n, st)) < 0) return r;
    if ((r = debug_stage(st, "pyr_chain")) < 0) return r;
  }
  if (ev) cudaEventRecord(ev[2], st);

  Detect2Params dp;
  memset(&dp, 0, sizeof(dp));
  for (int i = 0; i < numLevels; i++) {
    D2Level &L = dp.lev[i];
    L.w = lw[i]; L.h = lh[i];
    L.subsampling = (float)(1 << i);
    L.lowestScale = lowestScale / L.subsampling;                            // cudaSiftH.cu:213
    const float *k = lapTaps + (numOctaves - i) * 12 * 16;                  // octave index, :161,:1766
    for (int s = 0; s < CS_LAPLACE_S; s++)
      for (int j = 0; j < 5; j++) L.taps.k[s][j] = k[16 * s + j];
    dp.cellBase[i] = cellBase[i]; dp.cellsX[i] = cellsX[i];
    dp.lev0Img[i] = arena + levOff[i]; dp.levPitch[i] = lp[i];
  }
  dp.imgStride = (long long)perImage;
  const int hs = g_d2_hs > 0 ? g_d2_hs : (n >= 8 ? 96 : (n >= 2 ? 32 : 12));   // rows per stream
  if ((r = get_items(n, hs, &dp.items, &dp.numItems)) < 0) return r;
  dp.maps = d_maps;
  dp.thresh = thresh; dp.edgeLimit = 10.0f; dp.factor = 1.0f / CS_NUM_SCALES;   // cudaSiftH.cu:213
  dp.pts = d_pts; dp.ptsStride = ptsStride; dp.counters = d_counters; dp.sched = d_sched; dp.maxPts = maxPts;
  if (cap32_enabled()) { dp.cells = d_cells; dp.cellWords = cellWords; }
  dp.capLimit = g_cap_limit;
  if ((r = launch_detect2(dp, sms, st)) < 0) return r;
  if ((r = debug_stage(st, "detect2")) < 0) return r;
  if (cap32_enabled()) {
    if ((r = launch_cap32_fixup(dp, n, st)) < 0) return r;
    if ((r = debug_stage(st, "cap32_fixup")) < 0) return r;
  }
  if (ev) cudaEventRecord(ev[3], st);

  DescribeParams ds;
  memset(&ds, 0, sizeof(ds));
  ds.texArr = d_tex;
  ds.numLevels = numLevels; ds.numImages = n; ds.pts = d_pts; ds.ptsStride = ptsStride; ds.counters = d_counters;
  ds.cntStride = CS_CNT_STRIDE; ds.maxPts = maxPts;
  ds.finestSubsampling = 1.0f;
  ds.queue = d_sched + 1;
  if ((r = launch_describe(ds, st)) < 0) return r;
  if ((r = debug_stage(st, "describe")) < 0) return r;
  if (scaleUp)                                                             // cudaSiftH.cu:130
    for (int b = 0; b < n; b++)
      if ((r = launch_rescale(d_pts + (size_t)b * ptsStride, d_counters + (size_t)b * CS_CNT_STRIDE, maxPts, 0.5f, st)) < 0) return r;
  if (ev) cudaEventRecord(ev[4], st);
  if (rank) {
    RankParams rp = *rank;
    rp.in = d_pts; rp.inStride = ptsStride; rp.maxIn = maxPts; rp.counters = d_counters;
    if ((r = launch_rank(rp, n, sms, st)) < 0) return r;
    if ((r = debug_stage(st, "rank")) < 0) return r;
    if (ev) cudaEventRecord(ev[5], st);
  }
  return 0;
}

int Pipeline::enqueue_round1(const float *d_img, int pitch, double initBlur, float thresh, float lowestScale,
                             SiftPoint *d_pts, int maxPts, cudaStream_t st, cudaEvent_t *ev)
{
  int r;
  if (B != 1) { set_error("the round-1 kernels take one image at a time (pipeline built for %d)", B); return CS_E_ARG; }
  unsigned int *d_counters = counters(0), *d_sched = d_state + CS_CNT_STRIDE;
  // the counters (cudaSiftH.cu:77) and the scheduler words that follow them (describe's queue word)
  CS_CUDA(cudaMemsetAsync(d_counters, 0, (CS_CNT_STRIDE + 4) * sizeof(unsigned int), st));
  if (ev) cudaEventRecord(ev[0], st);
  Taps9 lp9;
  float sigma = (float)(initBlur > (double)0.001f ? initBlur : (double)0.001f);   // cudaSiftH.cu:112
  lowpass_taps(sigma, lp9.k);
  if (!scaleUp) {
    if ((r = launch_lowpass(d_img, pitch, level(0, 0), lp[0], lw[0], lh[0], lp9, st)) < 0) return r;
  } else {                                                                 // cudaSiftH.cu:119-123
    float *upImg = arena + upOff;
    if ((r = launch_scaleup(d_img, upImg, w0, h0, pitch, lp[0], st)) < 0) return r;
    if ((r = launch_lowpass(upImg, lp[0], level(0, 0), lp[0], lw[0], lh[0], lp9, st)) < 0) return r;
    lowestScale *= 2.0f;                                                   // cudaSiftH.cu:127
  }
  if (ev) cudaEventRecord(ev[1], st);
  for (int i = 1; i < numLevels; i++)                                      // cudaSiftH.cu:153-157
    if ((r = launch_scaledown(level(0, i - 1), level(0, i), lw[i - 1], lh[i - 1], lp[i - 1], lp[i], sdTaps, st)) < 0) return r;
  if (ev) cudaEventRecord(ev[2], st);

  DetectParams dp;
  memset(&dp, 0, sizeof(dp));
  int tiles = 0, nl = 0;
  for (int i = 0; i < numLevels; i++) {
    if (lw[i] < 3 || lh[i] < 3) continue;          // no interior pixel -> no extrema possible
    DetectLevel &L = dp.lev[nl++];
    L.img = level(0, i); L.w = lw[i]; L.h = lh[i]; L.pitch = lp[i];
    tiles += idivup(lw[i] - 2, CS_DETECT_TILE_W) * idivup(lh[i] - 2, CS_DETECT_TILE_H);   // see init (d_tiles)
    L.subsampling = (float)(1 << i);
    L.lowestScale = lowestScale / L.subsampling;                           // cudaSiftH.cu:213
    const float *k = lapTaps + (numOctaves - i) * 12 * 16;                 // octave index, :161,:1766
    for (int s = 0; s < CS_LAPLACE_S; s++)
      for (int j = 0; j < 5; j++) L.taps.set(s, j, k[16 * s + j]);
  }
  dp.numLevels = nl; dp.totalTiles = tiles; dp.tiles = d_tiles;
  if (tiles != numTiles) { set_error("detector tile list out of sync"); return CS_E_ARG; }
  dp.thresh = thresh; dp.edgeLimit = 10.0f; dp.factor = 1.0f / CS_NUM_SCALES;   // cudaSiftH.cu:213
  dp.pts = d_pts; dp.counters = d_counters; dp.maxPts = maxPts;
  if ((r = launch_detect(dp, st)) < 0) return r;
  if (ev) cudaEventRecord(ev[3], st);

  DescribeParams ds;
  memset(&ds, 0, sizeof(ds));
  for (int i = 0; i < numLevels; i++) ds.tex[i] = h_tex[i];
  ds.numLevels = numLevels; ds.numImages = 1; ds.pts = d_pts; ds.counters = d_counters; ds.maxPts = maxPts;
  ds.finestSubsampling = 1.0f;
  ds.queue = d_sched + 1;
  if ((r = launch_describe(ds, st)) < 0) return r;
  if (scaleUp)                                                             // cudaSiftH.cu:130
    if ((r = launch_rescale(d_pts, d_counters, maxPts, 0.5f, st)) < 0) return r;
  if (ev) cudaEventRecord(ev[4], st);
  return 0;
}

}  // namespace cs
