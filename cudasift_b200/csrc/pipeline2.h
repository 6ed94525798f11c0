// pipeline2.h -- host-side state of the batched extraction pipeline (pipeline2.cu).
#pragma once

#include "common.cuh"

#include <map>
#include <vector>

namespace cs {

struct Pipeline2 {
  int w0 = 0, h0 = 0, numOctaves = 0, numLevels = 0, B = 0, sms = 132;
  bool scaleUp = false;
  float *arena = nullptr;              // B consecutive per-image blocks: levels 0..n-1 [+ the up-scaled input]
  bool ownArena = false;
  size_t perImage = 0, levOff[CS_MAX_LEVELS] = {}, upOff = 0;   // in floats
  int lw[CS_MAX_LEVELS] = {}, lh[CS_MAX_LEVELS] = {}, lp[CS_MAX_LEVELS] = {};
  std::vector<cudaTextureObject_t> h_tex;
  cudaTextureObject_t *d_tex = nullptr;      // [image slot * CS_MAX_LEVELS + level]
  CUtensorMap *d_maps = nullptr;             // same indexing, box 256 x 1
  std::vector<CUtensorMap> upMaps;           // up-scaled inputs (scaleUp)
  unsigned int *d_state = nullptr;           // counters | scheduler | cap cells (one memset)
  size_t stateWords = 0;
  int cellWords = 0, cellBase[CS_MAX_LEVELS] = {}, cellsX[CS_MAX_LEVELS] = {};
  float lapTaps[8 * 12 * 16];
  Taps5 sdTaps;
  struct ItemList { uint4 *d; int n; };
  std::map<int, ItemList> items;             // detector work lists by (batch size, rows per stream)

  float *level(int b, int l) const { return arena + (size_t)b * perImage + levOff[l]; }
  unsigned int *counters(int b) const { return d_state + (size_t)b * CS_CNT_STRIDE; }

  int init(int w, int h, int octaves, bool up, int maxBatch, float *arenaPtr);
  void destroy();
  int get_items(int n, int hs, const uint4 **d_items, int *count);
  int fill_pyr_a(PyrAParams &pa, int n, const float *const *d_imgs, int pitch, double initBlur);
  // Enqueue the extraction of n images (device pointers, common pitch) on `st`.  Image i writes its records to
  // d_pts + i * ptsStride and its counters to counters(i).  ev (optional): 5 events at the stage boundaries
  // (start, after the level-0/1 kernel, after the chain, after detect, after describe).  paOut (optional)
  // receives the parameters of the first kernel (its tensor maps are the only per-call state of a captured graph).
  // rank (optional): d_pts is then the candidate area, and the ranking stage (rank.cu) writes each image's
  // rank->maxOut strongest records to rank->out + i * rank->outStride (ev: one more event, after ranking).
  int enqueue(int n, const float *const *d_imgs, int pitch, double initBlur, float thresh, float lowestScale,
              SiftPoint *d_pts, long long ptsStride, int maxPts, cudaStream_t st, cudaEvent_t *ev = nullptr,
              PyrAParams *paOut = nullptr, const RankParams *rank = nullptr);
};

void build_detector_items(const int *lw, const int *lh, int numLevels, int n, int hs, std::vector<uint4> &v);
extern int g_d2_hs, g_pa_rows, g_cap32, g_cap_limit, g_sd_split;

}  // namespace cs
