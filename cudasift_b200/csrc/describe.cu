// describe.cu -- fused orientation assignment + 128-D descriptor extraction.
//
// Behavioural spec: reference ComputeOrientationsCONST (cudaSiftD.cu:972-1057) and
// ExtractSiftDescriptorsCONSTNew (cudaSiftD.cu:308-417, FastAtan2 :295-306), host side
// cudaSiftH.cu:353-382.  The reference runs two persistent kernels per octave (10 launches
// per image) and accumulates both histograms with shared-memory float atomics, whose
// summation order -- and therefore the low-order bits of every descriptor -- change from
// run to run.  Here a single launch serves all octaves: one 128-thread CTA per keypoint
// computes the orientation histogram, its one or two peaks, and then one descriptor per
// peak.  Both histograms are accumulated without atomics in a fixed order (private partial
// histograms in shared memory, then a fixed-order reduction), so results are run-to-run
// deterministic; the summation order differs from the reference's only as much as the
// reference's own order differs between two of its runs.
//
// Image samples go through the texture unit exactly as in the reference (bilinear,
// clamp, unnormalised coordinates, cudaSiftH.cu:186-205), so the 1.8 fixed-point
// interpolation weights are the hardware's own.
//
// Scheduling: the keypoints of all images of a launch form one queue (image 0's, then image 1's, ...), and one
// resident wave of CTAs claims them from a counter.  A keypoint's chain of barriers is latency-bound, so what sets
// the stage's time is how many chains are in flight per SM and that no CTA idles while another image still has work.
#include "common.cuh"

namespace cs {

#define DS_THREADS 128
#define DS_MIN_CTAS 10      // resident CTAs per SM the register budget is set for (at most 48 registers a thread)

// cudaSiftD.cu:295-306, as scheduled in the reference's SASS.
__device__ __forceinline__ float fast_atan2(float y, float x)
{
  float absx = fabsf(x), absy = fabsf(y);
  float a = __fdiv_rn(fminf(absx, absy), fmaxf(absx, absy));
  float s = __fmul_rn(a, a);
  float r = __fmaf_rn(s, -0.0464964749f, 0.15931422f);
  r = __fmaf_rn(s, r, -0.327622764f);
  r = __fmul_rn(s, r);
  r = __fmaf_rn(r, a, a);
  r = (absy > absx ? __fsub_rn(1.57079637f, r) : r);
  r = (x < 0 ? __fsub_rn(3.14159274f, r) : r);
  r = (y < 0 ? -r : r);
  return r;
}

__global__ void __launch_bounds__(DS_THREADS, DS_MIN_CTAS)
describe_kernel(const __grid_constant__ DescribeParams P)
{
  __shared__ float s_gauss11[11];
  __shared__ float s_gauss16[16];
  __shared__ float s_ow[121];          // orientation sample weights
  __shared__ int s_obin[121];          // orientation sample bins
  // per-sample tables of the descriptor stage, row stride 17 (the accumulation reads them down the rows:
  // stride 16 would put every other row on the same bank)
  __shared__ float s_g2[4][16 * 17];             // descriptor votes per sample: ul, ll, ur, lr
  __shared__ float s_angf[16 * 17];
  __shared__ int s_angi[16 * 17];
  __shared__ float s_hp[32][33];       // orientation: private 32-bin histograms of warp 0's lanes
  __shared__ float s_pb[128][9];       // descriptor: private angle bins (+ Q22 overflow slot) per (cell, row)
  __shared__ float s_sums[2][4];       // the two norms of a descriptor: separate words, so no barrier between them
  __shared__ float s_ori[2];
  __shared__ int s_slot[2];
  __shared__ int s_nori;
  __shared__ int s_next;               // the keypoint this CTA takes after the current one

  const int tx = threadIdx.x, lane = tx & 31;
  if (tx < 16) s_gauss16[tx] = __expf(-(tx - 7.5f) * (tx - 7.5f) / 128.0f);   // cudaSiftD.cu:318
  for (int i = tx; i < 32 * 33; i += DS_THREADS) (&s_hp[0][0])[i] = 0.0f;

  // The queue: image i owns the batch-wide indices [end_{i-1}, end_i), end_i = sum over j <= i of
  // min(found_j, maxPts).  Every warp keeps end_lane in a register (lanes past the last image hold the total).
  unsigned int end = 0;
  if (lane < P.numImages) end = min(P.counters[(size_t)lane * P.cntStride], (unsigned)P.maxPts);
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned int t = __shfl_up_sync(0xffffffffu, end, o);
    if (lane >= o) end += t;
  }
  const int total = (int)__shfl_sync(0xffffffffu, end, 31);
  // claims run one keypoint ahead: the claim made during keypoint i is read while keypoint i + 1 runs
  unsigned int req = 0;
  if (tx == 0) req = gridDim.x + atomicAdd(P.queue, 1u);

  for (int g = blockIdx.x; g < total;) {
    const int img = __popc(__ballot_sync(0xffffffffu, end <= (unsigned)g));   // images that end at or before g
    const unsigned int first = img ? __shfl_sync(0xffffffffu, end, (img - 1) & 31) : 0u;
    const int numPrim = (int)(__shfl_sync(0xffffffffu, end, img) - first);
    const int pt = g - (int)first;
    SiftPoint *const pts = P.pts + (size_t)img * P.ptsStride;
    unsigned int *const counters = P.counters + (size_t)img * P.cntStride;
    SiftPoint *sp = pts + pt;
    const float px = sp->xpos, py = sp->ypos, pscale = sp->scale, psub = sp->subsampling;
    const int level = ((__float_as_int(psub) >> 23) & 0xff) - 127;   // subsampling = 2^level
    const cudaTextureObject_t tex = P.texArr ? P.texArr[img * CS_MAX_LEVELS + level] : P.tex[level];

    // ------------------------------------------------------------ orientation histogram
    {
      float i2sigma2 = __fdiv_rn(-1.0f, __fmul_rn(__fmul_rn(pscale, 4.5f), pscale));   // :982
      if (tx < 11) {
        float t = (float)(tx - 5);
        s_gauss11[tx] = expf(__fmul_rn(t, __fmul_rn(t, i2sigma2)));                     // :984
      }
    }
    __syncthreads();
    if (tx < 121) {
      int yd = tx / 11, xd = tx - yd * 11;
      float xf = __fadd_rn((float)xd, __fadd_rn(px, -4.5f));
      float yf = __fadd_rn((float)yd, __fadd_rn(py, -4.5f));
      float dx = __fsub_rn(tex2D<float>(tex, __fadd_rn(xf, 1.0f), yf), tex2D<float>(tex, __fadd_rn(xf, -1.0f), yf));
      float dy = __fsub_rn(tex2D<float>(tex, xf, __fadd_rn(yf, 1.0f)), tex2D<float>(tex, xf, __fadd_rn(yf, -1.0f)));
      int bin = __float2int_rz(__fadd_rn(__fdiv_rn(__fmul_rn(16.0f, atan2f(dy, dx)), 3.1416f), 16.5f));   // :997
      if (bin > 31) bin = 0;
      if (bin < 0) bin = 0;
      float grad = __fsqrt_rn(__fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
      s_ow[tx] = __fmul_rn(__fmul_rn(grad, s_gauss11[xd]), s_gauss11[yd]);
      s_obin[tx] = bin;
    }
    __syncthreads();
    if (tx < 32) {
      // warp 0: lane l accumulates samples l, l+32, l+64, l+96 into its private histogram, then
      // lane b sums column b over the 32 lanes in lane order (fixed order, no atomics)
      int touched[4];
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const int i = tx + 32 * k;
        touched[k] = -1;
        if (i < 121) {
          const int b = s_obin[i];
          s_hp[tx][b] = __fadd_rn(s_hp[tx][b], s_ow[i]);
          touched[k] = b;
        }
      }
      __syncwarp();
      float acc = 0.0f;
#pragma unroll 8
      for (int l = 0; l < 32; l++) acc = __fadd_rn(acc, s_hp[l][tx]);
      __syncwarp();
#pragma unroll
      for (int k = 0; k < 4; k++)
        if (touched[k] >= 0) s_hp[tx][touched[k]] = 0.0f;
      // :1004-1010 circular [1 4 6 4 1] smoothing, lane = bin
      const float h0 = acc;
      const float h1m = __shfl_sync(0xffffffffu, h0, (tx + 31) & 31), h1p = __shfl_sync(0xffffffffu, h0, (tx + 1) & 31);
      const float h2m = __shfl_sync(0xffffffffu, h0, (tx + 30) & 31), h2p = __shfl_sync(0xffffffffu, h0, (tx + 2) & 31);
      const float sm = __fadd_rn(__fmaf_rn(h0, 6.0f, __fmul_rn(4.0f, __fadd_rn(h1m, h1p))), __fadd_rn(h2m, h2p));
      const float smm = __shfl_sync(0xffffffffu, sm, (tx + 31) & 31), smp = __shfl_sync(0xffffffffu, sm, (tx + 1) & 31);
      const float pk = (sm > smm && sm >= smp ? sm : 0.0f);       // :1012-1015
      // :1018-1033: the serial scan keeps (largest, its first index) and (largest of the rest, its
      // first index); stated order-independently and evaluated with warp votes
      float m1 = pk;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, o));
      const unsigned b1 = __ballot_sync(0xffffffffu, pk == m1);
      const int i1 = (m1 > 0.0f) ? (__ffs(b1) - 1) : -1;
      float rest = (tx == i1) ? 0.0f : pk, m2 = rest;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m2 = fmaxf(m2, __shfl_xor_sync(0xffffffffu, m2, o));
      const unsigned b2 = __ballot_sync(0xffffffffu, rest == m2 && tx != i1);
      const int i2 = (m2 > 0.0f) ? (__ffs(b2) - 1) : -1;
      const float maxval1 = (i1 >= 0) ? m1 : 0.0f, maxval2 = (i2 >= 0) ? m2 : 0.0f;
      const float val1 = __shfl_sync(0xffffffffu, sm, (i1 + 1) & 31), val2 = __shfl_sync(0xffffffffu, sm, (i1 + 31) & 31);
      const float v1 = __shfl_sync(0xffffffffu, sm, (i2 + 1) & 31), v2 = __shfl_sync(0xffffffffu, sm, (i2 + 31) & 31);
      if (tx == 0) {   // :1034-1053
        s_next = (int)req;
        req = gridDim.x + atomicAdd(P.queue, 1u);
        float peak = __fadd_rn((float)i1, __fdiv_rn(__fmul_rn(0.5f, __fsub_rn(val1, val2)),
                                                    __fsub_rn(__fsub_rn(__fadd_rn(maxval1, maxval1), val1), val2)));
        s_ori[0] = __fmul_rn(11.25f, (peak < 0.0f ? __fadd_rn(peak, 32.0f) : peak));
        s_slot[0] = pt;
        int nori = 1;
        if (maxval2 > __fmul_rn(0.8f, maxval1)) {
          float pk2 = __fadd_rn((float)i2, __fdiv_rn(__fmul_rn(0.5f, __fsub_rn(v1, v2)),
                                                     __fsub_rn(__fsub_rn(__fadd_rn(maxval2, maxval2), v1), v2)));
          // Reference quirk Q1 (cudaSiftH.cu:115): secondary orientations of the finest
          // octave land beyond numPts and are never reported -> do not produce them.
          if (psub != P.finestSubsampling) {
            atomicMax(&counters[1], (unsigned)numPrim);
            unsigned int idx = atomicAdd(&counters[1], 1u);
            if (idx < (unsigned)P.maxPts) {
              s_ori[1] = __fmul_rn(11.25f, (pk2 < 0.0f ? __fadd_rn(pk2, 32.0f) : pk2));
              s_slot[1] = (int)idx;
              nori = 2;
            }
          }
        }
        s_nori = nori;
      }
    }
    __syncthreads();
    const int nori = s_nori;
    // read before any thread can pass the next keypoint's first two barriers, after which thread 0 rewrites it
    const int gnext = s_next;

    // ------------------------------------------------------------------ descriptors
    for (int k = 0; k < nori; k++) {
      const float orientation = s_ori[k];
      float theta = __fmul_rn(2.0f * 3.1415f / 360.0f, orientation);   // :330
      float sina = __sinf(theta), cosa = __cosf(theta);
      float scale = __fmul_rn(12.0f / 16.0f, pscale);
      float ssina = __fmul_rn(scale, sina), scosa = __fmul_rn(scale, cosa);
#pragma unroll
      for (int rep = 0; rep < 2; rep++) {
        const int sidx = tx + rep * DS_THREADS;     // sample index = y*16 + x
        const int y = sidx >> 4, x = sidx & 15;
        float tt = x - 7.5f, yy = y - 7.5f;
        // :338-339 as contracted in the reference's SASS
        float xpos = __fadd_rn(__fmaf_rn(-ssina, yy, __fadd_rn(__fmul_rn(tt, scosa), px)), 0.5f);
        float ypos = __fadd_rn(__fmaf_rn(scosa, yy, __fmaf_rn(tt, ssina, py)), 0.5f);
        float dx = __fsub_rn(tex2D<float>(tex, __fadd_rn(xpos, cosa), __fadd_rn(ypos, sina)),
                             tex2D<float>(tex, __fsub_rn(xpos, cosa), __fsub_rn(ypos, sina)));
        float dy = __fsub_rn(tex2D<float>(tex, __fsub_rn(xpos, sina), __fadd_rn(ypos, cosa)),
                             tex2D<float>(tex, __fadd_rn(xpos, sina), __fsub_rn(ypos, cosa)));
        float grad = __fmul_rn(__fmul_rn(s_gauss16[y], s_gauss16[x]),
                               __fsqrt_rn(__fmaf_rn(dx, dx, __fmul_rn(dy, dy))));
        float angf = __fmaf_rn(fast_atan2(dy, dx), 4.0f / 3.1415f, 4.0f);   // :345
        int hori = (x + 2) / 4 - 1;
        float horf = __fsub_rn(__fmul_rn(x - 1.5f, 0.25f), (float)hori), ihorf = __fsub_rn(1.0f, horf);
        int veri = (y + 2) / 4 - 1;
        float verf = __fsub_rn(__fmul_rn(y - 1.5f, 0.25f), (float)veri), iverf = __fsub_rn(1.0f, verf);
        int angi = __float2int_rz(angf);
        angf = __fsub_rn(angf, (float)angi);
        // Quirk Q22: for dy == +0, dx < 0 (edges of saturated areas) angf = 8.0001 and angi = 8;
        // the reference then adds its "iangf" vote at flat index 8*cell + 8, i.e. into angle
        // bin 0 of the NEXT cell (cudaSiftD.cu:353-384).  Reproduced in the accumulation below.
        float gl = __fmul_rn(ihorf, grad), gr = __fmul_rn(horf, grad);
        const int pidx = y * 17 + x;
        s_g2[0][pidx] = __fmul_rn(iverf, gl);
        s_g2[1][pidx] = __fmul_rn(verf, gl);
        s_g2[2][pidx] = __fmul_rn(iverf, gr);
        s_g2[3][pidx] = __fmul_rn(verf, gr);
        s_angf[pidx] = angf;
        s_angi[pidx] = angi;
      }
      __syncthreads();
      {  // deterministic accumulation.  Thread (cell, k): the k-th sample row of the cell's 8x8
         // window, summed over x into 8 private angle bins (+ slot 8 for quirk Q22: angi == 8
         // votes into angle bin 0 of the NEXT cell in flat order, cudaSiftD.cu:353-384).
        // The bins live in registers: each vote is a predicated add at a compile-time index, x ascending as before.
        // The loop has no branch: a (row, x) outside the 16x16 window votes +0.0f, which leaves every bin as it is
        // (a bin starts at +0, and a round-to-nearest sum that starts at +0 is never -0).
        const int cell = tx >> 3, kr = tx & 7;
        const int cy = cell >> 2, cx = cell & 3;
        const int y = 4 * cy - 2 + kr;
        const bool rowIn = (unsigned)y <= 15u;
        const int row = min(max(y, 0), 15) * 17;
        const int lower = kr < 4;                             // sample votes into its lower cell: ((y + 2) >> 2) - 1 != cy
        float pb[9];
#pragma unroll
        for (int a = 0; a < 9; a++) pb[a] = 0.0f;
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const int x = 4 * cx - 2 + j;                       // inside the window for j = 2..5 whatever cx is
          const bool edge = j < 2 || j > 5;
          const bool in = rowIn && (!edge || (unsigned)x <= 15u);
          const int sidx = row + (edge ? min(max(x, 0), 15) : x);
          const int angi = s_angi[sidx];
          const float af = s_angf[sidx];
          const float g2 = s_g2[(j < 4 ? 2 : 0) + lower][sidx];   // j < 4: ... into its right cell, ((x + 2) >> 2) - 1 != cx
          const float v1 = in ? __fmul_rn(__fsub_rn(1.0f, af), g2) : 0.0f;
          const float v2 = in ? __fmul_rn(af, g2) : 0.0f;
          const int a1 = min(angi, 8);
          // v1 goes to bin a1, v2 to bin angp = (angi < 7 ? angi + 1 : 0): bin a >= 1 when a1 == a - 1, bin 0 when
          // a1 >= 7.  a1 != angp, so no bin takes two votes of one sample.
          bool eq[9];
#pragma unroll
          for (int a = 0; a < 9; a++) eq[a] = (a1 == a);
#pragma unroll
          for (int a = 0; a < 9; a++)
            if (eq[a]) pb[a] = __fadd_rn(pb[a], v1);
          if (a1 >= 7) pb[0] = __fadd_rn(pb[0], v2);
#pragma unroll
          for (int a = 1; a < 8; a++)
            if (eq[a - 1]) pb[a] = __fadd_rn(pb[a], v2);
        }
#pragma unroll
        for (int a = 0; a < 9; a++) s_pb[tx][a] = pb[a];
      }
      __syncthreads();
      float v;
      {  // thread = output bin (cell, angle): fixed-order sum over the 8 rows
        const int cell = tx >> 3, a = tx & 7;
        float acc = 0.0f;
#pragma unroll
        for (int r = 0; r < 8; r++) acc = __fadd_rn(acc, s_pb[cell * 8 + r][a]);
        if (a == 0 && cell > 0) {
#pragma unroll
          for (int r = 0; r < 8; r++) acc = __fadd_rn(acc, s_pb[(cell - 1) * 8 + r][8]);
        }
        v = acc;
      }
      // :391-409 normalise, clamp at 0.2, renormalise
      float sum = __fmul_rn(v, v);
#pragma unroll
      for (int i = 16; i > 0; i /= 2) sum = __fadd_rn(sum, __shfl_down_sync(0xffffffffu, sum, i));
      if ((tx & 31) == 0) s_sums[0][tx >> 5] = sum;
      __syncthreads();
      float tsum1 = __fadd_rn(__fadd_rn(__fadd_rn(s_sums[0][0], s_sums[0][1]), s_sums[0][2]), s_sums[0][3]);
      float t1 = fminf(__fmul_rn(v, rsqrtf(tsum1)), 0.2f);
      sum = __fmul_rn(t1, t1);
#pragma unroll
      for (int i = 16; i > 0; i /= 2) sum = __fadd_rn(sum, __shfl_down_sync(0xffffffffu, sum, i));
      if ((tx & 31) == 0) s_sums[1][tx >> 5] = sum;
      __syncthreads();
      float tsum2 = __fadd_rn(__fadd_rn(__fadd_rn(s_sums[1][0], s_sums[1][1]), s_sums[1][2]), s_sums[1][3]);
      SiftPoint *out = pts + s_slot[k];
      out->data[tx] = __fmul_rn(t1, rsqrtf(tsum2));
      if (tx == 0) {
        out->xpos = __fmul_rn(px, psub);        // :410-414
        out->ypos = __fmul_rn(py, psub);
        out->scale = __fmul_rn(pscale, psub);
        out->orientation = orientation;
        if (k == 1) {                           // :1045-1051 (copy of the primary)
          out->sharpness = sp->sharpness;
          out->edgeness = sp->edgeness;
          out->subsampling = psub;
        }
      }
      // No barrier here: every shared word read since the last one is next written only after a later barrier
      // (the next orientation's first one, or the next keypoint's second one).
    }
    g = gnext;
  }
}

// One resident wave (resident_grid); a CTA whose first claim is past the end of the queue exits at once.
int launch_describe(const DescribeParams &p, cudaStream_t st)
{
  const int grid = resident_grid<describe_kernel, DS_THREADS>();
  if (grid < 0) return grid;
  describe_kernel<<<grid, DS_THREADS, 0, st>>>(p);
  count_launch();
  CS_CUDA(cudaGetLastError());
  return 0;
}

// cudaSiftD.cu:753-761 (RescalePositions) for the scaleUp path; count read on device.
__global__ void rescale_kernel(SiftPoint *pts, const unsigned int *counters, int maxPts, float f)
{
  unsigned int n = max(min(counters[0], (unsigned)maxPts), min(counters[1], (unsigned)maxPts));
  for (unsigned int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    pts[i].xpos = __fmul_rn(pts[i].xpos, f);
    pts[i].ypos = __fmul_rn(pts[i].ypos, f);
    pts[i].scale = __fmul_rn(pts[i].scale, f);
  }
}

int launch_rescale(SiftPoint *pts, const unsigned int *counters, int maxPts, float f, cudaStream_t st)
{
  rescale_kernel<<<64, 128, 0, st>>>(pts, counters, maxPts, f);
  count_launch();
  CS_CUDA(cudaGetLastError());
  return 0;
}

__global__ void tex_probe_kernel(cudaTextureObject_t tex, const float *xs, const float *ys, int n, float *out)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = tex2D<float>(tex, xs[i], ys[i]);
}

int launch_tex_probe(cudaTextureObject_t tex, const float *xs, const float *ys, int n, float *out, cudaStream_t st)
{
  tex_probe_kernel<<<idivup(n, 256), 256, 0, st>>>(tex, xs, ys, n, out);
  count_launch();
  CS_CUDA(cudaGetLastError());
  return 0;
}

int make_texture(cudaTextureObject_t *tex, const float *img, int w, int h, int pitch)
{ // cudaSiftH.cu:186-205
  cudaResourceDesc res = {};
  res.resType = cudaResourceTypePitch2D;
  res.res.pitch2D.devPtr = const_cast<float *>(img);
  res.res.pitch2D.width = w;
  res.res.pitch2D.height = h;
  res.res.pitch2D.pitchInBytes = (size_t)pitch * sizeof(float);
  res.res.pitch2D.desc = cudaCreateChannelDesc<float>();
  cudaTextureDesc td = {};
  td.addressMode[0] = cudaAddressModeClamp;
  td.addressMode[1] = cudaAddressModeClamp;
  td.filterMode = cudaFilterModeLinear;
  td.readMode = cudaReadModeElementType;
  td.normalizedCoords = 0;
  CS_CUDA(cudaCreateTextureObject(tex, &res, &td, NULL));
  return 0;
}

}  // namespace cs
