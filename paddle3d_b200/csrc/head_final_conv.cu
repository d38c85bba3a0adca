// Grouped 3x3 output convs of CenterHead's SeparateHeads (detection/centerpoint/center_head.py:80-117: per task and
// per head a Conv2D 64 -> {2, 1, 3, 2, 2, num_classes}, kernel 3, padding 1, with bias, no activation) as ONE launch on
// the CUDA cores.  With 1-3 output channels per conv the tensor-core kernel spends a whole 128 x 16 MMA pipeline "use"
// per 32 input channels of one head; here a block stages a 16 x 8 pixel tile (+ halo) of one head's 64 input channels
// in shared memory, channel-major, and every thread accumulates the <= 4 outputs of its pixel with exact fp32 FMAs in
// (tap, channel) order.
// Checked by tests/test_gpu_dense.py::test_batched_head_matches_per_layer_head.
//
//   input   pixel split rows [B*H*W][2][in_C]; group g reads channels [g*Cin, (g+1)*Cin) as hi + lo
//   weight  [groups][9][Cin][4] fp32 (outputs zero-padded to 4), bias [groups][4]
//   output  fp32 planes [B][planes][H][W]; group g writes planes plane0[g] .. plane0[g] + cnt[g] - 1
#include "common.cuh"
#include "p3d_b200.h"

namespace p3d {
namespace {

constexpr int kTW = 16, kTH = 8, kHW = (kTW + 2) * (kTH + 2);  // tile and haloed tile (180 pixels)
constexpr int kPitch = kHW + 1;  // odd channel pitch: the transposing stores of the staging loop hit 32 different banks
constexpr int kMaxGroups = 64;

struct FinalParams {
  int B, H, W, in_C, Cin, groups, planes;
  int tiles_x, tiles_y;
  int plane0[kMaxGroups];
  int cnt[kMaxGroups];
};

__global__ void __launch_bounds__(128) head_final_conv_kernel(const float *__restrict__ in_split, FinalParams p,
                                                              const float *__restrict__ weight,
                                                              const float *__restrict__ bias, float *__restrict__ out) {
  extern __shared__ float s_mem[];
  float *s_x = s_mem;                    // [Cin][kPitch]  channel-major haloed tile (hi + lo)
  float *s_w = s_mem + p.Cin * kPitch;   // [9][Cin][4]  (Cin % 4 == 0 keeps it 16-byte aligned)
  long long q = blockIdx.x;
  const int g = static_cast<int>(q % p.groups);
  q /= p.groups;
  const int tx0 = static_cast<int>(q % p.tiles_x) * kTW;
  q /= p.tiles_x;
  const int ty0 = static_cast<int>(q % p.tiles_y) * kTH;
  const int b = static_cast<int>(q / p.tiles_y);
  const int tid = threadIdx.x;
  // stage the haloed tile: consecutive threads read consecutive channels of one pixel (coalesced), store transposed
  for (int e = tid; e < kHW * p.Cin; e += blockDim.x) {
    const int px = e / p.Cin, c = e - px * p.Cin;
    const int y = ty0 - 1 + px / (kTW + 2), x = tx0 - 1 + px % (kTW + 2);
    float v = 0.f;
    if (y >= 0 && y < p.H && x >= 0 && x < p.W) {
      const size_t pix = (static_cast<size_t>(b) * p.H + y) * p.W + x;
      const float *row = in_split + pix * (2 * static_cast<size_t>(p.in_C));
      v = __ldg(row + g * p.Cin + c) + __ldg(row + p.in_C + g * p.Cin + c);
    }
    s_x[c * kPitch + px] = v;
  }
  for (int e = tid; e < 9 * p.Cin * 4; e += blockDim.x) s_w[e] = __ldg(weight + static_cast<size_t>(g) * 9 * p.Cin * 4 + e);
  __syncthreads();
  const int ly = tid / kTW, lx = tid % kTW;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int t = 0; t < 9; ++t) {
    const int px = (ly + t / 3) * (kTW + 2) + lx + t % 3;
    const float *w = s_w + t * p.Cin * 4;
    for (int c = 0; c < p.Cin; ++c) {
      const float xv = s_x[c * kPitch + px];
      const float4 wv = *reinterpret_cast<const float4 *>(w + c * 4);
      acc[0] = fmaf(xv, wv.x, acc[0]);
      acc[1] = fmaf(xv, wv.y, acc[1]);
      acc[2] = fmaf(xv, wv.z, acc[2]);
      acc[3] = fmaf(xv, wv.w, acc[3]);
    }
  }
  const int y = ty0 + ly, x = tx0 + lx;
  if (y < p.H && x < p.W) {
    for (int k = 0; k < p.cnt[g]; ++k)
      out[((static_cast<size_t>(b) * p.planes + p.plane0[g] + k) * p.H + y) * p.W + x] = acc[k] + __ldg(bias + g * 4 + k);
  }
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" int p3d_head_final_conv(const float *in_split, int B, int H, int W, int in_C, int Cin, int groups,
                                   const float *weight, const float *bias, const int32_t *plane0_host,
                                   const int32_t *cnt_host, int planes, float *out_nchw, p3d_stream_t stream) {
  if (!in_split || !weight || !bias || !plane0_host || !cnt_host || !out_nchw || B < 1 || H < 1 || W < 1)
    return P3D_ERR_INVALID_ARG;
  if (groups < 1 || groups > kMaxGroups || Cin < 4 || Cin % 4 || groups * Cin > in_C || planes < 1)
    return P3D_ERR_INVALID_ARG;
  FinalParams p;
  p.B = B;
  p.H = H;
  p.W = W;
  p.in_C = in_C;
  p.Cin = Cin;
  p.groups = groups;
  p.planes = planes;
  p.tiles_x = (W + kTW - 1) / kTW;
  p.tiles_y = (H + kTH - 1) / kTH;
  for (int g = 0; g < groups; ++g) {
    if (cnt_host[g] < 1 || cnt_host[g] > 4 || plane0_host[g] < 0 || plane0_host[g] + cnt_host[g] > planes)
      return P3D_ERR_INVALID_ARG;
    p.plane0[g] = plane0_host[g];
    p.cnt[g] = cnt_host[g];
  }
  const size_t smem = (static_cast<size_t>(Cin) * kPitch + 9 * static_cast<size_t>(Cin) * 4) * sizeof(float);
  if (smem > 200 * 1024) return P3D_ERR_UNSUPPORTED;
  const long long blocks = static_cast<long long>(B) * p.tiles_y * p.tiles_x * groups;
  P3D_CUDA_CHECK(cudaFuncSetAttribute(head_final_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      static_cast<int>(smem)));
  head_final_conv_kernel<<<static_cast<unsigned int>(blocks), 128, smem, static_cast<cudaStream_t>(stream)>>>(
      in_split, p, weight, bias, out_nchw);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}
