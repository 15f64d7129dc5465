// fp32 CUDA-core path of WaterNet.forward (WN_MODE_FP32_SIMT).
//
// Replaces /root/reference/waternet/net.py:45-56 (confidence maps), :75-80
// (refiners) and :99-108 (gated sum) with direct convolutions in plain fp32 FMA:
// no tensor cores, no operand rounding -- the arithmetic-exact mode the tensor-core
// path is compared against at sizes the CPU oracle cannot reach.
//
// Layout: activations are fp32 NCHW planes (what the API hands in and expects
// back).  One CTA computes a 32x8 pixel tile for up to 64 output channels;
// each warp owns 8 output channels, each lane one pixel column of 8 rows
// (64 accumulators).  Input halo tile and weights for a chunk of input
// channels are staged in shared memory; weights are read as warp-wide
// broadcasts, activations conflict-free (lane == x).
#include "common.cuh"

namespace wn {

constexpr int kTileW = 32;
constexpr int kTileH = 8;
constexpr int kCoutPerWarp = 8;

template <int KS>
struct SimtCfg {
  static constexpr int TH = kTileH + KS - 1;
  static constexpr int TW = kTileW + KS - 1;
  // input channels per shared-memory chunk, sized for ~60 KB with 64 couts
  static constexpr int CC = KS == 7 ? 4 : KS == 5 ? 8 : KS == 3 ? 16 : 32;
};

// act: 0 none, 1 relu, 2 sigmoid
template <int KS>
__global__ void __launch_bounds__(256)
conv_simt_kernel(const float* __restrict__ in, const float* __restrict__ wpk,
                 const float* __restrict__ bias, float* __restrict__ out, int cin, int cout,
                 int cout_pad, int H, int W, int act) {
  using C = SimtCfg<KS>;
  extern __shared__ __align__(16) float smem[];
  const int nwarps = blockDim.y;
  const int CB = nwarps * kCoutPerWarp;  // output channels of this CTA
  float* s_in = smem;                                  // [CC][TH][TW]
  float* s_w = smem + C::CC * C::TH * C::TW;           // [CC][KS*KS][CB]
  const int lane = threadIdx.x, warp = threadIdx.y;
  const int tid = warp * 32 + lane, nthreads = nwarps * 32;
  const int ncb = cout_pad / CB;
  const int n = blockIdx.z / ncb, cb = blockIdx.z % ncb;
  const int x0 = blockIdx.x * kTileW, y0 = blockIdx.y * kTileH;
  const size_t plane = (size_t)H * W;
  const float* in_n = in + (size_t)n * cin * plane;

  float acc[kTileH][kCoutPerWarp];
#pragma unroll
  for (int r = 0; r < kTileH; r++)
#pragma unroll
    for (int q = 0; q < kCoutPerWarp; q++) acc[r][q] = 0.f;

  for (int c0 = 0; c0 < cin; c0 += C::CC) {
    const int cc = min(C::CC, cin - c0);
    // stage the input halo tile (zero padding == padding="same")
    for (int i = tid; i < cc * C::TH * C::TW; i += nthreads) {
      int c = i / (C::TH * C::TW);
      int rem = i - c * (C::TH * C::TW);
      int ty = rem / C::TW, tx = rem - ty * C::TW;
      int gy = y0 + ty - KS / 2, gx = x0 + tx - KS / 2;
      float v = 0.f;
      if (gy >= 0 && gy < H && gx >= 0 && gx < W) v = in_n[(size_t)(c0 + c) * plane + (size_t)gy * W + gx];
      s_in[i] = v;
    }
    // stage weights [c][tap][CB]
    for (int i = tid; i < cc * KS * KS * CB; i += nthreads) {
      int row = i / CB, col = i - row * CB;  // row = c*KS*KS + tap
      s_w[i] = wpk[((size_t)c0 * KS * KS + row) * cout_pad + cb * CB + col];
    }
    __syncthreads();
    for (int c = 0; c < cc; c++) {
      const float* tin = s_in + c * C::TH * C::TW + lane;
      const float* tw = s_w + (size_t)c * KS * KS * CB + warp * kCoutPerWarp;
#pragma unroll
      for (int kx = 0; kx < KS; kx++) {
        float a[C::TH];
#pragma unroll
        for (int j = 0; j < C::TH; j++) a[j] = tin[j * C::TW + kx];
#pragma unroll
        for (int ky = 0; ky < KS; ky++) {
          const float4 w0 = *reinterpret_cast<const float4*>(tw + (ky * KS + kx) * CB);
          const float4 w1 = *reinterpret_cast<const float4*>(tw + (ky * KS + kx) * CB + 4);
          const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
          for (int r = 0; r < kTileH; r++)
#pragma unroll
            for (int q = 0; q < kCoutPerWarp; q++) acc[r][q] = fmaf(a[r + ky], wv[q], acc[r][q]);
        }
      }
    }
    __syncthreads();
  }

  const int gx = x0 + lane;
  if (gx >= W) return;
#pragma unroll
  for (int q = 0; q < kCoutPerWarp; q++) {
    const int co = cb * CB + warp * kCoutPerWarp + q;
    if (co >= cout) continue;
    const float bv = bias[co];
    float* o = out + ((size_t)n * cout + co) * plane;
#pragma unroll
    for (int r = 0; r < kTileH; r++) {
      const int gy = y0 + r;
      if (gy >= H) continue;
      float v = acc[r][q] + bv;
      if (act == 1) v = fmaxf(v, 0.f);
      else if (act == 2) v = 1.0f / (1.0f + expf(-v));
      o[(size_t)gy * W + gx] = v;
    }
  }
}

// OIHW fp32 -> [cin][ks*ks][cout_pad] (zero padded), bias -> [cout_pad]
__global__ void simt_pack_kernel(const float* __restrict__ w, const float* __restrict__ b,
                                 float* __restrict__ wpk, float* __restrict__ bpk, int cin,
                                 int cout, int cout_pad, int ks) {
  const int total = cin * ks * ks * cout_pad;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    int co = i % cout_pad;
    int row = i / cout_pad;
    int tap = row % (ks * ks), c = row / (ks * ks);
    wpk[i] = co < cout ? w[((size_t)co * cin + c) * ks * ks + tap] : 0.f;
  }
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < cout_pad; i += gridDim.x * blockDim.x)
    bpk[i] = i < cout ? b[i] : 0.f;
}

// torch.cat([x, wb, ce, gc], 1) with arbitrary input strides -> contiguous (N,12,H,W)
struct CatArgs {
  const float* p[4];
  long long s[4][4];
};
__global__ void cat_inputs_kernel(CatArgs a, float* __restrict__ out, int H, int W) {
  const int n = blockIdx.z, ch = blockIdx.y;  // ch in 0..11
  const int t = ch / 3, c = ch % 3;
  const int plane = H * W;
  for (int pix = blockIdx.x * blockDim.x + threadIdx.x; pix < plane; pix += gridDim.x * blockDim.x) {
    int y = pix / W, x = pix - y * W;
    out[((size_t)n * 12 + ch) * plane + pix] =
        a.p[t][n * a.s[t][0] + c * a.s[t][1] + y * a.s[t][2] + x * a.s[t][3]];
  }
}

// out = refined_wb*cm_wb + refined_ce*cm_ce + refined_gc*cm_gc   (net.py:104-108)
__global__ void gate_sum_kernel(const float* __restrict__ cm, const float* __restrict__ r0,
                                const float* __restrict__ r1, const float* __restrict__ r2,
                                float* __restrict__ out, int plane) {
  const int n = blockIdx.y;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= plane) return;
  const size_t base = (size_t)n * 3 * plane + pix;
  const float c0 = cm[base], c1 = cm[base + plane], c2 = cm[base + 2 * (size_t)plane];
#pragma unroll
  for (int c = 0; c < 3; c++) {
    size_t i = base + (size_t)c * plane;
    // same association as the reference: (a + b) + c, products rounded first
    out[i] = __fadd_rn(__fadd_rn(__fmul_rn(r0[i], c0), __fmul_rn(r1[i], c1)), __fmul_rn(r2[i], c2));
  }
}

// ---------------------------------------------------------------------------
static int layer_of(int idx, LayerDesc* d) {
  if (idx < 8) *d = kCmg[idx];
  else *d = kRef[(idx - 8) % 3];
  return 0;
}

int simt_pack_weights(wn_handle* h, const float* const* params, cudaStream_t stream) {
  for (int i = 0; i < kNumConvs; i++) {
    LayerDesc d;
    layer_of(i, &d);
    SimtLayer& L = h->simt[i];
    L.cin = d.cin;
    L.cout = d.cout;
    L.ks = d.ks;
    L.cout_pad = (d.cout + 7) / 8 * 8;
    size_t wn_ = (size_t)d.cin * d.ks * d.ks * L.cout_pad;
    if (!L.w) WN_CUDA(cudaMalloc(&L.w, wn_ * sizeof(float)));
    if (!L.bias) WN_CUDA(cudaMalloc(&L.bias, L.cout_pad * sizeof(float)));
    simt_pack_kernel<<<64, 256, 0, stream>>>(params[2 * i], params[2 * i + 1], L.w, L.bias, d.cin,
                                             d.cout, L.cout_pad, d.ks);
    WN_LAUNCH_CHECK(h);
  }
  return WN_OK;
}

void simt_free(wn_handle* h) {
  for (int i = 0; i < kNumConvs; i++) {
    if (h->simt[i].w) cudaFree(h->simt[i].w);
    if (h->simt[i].bias) cudaFree(h->simt[i].bias);
    h->simt[i].w = h->simt[i].bias = nullptr;
  }
}

template <int KS>
static int launch_conv(wn_handle* h, const SimtLayer& L, const float* in, float* out, int n, int H,
                       int W, int act, cudaStream_t stream) {
  using C = SimtCfg<KS>;
  int nwarps = L.cout_pad / kCoutPerWarp;
  if (nwarps > 8) nwarps = 8;
  int CB = nwarps * kCoutPerWarp;
  if (L.cout_pad % CB != 0) {
    set_error("cout_pad %d not a multiple of %d", L.cout_pad, CB);
    return WN_E_UNSUPPORTED;
  }
  size_t smem = (size_t)C::CC * (C::TH * C::TW + KS * KS * CB) * sizeof(float);
  WN_CUDA(cudaFuncSetAttribute(conv_simt_kernel<KS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)smem));
  dim3 grid((W + kTileW - 1) / kTileW, (H + kTileH - 1) / kTileH, n * (L.cout_pad / CB));
  if (grid.y > 65535 || grid.z > 65535) {
    set_error("grid too large for the SIMT path");
    return WN_E_UNSUPPORTED;
  }
  conv_simt_kernel<KS><<<grid, dim3(32, nwarps), smem, stream>>>(in, L.w, L.bias, out, L.cin,
                                                                 L.cout, L.cout_pad, H, W, act);
  WN_LAUNCH_CHECK(h);
  return WN_OK;
}

static int run_conv(wn_handle* h, int idx, const float* in, float* out, int n, int H, int W, int act,
                    cudaStream_t stream) {
  const SimtLayer& L = h->simt[idx];
  TimedScope ts(h, kSlotConv0 + idx, stream);
  switch (L.ks) {
    case 1: return launch_conv<1>(h, L, in, out, n, H, W, act, stream);
    case 3: return launch_conv<3>(h, L, in, out, n, H, W, act, stream);
    case 5: return launch_conv<5>(h, L, in, out, n, H, W, act, stream);
    case 7: return launch_conv<7>(h, L, in, out, n, H, W, act, stream);
  }
  set_error("unsupported kernel size %d", L.ks);
  return WN_E_UNSUPPORTED;
}

// workspace (floats per pixel per image): cat 12 | A 128 | B 128 | cm 3 | pair 6 | r32a 32 | r32b 32 | refined 9
static constexpr size_t kSimtFloatsPerPixel = 12 + 128 + 128 + 3 + 6 + 32 + 32 + 9;

// Images per pass: bounds the workspace (~1.4 KB per pixel) to a few GB at any batch size.
static int simt_chunk(int n, int h, int w) {
  long long per = (long long)h * w;
  long long nb = (4ll << 20) / (per > 0 ? per : 1);
  if (nb < 1) nb = 1;
  return nb < n ? (int)nb : n;
}

size_t simt_forward_workspace_bytes(int n, int h, int w) {
  return (size_t)simt_chunk(n, h, w) * h * w * kSimtFloatsPerPixel * sizeof(float) + 256;
}

// [x, other] -> contiguous (N,6,H,W): channels 0..2 and 3k..3k+2 of the 12-channel cat
__global__ void pair_kernel(const float* __restrict__ cat12, float* __restrict__ out, int which,
                            int plane) {
  const int n = blockIdx.z, ch = blockIdx.y;  // 0..5
  const int src = ch < 3 ? ch : 3 * which + (ch - 3);
  for (int pix = blockIdx.x * blockDim.x + threadIdx.x; pix < plane; pix += gridDim.x * blockDim.x)
    out[((size_t)n * 6 + ch) * plane + pix] = cat12[((size_t)n * 12 + src) * plane + pix];
}

static int simt_forward_chunk(wn_handle* h, const float* const in[4],
                              const int64_t in_strides[4][4], float* out, int n, int H, int W,
                              void* workspace, cudaStream_t stream, int dbg_layer = -1,
                              float* dbg_dst = nullptr, int stack = kStackAll, int which = 0);

int simt_forward(wn_handle* h, const float* const in[4], const int64_t in_strides[4][4], float* out,
                 int n, int H, int W, void* workspace, size_t workspace_bytes, cudaStream_t stream, int stack,
                 int which) {
  if (workspace_bytes < simt_forward_workspace_bytes(n, H, W)) {
    set_error("forward workspace too small: %zu < %zu", workspace_bytes,
              simt_forward_workspace_bytes(n, H, W));
    return WN_E_WORKSPACE;
  }
  const int nb = simt_chunk(n, H, W);
  for (int n0 = 0; n0 < n; n0 += nb) {
    const int cur = n - n0 < nb ? n - n0 : nb;
    const float* sub[4];
    for (int t = 0; t < 4; t++) sub[t] = in[t] + (long long)n0 * in_strides[t][0];
    int rc = simt_forward_chunk(h, sub, in_strides, out + (size_t)n0 * 3 * H * W, cur, H, W,
                                workspace, stream, -1, nullptr, stack, which);
    if (rc) return rc;
  }
  return WN_OK;
}

int simt_debug_layer(wn_handle* h, const float* const in[4], const int64_t in_strides[4][4], int n,
                     int H, int W, int layer, float* dst, void* workspace, size_t workspace_bytes,
                     cudaStream_t stream) {
  if (simt_chunk(n, H, W) != n || workspace_bytes < simt_forward_workspace_bytes(n, H, W)) {
    set_error("debug layer dump: batch too large for one pass or workspace too small");
    return WN_E_WORKSPACE;
  }
  return simt_forward_chunk(h, in, in_strides, nullptr, n, H, W, workspace, stream, layer, dst);
}

static int simt_forward_chunk(wn_handle* h, const float* const in[4],
                              const int64_t in_strides[4][4], float* out, int n, int H, int W,
                              void* workspace, cudaStream_t stream, int dbg_layer, float* dbg_dst, int stack,
                              int which) {
  const size_t px = (size_t)n * H * W;
  const int plane = H * W;
  float* ws = (float*)(((uintptr_t)workspace + 255) / 256 * 256);
  float* cat12 = ws;            ws += px * 12;
  float* bufA = ws;             ws += px * 128;
  float* bufB = ws;             ws += px * 128;
  float* cm = ws;               ws += px * 3;
  float* pair = ws;             ws += px * 6;
  float* r32a = ws;             ws += px * 32;
  float* r32b = ws;             ws += px * 32;
  float* refined = ws;          // 3 x (N,3,H,W)

  CatArgs ca;
  for (int t = 0; t < 4; t++) {
    ca.p[t] = in[t];
    for (int k = 0; k < 4; k++) ca.s[t][k] = in_strides[t][k];
  }
  int gx = (plane + 255) / 256;
  if (gx > 4096) gx = 4096;
  {
    TimedScope ts(h, kSlotPack, stream);
    cat_inputs_kernel<<<dim3(gx, 12, n), 256, 0, stream>>>(ca, cat12, H, W);
    WN_LAUNCH_CHECK(h);
  }

  // confidence-map generator: net.py:46-55
  int rc;
  const float* cur = cat12;
  float* pp[2] = {bufA, bufB};
  for (int i = 0; i < 8 && stack != kStackRefiners; i++) {
    float* dst = i == 7 ? (stack == kStackCmg ? out : cm) : pp[i & 1];
    if ((rc = run_conv(h, i, cur, dst, n, H, W, i == 7 ? 2 : 1, stream))) return rc;
    cur = dst;
    if (dbg_layer == i) {
      WN_CUDA(cudaMemcpyAsync(dbg_dst, dst, px * h->simt[i].cout * sizeof(float), cudaMemcpyDeviceToDevice, stream));
      return WN_OK;
    }
  }
  if (stack == kStackCmg) return WN_OK;  // ConfidenceMapGenerator.forward: the maps went straight to `out`
  // refiners: net.py:76-80, inputs cat[x, wb], cat[x, ce], cat[x, gc]
  for (int r = 0; r < 3; r++) {
    if (stack == kStackRefiners && r != which) continue;  // Refiner.forward of one refiner
    {
      TimedScope ts(h, kSlotPack, stream);
      pair_kernel<<<dim3(gx, 6, n), 256, 0, stream>>>(cat12, pair, r + 1, plane);
      WN_LAUNCH_CHECK(h);
    }
    float* refr = stack == kStackRefiners ? out : refined + (size_t)r * px * 3;
    if ((rc = run_conv(h, 8 + 3 * r + 0, pair, r32a, n, H, W, 1, stream))) return rc;
    if ((rc = run_conv(h, 8 + 3 * r + 1, r32a, r32b, n, H, W, 1, stream))) return rc;
    if (dbg_layer == 8 || dbg_layer == 9) {  // (N,32,H,W) -> channels 32r.. of (N,96,H,W)
      const float* src = dbg_layer == 8 ? r32a : r32b;
      WN_CUDA(cudaMemcpy2DAsync(dbg_dst + (size_t)r * 32 * plane, (size_t)96 * plane * sizeof(float), src,
                                (size_t)32 * plane * sizeof(float), (size_t)32 * plane * sizeof(float), n,
                                cudaMemcpyDeviceToDevice, stream));
      continue;
    }
    if ((rc = run_conv(h, 8 + 3 * r + 2, r32b, refr, n, H, W, 1, stream))) return rc;
    if (dbg_layer == 10)  // (N,3,H,W) -> channels 3r.. of (N,9,H,W)
      WN_CUDA(cudaMemcpy2DAsync(dbg_dst + (size_t)r * 3 * plane, (size_t)9 * plane * sizeof(float), refr,
                                (size_t)3 * plane * sizeof(float), (size_t)3 * plane * sizeof(float), n,
                                cudaMemcpyDeviceToDevice, stream));
  }
  if (dbg_layer >= 0 || stack == kStackRefiners) return WN_OK;
  TimedScope ts(h, kSlotGate, stream);
  gate_sum_kernel<<<dim3((plane + 255) / 256, n), 256, 0, stream>>>(
      cm, refined, refined + px * 3, refined + 2 * px * 3, out, plane);
  WN_LAUNCH_CHECK(h);
  return WN_OK;
}

}  // namespace wn
