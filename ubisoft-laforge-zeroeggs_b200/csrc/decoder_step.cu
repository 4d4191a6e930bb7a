// One teacher-forced step of the recurrent decoder (RecurrentDecoderNormal.forward, ZEGGS/modules.py:179-185):
//   u = [pose | speech | style];  a = ELU(W0 u + b0);  v = [a | u];  (h0', h1') = 2-layer GRU(v, (h0, h1));  y = W2 h1' + b2
// in fp32 (SIMT GEMMs, no bf16 anywhere): the tight per-step parity point SURVEY.md 8b/8d asks for (<= 1e-4 in normalised units)
// and the building block for streaming inference.  The window kernels (decoder_fwd*.cu) are the throughput path.
#include "decoder_common.cuh"

namespace zeggs {

// v[b] = [a[b] (H) | pose[b] (1134) | speech[b] (S) | style[b] (Z)];  u = v + H
__global__ void step_concat_kernel(int B, int H, int S, int Z, const float* __restrict__ pose, const float* __restrict__ speech,
                                   const float* __restrict__ style, float* __restrict__ v) {
  const int A = P_IN + S + Z, ld = H + A;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < B * A; i += gridDim.x * blockDim.x) {
    const int b = i / A, k = i % A;
    const float x = k < P_IN ? pose[(size_t)b * P_IN + k] : k < P_IN + S ? speech[(size_t)b * S + (k - P_IN)] : style[(size_t)b * Z + (k - P_IN - S)];
    v[(size_t)b * ld + H + k] = x;
  }
}
// nn.GRU cell gates (PyTorch order r, z, n; b_hn inside r * (...)): gi, gh [B,3H] (biases already added) -> h' = (1-z) n + z h
__global__ void step_gru_kernel(int B, int H, const float* __restrict__ gi, const float* __restrict__ gh, const float* __restrict__ h,
                                float* __restrict__ hn) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < B * H; i += gridDim.x * blockDim.x) {
    const int b = i / H, j = i % H;
    const float* gib = gi + (size_t)b * 3 * H; const float* ghb = gh + (size_t)b * 3 * H;
    const float r = sigmoid_f(gib[j] + ghb[j]);
    const float z = sigmoid_f(gib[H + j] + ghb[H + j]);
    const float n = tanhf(gib[2 * H + j] + r * ghb[2 * H + j]);
    hn[i] = (1.0f - z) * n + z * h[i];
  }
}

struct StepWs { float *v, *gi, *gh; size_t bytes; };
static StepWs step_ws(void* base, int B, int H, int S, int Z) {
  StepWs w; Arena a{(char*)base};
  w.v = a.take((size_t)B * (H + P_IN + S + Z)); w.gi = a.take((size_t)B * 3 * H); w.gh = a.take((size_t)B * 3 * H);
  w.bytes = a.off; return w;
}
extern "C" size_t zeggs_decoder_step_workspace_bytes(int B, int H, int S, int Z) {
  return (B < 1 || H < 1) ? 0 : step_ws(nullptr, B, H, S, Z).bytes;
}

extern "C" int zeggs_decoder_step_fwd(const zeggs_decoder_step_args* ap, void* stream_) {
  ZCHECK_ARG(ap, "decoder step: null args");
  const zeggs_decoder_step_args& a = *ap; cudaStream_t s = (cudaStream_t)stream_;
  const int B = a.B, H = a.H, S = a.S, Z = a.Z, A = P_IN + S + Z, ldv = H + A;
  ZCHECK_ARG(B >= 1 && H >= 1 && S >= 0 && Z >= 0, "decoder step: bad shape");
  ZCHECK_ARG(a.W0 && a.b0 && a.W_ih0 && a.b_ih0 && a.W_hh0 && a.b_hh0 && a.W_ih1 && a.b_ih1 && a.W_hh1 && a.b_hh1 && a.W2 && a.b2,
             "decoder step: null weight");
  ZCHECK_ARG(a.pose && a.speech && a.style && a.h_in && a.y && a.h_out, "decoder step: null tensor");
  StepWs w = step_ws(a.workspace, B, H, S, Z);
  ZCHECK_ARG(a.workspace && a.workspace_bytes >= w.bytes, "decoder step: workspace too small");
  const int g1 = ceil_div(B * A, 256), g2 = ceil_div(B * H, 256);
  step_concat_kernel<<<g1 > 592 ? 592 : g1, 256, 0, s>>>(B, H, S, Z, a.pose, a.speech, a.style, w.v); count_launch();
  int rc;
  // a = ELU(W0 u + b0) written straight into the first H columns of v
  rc = sgemm_launch(0, B, H, A, w.v + H, ldv, a.W0, A, a.b0, w.v, ldv, 1, 0, s); if (rc) return rc;
  rc = sgemm_launch(0, B, 3 * H, ldv, w.v, ldv, a.W_ih0, ldv, a.b_ih0, w.gi, 3 * H, 0, 0, s); if (rc) return rc;
  rc = sgemm_launch(0, B, 3 * H, H, a.h_in, H, a.W_hh0, H, a.b_hh0, w.gh, 3 * H, 0, 0, s); if (rc) return rc;
  step_gru_kernel<<<g2 > 592 ? 592 : g2, 256, 0, s>>>(B, H, w.gi, w.gh, a.h_in, a.h_out); count_launch();
  rc = sgemm_launch(0, B, 3 * H, H, a.h_out, H, a.W_ih1, H, a.b_ih1, w.gi, 3 * H, 0, 0, s); if (rc) return rc;
  rc = sgemm_launch(0, B, 3 * H, H, a.h_in + (size_t)B * H, H, a.W_hh1, H, a.b_hh1, w.gh, 3 * H, 0, 0, s); if (rc) return rc;
  step_gru_kernel<<<g2 > 592 ? 592 : g2, 256, 0, s>>>(B, H, w.gi, w.gh, a.h_in + (size_t)B * H, a.h_out + (size_t)B * H); count_launch();
  rc = sgemm_launch(0, B, P_OUT, H, a.h_out + (size_t)B * H, H, a.W2, H, a.b2, a.y, P_OUT, 0, 0, s); if (rc) return rc;
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

}  // namespace zeggs
