// Mel front end: reflect-pad -> symmetric-Hann STFT magnitude / n_fft -> Slaney mel filterbank -> clip ->
// dB -> [0,1] -> (optional) ln(10^(s/20)), 80->60 fps linear resample, energy channel.
// Replaces ZEGGS/audio/spectrograms.py:216-269, :161-183, :386-503, :57-131 and
// ZEGGS/data_pipeline.py:62-82 (one fused kernel; HBM-bound: each sample is read ~once, each output
// written once).
//
// See mel_kernel below: register-resident 32 x 25 split of an 800-point complex FFT carrying two real frames.
#include "library.cuh"
#include "mel_fft.cuh"

namespace zeggs {

constexpr int MEL_FT = 30;       // output frames per tile (+1 neighbour frame for the resampler = 31 -> 16 frame PAIRS)
constexpr int MEL_PAIRS = (MEL_FT + 2) / 2;
constexpr int MEL_WARPS = 8;
constexpr int MEL_N2 = 400;      // n_fft / 2: rfft bins 0..400
constexpr int MEL_TB = 25 * 33;  // per-warp transpose buffer, complex words (row stride 33: conflict-free both ways)

// One CTA = one clip x a tile of MEL_FT consecutive STFT frames.  The tile's samples are staged once in shared memory
// (coalesced, reflect padding resolved at load).  Each warp then takes frame PAIRS: frame A in the real part and frame B
// in the imaginary part of one 800-point complex FFT, split 32 x 25 -- every lane transforms 25 points in registers,
// the intermediate is transposed through shared memory, 25 lanes run a 32-point transform each, and the two real
// spectra are separated with one warp shuffle per bin pair (X_A[k] = (X[k] + conj X[800-k]) / 2, X_B likewise).
// Shared-memory traffic per frame pair: one 6.4 KB write + read (the 4-stage Stockham version moved 8x that).
__global__ void __launch_bounds__(MEL_WARPS * 32, 2) mel_kernel(zeggs_mel_args a, int L, double fpa) {
  extern __shared__ __align__(16) float sm[];
  const int n_fft = a.n_fft, hop = a.hop, nm = a.n_mels;
  const int nsamp_tile = (MEL_FT + 1) * hop + n_fft;            // frames f0 .. f0+MEL_FT+1
  float* samp = sm;                                             // [nsamp_tile]
  float* melt = samp + ((nsamp_tile + 3) & ~3);                 // [(FT+2)][nm]  log-mel m = s*ln10/20
  float* ener = melt + (MEL_FT + 2) * nm;                       // [(FT+2)]
  float* sdb = ener + ((MEL_FT + 2 + 3) & ~3);                  // [(FT+2)][nm]  s in [0,1] (only if mel_out)
  float2* twt = reinterpret_cast<float2*>(sdb + (a.mel_out ? (MEL_FT + 2) * nm : 0));   // [24][32] exp(-2 pi i lane k2 / 800)
  C2* tbuf = reinterpret_cast<C2*>(twt + 24 * 32);              // [warps][25][33]
  const int fbt = (a.fb_total > 0 && a.fb_total <= 4096) ? a.fb_total : 0;   // weights staged in shared memory when they fit
  float* fbw_s = reinterpret_cast<float*>(tbuf + MEL_WARPS * MEL_TB);     // [fbt] filterbank weights
  int* fbi = reinterpret_cast<int*>(fbw_s + ((fbt + 3) & ~3));            // [3][nm] start, len, offset
  const float* fbw = fbt ? fbw_s : a.fb_w;
  const int clip = blockIdx.y, f0 = blockIdx.x * MEL_FT;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* wav = a.wav ? a.wav + (size_t)clip * a.n_samples : nullptr;
  const short* wav16 = a.wav_i16 ? a.wav_i16 + (size_t)clip * a.n_samples : nullptr;
  const float gain = a.gain ? __ldg(a.gain + clip) : 1.0f;        // loudness normalisation folded into the load
  const int Ts = a.n_samples, Te = Ts < n_fft ? n_fft : Ts;     // spectrograms.py:233-234 zero-extends short clips
  // the 16-byte paths also need a 16-byte aligned base: a contiguous view with a storage offset need not have one
  const bool base16 = ((reinterpret_cast<uintptr_t>(a.wav ? (const void*)a.wav : (const void*)a.wav_i16) & 15) == 0);
  // ---- stage the tile's samples (reflect padding, spectrograms.py:237-239)
  {
    const int o0 = f0 * hop - n_fft / 2;
    if (wav && base16 && o0 >= 0 && o0 + nsamp_tile <= Ts && ((o0 & 3) == 0) && ((a.n_samples & 3) == 0) && ((nsamp_tile & 3) == 0)) {
      // interior tile: straight 16-byte copies
      const float4* src4 = reinterpret_cast<const float4*>(wav + o0);
      float4* dst4 = reinterpret_cast<float4*>(samp);
      for (int i = tid; i < nsamp_tile / 4; i += blockDim.x) {
        float4 v = __ldg(src4 + i);
        v.x *= gain; v.y *= gain; v.z *= gain; v.w *= gain;
        dst4[i] = v;
      }
    } else if (wav16 && base16 && o0 >= 0 && o0 + nsamp_tile <= Ts && ((o0 & 7) == 0) && ((a.n_samples & 7) == 0) && ((nsamp_tile & 7) == 0)) {
      // interior tile of int16 PCM: 16-byte loads of 8 samples, x / 32768 (audio_files.py:211-236)
      const uint4* src8 = reinterpret_cast<const uint4*>(wav16 + o0);
      const float sc = gain * (1.0f / 32768.0f);
      for (int i = tid; i < nsamp_tile / 8; i += blockDim.x) {
        const uint4 v = __ldg(src8 + i);
        const unsigned w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int h = 0; h < 4; ++h) {
          samp[8 * i + 2 * h] = (float)(short)(w[h] & 0xffffu) * sc;
          samp[8 * i + 2 * h + 1] = (float)(short)(w[h] >> 16) * sc;
        }
      }
    } else {
      for (int i = tid; i < nsamp_tile; i += blockDim.x) {
        int o = o0 + i;
        if (o < 0) o = -o;
        if (o >= Te) o = 2 * (Te - 1) - o;
        float v = 0.f;
        if (o >= 0 && o < Ts) v = wav ? __ldg(wav + o) : (float)__ldg(wav16 + o) * (1.0f / 32768.0f);
        samp[i] = v * gain;
      }
    }
  }
  {
    // exp(-2 pi i n1 k2 / 800) from the host table tw2[k] = exp(-2 pi i k / 800), k = 0..400 (second half by symmetry)
    const float2* tw2 = reinterpret_cast<const float2*>(a.twiddle) + MEL_N2;
    for (int i = tid; i < 24 * 32; i += blockDim.x) {
      const int k2 = 1 + i / 32, n1 = i & 31;
      const int m = (n1 * k2) % 800;
      float2 w = __ldg(tw2 + (m <= MEL_N2 ? m : m - MEL_N2));
      if (m > MEL_N2) { w.x = -w.x; w.y = -w.y; }
      twt[i] = w;
    }
    for (int i = tid; i < fbt; i += blockDim.x) fbw_s[i] = __ldg(a.fb_w + i);
    for (int i = tid; i < nm; i += blockDim.x) { fbi[i] = a.fb_start[i]; fbi[nm + i] = a.fb_len[i]; fbi[2 * nm + i] = a.fb_off[i]; }
  }
  float wr[25];                                                 // Hann window taps of this lane (spectrograms.py:230)
#pragma unroll
  for (int j = 0; j < 25; ++j) wr[j] = __ldg(a.window + lane + 32 * j);
  __syncthreads();
  C2* tb = tbuf + warp * MEL_TB;
  float* amp = reinterpret_cast<float*>(tb);                    // [2][401] magnitudes / n_fft, aliases the transpose buffer
  const float inv_nfft = 1.0f / (float)n_fft;
  const float R_db = -20.0f * log10f(a.min_amp);                // spectrograms.py:127
  const int rl = lane < 25 ? lane : 24;                         // row this lane transforms (lanes 25..31 shadow row 24)
  const int src = lane == 0 ? 0 : (lane < 25 ? 25 - lane : lane);
#pragma unroll 1
  for (int pr = warp; pr < MEL_PAIRS; pr += MEL_WARPS) {
    const int fl = 2 * pr;
    if (f0 + fl >= L) break;
    {
      const float* xa = samp + fl * hop + lane;
      const float* xb = xa + hop;
      C2 v[25];
#pragma unroll
      for (int j = 0; j < 25; ++j) v[j] = c2(xa[32 * j] * wr[j], xb[32 * j] * wr[j]);
      dft25(v);
#pragma unroll
      for (int p = 0; p < 25; ++p) {
        const int k2 = dft25_freq_of_pos(p);
        C2 y = v[p];
        if (k2 > 0) { const float2 w = twt[(k2 - 1) * 32 + lane]; y = cmul(y, c2(w.x, w.y)); }
        tb[k2 * 33 + lane] = y;
      }
    }
    __syncwarp();
    C2 u[32];
#pragma unroll
    for (int n1 = 0; n1 < 32; ++n1) u[n1] = tb[rl * 33 + n1];
    dft32(u);
    __syncwarp();
    // ---- separate the two real spectra: bin k = lane + 25 k1 pairs with 800 - k = (25 - lane) + 25 (31 - k1)  (lane 0: 25 (32 - k1))
#pragma unroll
    for (int k1 = 0; k1 <= 16; ++k1) {
      const C2 P = u[brev5(k1)];
      C2 Q;
      Q.re = __shfl_sync(0xffffffffu, u[brev5(31 - k1)].re, src);
      Q.im = __shfl_sync(0xffffffffu, u[brev5(31 - k1)].im, src);
      if (lane == 0) Q = u[brev5((32 - k1) & 31)];
      const int k = lane + 25 * k1;
      if (lane < 25 && k <= MEL_N2) {
        const float are = 0.5f * (P.re + Q.re), aim = 0.5f * (P.im - Q.im);
        const float bre = 0.5f * (P.im + Q.im), bim = 0.5f * (P.re - Q.re);
        amp[k] = sqrtf(are * are + aim * aim) * inv_nfft;
        amp[MEL_N2 + 1 + k] = sqrtf(bre * bre + bim * bim) * inv_nfft;
      }
    }
    __syncwarp();
    // ---- sparse Slaney filterbank -> clip -> dB -> [0,1] -> ln(10^(s/20)), energy; both frames share the weight loads
    float esa = 0.f, esb = 0.f;
    for (int band = lane; band < nm; band += 32) {
      const int st = fbi[band], ln = fbi[nm + band];
      const float* wgt = fbw + fbi[2 * nm + band];
      const float* pa = amp + st;
      const float* pb = amp + MEL_N2 + 1 + st;
      float acca = 0.f, accb = 0.f, acca2 = 0.f, accb2 = 0.f;
      int i = 0;
      for (; i + 4 <= ln; i += 4) {
        const float w0 = wgt[i], w1 = wgt[i + 1], w2 = wgt[i + 2], w3 = wgt[i + 3];
        acca = fmaf(w0, pa[i], acca); accb = fmaf(w0, pb[i], accb);
        acca2 = fmaf(w1, pa[i + 1], acca2); accb2 = fmaf(w1, pb[i + 1], accb2);
        acca = fmaf(w2, pa[i + 2], acca); accb = fmaf(w2, pb[i + 2], accb);
        acca2 = fmaf(w3, pa[i + 3], acca2); accb2 = fmaf(w3, pb[i + 3], accb2);
      }
      for (; i < ln; ++i) { const float wv = wgt[i]; acca = fmaf(wv, pa[i], acca); accb = fmaf(wv, pb[i], accb); }
      acca += acca2; accb += accb2;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float acc = h ? accb : acca;
        const float v = fmaxf(fabsf(acc), a.min_amp);                         // spectrograms.py:110-116
        const float sv = (20.0f * log10f(v) + R_db) / R_db;                   // :119, :127-129
        const float mm = sv * 0.11512925464970229f;                           // ln(10^(s/20)), data_pipeline.py:62-63
        melt[(fl + h) * nm + band] = mm;
        if (a.mel_out) sdb[(fl + h) * nm + band] = sv;
        const float ex = expf(mm);
        if (h) esb = fmaf(ex, ex, esb); else esa = fmaf(ex, ex, esa);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { esa += __shfl_xor_sync(0xffffffffu, esa, o); esb += __shfl_xor_sync(0xffffffffu, esb, o); }
    if (lane == 0) { ener[fl] = sqrtf(esa); ener[fl + 1] = sqrtf(esb); }      // data_pipeline.py:28-30
    __syncwarp();
  }
  __syncthreads();
  // ---- mel_out[clip][band][f] (frames contiguous)
  if (a.mel_out) {
    for (int i = tid; i < nm * MEL_FT; i += blockDim.x) {
      int band = i / MEL_FT, fl = i % MEL_FT;
      if (f0 + fl < L) a.mel_out[((size_t)clip * nm + band) * L + f0 + fl] = sdb[fl * nm + band];
    }
  }
  // ---- 60 fps resample (data_pipeline.py:65-82): rows k with clamp(floor(k*fpa), 0, L-2) in [f0, f0+MEL_FT)
  if (a.feat_out) {
    int k_lo = (int)floor((double)f0 / fpa) - 1;
    int k_hi = (int)ceil((double)(f0 + MEL_FT) / fpa) + 1;
    if (k_lo < 0) k_lo = 0;
    if (k_hi > a.anim_length) k_hi = a.anim_length;
    const int nch = nm + 1;
    for (int k = k_lo + warp; k < k_hi; k += MEL_WARPS) {          // one warp per 60 fps row: the index math once per row
      const double pos = (double)k * fpa;
      int i0 = (int)floor(pos);
      if (i0 > L - 2) i0 = L - 2;
      if (i0 < 0) i0 = 0;
      if (i0 < f0 || i0 >= f0 + MEL_FT) continue;
      const float wgt = (float)(pos - (double)i0);
      const int fl = i0 - f0;
      float* dst = a.feat_out + ((size_t)clip * a.anim_length + k) * nch;
      for (int ch = lane; ch < nch; ch += 32) {
        float v0, v1;
        if (ch < nm) { v0 = melt[fl * nm + ch]; v1 = (L > 1) ? melt[(fl + 1) * nm + ch] : v0; }
        else { v0 = ener[fl]; v1 = (L > 1) ? ener[fl + 1] : v0; }
        dst[ch] = v0 + (v1 - v0) * wgt;
      }
    }
  }
}

extern "C" int zeggs_mel_num_frames(int n_samples, int n_fft, int hop) {
  // spectrograms.py:233-245 (centered)
  if (n_samples < 1 || n_fft < 2 || hop < 1) return -1;
  long long n = n_samples < n_fft ? n_fft : n_samples;
  n += 2 * (n_fft / 2);
  long long L = (n - n_fft) / hop;
  if (n % hop != 0) L += 1;
  return (int)L;
}

extern "C" int zeggs_mel_forward(const zeggs_mel_args* ap, void* stream_) {
  ZCHECK_ARG(ap != nullptr, "mel: null args");
  const zeggs_mel_args& a = *ap;
  cudaStream_t stream = (cudaStream_t)stream_;
  if (a.n_fft != 2 * MEL_N2) { set_error("mel: n_fft=%d unsupported (this build transforms n_fft=800 only)", a.n_fft); return ZEGGS_ERR_UNSUPPORTED; }
  ZCHECK_ARG(a.n_clips >= 0 && a.n_samples >= 1 && a.hop >= 1 && a.hop <= 800 && a.n_mels >= 1 && a.n_mels <= 256, "mel: bad shape");
  ZCHECK_ARG(a.n_clips <= 65535, "mel: n_clips=%d exceeds 65535, the grid's y limit (one grid row per clip); split the batch", a.n_clips);
  ZCHECK_ARG((a.wav != nullptr) != (a.wav_i16 != nullptr), "mel: exactly one of wav (f32) / wav_i16 (int16 PCM)");
  ZCHECK_ARG(a.window && a.twiddle && a.fb_start && a.fb_len && a.fb_off && a.fb_w, "mel: null table/input pointer");
  ZCHECK_ARG(a.mel_out || a.feat_out, "mel: no output requested");
  ZCHECK_ARG(a.n_samples >= a.n_fft / 2 + 1, "mel: clip shorter than n_fft/2+1 samples cannot be reflect-padded");
  if (a.n_clips == 0) return ZEGGS_OK;
  const int L = zeggs_mel_num_frames(a.n_samples, a.n_fft, a.hop);
  ZCHECK_ARG(L >= 1, "mel: no frames");
  if (a.feat_out) {
    ZCHECK_ARG(a.anim_length >= 1 && a.frames_per_anim > 0.0, "mel: bad resample parameters");
    ZCHECK_ARG((double)(a.anim_length - 1) * a.frames_per_anim <= (double)(L - 1) + 1e-9,
               "mel: anim_length %d needs frames beyond L=%d (reference would produce NaN, data_pipeline.py:473)", a.anim_length, L);
  }
  const int nsamp_tile = (MEL_FT + 1) * a.hop + a.n_fft;
  const size_t smem_rest = (size_t)(((nsamp_tile + 3) & ~3) + (MEL_FT + 2) * a.n_mels * (a.mel_out ? 2 : 1) + ((MEL_FT + 2 + 3) & ~3)) * sizeof(float)
                         + (size_t)24 * 32 * sizeof(float2) + (size_t)MEL_WARPS * MEL_TB * sizeof(C2) + (size_t)3 * a.n_mels * sizeof(int);
  const size_t smem_fb = (size_t)(((a.fb_total > 0 && a.fb_total <= 4096 ? a.fb_total : 0) + 3) & ~3) * sizeof(float);
  DeviceLimits lim;
  RC(device_limits(&lim));
  // Large hops with many bands and mel_out (hop 800, 256 bands: 233,088 B with the shipped 752 weights) exceed the
  // opt-in limit (232,448 B on an H100): there the kernel reads the filterbank weights from global memory instead.
  zeggs_mel_args la = a;
  size_t smem = smem_rest + smem_fb;
  if (smem > lim.smem_optin) { la.fb_total = 0; smem = smem_rest; }
  ZCHECK_ARG(smem <= lim.smem_optin, "mel: hop=%d with n_mels=%d needs %zu B of shared memory per block, above the device's %zu B",
             a.hop, a.n_mels, smem, lim.smem_optin);
  RC(set_max_dynamic_smem(mel_kernel, smem));
  dim3 grid(ceil_div(L, MEL_FT), a.n_clips);
  ScopedTimer tm("mel", stream);
  mel_kernel<<<grid, MEL_WARPS * 32, smem, stream>>>(la, L, a.frames_per_anim);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

}  // namespace zeggs
