// Mel front-end tail: |STFT|^2 -> HTK mel filterbank -> log -> affine.
//
// Reference: FAquantizer.preprocess modules/quantize.py:239-242 over
// torchaudio.transforms.MelSpectrogram(sample_rate=24000, n_fft=2048, win_length=1200,
// hop_length=300, n_mels=80) (modules/quantize.py:228-230).
//
// The windowed DFT itself runs in conv_simt.cu as a K=1200-tap, stride-300, Cin=1 "conv" of the
// waveform against a [1200][2*1025] cos/-sin basis with the Hann window folded in (engine.cu
// builds the basis in fp64); reflect padding of the centre=True STFT is the conv's index map.
// This kernel consumes its output: spec[b][f][2*bin] = Re, [2*bin+1] = Im.
#include "common.cuh"
#include "kernels.h"

namespace fac {

constexpr int MEL_BINS = 1025;
constexpr int MEL_N = 80;

__global__ void __launch_bounds__(128) mel_from_spec_kernel(const float* __restrict__ spec, int ldspec,
                                                            const float* __restrict__ fb, float* __restrict__ mel,
                                                            int F, int Tm) {
    __shared__ float pw[MEL_BINS + 3];
    const int b = blockIdx.y, f = blockIdx.x;
    const float* row = spec + ((size_t)b * F + f) * ldspec;
    for (int i = threadIdx.x; i < MEL_BINS; i += blockDim.x) {
        float2 c = *reinterpret_cast<const float2*>(row + 2 * i);
        pw[i] = c.x * c.x + c.y * c.y;   // spec.abs().pow(2)
    }
    __syncthreads();
    const int m = threadIdx.x;
    if (m < MEL_N) {
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        int i = 0;
        for (; i + 3 < MEL_BINS; i += 4) {
            a0 = fmaf(pw[i], __ldg(fb + (size_t)i * MEL_N + m), a0);
            a1 = fmaf(pw[i + 1], __ldg(fb + (size_t)(i + 1) * MEL_N + m), a1);
            a2 = fmaf(pw[i + 2], __ldg(fb + (size_t)(i + 2) * MEL_N + m), a2);
            a3 = fmaf(pw[i + 3], __ldg(fb + (size_t)(i + 3) * MEL_N + m), a3);
        }
        for (; i < MEL_BINS; ++i) a0 = fmaf(pw[i], __ldg(fb + (size_t)i * MEL_N + m), a0);
        float v = (a0 + a1) + (a2 + a3);
        // (log(1e-5 + mel) - mean) / std with mean=-4, std=4
        mel[((size_t)b * Tm + f) * MEL_N + m] = (logf(1e-5f + v) + 4.0f) / 4.0f;
    }
}

// Frame gather for the tensor-core DFT: frames[b][f][j] = wave[b][reflect((f_first + f)*hop - pad + j)], j < win, f < F.  The hop
// (300) is not a multiple of the 16-channel chunk of the tensor-core conv, so the strided "conv" view of the STFT cannot feed
// it directly; the explicit [B*F][1200] matrix (49 MB at B=32) can, as a plain K=1 GEMM against the folded basis.
// `wave` is [B][T] (row pitch T) and is reflected at both of its edges.  The streaming compressor passes a [history | chunk]
// window of the utterance with f_first > 0: it only asks for a frame that reaches past a window edge when that edge is the
// utterance's true start or end, so the reflection is the offline one.
__global__ void __launch_bounds__(256) stft_frames_kernel(const float* __restrict__ wave, float* __restrict__ frames, int T,
                                                          int F, int f_first, int hop, int win, int pad,
                                                          const int* __restrict__ lane_len) {
    const int b = blockIdx.y, f = blockIdx.x;
    const PadMap pm = PadMap::lane(lane_len, b, T, pad, pad, 1);
    const float* w = wave + (size_t)b * T;
    float* o = frames + ((size_t)b * F + f) * win;
    for (int j = threadIdx.x; j < win; j += blockDim.x) {
        const int src = pm.src((f_first + f) * hop - pad + j);
        o[j] = src >= 0 ? __ldg(w + src) : 0.f;
    }
}
cudaError_t launch_stft_frames(const float* wave, float* frames, int B, int T, int F, int hop, int win, int pad, cudaStream_t st,
                               int f_first, const int* lane_len) {
    if (B <= 0 || F <= 0) return cudaSuccess;
    stft_frames_kernel<<<dim3(F, B), 256, 0, st>>>(wave, frames, T, F, f_first, hop, win, pad, lane_len);
    return cudaGetLastError();
}

cudaError_t launch_mel_from_spec(const float* spec, int ldspec, const float* fb, float* mel, int B, int F, int Tm,
                                 cudaStream_t st) {
    if (B <= 0 || Tm <= 0) return cudaSuccess;
    dim3 grid(Tm, B);
    mel_from_spec_kernel<<<grid, 128, 0, st>>>(spec, ldspec, fb, mel, F, Tm);
    return cudaGetLastError();
}

// ---- losses.py:65-89 reconstruction_loss: the per-frame tail of one mel scale ----------------------------------------
// spec holds the windowed DFT of 2B signals (rows [0, B*F): x, rows [B*F, 2*B*F): G_x), [row][2*bin] = Re, [2*bin+1] = Im.
// One CTA per (frame, utterance): power spectra of both signals -> 64 HTK mel bands each (torchaudio MelSpectrogram,
// power = 2) -> this frame's share of  l1 = mean |S_x - S_G|  and of
// l2 = mean_{b,frame} sqrt(mean_mel (log(|S_x| + eps) - log(|S_G| + eps))^2):   terms[(b*F+f)*2] = sum_mel |dS|,
// terms[.. + 1] = sqrt(sum_mel dlog^2 / 64).
constexpr int LOSS_MELS = 64;
__global__ void __launch_bounds__(128) mel_loss_terms_kernel(const float* __restrict__ spec, int ldspec, int nb,
                                                             const float* __restrict__ fb, int B, int F, float eps,
                                                             float* __restrict__ terms) {
    extern __shared__ float pw[];                    // [2][nb] power spectra
    __shared__ float mels[2][LOSS_MELS];
    __shared__ float red[2][2];
    const int b = blockIdx.y, f = blockIdx.x, tid = threadIdx.x;
    const float* rx = spec + ((size_t)b * F + f) * ldspec;
    const float* rg = spec + ((size_t)(B + b) * F + f) * ldspec;
    for (int i = tid; i < nb; i += blockDim.x) {
        const float2 cx = *reinterpret_cast<const float2*>(rx + 2 * i), cg = *reinterpret_cast<const float2*>(rg + 2 * i);
        pw[i] = cx.x * cx.x + cx.y * cx.y;
        pw[nb + i] = cg.x * cg.x + cg.y * cg.y;
    }
    __syncthreads();
    {
        const int sig = tid >> 6, m = tid & 63;
        const float* q = pw + sig * nb;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        int i = 0;
        for (; i + 3 < nb; i += 4) {
            a0 = fmaf(q[i], __ldg(fb + (size_t)i * LOSS_MELS + m), a0);
            a1 = fmaf(q[i + 1], __ldg(fb + (size_t)(i + 1) * LOSS_MELS + m), a1);
            a2 = fmaf(q[i + 2], __ldg(fb + (size_t)(i + 2) * LOSS_MELS + m), a2);
            a3 = fmaf(q[i + 3], __ldg(fb + (size_t)(i + 3) * LOSS_MELS + m), a3);
        }
        for (; i < nb; ++i) a0 = fmaf(q[i], __ldg(fb + (size_t)i * LOSS_MELS + m), a0);
        mels[sig][m] = (a0 + a1) + (a2 + a3);
    }
    __syncthreads();
    if (tid < LOSS_MELS) {
        const float sx = mels[0][tid], sg = mels[1][tid];
        float d1 = fabsf(sx - sg);
        const float dl = logf(fabsf(sx) + eps) - logf(fabsf(sg) + eps);
        float d2 = dl * dl;
        d1 = warp_sum(d1); d2 = warp_sum(d2);
        if ((tid & 31) == 0) { red[tid >> 5][0] = d1; red[tid >> 5][1] = d2; }
    }
    __syncthreads();
    if (tid == 0) {
        terms[((size_t)b * F + f) * 2] = red[0][0] + red[1][0];
        terms[((size_t)b * F + f) * 2 + 1] = sqrtf((red[0][1] + red[1][1]) / (float)LOSS_MELS);
    }
}
cudaError_t launch_mel_loss_terms(const float* spec, int ldspec, int nb, const float* fb, int B, int F, float eps, float* terms,
                                  cudaStream_t st) {
    if (B <= 0 || F <= 0) return cudaSuccess;
    if (B > 65535) return cudaErrorInvalidValue;
    mel_loss_terms_kernel<<<dim3(F, B), 128, (size_t)2 * nb * sizeof(float), st>>>(spec, ldspec, nb, fb, B, F, eps, terms);
    return cudaGetLastError();
}

// Deterministic fp64 sums (fixed partition, fixed tree): out[0] = sum of in[i*stride] * scale, i < n -- one CTA.
__global__ void __launch_bounds__(1024) strided_sum_kernel(const float* __restrict__ in, long long n, int stride, double scale,
                                                           double* __restrict__ out) {
    __shared__ double sh[1024];
    double a = 0.0;
    for (long long i = threadIdx.x; i < n; i += 1024) a += (double)in[i * stride];
    sh[threadIdx.x] = a;
    __syncthreads();
    for (int o = 512; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[0] = sh[0] * scale;
}
cudaError_t launch_strided_sum(const float* in, long long n, int stride, double scale, double* out, cudaStream_t st) {
    strided_sum_kernel<<<1, 1024, 0, st>>>(in, n, stride, scale, out);
    return cudaGetLastError();
}

// squared error of two [n] signals: per-block fp64 partials (fixed partition), then strided_sum over the partials
__global__ void __launch_bounds__(256) sqdiff_partial_kernel(const float* __restrict__ a, const float* __restrict__ b, long long n,
                                                             float* __restrict__ part) {
    __shared__ double sh[256];
    double acc = 0.0;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        const double d = (double)a[i] - (double)b[i];
        acc += d * d;
    }
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) part[blockIdx.x] = (float)sh[0];
}
cudaError_t launch_sqdiff_partial(const float* a, const float* b, long long n, float* part, int nblocks, cudaStream_t st) {
    sqdiff_partial_kernel<<<nblocks, 256, 0, st>>>(a, b, n, part);
    return cudaGetLastError();
}

// L = 100 * mse + sum_i (l1_i + sqrt(s_i / 2) * l2_i), s_i = 64 << i  (losses.py:65-89, accumulated in fp32 in that order)
__global__ void loss_combine_kernel(const double* __restrict__ v /* [1 + 2*6]: mse, then (l1, l2) per scale */,
                                    float* __restrict__ loss, float* __restrict__ terms) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    float L = 100.0f * (float)v[0];
    if (terms) terms[0] = (float)v[0];
    for (int i = 0; i < 6; ++i) {
        const float l1 = (float)v[1 + 2 * i], l2 = (float)v[2 + 2 * i];
        const float alpha = sqrtf((float)(64 << i) * 0.5f);
        L += l1 + alpha * l2;
        if (terms) { terms[1 + 2 * i] = l1; terms[2 + 2 * i] = l2; }
    }
    loss[0] = L;
}
cudaError_t launch_loss_combine(const double* v, float* loss, float* terms, cudaStream_t st) {
    loss_combine_kernel<<<1, 32, 0, st>>>(v, loss, terms);
    return cudaGetLastError();
}

__global__ void __launch_bounds__(256) add3_kernel(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ c,
                                                   long long n, float* __restrict__ out) {
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        float v = a[i] + b[i];
        if (c) v += c[i];
        out[i] = v;
    }
}
cudaError_t launch_add3(const float* a, const float* b, const float* c, long long n, float* out, cudaStream_t st) {
    long long blocks = (n + 255) / 256;
    if (blocks > 148 * 16) blocks = 148 * 16;
    add3_kernel<<<(unsigned)blocks, 256, 0, st>>>(a, b, c, n, out);
    return cudaGetLastError();
}

// ---- dac/nn/loss.py:142-327 MultiScaleSTFTLoss / MelSpectrogramLoss: the per-frame tail of one scale ----------------
// spec as for mel_loss_terms_kernel (rows of x, then rows of y).  Per (frame, utterance): magnitudes |X|, |Y| (audiotools
// AudioSignal.magnitude = abs(stft)); with a filterbank fb [nb][n_out] the mel spectra mag @ fb (AudioSignal.mel_spectrogram),
// else n_out = nb and the values are the magnitudes themselves.  terms[(b*F+f)*2] = sum_o |vx - vy| (the mag_weight term),
// terms[.. + 1] = sum_o |log10(clamp(vx, eps)^pw) - log10(clamp(vy, eps)^pw)| (the log_weight term); both are means over
// (utterance, o, frame) in the reference (nn.L1Loss), formed by the caller's fixed-order fp64 sums.
__global__ void __launch_bounds__(128) spec_loss_terms_kernel(const float* __restrict__ spec, int ldspec, int nb, const float* __restrict__ fb,
                                                              int n_out, int B, int F, float eps, float pw, float* __restrict__ terms) {
    extern __shared__ float mg[];                    // [2][nb] magnitudes
    __shared__ float red[4][2];
    const int b = blockIdx.y, f = blockIdx.x, tid = threadIdx.x;
    const float* rx = spec + ((size_t)b * F + f) * ldspec;
    const float* ry = spec + ((size_t)(B + b) * F + f) * ldspec;
    for (int i = tid; i < nb; i += blockDim.x) {
        const float2 cx = *reinterpret_cast<const float2*>(rx + 2 * i), cy = *reinterpret_cast<const float2*>(ry + 2 * i);
        mg[i] = sqrtf(cx.x * cx.x + cx.y * cx.y);
        mg[nb + i] = sqrtf(cy.x * cy.x + cy.y * cy.y);
    }
    __syncthreads();
    float d1 = 0.f, d2 = 0.f;
    for (int o = tid; o < n_out; o += blockDim.x) {
        float vx, vy;
        if (fb) {
            float a0 = 0.f, a1 = 0.f, c0 = 0.f, c1 = 0.f;
            int i = 0;
            for (; i + 1 < nb; i += 2) {
                const float w0 = __ldg(fb + (size_t)i * n_out + o), w1 = __ldg(fb + (size_t)(i + 1) * n_out + o);
                a0 = fmaf(mg[i], w0, a0); a1 = fmaf(mg[i + 1], w1, a1);
                c0 = fmaf(mg[nb + i], w0, c0); c1 = fmaf(mg[nb + i + 1], w1, c1);
            }
            if (i < nb) { const float w0 = __ldg(fb + (size_t)i * n_out + o); a0 = fmaf(mg[i], w0, a0); c0 = fmaf(mg[nb + i], w0, c0); }
            vx = a0 + a1; vy = c0 + c1;
        } else {
            vx = mg[o]; vy = mg[nb + o];
        }
        d1 += fabsf(vx - vy);
        float lx = fmaxf(vx, eps), ly = fmaxf(vy, eps);
        if (pw == 2.0f) { lx *= lx; ly *= ly; }
        else if (pw != 1.0f) { lx = powf(lx, pw); ly = powf(ly, pw); }
        d2 += fabsf(log10f(lx) - log10f(ly));
    }
    d1 = warp_sum(d1); d2 = warp_sum(d2);
    if ((tid & 31) == 0) { red[tid >> 5][0] = d1; red[tid >> 5][1] = d2; }
    __syncthreads();
    if (tid == 0) {
        terms[((size_t)b * F + f) * 2] = (red[0][0] + red[1][0]) + (red[2][0] + red[3][0]);
        terms[((size_t)b * F + f) * 2 + 1] = (red[0][1] + red[1][1]) + (red[2][1] + red[3][1]);
    }
}
cudaError_t launch_spec_loss_terms(const float* spec, int ldspec, int nb, const float* fb, int n_out, int B, int F, float eps, float pw,
                                   float* terms, cudaStream_t st) {
    if (B <= 0 || F <= 0) return cudaSuccess;
    if (B > 65535) return cudaErrorInvalidValue;
    spec_loss_terms_kernel<<<dim3(F, B), 128, (size_t)2 * nb * sizeof(float), st>>>(spec, ldspec, nb, fb, n_out, B, F, eps, pw, terms);
    return cudaGetLastError();
}

// sum |a - b| over [n]: per-block fp64 partials (fixed partition); strided_sum over the partials gives the L1 loss
__global__ void __launch_bounds__(256) absdiff_partial_kernel(const float* __restrict__ a, const float* __restrict__ b, long long n,
                                                              float* __restrict__ part) {
    __shared__ double sh[256];
    double acc = 0.0;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256)
        acc += fabs((double)a[i] - (double)b[i]);
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) part[blockIdx.x] = (float)sh[0];
}
cudaError_t launch_absdiff_partial(const float* a, const float* b, long long n, float* part, int nblocks, cudaStream_t st) {
    absdiff_partial_kernel<<<nblocks, 256, 0, st>>>(a, b, n, part);
    return cudaGetLastError();
}

// ---- gradients of the spectral losses (fac_spectral_loss_grad) -------------------------------------------------------
// One CTA per (frame, utterance), run after spec_loss_terms_kernel has read `spec`.  Recomputes |X|, |Y| and (mel scales)
// v = |.| @ fb with the terms kernel's arithmetic, so every sign below is the one the returned loss saw, then forms per
// requested signal
//   dL/dvx = mag_scale * sgn(vx - vy) + log_scale * sgn(log10 lx - log10 ly) * pw / (vx ln 10)   (log part only where vx >= eps)
// (dL/dvy the same with the signs negated and vy; mag_scale = mag_weight / N, log_scale = log_weight / N, N = B * F * n_out:
// the nn.L1Loss means), chains it through the filterbank transpose (d|X|_k = sum_o fb[k][o] dv_o, one warp per k, fixed
// butterfly order) and the complex magnitude (dRe = d|X| Re / |X|, dIm = d|X| Im / |X|, 0 where |X| = 0, as torch's sgn),
// and writes dRe, dIm in place over that signal's spec row; columns >= 2 * nb are zeroed.
// Each row is written scaled by a power of two 2^k chosen from the frame's largest |dL/d|.||, which bounds every |dRe|,
// |dIm| of the row: the scaled row's largest entry lies in [2^13, 2^14).  The gradients carry the loss's 1 / N mean factor
// (1e-9 ... 1e-6 at the benchmark shape), below fp16's normal range, and the gradient GEMM's promoted class splits its
// activations into fp16 hi + 2^11-scaled fp16 lo without a scale of its own; scaled, they keep its 22 significant bits.
// inv_scale[row] = 2^-k (rows as in spec: x, then y) is applied by the overlap-add.  Both scalings are exact in fp32.
__global__ void __launch_bounds__(128) spec_loss_grad_kernel(float* __restrict__ spec, int ldspec, int nb, const float* __restrict__ fb,
                                                             int n_out, int B, int F, float eps, float pw, float mag_scale, float log_scale,
                                                             int want_x, int want_y, float* __restrict__ inv_scale) {
    extern __shared__ float sg[];
    float* mg = sg;                                  // [2][nb] magnitudes
    float* dv = sg + 2 * nb;                         // [2][n_out] dL/dv of x, y (no filterbank: dL/d|.| itself)
    float* dm = fb ? dv + 2 * n_out : dv;            // [2][nb] dL/d|.|
    const int b = blockIdx.y, f = blockIdx.x, tid = threadIdx.x;
    float* rx = spec + ((size_t)b * F + f) * ldspec;
    float* ry = spec + ((size_t)(B + b) * F + f) * ldspec;
    for (int i = tid; i < nb; i += blockDim.x) {
        const float2 cx = *reinterpret_cast<const float2*>(rx + 2 * i), cy = *reinterpret_cast<const float2*>(ry + 2 * i);
        mg[i] = sqrtf(cx.x * cx.x + cx.y * cx.y);
        mg[nb + i] = sqrtf(cy.x * cy.x + cy.y * cy.y);
    }
    __syncthreads();
    const float inv_ln10 = 0.43429448190325182f;
    for (int o = tid; o < n_out; o += blockDim.x) {
        float vx, vy;
        if (fb) {
            float a0 = 0.f, a1 = 0.f, c0 = 0.f, c1 = 0.f;
            int i = 0;
            for (; i + 1 < nb; i += 2) {
                const float w0 = __ldg(fb + (size_t)i * n_out + o), w1 = __ldg(fb + (size_t)(i + 1) * n_out + o);
                a0 = fmaf(mg[i], w0, a0); a1 = fmaf(mg[i + 1], w1, a1);
                c0 = fmaf(mg[nb + i], w0, c0); c1 = fmaf(mg[nb + i + 1], w1, c1);
            }
            if (i < nb) { const float w0 = __ldg(fb + (size_t)i * n_out + o); a0 = fmaf(mg[i], w0, a0); c0 = fmaf(mg[nb + i], w0, c0); }
            vx = a0 + a1; vy = c0 + c1;
        } else {
            vx = mg[o]; vy = mg[nb + o];
        }
        float lx = fmaxf(vx, eps), ly = fmaxf(vy, eps);
        if (pw == 2.0f) { lx *= lx; ly *= ly; }
        else if (pw != 1.0f) { lx = powf(lx, pw); ly = powf(ly, pw); }
        const float dl = log10f(lx) - log10f(ly);
        const float s_mag = (float)((vx > vy) - (vx < vy)), s_log = (float)((dl > 0.f) - (dl < 0.f));
        float gx = mag_scale * s_mag, gy = -gx;
        if (vx >= eps) gx += log_scale * s_log * (pw * inv_ln10 / vx);
        if (vy >= eps) gy -= log_scale * s_log * (pw * inv_ln10 / vy);
        dv[o] = gx; dv[n_out + o] = gy;
    }
    __syncthreads();
    if (fb) {
        const int warp = tid >> 5, lane = tid & 31;
        for (int k = warp; k < nb; k += blockDim.x >> 5) {
            const float* row = fb + (size_t)k * n_out;
            float ax = 0.f, ay = 0.f;
            for (int o = lane; o < n_out; o += 32) {
                const float w = __ldg(row + o);
                ax = fmaf(w, dv[o], ax); ay = fmaf(w, dv[n_out + o], ay);
            }
            ax = warp_sum(ax); ay = warp_sum(ay);
            if (lane == 0) { dm[k] = ax; dm[nb + k] = ay; }
        }
        __syncthreads();
    }
    // per-signal power-of-two row scale from max |dL/d|.||
    __shared__ float red[4][2];
    __shared__ float row_scale[2];
    float mx = 0.f, my = 0.f;
    for (int i = tid; i < nb; i += blockDim.x) { mx = fmaxf(mx, fabsf(dm[i])); my = fmaxf(my, fabsf(dm[nb + i])); }
    for (int o = 16; o > 0; o >>= 1) {
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        my = fmaxf(my, __shfl_xor_sync(0xffffffffu, my, o));
    }
    if ((tid & 31) == 0) { red[tid >> 5][0] = mx; red[tid >> 5][1] = my; }
    __syncthreads();
    if (tid < 2) {
        const float m = fmaxf(fmaxf(red[0][tid], red[1][tid]), fmaxf(red[2][tid], red[3][tid]));
        int k = 0;
        if (m > 0.f) {
            int e;
            frexpf(m, &e);                               // m in [2^(e-1), 2^e)
            k = min(max(14 - e, -126), 126);
        }
        row_scale[tid] = ldexpf(1.f, k);
        if ((tid == 0 && want_x) || (tid == 1 && want_y)) inv_scale[(size_t)(tid * B + b) * F + f] = ldexpf(1.f, -k);
    }
    __syncthreads();
    const float sx = row_scale[0], sy = row_scale[1];
    for (int i = tid; i < nb; i += blockDim.x) {
        if (want_x) {
            const float2 c = *reinterpret_cast<const float2*>(rx + 2 * i);
            const float m = mg[i], g = dm[i] * sx;
            *reinterpret_cast<float2*>(rx + 2 * i) = m > 0.f ? make_float2(g * (c.x / m), g * (c.y / m)) : make_float2(0.f, 0.f);
        }
        if (want_y) {
            const float2 c = *reinterpret_cast<const float2*>(ry + 2 * i);
            const float m = mg[nb + i], g = dm[nb + i] * sy;
            *reinterpret_cast<float2*>(ry + 2 * i) = m > 0.f ? make_float2(g * (c.x / m), g * (c.y / m)) : make_float2(0.f, 0.f);
        }
    }
    for (int j = 2 * nb + tid; j < ldspec; j += blockDim.x) {
        if (want_x) rx[j] = 0.f;
        if (want_y) ry[j] = 0.f;
    }
}
cudaError_t launch_spec_loss_grad(float* spec, int ldspec, int nb, const float* fb, int n_out, int B, int F, float eps, float pw,
                                  float mag_scale, float log_scale, int want_x, int want_y, float* inv_scale, cudaStream_t st) {
    if (B <= 0 || F <= 0 || !(want_x || want_y)) return cudaSuccess;
    if (B > 65535) return cudaErrorInvalidValue;
    const size_t smem = (size_t)(2 * nb + 2 * n_out + (fb ? 2 * nb : 0)) * sizeof(float);
    if (smem > 48 * 1024) return cudaErrorInvalidValue;
    spec_loss_grad_kernel<<<dim3(F, B), 128, smem, st>>>(spec, ldspec, nb, fb, n_out, B, F, eps, pw, mag_scale, log_scale, want_x, want_y,
                                                         inv_scale);
    return cudaGetLastError();
}

// Adjoint of stft_frames_kernel (f_first = 0): a deterministic gather, no atomics.  out[b][t] is the sum of
// dframes[b][f][j] * inv_scale[b][f] (the row scales of spec_loss_grad_kernel) over every (f, j) that read sample t: padded
// position t + pad itself and, for the reflect padding, the mirrored positions pad - t (left edge, 1 <= t <= pad) and
// pad + 2 (T - 1) - t (right edge, T - 1 - pad <= t <= T - 2), in that order, frames ascending -- the fold torch's
// reflect-pad backward does.  accumulate = 0 writes, 1 adds (the later scales of one loss).
__global__ void __launch_bounds__(256) stft_overlap_add_grad_kernel(const float* __restrict__ dframes, const float* __restrict__ inv_scale,
                                                                    float* __restrict__ out, int T, int F, int hop, int win, int pad,
                                                                    int accumulate) {
    const int b = blockIdx.y, t = blockIdx.x * 256 + threadIdx.x;
    if (t >= T) return;
    const float* d = dframes + (size_t)b * F * win;
    const float* is = inv_scale + (size_t)b * F;
    int pos[3], n = 0;
    pos[n++] = t + pad;
    if (t >= 1 && t <= pad) pos[n++] = pad - t;
    if (t >= T - 1 - pad && t <= T - 2) pos[n++] = pad + 2 * (T - 1) - t;
    float s = 0.f;
    for (int q = 0; q < n; ++q) {
        const int P = pos[q];
        const int f0 = P - win + 1 > 0 ? (P - win + hop) / hop : 0;     // first frame reaching P
        const int f1 = P / hop < F - 1 ? P / hop : F - 1;               // last frame starting at or before P
        for (int fr = f0; fr <= f1; ++fr) s += d[(size_t)fr * win + (P - fr * hop)] * __ldg(is + fr);
    }
    float* o = out + (size_t)b * T + t;
    *o = accumulate ? *o + s : s;
}
cudaError_t launch_stft_overlap_add_grad(const float* dframes, const float* inv_scale, float* out, int B, int T, int F, int hop, int win,
                                         int pad, int accumulate, cudaStream_t st) {
    if (B <= 0 || T <= 0) return cudaSuccess;
    if (B > 65535) return cudaErrorInvalidValue;
    stft_overlap_add_grad_kernel<<<dim3((T + 255) / 256, B), 256, 0, st>>>(dframes, inv_scale, out, T, F, hop, win, pad, accumulate);
    return cudaGetLastError();
}

// d/da mean |a - b| = sgn(a - b) / n (torch's sign: 0 where a == b); db = -da.  da / db may each be null.
__global__ void __launch_bounds__(256) l1_grad_kernel(const float* __restrict__ a, const float* __restrict__ b, long long n, float inv_n,
                                                      float* __restrict__ da, float* __restrict__ db) {
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        const float d = a[i] - b[i];
        const float g = d > 0.f ? inv_n : (d < 0.f ? -inv_n : 0.f);
        if (da) da[i] = g;
        if (db) db[i] = -g;
    }
}
cudaError_t launch_l1_grad(const float* a, const float* b, long long n, float inv_n, float* da, float* db, cudaStream_t st) {
    if (n <= 0 || !(da || db)) return cudaSuccess;
    long long blocks = (n + 255) / 256;
    if (blocks > 148 * 16) blocks = 148 * 16;
    l1_grad_kernel<<<(unsigned)blocks, 256, 0, st>>>(a, b, n, inv_n, da, db);
    return cudaGetLastError();
}

// loss = sum over scales of (log_weight * v[2i+1] + mag_weight * v[2i]) accumulated in fp32 in the reference's order
// (dac/nn/loss.py:217-226: the log term first); n = 0: loss = (float)v[0] (L1Loss)
__global__ void spec_loss_combine_kernel(const double* __restrict__ v, int n, float mag_weight, float log_weight, float* __restrict__ loss) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    if (n == 0) { loss[0] = (float)v[0]; return; }
    float L = 0.0f;
    for (int i = 0; i < n; ++i) {
        L += log_weight * (float)v[2 * i + 1];
        L += mag_weight * (float)v[2 * i];
    }
    loss[0] = L;
}
cudaError_t launch_spec_loss_combine(const double* v, int n, float mag_weight, float log_weight, float* loss, cudaStream_t st) {
    spec_loss_combine_kernel<<<1, 32, 0, st>>>(v, n, mag_weight, log_weight, loss);
    return cudaGetLastError();
}

}  // namespace fac
