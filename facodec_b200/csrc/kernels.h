// Internal kernel launch interfaces (C++ only; the public C-ABI is include/facodec_b200.h).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace fac {

struct ConvParams {
    const float* x = nullptr;          // [B][Tin][Cin]
    const float* w = nullptr;          // [K*Cin][ldw]
    const float* bias = nullptr;       // [Cout] or null
    const float* in_alpha = nullptr;   // [Cin] snake on input, or null
    const float* in_inv_alpha = nullptr;
    const float* out_alpha = nullptr;  // [Cout] when out_act == ACT_SNAKE
    const float* out_inv_alpha = nullptr;
    const float* res = nullptr;        // residual, same layout as y, or null
    const int* valid_len = nullptr;    // [B] rows >= valid_len[b] are written as 0, or null
    const int* lane_len = nullptr;     // [B] input rows of each lane (PadMap::lane), or null: Tin for every lane
    float* y = nullptr;                // [B][Tout][ldy] (or [B][Cout][Tout] when y_transposed)
    int B = 0, Tin = 0, Cin = 0, Tout = 0, Cout = 0;
    int K = 1, dil = 1, stride = 1, pad_left = 0, pad_right = 0, pad_reflect = 0;
    int ldw = 0, ldy = 0, ldx = 0;   // ldx = input row stride (>= Cin)
    int out_act = 0;
    int y_transposed = 0;
    size_t x_bstride = 0, y_bstride = 0;
};
cudaError_t launch_conv(const ConvParams& p, cudaStream_t st);

// ---- wgmma tensor-core conv (conv_tc.cu) -----------------------------------------------------
struct TcConvParams {
    const float* x = nullptr;          // [B][Tin][ldx] channels-last samples
    const float* wblob = nullptr;      // [ntile][chunk][tap][hi|lo][k-piece][N][16 B] (tc_pack_blob)
    const float* bias = nullptr;
    const float* in_alpha = nullptr;   // [Cin] Snake on the input or null
    const float* in_inv_alpha = nullptr;
    const float* out_alpha = nullptr;  // [Cout] when out_act == ACT_SNAKE
    const float* out_inv_alpha = nullptr;
    const float* res = nullptr;        // [B][Tout][ldy] or null
    float* y = nullptr;                // [B][Tout][ldy]
    int B = 0, Tin = 0, Cin = 0, ldx = 0;
    int vf = 1;                        // samples per A row (down-conv stride; 1 otherwise)
    int Kr = 1, dil = 1, PLr = 0;      // taps / dilation / left pad, in rows
    int pad_left_s = 0, pad_right_s = 0, reflect = 0;   // sample-level padding (PadMap)
    const int* lane_len = nullptr;     // [B] input samples of each lane (PadMap::lane), or null: Tin for every lane
    int Tout = 0, Cout = 0, ldy = 0;
    int out_act = 0;
    int promoted = 0;                  // 1 = promoted accumulation, windows into a master in shared memory (upstream of the VQ)
    int bf16 = 0;                      // 1 = bf16 hi/lo split (K = 16 MMAs) instead of tf32 hi/lo; downstream of the VQ only
    int g1f16 = 0;                     // with bf16 = 1 (downstream only): the layer's own GEMM (the k-tap conv; GEMM 1 of a fused unit) takes
                                       // ONE fp16 pass (10-bit operands, fp32 accumulation) instead of the 3-pass bf16 hi/lo split
    int f16x2 = 0;                     // promoted only: fp16 hi + 2^11-scaled fp16 lo split (K = 16 MMAs) instead of tf32 hi/lo
    int fused = 0;                     // 1 = whole ResidualUnit: conv7 -> +b7 -> Snake -> 1x1 conv -> +b1 -> +x
    int tt = 0;                        // f16x2 only: transposed formulation (weights = wgmma A operand, time = wgmma N)
    int occ2_maxn = 0;                 // > 0: tiles with N <= occ2_maxn are planned for two resident CTAs per SM
    int max_group = 4;                 // largest `group` the plan may take (1: the one-chunk reference of the tests)
    const float* wblob2 = nullptr;     // 1x1 conv weight blob (same tile N), when fused
    const float* bias2 = nullptr;
    int nchunk2 = 0;
    // plan (tc_conv_plan)
    int promote_every = 1;             // promoted: chunks per accumulation window
    int N = 0, nchunk = 0, Rpad = 0, stagesB = 0;
    int group = 1;                     // 16-channel chunks per K-loop step (1, 2 or 4; divides nchunk and promote_every)
    int MT = 2;                        // 2: tile = 128 rows x N (warpgroups split rows); 1: 64 rows x N (they split channels)
    int b_slot = 0;                    // bytes of one weight-ring slot
    int occ2 = 0;                      // planned for two resident CTAs per SM
    int R2pad = 0;                     // fused: row pitch (rows) of the resident GEMM-2 operand
    size_t smem_bytes = 0;
    size_t x_bstride = 0, y_bstride = 0;
    int row2d = 0;                     // > 0: 3x3 Conv2d over [T][row2d][C] maps (Kr = 9, conv2d_tc_kernel); see conv_tc_body
};
bool tc_conv_plan(TcConvParams& p);
size_t tc_blob_floats(const TcConvParams& p);
void tc_pack_blob(const TcConvParams& p, const float* wp, int ldw, float* blob);
cudaError_t launch_conv_tc(const TcConvParams& p, cudaStream_t st);

// ---- LSTM recurrence (lstm.cu) -----------------------------------------------------------
// One nn.LSTM layer over all T steps for up to 32 sequences (dac/model/encodec.py:272-288).
struct LstmParams {
    const float* xg = nullptr;    // [B][T][4H] = x W_ih^T + b_ih + b_hh, gate order i,f,g,o
    const float* whh_p = nullptr; // packed per CTA: [G][H][4U]  (r = gate*U + u)
    const float* whh_p16 = nullptr; // bf16 split: [G][H/16][hi|lo][8 k-pairs][4U] 32-bit words (k even in the low half)
    int bf16 = 0;                 // 1 = bf16 hi/lo recurrence (downstream of the VQ only)
    // second-generation kernel (lstm2.cu): W_hh resident in shared memory as fp16 words, h exchanged pre-split
    const uint32_t* whh_p2 = nullptr;   // lstm2_pack layout
    uint32_t* h16 = nullptr;            // scratch [2 parities][planes][H/2][32] words
    int pass3 = 0;                      // 1 = fp16 hi + scaled-lo 3-pass (upstream of the VQ); 0 = one fp16 pass
    // streaming (lstm2 only): state carried between chunks, updated in place; null = zero initial state, nothing saved
    uint32_t* state_h = nullptr;        // [planes][H/2][32] words (h in the published fp16 layout)
    float* state_c = nullptr;           // [G][32][U] cell state
    const float* skip = nullptr;  // [B][T][H] added to the output (SLSTM skip) or null
    float* y = nullptr;           // [B][T][H]
    float* hT = nullptr;          // scratch [2][H][32]
    unsigned int* bar = nullptr;  // grid barrier counter (zeroed by the launcher)
    int B = 0, T = 0, H = 0, U = 0, G = 0;
};
// Per-lane step counts of the resident-W kernel (a stream chunk whose lanes end at different frames): lane b updates (h, c)
// for t < len[b] only and then carries them unchanged, so the state left behind is the one after len[b] steps; its output
// rows t >= len[b] are finite don't-cares.  One-pass class (pass3 = 0) only; launches without them run a kernel
// instantiation of their own.
struct LstmLaneLens { int len[32]; };
cudaError_t launch_lstm_layer(const LstmParams& p, cudaStream_t st);
// reverse = true: the reverse direction of a bidirectional layer, lane b from frame lens->len[b] - 1 down to 0 (pass3, lens
// required, no stream state); its rows t >= len[b] are finite don't-cares
cudaError_t launch_lstm2_layer(const LstmParams& p, cudaStream_t st, const LstmLaneLens* lens = nullptr, bool reverse = false);
size_t lstm2_pack_words(int H, int U, int pass3);
void lstm2_pack(const float* whh, int H, int U, int pass3, uint32_t* out);
size_t lstm2_smem_bytes(int H, int U, int pass3);
// sizes of one layer's carried stream state: state_h words and state_c floats
void lstm2_state_sizes(int H, int U, int pass3, size_t* h_words, size_t* c_floats);
cudaError_t lstm2_read_phase_clocks(long long* out4);
// One batch lane's carry of one layer is PL * H/2 h words + H c floats (PL = 2 when pass3).  lstm2_lane_map writes, for word
// j of lane b's carry, its position in [state_h words | state_c floats] (state_h first, then state_c at offset h_words).
void lstm2_lane_map(int H, int U, int pass3, int b, long long* pos);
// Moves the carries of lanes [0, n) between state (state_h, state_c) and n packed per-session slots of lstm2_lane_map order
// (to_lanes = 1: slot[b] -> lane b; 0: lane b -> slot[b]), raw 32-bit words.
constexpr int kLaneMax = 32;
struct LaneCarryParams {
    uint32_t* slot[kLaneMax];
    uint32_t* state_h = nullptr;
    float* state_c = nullptr;
    int n = 0, H = 0, U = 0, pass3 = 0, to_lanes = 0;
};
cudaError_t launch_lstm2_lane_carry(const LaneCarryParams& p, cudaStream_t st);
// dst[b][0, words[b]) = src[b][0, words[b]) for lanes b < n (32-bit words; pool.cu): the slot <-> lane moves of the stream
// pools (N = kLaneMax), and the slot <-> state-payload moves of a session export or import (N = kMoveLanes, one launch per
// state region for up to that many sessions; the 24 KB parameter block stays under sm_90's 32 764-byte limit).
constexpr int kMoveLanes = 1024;
template <int N>
struct LaneCopyParamsN {
    const uint32_t* src[N];
    uint32_t* dst[N];
    long long words[N];
    int n = 0;
};
using LaneCopyParams = LaneCopyParamsN<kLaneMax>;
cudaError_t launch_lane_copy(const LaneCopyParamsN<kLaneMax>& p, cudaStream_t st);
cudaError_t launch_lane_copy(const LaneCopyParamsN<kMoveLanes>& p, cudaStream_t st);
int lstm_units_per_cta(int H);
cudaError_t lstm_read_phase_clocks(long long* out4);   // CTA-0 accumulated phase clocks of the last launch  // U such that H % U == 0 and H / U <= resident CTAs

// ---- mel front-end (frontend.cu) -----------------------------------------------------------
// spec [B][F][ldspec] (re at 2*bin, im at 2*bin+1) -> mel [B][Tm][80] = (log(1e-5 + |.|^2 fb)+4)/4
// frames [f_first, f_first + F) of the centred STFT of wave [B][T], reflected at both ends of the T samples (lane_len [B]
// device: at both ends of lane b's own lane_len[b] samples)
cudaError_t launch_stft_frames(const float* wave, float* frames /*[B][F][win]*/, int B, int T, int F, int hop, int win, int pad,
                               cudaStream_t st, int f_first = 0, const int* lane_len = nullptr);
cudaError_t launch_mel_from_spec(const float* spec, int ldspec, const float* fb /*[1025][80]*/, float* mel,
                                 int B, int F, int Tm, cudaStream_t st);

// ---- quantizer-side kernels (quant.cu) -----------------------------------------------------
struct VqWeights {           // one dac/nn/quantize.py VectorQuantize, folded
    const float* w_in;       // [8][1024]
    const float* b_in;       // [8]
    const float* cb;         // [1024][8] raw codebook
    const float* cbn;        // [1024][8] F.normalize(codebook)
    const float* cbn2;       // [1024] sum(cbn^2)
    const float* w_out;      // [8][1024]  (transposed for coalescing: w_out_t[k][c])
    const float* b_out;      // [1024]
};
struct FaqParams {
    const float* f0 = nullptr;   // [B][Tq][1024] prosody features (channels-last)
    const float* z = nullptr;    // [B][Tz][1024] encoder latents (channels-last)
    VqWeights vq[6];             // prosody, content0, content1, residual0..2
    int n_c = 1;
    const float* gamma_beta = nullptr;  // [B][2048] timbre_linear(timbre)
    float* outs = nullptr;       // [B][Tq][1024]
    float* zp = nullptr, *zc = nullptr, *zr = nullptr;  // [B][Tq][1024] each (may be null)
    int64_t* codes_p = nullptr;  // [B][1][Tq]
    int64_t* codes_c = nullptr;  // [B][n_c][Tq]
    int64_t* codes_r = nullptr;  // [B][3][Tq]
    float* sqerr = nullptr;      // [6][B*Tq] per-frame sum (z_e - z_q)^2
    int B = 0, Tq = 0, Tz = 0, Tf0 = 0;   // Tz / Tf0 = frames per utterance of z / f0 (>= Tq)
};
cudaError_t launch_fa_quantize(const FaqParams& p, cudaStream_t st);
// the codes alone (f0, z, vq, n_c, codes_*, B, Tq, Tz, Tf0 read; gamma_beta, outs, the parts and sqerr neither read nor written)
cudaError_t launch_fa_codes(const FaqParams& p, cudaStream_t st);
// FAquantizer from codes: the same six VectorQuantizes' out_proj(codebook[code]) + the AdaLN, no search
struct DeqParams {
    const int64_t* codes_p = nullptr;   // [B][1][T]
    const int64_t* codes_c = nullptr;   // [B][n_c][T], n_c = 1 or 2
    const int64_t* codes_r = nullptr;   // [B][n_r][T], n_r = 0..3 (unread when 0)
    int n_c = 1, n_r = 3;
    VqWeights vq[6];                    // as FaqParams
    const float* gamma_beta = nullptr;  // [B][2048] timbre_linear(timbre)
    float* outs = nullptr;              // [B][T][1024]
    float* zp = nullptr, *zc = nullptr, *zr = nullptr;  // [B][T][1024] each (may be null)
    int B = 0, T = 0;
};
cudaError_t launch_dequantize(const DeqParams& p, cudaStream_t st);
// the same per lane of a decode-pool batch (n <= 32 lanes): lane b reads codes_p[b] [1][F[b]], codes_c[b] [n_c[b]][F[b]],
// codes_r[b] [n_r[b]][F[b]] and gamma_beta[b] [2048], and writes outs [n][Fmax][1024] (frames t >= F[b] zero).  ld > 0:
// every lane's code rows are ld codes apart instead of F[b] (lanes of one [B][rows][ld] tensor, a ragged offline batch).
struct DeqLaneParams {
    const int64_t* codes_p[32];
    const int64_t* codes_c[32];
    const int64_t* codes_r[32];
    const float* gamma_beta[32];
    int n_c[32], n_r[32], F[32];
    VqWeights vq[6];
    float* outs = nullptr;
    int n = 0, Fmax = 0, ld = 0;
};
cudaError_t launch_dequantize_lanes(const DeqLaneParams& p, cudaStream_t st);
// losses[0] = commitment, losses[1] = codebook (identical in forward), from sqerr
cudaError_t launch_vq_loss_reduce(const float* sqerr, int nq, int B, int Tq, float* losses2, cudaStream_t st);

// generic residual VQ over [N frames][D] with D == 1024, codebook_dim == 8 (quantize/rvq.py)
struct RvqParams {
    const float* x = nullptr;    // [B][T][1024] channels-last
    VqWeights vq[8];
    int nq = 0;
    float* qout = nullptr;       // [B][T][1024] quantized_out
    float* allq = nullptr;       // [nq][B][T][1024] or null
    int64_t* idx = nullptr;      // [nq][B][T]
    int B = 0, T = 0;
};
cudaError_t launch_rvq(const RvqParams& p, cudaStream_t st);

// elementwise / small ops
// losses.py:65-89 reconstruction_loss tail (frontend.cu)
cudaError_t launch_mel_loss_terms(const float* spec, int ldspec, int nb, const float* fb /*[nb][64]*/, int B, int F, float eps,
                                  float* terms /*[B*F][2]*/, cudaStream_t st);
cudaError_t launch_strided_sum(const float* in, long long n, int stride, double scale, double* out, cudaStream_t st);
cudaError_t launch_sqdiff_partial(const float* a, const float* b, long long n, float* part, int nblocks, cudaStream_t st);
// dac/nn/loss.py:142-327 spectral losses (frontend.cu)
cudaError_t launch_spec_loss_terms(const float* spec, int ldspec, int nb, const float* fb /*[nb][n_out] or null*/, int n_out, int B, int F,
                                   float eps, float pw, float* terms /*[B*F][2]*/, cudaStream_t st);
cudaError_t launch_absdiff_partial(const float* a, const float* b, long long n, float* part, int nblocks, cudaStream_t st);
cudaError_t launch_spec_loss_combine(const double* v, int n, float mag_weight, float log_weight, float* loss, cudaStream_t st);
// their gradients (fac_spectral_loss_grad / fac_l1_loss_grad): dL/d(Re, Im) in place over the spec rows of the requested
// signals, each row scaled by a power of two whose inverse goes to inv_scale [2*B*F]; the adjoint of launch_stft_frames
// (f_first = 0) over those scaled rows into out [B][T] (accumulate: add instead of write); sgn(a - b) / n
cudaError_t launch_spec_loss_grad(float* spec, int ldspec, int nb, const float* fb, int n_out, int B, int F, float eps, float pw,
                                  float mag_scale, float log_scale, int want_x, int want_y, float* inv_scale, cudaStream_t st);
cudaError_t launch_stft_overlap_add_grad(const float* dframes /*[B][F][win]*/, const float* inv_scale /*[B][F]*/, float* out, int B, int T,
                                         int F, int hop, int win, int pad, int accumulate, cudaStream_t st);
cudaError_t launch_l1_grad(const float* a, const float* b, long long n, float inv_n, float* da, float* db, cudaStream_t st);
cudaError_t launch_add3(const float* a, const float* b, const float* c /* or null */, long long n, float* out, cudaStream_t st);
cudaError_t launch_loss_combine(const double* v13, float* loss, float* terms, cudaStream_t st);
cudaError_t launch_transpose(const float* in, float* out, int B, int R, int C, cudaStream_t st);  // [B][R][C]->[B][C][R]
// tanh(a + g_a) * sigmoid(b + g_b); g = null or one [2*hidden] conditioning row per utterance (rows_per_utt rows each, g_stride floats apart)
cudaError_t launch_wn_gate(const float* xin, float* acts, size_t n_rows, int hidden, cudaStream_t st, const float* g = nullptr,
                           size_t rows_per_utt = 0, size_t g_stride = 0);
cudaError_t launch_wn_update(const float* rs, float* x, float* out, size_t n_rows, int hidden, int last, cudaStream_t st);
cudaError_t launch_glu_res(const float* y, float* x, int B, int T, int C, const int* valid_len, cudaStream_t st);  // x = x + y1*sig(y2) (masked)
// lane_len (a ragged batch; device [B], with its host copy lane_len_host): lane b is the attention of its own first lane_len[b]
// rows, as a call with T = lane_len[b] computes it, bit for bit, in the variant that call takes; its other rows of o are 0.
cudaError_t launch_attention(const float* q, const float* k, const float* v, float* o, int B, int T, int heads,
                             int dk, const int* valid_len, cudaStream_t st, int force_stream = 0, const int* lane_len = nullptr,
                             const int* lane_len_host = nullptr);
// mean over T frames (sum over all T / valid_len[b] when valid_len); lane_len [B] device: lane b's first lane_len[b] frames
// only, summed as a call with T = lane_len[b] sums them
cudaError_t launch_mean_pool(const float* x, float* out, int B, int T, int C, const int* valid_len, cudaStream_t st,
                             const int* lane_len = nullptr);
cudaError_t launch_fill_u32(unsigned int* p, unsigned int v, size_t n, cudaStream_t st);

// JDCNet eval-mode pieces and train.py's targets (jdc.cu); maps are [B][T][F + 2][C] with zero pad columns, lens [B] device
// frames per lane (null: T each)
cudaError_t launch_jdc_conv_in(const float* mel /*[B][80][T]*/, const float* w /*[9][64]*/, const float* bias, float* y, int B, int T,
                               const int* lens, cudaStream_t st);
cudaError_t launch_jdc_pre_pool(const float* x, const float* sc, const float* sh, float* y, int B, int T, int F, int C, cudaStream_t st);
cudaError_t launch_jdc_pool_block(const float* x, const float* sc, const float* sh, float* gan, float* pool, float* lstm_in, int B,
                                  int T, const int* lens, cudaStream_t st);
cudaError_t launch_jdc_head(const float* yf, const float* yb, const float* w, const float* bias, float* f0, int B, int T,
                            const int* lens, cudaStream_t st);
cudaError_t launch_f0_targets(const float* f0, const int* lens, int B, int T, float* out, float* glob, cudaStream_t st);
cudaError_t launch_log_norm(const float* mel, int B, int T, float* out, cudaStream_t st);

// alias-free activation (alias_free_torch/act.py:24-29): up x2 -> snake-beta/identity -> down x2
cudaError_t launch_alias_free_act(const float* x, float* y, int B, int C, int T, const float* filt12,
                                  const float* alpha, const float* inv_beta, cudaStream_t st);

}  // namespace fac
