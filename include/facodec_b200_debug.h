/* facodec_b200 -- kernel-level test hooks, host-only packing/plan probes and per-launch profiling.
 *
 * NOT part of the drop-in surface (that is include/facodec_b200.h = SURVEY.md section 8b): these entry points exist
 * for tests/test_gpu_kernels.py, tests/test_host.py, scripts/ and bench.py's roofline pass.  Same library, same
 * conventions (plain pointers and sizes, negative fac_status on error).
 */
#ifndef FACODEC_B200_DEBUG_H
#define FACODEC_B200_DEBUG_H

#include "facodec_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Kernel-level test hooks (used by tests/test_gpu_kernels.py; not part of the drop-in surface).
 * fac_debug_conv runs the generic channels-last conv kernel on one layer: x [B,Tin,Cin] and
 * y [B,Tout,Cout] are DEVICE channels-last buffers, w_host is a HOST nn.Conv1d weight
 * [Cout,Cin,K] (already weight-normed), bias/in_alpha/out_alpha HOST vectors or NULL,
 * res a DEVICE tensor like y or NULL; act: 0 none, 1 tanh, 2 mish.
 * fac_debug_slstm runs SLSTM (2 layers + skip) on x [B,T,H] DEVICE with HOST nn.LSTM weights
 * w[8] = {w_ih_l0, w_hh_l0, b_ih_l0, b_hh_l0, w_ih_l1, ...}. */
int fac_debug_conv(fac_handle* h, const float* x, const float* w_host, const float* bias_host, int B, int Tin,
                   int Cin, int Cout, int K, int dil, int stride, int pad_left, int pad_right, int reflect,
                   const float* in_alpha_host, const float* out_alpha_host, int act, const float* res,
                   float* y, int Tout, void* stream);
/* Same contract as fac_debug_conv, forced through the wgmma conv kernel: promoted = 0 -> 3xTF32, one accumulator,
 * 1 -> 3xTF32 with each window of <= 48 chained MMAs promoted into an fp32 master accumulator, 2 -> bf16 hi/lo split
 * (decoder-only precision class), 3 -> promoted fp16 hi + 2^11-scaled fp16 lo split (the class used upstream of the
 * VQ), 4 -> 3 in the transposed formulation (weights as the wgmma A operand, time as wgmma N), 5 -> ONE fp16 pass (the
 * k = 7 convs downstream of the VQ).  The handle's "tc_occ2_maxn" applies.  Returns FAC_ERR_UNSUPPORTED when the layer
 * geometry is not eligible (Cin % 16, Cout % 16, stride) and for any other mode. */
int fac_debug_conv_tc(fac_handle* h, const float* x, const float* w_host, const float* bias_host, int B, int Tin,
                      int Cin, int Cout, int K, int dil, int stride, int pad_left, int pad_right, int reflect,
                      const float* in_alpha_host, const float* out_alpha_host, int act, const float* res,
                      float* y, int Tout, int promoted, void* stream);
/* fac_debug_conv_tc with the layer's K loop stepped one 16-channel chunk at a time (the planner groups 2 or 4 chunks per
 * step on layers of 1-3 taps): the reference a grouped launch must equal bit for bit.  *group receives the number of
 * chunks per step the layer's own plan takes. */
int fac_debug_conv_tc_group1(fac_handle* h, const float* x, const float* w_host, const float* bias_host, int B, int Tin,
                             int Cin, int Cout, int K, int dil, int stride, int pad_left, int pad_right, int reflect,
                             const float* in_alpha_host, const float* out_alpha_host, int act, const float* res,
                             float* y, int Tout, int promoted, void* stream, int* group);
/* One layer of a ragged batch: fac_debug_conv_tc's arguments with lane_len_host (HOST, B entries, or NULL: Tin each)
 * the input rows of each lane, each padded about its own end as ConvParams::lane_len / TcConvParams::lane_len do.
 * path = -1 runs launch_conv (the fp32 FMA kernels: it picks the cin1, cout1 or generic kernel itself), path = 0..5 the
 * tensor-core classes of fac_debug_conv_tc.  A length outside [1, Tin] returns FAC_ERR_INVALID before anything is
 * launched. */
int fac_debug_conv_lanes(fac_handle* h, const float* x, const float* w_host, const float* bias_host, int B, int Tin,
                         int Cin, int Cout, int K, int dil, int stride, int pad_left, int pad_right, int reflect,
                         const float* in_alpha_host, const float* out_alpha_host, int act, const float* res,
                         float* y, int Tout, int path, const int* lane_len_host, void* stream);
/* One ResidualUnit (dac/model/dac.py:25-42) y = x + conv1(snake(conv7_d(snake(x)))) on DEVICE channels-last
 * x, y [B,T,C] with HOST folded weights w7 [C,C,7], w1 [C,C,1].  mode 0: fp32 FMA kernels, 1: two tensor-core
 * launches, 2: the single fused tensor-core launch (FAC_ERR_UNSUPPORTED if the geometry cannot be fused);
 * 3 / 4: as 1 / 2 with the bf16 hi/lo split; 5 / 6: as 3 / 4 with the k = 7 conv in one fp16 pass; 7 / 8: as 1 / 2 for
 * an encoder unit (weights packed for the promoted class, run upstream of the VQ: fp16 hi + 2^11-scaled lo, two CTAs per
 * SM; 8 only at C = 64 and 128).  Any other mode returns FAC_ERR_INVALID.  Causal. */
int fac_debug_resunit(fac_handle* h, const float* x, const float* w7_host, const float* b7_host, const float* w1_host,
                      const float* b1_host, const float* alpha1_host, const float* alpha2_host, int B, int T, int C,
                      int dil, int mode, float* y, void* stream);
/* fac_debug_resunit with the unit's padding chosen by causal (0: the non-causal split of the redecoder's decoder,
 * reflected at both ends) and lane_len_host (HOST, B entries in [1, T], or NULL) each lane's own rows, as the ragged
 * decoder passes them.  A length outside [1, T] returns FAC_ERR_INVALID before anything is launched. */
int fac_debug_resunit_lanes(fac_handle* h, const float* x, const float* w7_host, const float* b7_host,
                            const float* w1_host, const float* b1_host, const float* alpha1_host,
                            const float* alpha2_host, int B, int T, int C, int dil, int mode, int causal,
                            const int* lane_len_host, float* y, void* stream);
/* clock64() phase timestamps written by one probe CTA of the most recent conv_tc_kernel launch:
 * [0] start, [1] all activation chunks produced, [2] GEMM 1 retired, [3] GEMM-2 operand produced (fused),
 * [4] GEMM 2 retired (fused), [5] epilogue done.  Kernel-tuning aid. */
int fac_debug_tc_phase_clocks(fac_handle* h, long long* out8);
/* Probe producer thread of the same launch, cycles summed over the tile's chunks: [0] waiting for a free operand buffer,
 * [1] waiting for the chunk's global loads, [2] Snake + split + stores + arrive, [3] number of chunks. */
int fac_debug_tc_producer_clocks(fac_handle* h, long long* out4);
/* Per-chunk timeline of the same probe CTA, out80 = [5][16] absolute clock64 values for chunks 0..15: [0] MMA warp saw the
 * chunk's operands, [1] MMA warp finished issuing the chunk, [2] producer thread 0 saw the operand buffer free,
 * [3] producer thread 0 arrived (chunk stored), [4] cycles the MMA warp waited for weights inside the chunk. */
int fac_debug_tc_trace(fac_handle* h, long long* out80);
/* Host-only: the recurrent-weight packing of lstm_rec_kernel for one nn.LSTM weight_hh [4H][H] (HOST, gate order
 * i,f,g,o): bf16 = 0 -> fp32 [G][H][4U] (row r = gate*U + u of the CTA owning hidden units g*U..g*U+U-1);
 * bf16 = 1 -> [G][H/16][hi|lo][8 k-pairs][4U] words of two bf16 (even k in the low half), lo = rn_bf16(w - hi).
 * bf16 = 2 / 3 -> the resident-W kernel's layouts (lstm2.cu): one fp16 plane [G][H/16][8][4U] / fp16 hi + 2^11-scaled lo planes
 * [G][H/16][hi|lo][8][4U], column of row r of k pair k2 = r ^ swizzle(k2) (conflict-free fragment loads).
 * Returns the number of 32-bit words (G*H*4U) also when out is NULL/too small; info3 = {U, G, 4U}. */
long long fac_debug_lstm_pack(const float* whh_host, int H, int bf16, float* out, long long capacity_floats, int* info3);
/* Host-only: the launch plan of one stream-pool step.  kind 0 (codes pool): counters[4 i ..] = {samples encoded, x history
 * length, LSTM-output history length, frames emitted} of session i, lengths[i] = its chunk in samples; kind 1 (voice-conversion
 * pool): counters[3 i ..] = {code frames received, z frames final, output frames emitted}, lengths[i] = its chunk in frames;
 * kind 2 (decode pool): counters[i] = frames decoded by session i, lengths[i] = its chunk in frames; kind 3 (voice-conversion
 * pool with switches): counters[4 i ..] = kind 1's and 1 for a session whose timbre changed since its last step.
 * group[i] receives the group of session i (sessions whose launch sequences are identical; groups numbered in order of first
 * appearance), batch[i] its batch (each group cut into batches of <= 32 in input order).  Returns the number of batches. */
int fac_debug_pool_plan(int kind, int n, const long long* counters, const int* lengths, int* group, int* batch);
/* Host-only: the plan of one voice-conversion step on a stream at (N code frames received, Zf z frames final, Yf output
 * frames emitted) fed F frames (F = 0 exactly when finish), stale = 1 after a timbre switch.  out16 = {F, codes window
 * frames, of them history, z window frames, of them history, first kept z row in the codes window, kept z rows, output
 * frames, first output frame in the z window, first z row kept after the step, z rows kept, stale (0 when the z history is
 * empty), N, Zf and Yf after the step, code frames the stream keeps}.  Returns 16. */
int fac_debug_vc_plan(long long N, long long Zf, long long Yf, int F, int finish, int stale, long long* out16);
/* Host-only: the header checks fac_*_pool_import runs before it touches a pool, for a pool of `kind` (FAC_STATE_*) whose
 * weights give `fingerprint` and whose handle has options[FAC_STATE_OPTIONS], given payload_bytes of payload: the status
 * the import would return for the header, and on success the header's counters in counters_out[FAC_STATE_COUNTERS] (may
 * be NULL).  The pool-side checks (counters, n_c, quantum, capacity, device) are not part of it. */
int fac_debug_state_header(const void* header, size_t header_bytes, int kind, uint64_t fingerprint, const int64_t* options,
                           size_t payload_bytes, long long* counters_out);
/* Host-only: the StyleEncoder batches of fac_codes_pool_timbre over n sessions of frames[i] mel frames: batch[i] = the
 * batch of session i (batches in launch order); returns the number of batches. */
int fac_debug_timbre_plan(int n, const int* frames, int* batch);
/* Host-only: where one batch lane's carry of one resident-W LSTM layer (H = 1024 or 1536; pass3 = 1: hi | lo h planes) sits
 * in a stream's state: pos[j] for word j (h words first, then the c floats) is its index in [state_h words | state_c floats].
 * The pools move exactly these words between a session's slot and any lane.  Returns the word count (also when pos is
 * NULL or capacity too small). */
long long fac_debug_lstm_lane_map(int H, int pass3, int lane, long long* pos, long long capacity);
/* Host-only: the padding index map every conv kernel applies instead of materialising a padded copy
 * (dac/model/encodec.py:96-113 pad1d incl. the short-input branch): out[i] = source row of padded position
 * i - pad_left, or -1 where the padded value is zero; n must be pad_left + L + pad_right. */
int fac_debug_pad_map(int L, int pad_left, int pad_right, int reflect, int* out, int n);
/* Host-only: that map for each lane of a ragged batch, as the conv kernels build it from per-lane lengths: lane b (of B)
 * pads its own lane_len[b] <= Tin rows (lane_len NULL: Tin each).  out [B][n], n = pad_left + Tin + pad_right; positions
 * past the lane's own padded length hold rows the lane's outputs never read, each -1 or below lane_len[b]. */
int fac_debug_lane_pad_map(const int* lane_len, int B, int Tin, int pad_left, int pad_right, int reflect, int* out, int n);
/* Host-only (no GPU, no handle): the tile plan of the wgmma conv kernel for one layer geometry.  mode: 0 TF32,
 * 1 promoted TF32, 2 bf16, 3 promoted fp16 hi + scaled lo, 4 fused ResidualUnit bf16, 5 fused TF32, 6 mode 3 in the
 * transposed formulation, 7 ONE fp16 pass (the k = 7 convs downstream of the VQ), 8 fused ResidualUnit with its k = 7
 * conv in one fp16 pass, 9 fused ResidualUnit in the class of mode 3 (N = C and two CTAs per SM, or unsupported).
 * occ2_maxn as the "tc_occ2_maxn" option.  Tout may be 0 (unknown).  out8 = {N, MT (2: warpgroups split 128 rows, 1: they split N over 64 rows),
 * K chunks, weight-ring stages, rows per tile, dynamic shared-memory bytes, padded rows of the operand buffer,
 * chunks per promotion}.  FAC_ERR_UNSUPPORTED when the layer is not eligible. */
int fac_debug_tc_plan(int Cin, int Cout, int K, int dil, int stride, int Tout, int mode, int occ2_maxn, int* out8);
/* Host-only: 16-channel chunks per K-loop step (1, 2 or 4) of the same plan, or the negative status of fac_debug_tc_plan.
 * smem2 (or NULL) receives the dynamic shared-memory bytes of that plan and of the layer's one-chunk-per-step plan. */
int fac_debug_tc_plan_group(int Cin, int Cout, int K, int dil, int stride, int Tout, int mode, int occ2_maxn, int* smem2);
/* Host-only: packs nn.Conv1d weights [Cout][Cin][K] (HOST) into the tensor-core blob of mode 0..3 (see
 * fac_debug_tc_plan): [Cout/N][K chunks][taps][hi|lo][k-groups][N][16 bytes], hi|lo = TF32 pair (4 k-groups of 4 fp32
 * words), bf16 pair or fp16 hi / 2^11-scaled lo (2 k-groups of 8 halves).  Returns the blob size in 32-bit words (also
 * when blob_out is NULL or too small), or a negative status. */
long long fac_debug_tc_pack(const float* w_host, int Cin, int Cout, int K, int stride, int mode, float* blob_out,
                            long long capacity_floats);
/* clock64() totals of CTA 0 of the most recent lstm_rec_kernel launch, summed over all steps:
 * [0] grid-barrier wait, [1] W_hh/h streaming + MMAs, [2] cross-warp reduce + gate math, [3] publish. */
int fac_debug_lstm_phase_clocks(fac_handle* h, long long* out4);
/* Host-only: see engine.cu -- the conv form of a ConvTranspose1d(k = 2s, stride s) weight [Cin][Cout][2s]: causal -> 2 taps,
 * non-causal -> 3 taps, out [taps][Cin][s*Cout] (phase-major channels); returns the float count. */
long long fac_debug_convtr_pack(const float* w_host, int Cin, int Cout, int stride, int causal, float* out,
                                long long capacity_floats);
/* fac_debug_slstm (synchronous) runs the LSTM with the precision options set on h.  upstream = 1: packed and run as the
 * encoder's LSTM (promoted input projection, 3-pass recurrence); 0: as the decoder's.  chunks = NULL or n_chunks = 0: one
 * pass over all T.  Otherwise chunks (HOST, n_chunks lengths summing to T) runs T chunk by chunk, carrying the LSTM state
 * from a zero state as the streaming calls do: needs B <= 32 and the resident-W kernel (FAC_ERR_UNSUPPORTED otherwise).
 * Bad chunk lists return FAC_ERR_INVALID.  Both errors are returned before anything is launched. */
int fac_debug_slstm(fac_handle* h, const float* x, const float* const* w_host, int B, int T, int H, int upstream,
                    const int* chunks, int n_chunks, float* y, void* stream);
/* fac_debug_slstm_lanes (synchronous): the same LSTM over all T steps as a stream chunk with per-lane step counts, B <= 32
 * (the resident-W kernel).  carry (DEVICE [B][2 layers][words], words = fac_debug_lstm_lane_map's count for H and the
 * class's pass3) holds each row's (h, c) in lane-map order: read as the initial state, overwritten with the final one.
 * lens (HOST, B entries in [0, T], or NULL for T each): row b steps lens[b] times and its carry is the state after them;
 * its rows of y past lens[b] are finite but meaningless.  With lens NULL the kernel runs without per-lane counts.  Lengths
 * run the decoder's one-pass class only (upstream = 0; FAC_ERR_UNSUPPORTED otherwise). */
int fac_debug_slstm_lanes(fac_handle* h, const float* x, const float* const* w_host, int B, int T, int H, int upstream,
                          const int* lens, uint32_t* carry, float* y, void* stream);
/* fa_quantize_kernel + vq_loss_reduce_kernel on caller-given features, the six VectorQuantizes and the AdaLN of
 * FAquantizer.forward_v2 (synchronous).  DEVICE f0 [B][Tf0][1024], z [B][Tz][1024] (Tf0, Tz >= Tq: frame t of
 * utterance b is row b*Tf0 + t / b*Tz + t), gamma_beta [B][2048].  vq_host[i] = HOST {in_w [8][1024], in_b [8],
 * out_w [1024][8], out_b [1024], codebook [1024][8]} of VQ i = prosody, content 0, content 1, residual 0..2 (weights
 * already weight-normed), packed as the product packs them.  DEVICE outputs as FaqParams: outs / zp / zc / zr
 * [B][Tq][1024] (zp, zc, zr may be NULL), codes_p [B][1][Tq], codes_c [B][n_c][Tq], codes_r [B][3][Tq] int64,
 * sqerr [6][B*Tq], losses2 [2]. */
int fac_debug_fa_quantize(fac_handle* h, const float* f0, const float* z, const float* const vq_host[6][5],
                          const float* gamma_beta, int n_c, int B, int Tq, int Tz, int Tf0, float* outs, float* zp,
                          float* zc, float* zr, int64_t* codes_p, int64_t* codes_c, int64_t* codes_r, float* sqerr,
                          float* losses2, void* stream);
/* The StyleEncoder's self-attention (launch_attention, synchronous) on DEVICE channels-last q, k, v, o
 * [B][T][heads*256]; valid_len DEVICE int [B] (keys and queries t >= valid_len[b] masked) or NULL.
 * force_stream = 0 keeps launch_attention's choice (stored scores up to 200 KB of shared memory), 1 forces the
 * kernel that recomputes the scores. */
int fac_debug_attention(fac_handle* h, const float* q, const float* k, const float* v, float* o, int B, int T,
                        int heads, const int* valid_len, int force_stream, void* stream);
/* Registers (dst != NULL) or clears a named tap: the next forward copies that channels-last
 * intermediate into dst (DEVICE, up to capacity_floats).  Names: enc_conv0, enc_block1..4 (after the down-sampling conv),
 * enc_block<i>.res<j> (after ResidualUnit j = 0..2 of EncoderBlock i), enc_lstm, mel80, f0_input, gamma_beta, dec_conv0,
 * dec_lstm, dec_block<i>.up (after DecoderBlock i's up-sampling conv), dec_block<i>.res<j>, dec_block1..4 (the block's
 * output, = dec_block<i>.res2); the dec_* names also fire in the redecoder's decoder.  dec_pool.latents: the per-lane dequantized
 * latents [n][Fmax][1024] of a fac_dec_pool_decode_codes batch (each batch overwrites it; frames past a lane's F are 0).
 * Per scale i of fac_reconstruction_loss ("recon.") and fac_spectral_loss ("spec."): recon.dft.<i> / spec.dft.<i> the
 * DFT GEMM output [2*B*F][ld] (rows [0, B*F) of x, then those of the second signal; Re at column 2k, Im at 2k + 1,
 * columns >= 2*nb zero), recon.terms.<i> / spec.terms.<i> the per-frame terms [B*F][2], and recon.fb.<i> / spec.fb.<i>
 * (mel scales only) the filterbank [nb][n_mels] as the terms kernel reads it.  fac_spectral_loss_grad adds spec.dframes.<i>:
 * the frames buffer [2*B*F][w] after the transposed DFT GEMM, whose rows of each signal with a requested gradient hold
 * dL/dframes scaled by a per-row power of two (the other signal's rows still hold its frames), and spec.dscale.<i> [2*B*F]
 * the inverse row scales: dL/dframes = row * dscale[row].  fac_jdc_forward's taps, maps channels-last [B][T][F + 2][C]
 * with zero pad columns: jdc.conv_in (conv_block.0-2, F = 80), jdc.conv_block (conv_block.3), jdc.res<i>.pre (res_block<i>
 * pre_conv), jdc.res<i>.conv1 (conv.0-2), jdc.res<i> (the block's output); jdc.lstm_in [B][T][512], jdc.lstm.xg_fwd /
 * jdc.lstm.xg_rev [B][T][1024] (input GEMMs, gate order i, f, g, o, b_ih + b_hh added), jdc.lstm.fwd / jdc.lstm.rev [B][T][256]. */
int fac_debug_tap(fac_handle* h, const char* name, float* dst, size_t capacity_floats);

/* Per-kernel-family device timing for bench.py's roofline object: when enabled, every launch of
 * the forward paths is bracketed by CUDA events on the launching stream.  Families: "conv"
 * (conv_cl_kernel, fp32 FMA), "conv_tc" / "conv_tcp" (conv_tc_kernel, plain / promoted), "lstm_rec", "fa_quantize",
 * "dequantize" (decoding from codes).  fac_profile_get returns
 * the accumulated device milliseconds, ALGORITHMIC flops (2*MACs) and bytes (in + out + weights
 * once) and launch count since the last fac_profile_reset (it synchronises the device). */
int fac_profile_enable(fac_handle* h, int on);
int fac_profile_reset(fac_handle* h);
int fac_profile_get(fac_handle* h, const char* family, double* ms, double* flops, double* bytes,
                    long long* launches);
/* Per-call-site breakdown as text lines "key<TAB>ms<TAB>GFLOP<TAB>GB<TAB>launches"; returns the
 * buffer size needed (call with buf = NULL first). */
size_t fac_profile_dump(fac_handle* h, char* buf, size_t cap);

#ifdef __cplusplus
}
#endif
#endif /* FACODEC_B200_DEBUG_H */
