/* facodec_b200 -- C-ABI of the B200-native FAcodec encode -> quantize -> decode hot path.
 *
 * The reference (Plachtaa/FAcodec) has no FFI layer: its boundary is the Python nn.Module call
 * surface  model.encoder(x) / model.quantizer(z, wave, ...) / model.decoder(z)  on the Munch
 * returned by build_model (modules/commons.py:283-348).  Each entry point below names the
 * reference interface it replaces; facodec_b200/modules.py is the thin ctypes shim that puts the
 * nn.Module surface back on top (INTEGRATION.md shows the binding).
 *
 * Conventions: plain pointers and sizes only; every tensor argument is a DEVICE pointer in the
 * reference's own layout (float32 [B, C, T] contiguous, int64 codes) unless the name ends in
 * _host; outputs are caller-allocated; `stream` is a cudaStream_t (0 = legacy default stream);
 * calls on one handle must be serialised by the caller.  Every function returns 0 on success or
 * a negative fac_status; fac_last_error() gives the text.  No exceptions cross the ABI.
 * Scratch memory is a grow-only device arena owned by the handle (fac_workspace_bytes).
 */
#ifndef FACODEC_B200_H
#define FACODEC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct fac_handle fac_handle;

enum fac_status {
    FAC_OK = 0,
    FAC_ERR_INVALID = -1,   /* bad argument / shape */
    FAC_ERR_STATE = -2,     /* weights missing or not finalized */
    FAC_ERR_CUDA = -3,      /* CUDA runtime error (text in fac_last_error) */
    FAC_ERR_UNSUPPORTED = -4
};

/* FAC_REDECODER / FAC_REDECODER_DECODER: the voice-conversion model of build_model(args, stage='redecoder')
 * (modules/commons.py:385-412): modules/redecoder.py Redecoder (wavenet) and its Decoder(causal=False, lstm=0). */
enum fac_module { FAC_ENCODER = 0, FAC_QUANTIZER = 1, FAC_DECODER = 2, FAC_REDECODER = 3, FAC_REDECODER_DECODER = 4,
                  FAC_NUM_MODULES = 5 };

/* Library/ABI version (bumped on any signature change). */
int fac_abi_version(void);

/* Create / destroy an engine bound to CUDA device `device`. */
int fac_create(fac_handle** out, int device);
int fac_destroy(fac_handle* h);
const char* fac_last_error(const fac_handle* h);

/* Checkpoint loading.  Replaces  model[key].load_state_dict(ckpt[key])  (reconstruct.py:30-34,
 * modules/commons.py:446-471): feed every tensor of the reference state_dict of `module`
 * (reference key names, e.g. "block.1.block.0.block.1.conv.conv.weight_v"), HOST float32 data,
 * then call fac_finalize once.  fac_finalize folds weight-norm (g * v / ||v||, encodec.py:42-51),
 * Snake 1/(alpha+1e-9), LSTM biases, normalises the VQ codebooks, builds the STFT basis from
 * "to_mel.spectrogram.window", packs everything into kernel layouts and uploads it.
 * Modules whose tensors were never loaded stay unavailable (their entry points return
 * FAC_ERR_STATE). */
int fac_load_tensor(fac_handle* h, int module, const char* key, const float* data_host,
                    const int64_t* shape, int ndim);
int fac_finalize(fac_handle* h);

/* Replicated deployment (one process per GPU): rank 0 reads the checkpoint and broadcasts the raw
 * tensors as ONE flat fp32 buffer (ncclBroadcast through torch.distributed, see
 * facodec_b200/distributed.py); every rank then runs fac_load_tensor + fac_finalize locally.
 * There is no collective on the hot path. */

/* model.encoder(x): dac/model/dac.py:103-104 Encoder.forward.
 * x [B,1,T] -> z [B,1024,ceil(T/300)]. */
int fac_encode(fac_handle* h, const float* x, int B, int T, float* z, void* stream);
int fac_encode_frames(int T);   /* ceil-div chain of the strided convs = output frames */

/* model.quantizer(z, wave, n_c, n_t, full_waves, wave_lens, return_codes):
 * modules/quantize.py:375-454 FAquantizer.forward_v2 in eval mode.
 * z [B,1024,Tz], wave [B,1,T]; Tq = min(T/300, Tz).  full_waves [B,T_full] + wave_lens[B]
 * (int64, device) may be NULL (then the timbre comes from `wave`).  Outputs (any of zp/zc/zr/
 * codes_* may be NULL): outs, zp, zc, zr [B,1024,Tq]; losses2[2] = {commitment, codebook};
 * timbre [B,1024]; codes_p [B,1,Tq], codes_c [B,n_c,Tq], codes_r [B,3,Tq] int64. */
int fac_quantize(fac_handle* h, const float* z, const float* wave, int B, int T, int Tz, int n_c,
                 const float* full_waves, int T_full, const int64_t* wave_lens,
                 float* outs, float* zp, float* zc, float* zr, float* losses2, float* timbre,
                 int64_t* codes_p, int64_t* codes_c, int64_t* codes_r, void* stream);

/* model.decoder(z): dac/model/dac.py:164-165 Decoder.forward.  z [B,1024,Tf] -> y [B,1,300*Tf]. */
int fac_decode(fac_handle* h, const float* z, int B, int Tf, float* y, void* stream);

/* reconstruct.py:56-61 in one call, device buffers: encoder -> quantizer(n_c) -> decoder with the
 * latents kept channels-last on the device (no boundary transposes).  codes_* / timbre may be NULL. */
int fac_codec_forward(fac_handle* h, const float* x, int B, int T, int n_c, float* y,
                      int64_t* codes_p, int64_t* codes_c, int64_t* codes_r, float* timbre, void* stream);

/* Same, HOST buffers (pinned recommended): H2D of x, forward, D2H of y + codes, stream sync. */
int fac_codec_forward_host(fac_handle* h, const float* x_host, int B, int T, int n_c, float* y_host,
                           int64_t* codes_p_host, int64_t* codes_c_host, int64_t* codes_r_host, void* stream);

/* Compress only: fac_codec_forward without the decoder (encoder -> quantizer(n_c), the quantizer's waveform-only front
 * forked beside the encoder): the same codes and timbre as fac_codec_forward, bit for bit.  codes_p [B,1,Tq],
 * codes_c [B,n_c,Tq], codes_r [B,3,Tq] int64 are required; timbre [B,1024] may be NULL. */
int fac_codec_encode(fac_handle* h, const float* x, int B, int T, int n_c, int64_t* codes_p, int64_t* codes_c,
                     int64_t* codes_r, float* timbre, void* stream);
/* Ragged batches: fac_codec_forward_lens and fac_codec_encode_lens take lengths, a HOST array of B sample counts in
 * (1024, T] (NULL: T each).  Lane b computes x[b, 0, :lengths[b]] exactly as its own B = 1 call does, bit for bit: its
 * F_b = min(lengths[b] / 300, fac_encode_frames(lengths[b])) code frames, timbre and 300 * F_b samples.  Outputs keep the
 * shapes of the call without lengths; codes past F_b are -1 and y past 300 * F_b is 0.  Samples past a lane's length are
 * never read.  A length out of range is FAC_ERR_INVALID before anything is queued; lengths that all equal T make the
 * call without them. */
int fac_codec_forward_lens(fac_handle* h, const float* x, int B, int T, const int* lengths, int n_c, float* y,
                           int64_t* codes_p, int64_t* codes_c, int64_t* codes_r, float* timbre, void* stream);
int fac_codec_encode_lens(fac_handle* h, const float* x, int B, int T, const int* lengths, int n_c, int64_t* codes_p,
                          int64_t* codes_c, int64_t* codes_r, float* timbre, void* stream);
/* Timbre only: the timbre [B,1024] fac_codec_encode_lens writes for the same x and lengths (any n_c), bit for bit, from
 * the launches it runs for it alone -- the mel front-end and the StyleEncoder (modules/quantize.py:377-379), with the
 * same lanes -- and no encoder, prosody or VQ launch.  Needs only the quantizer; the rules on T and lengths are those of
 * fac_codec_encode_lens. */
int fac_codec_timbre_lens(fac_handle* h, const float* x, int B, int T, const int* lengths, float* timbre, void* stream);

/* Decompress.  The reference has no single call for it (FAquantizer.decode, modules/quantize.py:245-254, needs the
 * timbre quantizer that timbre_norm = True leaves out); it is ResidualVectorQuantize.from_codes (dac/nn/quantize.py:200-220:
 * out_proj(codebook[code]) summed over a quantizer's rows) on the prosody, content and residual quantizers, then
 * outs = LayerNorm((z_p + z_c) + z_r) * gamma + beta with gamma | beta = timbre_linear(timbre) (modules/quantize.py:437-449).
 * codes_p [B,1,T], codes_c [B,n_c_rows,T] (n_c_rows = 1 or 2), codes_r [B,n_r_rows,T] (n_r_rows = 0..3; NULL allowed when
 * 0: z_r is left out, as the training-time res_mask = 0 does) int64, timbre [B,1024] -- any utterance's timbre, so codes of
 * one speaker decode in the voice of another.  A code outside [0, 1024) is never read past the codebook: it makes its
 * frame's outputs NaN.
 * fac_dequantize: outs [B,1024,T]; zp / zc / zr [B,1024,T] may be NULL.
 * fac_codes_decode: the same, then the codec's decoder with the latents kept channels-last: y [B,1,300*T]. */
int fac_dequantize(fac_handle* h, const int64_t* codes_p, const int64_t* codes_c, int n_c_rows, const int64_t* codes_r,
                   int n_r_rows, const float* timbre, int B, int T, float* outs, float* zp, float* zc, float* zr, void* stream);
int fac_codes_decode(fac_handle* h, const int64_t* codes_p, const int64_t* codes_c, int n_c_rows, const int64_t* codes_r,
                     int n_r_rows, const float* timbre, int B, int T, float* y, void* stream);
/* Ragged batches: fac_codes_decode_lens and fac_voice_convert_lens take frames, a HOST array of B frame counts in [1, T]
 * (NULL: T each).  Lane b decodes its first frames[b] frames exactly as its own B = 1 call on codes[..., :frames[b]] does,
 * bit for bit; codes past them are neither read nor checked, and y[b, 0, 300 * frames[b]:] is 0.  A count out of range is
 * FAC_ERR_INVALID before anything is queued.  Counts that all equal T make the call without them. */
int fac_codes_decode_lens(fac_handle* h, const int64_t* codes_p, const int64_t* codes_c, int n_c_rows, const int64_t* codes_r,
                          int n_r_rows, const float* timbre, int B, int T, const int* frames, float* y, void* stream);

/* Voice conversion (reconstruct_redecoder.py:108-122, webui.py:68-81).
 * fac_redecode = model.encoder(p_code, c_code, timbre, use_p_code, use_c_code, n_c) of the redecoder model,
 * modules/redecoder.py:35-48: codes_p [B,1,T], codes_c [B,n_c_rows,T] int64 (device; the codec's codes[0], codes[1]),
 * timbre [B,1024] -> z [B,1024,T].  n_c <= n_c_rows <= 2 content codebooks are summed.
 * fac_redecoder_decode = that model's decoder (non-causal, no SLSTM: config_redecoder.yml decoder_causal / decoder_lstm),
 * z [B,1024,Tf] -> y [B,1,300*Tf].  fac_voice_convert runs both with the latents kept channels-last on the device.
 * A code the call reads (codes_p when use_p_code, content rows < n_c when use_c_code) outside [0, 1024) is never read past the
 * embedding tables: it makes its frame's embedding NaN, which the WN spreads to the z frames within 32 of it. */
int fac_redecode(fac_handle* h, const int64_t* codes_p, const int64_t* codes_c, int n_c_rows, const float* timbre,
                 int B, int T, int use_p_code, int use_c_code, int n_c, float* z, void* stream);
int fac_redecoder_decode(fac_handle* h, const float* z, int B, int Tf, float* y, void* stream);
int fac_voice_convert(fac_handle* h, const int64_t* codes_p, const int64_t* codes_c, int n_c_rows, const float* timbre,
                      int B, int T, int use_p_code, int use_c_code, int n_c, float* y, void* stream);
int fac_voice_convert_lens(fac_handle* h, const int64_t* codes_p, const int64_t* codes_c, int n_c_rows, const float* timbre,
                           int B, int T, int use_p_code, int use_c_code, int n_c, const int* frames, float* y, void* stream);

/* Voice conversion in chunks, bit-identical to fac_voice_convert on the whole utterance.  The redecoder and its decoder are
 * non-causal but hold no LSTM, so the output needs a fixed look-ahead and no recurrent state.  z frame t reads codes
 * [t - 32, t + 32] (16 WN layers of k = 5 convs, reflect-padded 2 frames per side), and output frame t (samples
 * [300 t, 300 t + 300)) reads z frames [t - 12, t + 12] (the decoder's centred convs and 3-tap transposed convs).  Output
 * frame t is therefore final once codes up to frame t + 44 have arrived: fac_vc_stream_lookahead() = 44 frames, 550 ms at
 * 24 kHz.  Each call recomputes the redecoder over <= 32 frames of code history plus 32 of look-ahead, and the decoder over
 * <= 12 + 12 frames of z; windows reflect only at the utterance's true start (frame 0) and, at finish, its true end.
 * fac_vc_stream_begin(B <= 32, timbre [B,1024] device, use_p_code, use_c_code, n_c <= 2) -> stream id (>= 0) or a negative
 * status; the timbre's cond layer runs once here.
 * fac_vc_stream_convert: codes_p [B,1,F], codes_c [B,n_c_rows,F] int64 (device; the codec's codes[0], codes[1], e.g. a chunk
 * of fac_stream_encode_codes), F >= 1 new frames -> returns k (0 <= k <= F; 0 for the first 44 frames received) and writes the
 * next k output frames to y as [B,1,300*k] (capacity B*300*F floats).
 * fac_vc_stream_finish: the end of the utterance -> returns k <= 44 (k = min(N, 44) for N frames received) and writes the
 * last k frames to y as [B,1,300*k] (capacity B*300*44 floats).  A stream shorter than the look-ahead emits everything here.
 * fac_vc_stream_set_timbre(timbre [B,1024] device): converts to this voice from the next call on; the cond layer runs here.
 * The next call recomputes the z frames the decoder still reads ([Yf - 12, Zf) of the output frames emitted Yf and z
 * frames final Zf) from the code history under the new cond, so every sample emitted from then on, finish included, equals
 * fac_voice_convert of the whole utterance with the new timbre, and everything emitted before equals it with the old one.
 * The stream keeps the last 2 * (32 + 12) code frames for this.  Switching to the same timbre changes nothing.
 * FAC_ERR_STATE: convert after finish, finish twice, finish with nothing received, set_timbre after finish;
 * FAC_ERR_INVALID: bad B, F <= 0, n_c > n_c_rows, a null timbre.  A rejected call leaves the stream as it was (its cond
 * included: set_timbre computes into workspace, then copies).  Out-of-range codes behave as in fac_voice_convert. */
int fac_vc_stream_lookahead(void);
int fac_vc_stream_begin(fac_handle* h, int B, const float* timbre, int use_p_code, int use_c_code, int n_c, void* stream);
int fac_vc_stream_convert(fac_handle* h, int stream_id, const int64_t* codes_p, const int64_t* codes_c, int n_c_rows, int F,
                          float* y, void* stream);
int fac_vc_stream_finish(fac_handle* h, int stream_id, float* y, void* stream);
int fac_vc_stream_set_timbre(fac_handle* h, int stream_id, const float* timbre, void* stream);
int fac_vc_stream_end(fac_handle* h, int stream_id);

/* Streaming (SURVEY.md section 8f rank 4; README.md:105-107 "causal ... can be used for streaming"): the encoder and the codec's
 * decoder are causal, so a long utterance can be processed in chunks with the SAME results as one offline call
 * (dac/model/dac.py:103-104, :164-165).  The reference ships no streaming driver; these entry points carry what the
 * causal graph needs between chunks on the device: the conv stacks' left context (6000 samples / 20 latent frames) and the
 * SLSTM (h, c) states (dac/model/encodec.py:272-288: the SLSTM itself keeps none; it is explicit here).
 * fac_stream_begin(B <= 32) -> stream id (>= 0) or a negative status; one stream holds one encoder and one decoder state.
 * fac_stream_encode: x_chunk [B,1,T] (device; T a multiple of 300, the first chunk >= 3000) -> z_chunk [B,1024,T/300].
 * fac_stream_decode: z_chunk [B,1024,Fc] (device; first chunk >= 10 frames) -> y_chunk [B,1,300*Fc].
 * fac_quantize on each z chunk is NOT exact: only the content codes are per frame of z.  The prosody branch reads a centred
 * STFT (600 samples of look-ahead per frame, reflected at the wave's ends) through an 8-layer causal WaveNet whose convs
 * reflect-pad at their left edge, and the residual codes read z - z_p - z_c; the timbre pools over the whole utterance
 * (modules/quantize.py:228-242, :375-454).  fac_stream_encode_codes / fac_stream_finish_codes carry what that needs.
 * fac_stream_decode_codes: fac_stream_decode on a chunk of codes (Fc frames, arguments as fac_codes_decode); it advances
 * the same decoder state, so one stream should be fed either latents or codes.
 *
 * Compression to codes in chunks, with codes and timbre bit-identical to fac_codec_encode on the whole utterance:
 * fac_stream_encode_codes: x_chunk [B,1,T] (chunk rules of fac_stream_encode), n_c = 1 or 2 for the whole stream ->
 * codes_p [B,1,F_out], codes_c [B,n_c,F_out], codes_r [B,3,F_out] int64 (device), F_out = T/300 - 1 on the first call and
 * T/300 after it; returns F_out.  The codes run ONE frame behind the samples: mel frame t reads samples up to 300 t + 600,
 * so the last frame seen is final only when the stream ends.  fac_stream_finish_codes writes that held-back frame
 * (codes [B,rows,1]) and, unless `timbre` is NULL, timbre [B,1024] (StyleEncoder over every mel frame of the utterance);
 * returns 1 and closes the encoder half (the decoder half is untouched: fac_stream_decode_codes may run alongside).
 * The stream keeps every mel80 row until fac_stream_end: 320 B per frame per utterance, ~92 MB per utterance-hour.
 * Each chunk recomputes the encoder over a 6000-sample history and the prosody net over <= 32 frames of history.
 * FAC_ERR_STATE: encode_codes on a stream fed by fac_stream_encode or the reverse, any encode after finish, finish with
 * nothing encoded; FAC_ERR_INVALID: n_c changed mid-stream; FAC_ERR_UNSUPPORTED unless "tensor_cores" is 2 (the only mel
 * path that cuts the STFT frames explicitly).  A rejected call leaves the stream as it was.
 * fac_stream_timbre: the timbre [B,1024] fac_stream_finish_codes would write if the utterance ended now -- fac_codec_encode's
 * on every sample fed so far, bit for bit -- without ending it: the last mel frame is cut from the sample history reflected
 * at the current end into workspace, and the StyleEncoder runs over the samples / 300 rows.  Nothing the stream emits
 * later changes.  Rejected (stream unchanged) as fac_stream_finish_codes is: FAC_ERR_STATE before the first
 * fac_stream_encode_codes chunk, on a stream fed by fac_stream_encode, after finish; FAC_ERR_UNSUPPORTED unless
 * "tensor_cores" is 2. */
int fac_stream_begin(fac_handle* h, int B);
int fac_stream_encode(fac_handle* h, int stream_id, const float* x, int T, float* z, void* stream);
int fac_stream_decode(fac_handle* h, int stream_id, const float* z, int Fc, float* y, void* stream);
int fac_stream_decode_codes(fac_handle* h, int stream_id, const int64_t* codes_p, const int64_t* codes_c, int n_c_rows,
                            const int64_t* codes_r, int n_r_rows, const float* timbre, int Fc, float* y, void* stream);
int fac_stream_encode_codes(fac_handle* h, int stream_id, const float* x, int T, int n_c, int64_t* codes_p, int64_t* codes_c,
                            int64_t* codes_r, void* stream);
int fac_stream_finish_codes(fac_handle* h, int stream_id, int64_t* codes_p, int64_t* codes_c, int64_t* codes_r, float* timbre,
                            void* stream);
int fac_stream_timbre(fac_handle* h, int stream_id, float* timbre, void* stream);
int fac_stream_end(fac_handle* h, int stream_id);

/* Stream pools: many live sessions, each behaving exactly like its own B = 1 stream, stepped in shared launches.  A pool
 * owns the state of up to `capacity` sessions; a step names any subset of them, each at most once, with its own chunk.
 * Sessions at the same stage of their windows (after a short warm-up, those fed equal chunk lengths) share one launch
 * sequence, up to 32 per batch (the LSTM's batch tile); larger groups run as several batches.  A session's outputs are
 * bit-identical to those of a B = 1 stream fed the same chunks, whoever shares its launches.
 * Every step validates all its arguments before it launches anything: a rejected step returns a negative status and leaves
 * every session of the pool as it was.  Per-session buffers are device pointers, the arrays holding them host arrays.
 * FAC_ERR_INVALID: an unknown, closed or repeated session, a null buffer, the chunk rules of the stream entries;
 * FAC_ERR_STATE: a session in the wrong state for the call (as the stream entries), open on a full pool.
 *
 * fac_codes_pool_create(capacity >= 1, n_c = 1 or 2 for every session) -> pool id; needs the encoder and the quantizer.
 * fac_codes_pool_open -> session id (a slot, reused after close), a fresh fac_stream_encode_codes stream.
 * fac_codes_pool_encode_codes: for i < n, session sessions[i] takes x[i] [1,1,T[i]] (rules of fac_stream_encode_codes) and
 * writes codes_p[i] [1,1,F], codes_c[i] [1,n_c,F], codes_r[i] [1,3,F]; frames[i] = F (T/300 - 1 on a first chunk, T/300 after).
 * fac_codes_pool_finish_codes: fac_stream_finish_codes per session (one frame each; timbre may be NULL, or timbre[i] NULL).
 * The session's mel rows are kept until the pool is destroyed and reused by the next session of the slot.
 * fac_codes_pool_timbre: fac_stream_timbre per session into timbre[i] [1,1024], without ending any of them.  The sessions
 * run as lanes of ragged StyleEncoder batches (<= 32 lanes, ordered by frame count, lanes x longest lane <= 32768 mel
 * frames; a longer session runs alone), each lane bit-identical to its session's own B = 1 fac_stream_timbre.  A session
 * that is not open, named twice, finished or has nothing encoded rejects the whole call before anything is queued.
 * fac_last_launch_count counts the launches of all its batches.
 * fac_vc_pool_create(capacity >= 1, use_p_code, use_c_code, 0 <= n_c <= 2) -> pool id; needs the redecoder and its decoder.
 * The options are the defaults of fac_vc_pool_open.
 * fac_vc_pool_open(timbre [1,1024] device) -> session id; the timbre's cond layer runs here.
 * fac_vc_pool_open_mode(timbre, use_p_code, use_c_code, 0 <= n_c <= 2): fac_vc_pool_open with the session's own mode.
 * Sessions of different modes share batches: each lane embeds its codes in its own mode, bit for bit as a B = 1 stream of
 * that mode, and the rest of the launch sequence does not depend on the mode.
 * fac_vc_pool_set_timbre(session, timbre [1,1024] device): fac_vc_stream_set_timbre on one session.  Until its next step
 * has run, the session batches only with other switched sessions (that step recomputes its z history on a wider window).
 * FAC_ERR_INVALID for a session not open, FAC_ERR_STATE after its finish.
 * fac_vc_pool_convert: session sessions[i] takes codes_p[i] [1,1,F[i]], codes_c[i] [1,n_c_rows[i],F[i]] (as
 * fac_vc_stream_convert) and writes frames[i] = k output frames to y[i] [1,1,300*k] (capacity 300*F[i] floats).
 * fac_last_launch_count counts the launches of all its batches.
 * fac_vc_pool_finish: fac_vc_stream_finish per session; y[i] holds 300*44 floats.
 * fac_dec_pool_create(capacity >= 1) -> pool id; needs the quantizer and the decoder.
 * fac_dec_pool_open(timbre [1,1024] device) -> session id, a fresh fac_stream_decode_codes stream decoding with that timbre;
 * gamma | beta = timbre_linear(timbre) is computed once here.
 * fac_dec_pool_decode_codes: session sessions[i] takes codes_p[i] [1,1,F[i]], codes_c[i] [1,n_c_rows[i],F[i]] and
 * codes_r[i] [1,n_r_rows[i],F[i]] (1 <= n_c_rows <= 2, 0 <= n_r_rows <= 3, codes_r[i] unread when 0; a session's first chunk
 * >= 10 frames) and writes y[i] [1,1,300*F[i]].  The decoder is causal, so every frame is final when it arrives (no finish).
 * Sessions that have decoded equally many frames (20 or more: any two in steady state) share a batch whatever their chunk
 * lengths and code rows.  Out-of-range codes give NaN samples, as fac_codes_decode.
 * fac_dec_pool_set_timbre(session, timbre [1,1024] device): the session decodes with this timbre from its next chunk on
 * (gamma | beta recomputed by fac_dec_pool_open's launch); its decoder state and every other session are untouched.
 * fac_*_pool_close frees a session's slot; fac_*_pool_destroy frees the pool (and runs at fac_destroy). */
int fac_codes_pool_create(fac_handle* h, int capacity, int n_c);
int fac_codes_pool_open(fac_handle* h, int pool_id, void* stream);
int fac_codes_pool_encode_codes(fac_handle* h, int pool_id, int n, const int* sessions, const int* T, const float* const* x,
                                int64_t* const* codes_p, int64_t* const* codes_c, int64_t* const* codes_r, int* frames,
                                void* stream);
int fac_codes_pool_finish_codes(fac_handle* h, int pool_id, int n, const int* sessions, int64_t* const* codes_p,
                                int64_t* const* codes_c, int64_t* const* codes_r, float* const* timbre, void* stream);
int fac_codes_pool_timbre(fac_handle* h, int pool_id, int n, const int* sessions, float* const* timbre, void* stream);
int fac_codes_pool_close(fac_handle* h, int pool_id, int session);
int fac_codes_pool_destroy(fac_handle* h, int pool_id);
int fac_vc_pool_create(fac_handle* h, int capacity, int use_p_code, int use_c_code, int n_c);
int fac_vc_pool_open(fac_handle* h, int pool_id, const float* timbre, void* stream);
int fac_vc_pool_open_mode(fac_handle* h, int pool_id, const float* timbre, int use_p_code, int use_c_code, int n_c,
                          void* stream);
int fac_vc_pool_set_timbre(fac_handle* h, int pool_id, int session, const float* timbre, void* stream);
int fac_vc_pool_convert(fac_handle* h, int pool_id, int n, const int* sessions, const int* F, const int64_t* const* codes_p,
                        const int64_t* const* codes_c, const int* n_c_rows, float* const* y, int* frames, void* stream);
int fac_vc_pool_finish(fac_handle* h, int pool_id, int n, const int* sessions, float* const* y, int* frames, void* stream);
int fac_vc_pool_close(fac_handle* h, int pool_id, int session);
int fac_vc_pool_destroy(fac_handle* h, int pool_id);
int fac_dec_pool_create(fac_handle* h, int capacity);
int fac_dec_pool_open(fac_handle* h, int pool_id, const float* timbre, void* stream);
int fac_dec_pool_decode_codes(fac_handle* h, int pool_id, int n, const int* sessions, const int* F, const int64_t* const* codes_p,
                              const int64_t* const* codes_c, const int* n_c_rows, const int64_t* const* codes_r,
                              const int* n_r_rows, float* const* y, void* stream);
int fac_dec_pool_set_timbre(fac_handle* h, int pool_id, int session, const float* timbre, void* stream);
int fac_dec_pool_close(fac_handle* h, int pool_id, int session);
int fac_dec_pool_destroy(fac_handle* h, int pool_id);

/* Sample-rate conversion: torchaudio.functional.resample(x, orig, new) with its defaults (sinc_interp_hann,
 * lowpass_filter_width 6, rolloff 0.99).  Rates are integers in [8000, 192000]; with the pair reduced by its gcd,
 * width = ceil(6 orig / (min(orig, new) * 0.99)) and the table holds K = 2 width + orig taps for each of `new` phases; pairs
 * with K * new > 65536 are FAC_ERR_INVALID (every pair between 24 kHz and 8, 11.025, 16, 22.05, 32, 44.1, 48, 96 or 192 kHz
 * fits).  n input samples give ceil(new n / orig) outputs; output j sums its K taps in fp32 with fmaf in ascending order,
 * and that order depends on j alone, so a lane of a batch and every session of a pool equal their own offline B = 1 call bit
 * for bit.  Equal rates copy.
 * fac_resample_geometry: host only; out4 = {reduced orig, reduced new, width, K}.
 * fac_resample_out_len: host only; ceil(new n / orig), or a negative status.
 * fac_resample_table: registers the float32 filter table [new][K] of a pair (reduced, as fac_resample_geometry gives it) and
 * uploads it once per handle; later calls for the pair are no-ops.  The table is torchaudio's _get_sinc_resample_kernel(...,
 * dtype=torch.float32) bit for bit, whose sin / cos are torch's own: a C++ build of the same formula with the C library's
 * sinf / cosf differs in the last bit in about 0.7 % of the taps.  facodec_b200.modules.resample_table builds it (its
 * recipe, 15 lines of torch ops, is the reference for any other host); a C caller computes it once per pair that way or
 * takes it from torchaudio, and registers it here.  The other calls return FAC_ERR_STATE for a pair without a table.
 * fac_resample: x [B,T] (device) -> y [B,ceil(new T / orig)].  lengths: NULL or a HOST array of B counts in [0, T]; lane b
 * resamples x[b, :lengths[b]] and writes 0 past its ceil(new lengths[b] / orig) outputs.
 * Resampler pools: live sessions, each with its own rate pair, stepped in one launch (up to 256 lanes per launch).
 * fac_rs_pool_create(capacity, quantum >= 1) -> pool id.  fac_rs_pool_open(orig, new) -> session id.
 * fac_rs_pool_push: session sessions[i] takes x[i] [T[i]] (T >= 0) and writes counts[i] outputs to y[i]: every output whose
 * whole window lies inside the input so far (fac_resample_ready), rounded down to a multiple of the quantum.
 * fac_resample_ready: host only; that count for a session that has seen `seen` samples and returned `emitted` outputs.
 * fac_rs_pool_finish: the end of the sessions' input, after an optional last chunk (T / x may be NULL): writes the rest,
 * counts[i] = ceil(new seen / orig) - emitted, with the input zero-padded as fac_resample pads it.  A finished session takes
 * no more input until it is closed.  Concatenated, a session's outputs equal fac_resample of its concatenated input.
 * fac_rs_pool_undo: takes back each named session's last push or finish (the outputs it wrote are to be discarded), for a
 * caller whose own step on those outputs was rejected; a session can take back one step, and open / close forget it.
 * A slot keeps the input from the window of its first output not yet returned (at most K + orig ceil((quantum - 1) / new)
 * samples) in two buffers: a step writes the other one and the slot flips once the launch is queued, so a rejected step
 * leaves every session as it was.  Counts follow from the pushed lengths alone: no call synchronises with the device.
 * fac_last_launch_count after fac_resample / fac_rs_pool_push / fac_rs_pool_finish counts that call's launches alone
 * (1 for up to 256 lanes). */
int fac_resample_geometry(int orig, int new_rate, int* out4);
long long fac_resample_out_len(int orig, int new_rate, long long n);
long long fac_resample_ready(int orig, int new_rate, int quantum, long long seen, long long emitted);
int fac_resample_table(fac_handle* h, int orig, int new_rate, const float* table_host);
int fac_resample(fac_handle* h, const float* x, int B, int T, const int* lengths, int orig, int new_rate, float* y, void* stream);
int fac_rs_pool_create(fac_handle* h, int capacity, int quantum);
int fac_rs_pool_open(fac_handle* h, int pool_id, int orig, int new_rate);
int fac_rs_pool_push(fac_handle* h, int pool_id, int n, const int* sessions, const int* T, const float* const* x, float* const* y,
                     int* counts, void* stream);
int fac_rs_pool_finish(fac_handle* h, int pool_id, int n, const int* sessions, const int* T, const float* const* x,
                       float* const* y, int* counts, void* stream);
int fac_rs_pool_undo(fac_handle* h, int pool_id, int n, const int* sessions);
int fac_rs_pool_close(fac_handle* h, int pool_id, int session);
int fac_rs_pool_destroy(fac_handle* h, int pool_id);

/* Session state: a live pool session taken out of its pool and put into another pool of the same kind, model and options,
 * on the same device or another one, in this process or another.  After import the session continues bit for bit as it
 * would have in its source pool, and shares batches with native sessions under the usual plan keys.
 *
 * A state is a host header (fac_state_header, native little-endian byte order) and one device payload of
 * header.payload_bytes, which holds the slot's regions back to back in the order listed below, each region_bytes[r] long
 * (every size a multiple of 4).  Counters and regions per kind:
 *   FAC_STATE_CODES  counters {n_c of the pool, mode (0 fresh, 2 coding), samples, frames emitted, sample history length,
 *                    encoder-LSTM output history length}; regions {sample history [6000] f32, LSTM output history
 *                    [2][1024] f32, held latent [1024] f32, LSTM carry [2][2 048] words, mel rows [emitted][80] f32}.
 *                    The mel rows make the payload grow with the call: 320 B per frame, about 1.5 MB after 60 s.
 *   FAC_STATE_VC     counters {use_p_code, use_c_code, n_c, stale, N, Zf, Yf}; regions {cond [16 384] f32, code history
 *                    [3][88] i64, z history [24][1024] f32}.
 *   FAC_STATE_DEC    counters {frames}; regions {latent history [6][1024] f32, LSTM output history [20][1536] f32, LSTM
 *                    carry [2][2 304] words, gamma | beta [2048] f32}.
 *   FAC_STATE_RS     counters {quantum, reduced orig, reduced new, width, K, samples seen, outputs emitted, first history
 *                    sample, history length}; regions {history [history length] f32}.
 * fingerprint: a 64-bit hash of the host weights of the modules a kind runs (codes: encoder + quantizer; dec: quantizer +
 * decoder; vc: redecoder + its decoder; rs: 0), taken at fac_finalize: the same state dicts give the same value in any
 * handle, device or process.  options: the fac_set_option values in the order tensor_cores, fuse_resunit, lstm_v2,
 * decoder_lstm_fp16, attention_stream, decoder_conv7_fp16, encoder_f16x2, encoder_tt, tc_occ2_maxn, decoder_bf16,
 * overlap_front.  checksum:
 * FNV-1a 64 of every header byte before it.
 * FAC_STATE_VERSION moves with any change to a slot struct (EncHalf, VcStream, DecHalf in engine.cu, RsSlot in resample.cu),
 * to the regions or to the counters; states of another version are refused.
 *
 * fac_*_pool_export_size: host only; the header and payload bytes of one open session.
 * fac_*_pool_export: writes sessions[i]'s header to headers[i] (host, sizeof(fac_state_header)) and its payload to
 * payloads[i] (device memory of the handle's device, 4-byte aligned, export_size bytes), in one launch per region for up to
 * 1024 sessions.  The sessions stay open and unchanged: export, import and close moves a session; export and two imports
 * fork it.  FAC_ERR_INVALID for an unknown, closed or repeated session or a bad buffer; FAC_ERR_STATE for a session
 * finished by fac_codes_pool_finish_codes, fac_vc_pool_finish or fac_rs_pool_finish.
 * fac_*_pool_import: opens a slot holding the state and returns its session id.  Everything is checked before anything is
 * written, and a rejected import changes neither pool: FAC_ERR_INVALID for a short, corrupt or foreign header (magic,
 * checksum, kind, sizes that disagree with the counters or the payload) or a payload not on the handle's device;
 * FAC_ERR_STATE for another format version, other weights, other options, another pool n_c or quantum, a full pool or, for
 * a resampler state, a rate pair without a registered table.  An imported resampler session has no step to take back
 * (fac_rs_pool_undo).  Bit equality across devices assumes the same GPU model; the SM count is not checked.
 * fac_last_launch_count after an export or import counts one launch per region. */
#define FAC_STATE_MAGIC 0x54534346u     /* "FCST" */
#define FAC_STATE_VERSION 1
#define FAC_STATE_OPTIONS 12
#define FAC_STATE_COUNTERS 12
#define FAC_STATE_REGIONS 6
enum { FAC_STATE_CODES = 1, FAC_STATE_VC = 2, FAC_STATE_DEC = 3, FAC_STATE_RS = 4 };
typedef struct fac_state_header {
    uint32_t magic, version, kind, header_bytes;
    uint64_t fingerprint;
    int64_t options[FAC_STATE_OPTIONS];         /* unused entries 0 */
    int64_t counters[FAC_STATE_COUNTERS];       /* unused entries 0 */
    int64_t region_bytes[FAC_STATE_REGIONS];    /* unused entries 0 */
    uint64_t payload_bytes;
    uint64_t checksum;
} fac_state_header;
int fac_codes_pool_export_size(fac_handle* h, int pool_id, int session, size_t* header_bytes, size_t* payload_bytes);
int fac_codes_pool_export(fac_handle* h, int pool_id, int n, const int* sessions, void* const* headers, void* const* payloads,
                          void* stream);
int fac_codes_pool_import(fac_handle* h, int pool_id, const void* header, size_t header_bytes, const void* payload,
                          size_t payload_bytes, void* stream);
int fac_vc_pool_export_size(fac_handle* h, int pool_id, int session, size_t* header_bytes, size_t* payload_bytes);
int fac_vc_pool_export(fac_handle* h, int pool_id, int n, const int* sessions, void* const* headers, void* const* payloads,
                       void* stream);
int fac_vc_pool_import(fac_handle* h, int pool_id, const void* header, size_t header_bytes, const void* payload,
                       size_t payload_bytes, void* stream);
int fac_dec_pool_export_size(fac_handle* h, int pool_id, int session, size_t* header_bytes, size_t* payload_bytes);
int fac_dec_pool_export(fac_handle* h, int pool_id, int n, const int* sessions, void* const* headers, void* const* payloads,
                        void* stream);
int fac_dec_pool_import(fac_handle* h, int pool_id, const void* header, size_t header_bytes, const void* payload,
                        size_t payload_bytes, void* stream);
int fac_rs_pool_export_size(fac_handle* h, int pool_id, int session, size_t* header_bytes, size_t* payload_bytes);
int fac_rs_pool_export(fac_handle* h, int pool_id, int n, const int* sessions, void* const* headers, void* const* payloads,
                       void* stream);
int fac_rs_pool_import(fac_handle* h, int pool_id, const void* header, size_t header_bytes, const void* payload,
                       size_t payload_bytes, void* stream);

/* quantize/rvq.py:27-75 ResidualVQ.forward (eval) over quantize/fvq.py FactorizedVectorQuantize,
 * dim=1024, codebook_dim=8, 2^10 entries (BASELINE configs[3]).  Parameters are passed directly
 * (already weight-normed, HOST): per quantizer q: in_w [8,1024], in_b [8], out_w [1024,8],
 * out_b [1024], codebook [1024,8].  fac_rvq_create returns an id usable with fac_rvq_forward:
 * x [B,1024,T] -> quantized_out [B,1024,T], indices [nq,B,T] int64, all_quantized [nq,B,1024,T]
 * (may be NULL).  x_channels_last != 0 means x / outputs are [B,T,1024] (no transposes). */
int fac_rvq_create(fac_handle* h, int nq, const float* const* in_w, const float* const* in_b,
                   const float* const* out_w, const float* const* out_b, const float* const* codebook);
int fac_rvq_destroy(fac_handle* h, int rvq_id);   /* frees that set's device arena (e.g. before re-creating it with new weights) */
int fac_rvq_forward(fac_handle* h, int rvq_id, const float* x, int B, int T, int x_channels_last,
                    float* quantized_out, int64_t* indices, float* all_quantized, void* stream);

/* alias_free_torch/act.py:24-29 Activation1d.forward with up/down ratio 2, 12-tap Kaiser-sinc
 * filters (filter.py:27-58).  x, y [B,C,T].  act: 0 = identity, 1 = SnakeBeta with per-channel
 * alpha / beta given as already-exponentiated values (modules/quantize.py:29-79). */
int fac_alias_free_act(fac_handle* h, const float* x, int B, int C, int T, int act,
                       const float* alpha, const float* beta, float* y, void* stream);

/* Dataset-side mel: meldataset.py:37-47 preprocess (PseudoDataset.__getitem__ :64-71) -- torchaudio MelSpectrogram(n_mels=80,
 * n_fft=2048, win_length=1200, hop_length=300) with its default sample_rate=16000 filterbank, centre=True, then
 * (log(1e-5 + mel) + 4) / 4.  wave [B,T] (device, T > 1024) -> mel [B,80,T/300+1]. */
int fac_dataset_mel(fac_handle* h, const float* wave, int B, int T, float* mel, void* stream);

/* Training-side reconstruction loss, forward only: losses.py:65-89 reconstruction_loss(x, G_x) =
 * 100 * mse(x, G_x) + sum over s in {64, 128, ..., 2048} of (l1_s + sqrt(s/2) * l2_s) between the 64-band mel spectrograms
 * torchaudio MelSpectrogram(sample_rate=16000, n_fft=max(s,512), win_length=s, hop_length=s/4, n_mels=64) gives for x and G_x:
 * l1 = mean |S_x - S_G|, l2 = mean over (utterance, frame) of sqrt(mean over bands of (log(|S_x|+1e-7) - log(|S_G|+1e-7))^2).
 * x, gx [B,T] (device, T > 1024).  loss: 1 float (device).  terms: NULL or 13 floats (device): mse, then (l1, l2) per scale. */
int fac_reconstruction_loss(fac_handle* h, const float* x, const float* gx, int B, int T, float* loss, float* terms, void* stream);

/* dac/nn/loss.py:142-327 MultiScaleSTFTLoss (n_mels = NULL) / MelSpectrogramLoss and :11-47 L1Loss, forward values.  The
 * reference evaluates them on audiotools AudioSignal objects; audiotools / librosa are not vendored (SURVEY.md 8c: parity
 * UNPINNED), so their published semantics are restated: torch.stft(n_fft = window_length, hop = window_length/4, periodic Hann,
 * centre = True, reflect), magnitude = |stft|, mel = magnitude @ librosa.filters.mel(sample_rate, n_fft, n_mels, fmin, fmax)^T
 * (Slaney scale + area normalisation); loss = sum over scales of log_weight * mean|log10(clamp(v,eps)^pow) differences| +
 * mag_weight * mean|v differences|.  x, y [B,T] (device).  window_lengths: powers of two in [16, 4096]; mel_fmax[i] <= 0 means
 * sample_rate / 2.  loss: 1 float (device).  The (sample_rate, scales) configuration is cached on the handle. */
int fac_spectral_loss(fac_handle* h, const float* x, const float* y, int B, int T, int sample_rate, int n_scales,
                      const int* window_lengths, const int* n_mels, const float* mel_fmin, const float* mel_fmax, float clamp_eps,
                      float mag_weight, float log_weight, float pow, float* loss, void* stream);
int fac_l1_loss(fac_handle* h, const float* x, const float* y, long long n, float* loss, void* stream);
/* The same losses with their gradients for back-propagation: arguments and errors as above, plus dx / dy ([B,T] device, each
 * may be NULL) receiving dL/dx and dL/dy (upstream gradient 1; L is a scalar, so a caller scales them by its own).  *loss is
 * bit-identical to the forward call's; with dx = dy = NULL the call is the forward call.  Gradients are bit-reproducible
 * (fixed summation orders, no atomics).  The spectral gradient follows torch autograd of the restated loss: sgn(0) = 0 in
 * the L1 terms, clamp passes the gradient where v >= eps, d|z|/dz = 0 at z = 0, reflect padding folded back. */
int fac_spectral_loss_grad(fac_handle* h, const float* x, const float* y, int B, int T, int sample_rate, int n_scales,
                           const int* window_lengths, const int* n_mels, const float* mel_fmin, const float* mel_fmax, float clamp_eps,
                           float mag_weight, float log_weight, float pow, float* loss, float* dx, float* dy, void* stream);
int fac_l1_loss_grad(fac_handle* h, const float* x, const float* y, long long n, float* loss, float* dx, float* dy, void* stream);

/* Predictor heads: modules/quantize.py:106-125 CNNLSTM(indim, outdim, head, global_pred) forward (3 ResidualUnits of
 * alias-free SnakeBeta + weight-normed Conv1d k7 (dilation 1, 2, 3, zero padding) / k1, a final alias-free SnakeBeta,
 * `nheads` nn.Linear layers; mean over time first when global_pred).  fac_head_begin returns a head id; feed the reference
 * state_dict tensors (keys "model.0.block.0.act.alpha", "model.0.block.1.weight_g", ..., "heads.0.weight"; the registered
 * filter buffers are ignored) with fac_head_tensor, then fac_head_finalize.  fac_head_forward: x [B,indim,T] (device) ->
 * outs[i] [B,T,outdim] (or [B,outdim] when global_pred), i < nheads, caller-allocated device buffers.
 * global_pred = 2 makes the head a plain nn.Linear(indim, outdim) (FApredictors.timbre_predictor under timbre_norm,
 * modules/quantize.py:470-473): stage "linear.weight" [outdim][indim] and "linear.bias", nheads = 1; fac_head_forward then
 * takes x as [B*T rows][indim] and writes outs[0] [B*T][outdim].
 * fac_add3: out = a + b (+ c when c is not NULL), n floats on the device: the latent sums FApredictors.forward_v2 feeds
 * its gradient-reversal heads (modules/quantize.py:571-586). */
int fac_head_begin(fac_handle* h);
int fac_head_tensor(fac_handle* h, int head_id, const char* key, const float* data_host, const int64_t* shape, int ndim);
int fac_head_finalize(fac_handle* h, int head_id, int indim, int outdim, int nheads, int global_pred);
int fac_head_forward(fac_handle* h, int head_id, const float* x, int B, int T, float* const* outs, void* stream);
int fac_add3(fac_handle* h, const float* a, const float* b, const float* c, long long n, float* out, void* stream);

/* JDCNet pitch extractor (modules/JDC/model.py JDCNet(num_class=1), eval mode; the model train.py's load_F0_models loads).
 * fac_jdc_begin returns an id; stage the reference state_dict tensors (the ['net'] dict of bst.t7: "conv_block.0.weight",
 * "res_block1.pre_conv.0.running_mean", "bilstm_classifier.weight_ih_l0_reverse", "classifier.bias", ...; the detector
 * branch's keys are accepted and unused) with fac_jdc_tensor, then fac_jdc_finalize, which folds every BatchNorm (eval:
 * running statistics, eps 1e-5).  fac_jdc_forward: mel [B,1,80,T] (device) -> f0 [B,T], gan_feature [B,256,10,T] and
 * pool_out [B,256,T,2] (caller-allocated device buffers), model.py:102-137 with Dropout as the identity.  lengths (HOST,
 * B ints in [1, T], or NULL): lane b is its own first lengths[b] frames -- every 3x3 conv zero-pads time at the lane's own
 * end and the reverse LSTM starts at its last frame -- bit-identical to a B = 1 call on them; outputs past lengths[b] are 0.
 * fac_f0_targets (train.py:219-251, norm_f0): f0 [B,T] (device) -> targets [B,T] and glob_f0 [B]; lengths (HOST, in [0, T],
 * or NULL) limits lane b to its first lengths[b] frames (the others are -10).  fac_log_norm (modules/commons.py:176-181,
 * mean -4, std 4): mel [B,80,T] -> out [B,T] = log(||exp(4 mel - 4)||_2 over the 80 bins). */
int fac_jdc_begin(fac_handle* h);
int fac_jdc_tensor(fac_handle* h, int jdc_id, const char* key, const float* data_host, const int64_t* shape, int ndim);
int fac_jdc_finalize(fac_handle* h, int jdc_id);
int fac_jdc_forward(fac_handle* h, int jdc_id, const float* mel, int B, int T, const int* lengths, float* f0, float* gan_feature,
                    float* pool_out, void* stream);
int fac_f0_targets(fac_handle* h, const float* f0, int B, int T, const int* lengths, float* targets, float* glob_f0, void* stream);
int fac_log_norm(fac_handle* h, const float* mel, int B, int T, float* out, void* stream);

/* Engine options.  "tensor_cores": 0 = fp32 FMA kernels everywhere; 1 = wgmma split-operand
 * kernel for every eligible layer downstream of the VQ (decoder, timbre branch), fp32 FMA upstream
 * (encoder, prosody branch); 2 (default) = wgmma everywhere, with the promoted accumulation
 * variant upstream of the VQ where the bit-exact argmin needs fp32-grade sums.
 * "fuse_resunit": 1 (default) runs each decoder ResidualUnit whose channels fit one CTA tile as a single
 * fused launch (conv7 -> Snake -> 1x1 conv -> +x with the intermediate kept in shared memory), and so each encoder
 * ResidualUnit of 64 or 128 channels when it runs the promoted fp16 hi + scaled-lo class ("tensor_cores" 2,
 * "encoder_f16x2" 1, "encoder_tt" 0; bit-identical to its two launches); 0 = two launches; 2 = fuse only units of at
 * most 128 channels.
 * "decoder_bf16": 1 (default) = layers downstream of the VQ split operands into bf16 hi + bf16 lo
 * (K = 16 MMAs: half the MMAs and half the operand bytes of the TF32 split; waveform error
 * ~1e-5 RMS against the 1e-4 bar, measured on the oracle), evaluate Snake with the SFU sine and run the LSTM recurrence on bf16 hi/lo
 * mma.sync tiles; 0 = TF32 hi/lo everywhere.  Never applied upstream of the VQ.
 * "encoder_f16x2": 1 (default) = layers upstream of the VQ split operands into fp16 hi + fp16 lo scaled by 2^11
 * (K = 16 MMAs at twice the TF32 rate, cross terms in their own accumulator, scaled back at promotion): the same
 * 22 mantissa bits as the TF32 pair, but operands must stay below fp16's 65504; 0 = TF32 hi/lo pairs.
 * "encoder_tt": 0 (default) / 1 = those layers in the transposed formulation (weights as the wgmma A operand, time as
 * wgmma N); same arithmetic, another tiling.
 * "tc_occ2_maxn": tiles of at most this many channels with plain accumulation are planned for TWO resident CTAs per SM
 * (<= 113 KB shared memory, <= 128 registers per thread) so one CTA's MMAs overlap the other's operand production and
 * epilogue; 0 (default) = off. */
int fac_set_option(fac_handle* h, const char* name, int value);

size_t fac_workspace_bytes(const fac_handle* h);
/* number of kernel launches issued by the last forward call (bench.py "gpu_launches") */
int fac_last_launch_count(const fac_handle* h);

#ifdef __cplusplus
}
#endif
#endif /* FACODEC_B200_H */
