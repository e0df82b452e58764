// Engine + C-ABI (include/facodec_b200.h): checkpoint folding/packing, workspace, and the
// launch sequences of Encoder.forward (dac/model/dac.py:69-104), FAquantizer.forward_v2
// (modules/quantize.py:375-454) and Decoder.forward (dac/model/dac.py:131-165).
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <initializer_list>
#include <map>
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/facodec_b200.h"
#include "../../include/facodec_b200_debug.h"
#include "common.cuh"
#include "kernels.h"
#include "resample.h"

using namespace fac;

namespace {

constexpr int HOP = 300;
constexpr int LATENT = 1024;
constexpr int N_FFT = 2048;
constexpr int WIN = 1200;
constexpr int N_BINS = 1025;
constexpr int SPEC_LD = 2052;   // 2*1025 rounded up to a multiple of 4
constexpr int SPEC_TC_LD = 2176; // ... and to 17 channel tiles of 128 for the tensor-core DFT
constexpr int N_MELS = 80;

struct HostTensor {
    std::vector<float> data;
    std::vector<int64_t> shape;
    size_t numel() const { size_t n = 1; for (auto s : shape) n *= (size_t)s; return n; }
};
using TensorMap = std::map<std::string, HostTensor>;

struct ConvW {
    size_t w = 0, b = 0; int Cin = 0, Cout = 0, K = 1, ldw = 0;
    // tensor-core blob (conv_tc.cu): present when the layer is eligible
    bool tc = false; size_t tcw = 0; int vf = 1, Kr = 0, tcN = 0;   // tcN: channel tile the blob was laid out for
    bool promoted = false;   // blob built for conv_tcp_kernel (layers upstream of the VQ)
    bool has16 = false; size_t tcw16 = 0;   // 16-bit-operand blob: bf16 hi/lo (non-promoted layers) or fp16 hi / scaled lo (promoted)
    bool has_f16s = false; size_t tcw_f16s = 0;   // hi-only fp16 blob: the one-pass class of the k = 7 convs downstream of the VQ
};
struct SnakeW { size_t a = 0, ia = 0; int C = 0; };
struct LstmW { ConvW ih[2]; size_t whh[2] = {0, 0}; size_t whh16[2] = {0, 0}; bool has16 = false; int H = 0, U = 0, G = 0;
               size_t whh2[2][2] = {{0, 0}, {0, 0}}; bool has2[2] = {false, false}; };   // lstm2 packs: [layer][pass3]
struct ResW { SnakeW s1; ConvW c7; SnakeW s2; ConvW c1; int dil = 1; };
struct VqW { size_t w_in, b_in, cb, cbn, cbn2, w_out, b_out; };

struct EncW {
    ConvW conv0;
    struct Block { ResW res[3]; SnakeW snake; ConvW down; int stride; } blk[4];
    LstmW lstm; SnakeW snake; ConvW conv_out;
};
struct DecW {
    ConvW conv0; LstmW lstm;
    struct Block { SnakeW snake; ConvW up; int stride; int cout; ResW res[3]; } blk[4];
    SnakeW snake; ConvW conv_out;
    bool causal = true, has_lstm = true;   // the redecoder's decoder: causal = false, no SLSTM (config_redecoder.yml)
};
// modules/redecoder.py Redecoder(encoder_type = "wavenet"): embeddings + WN(512, k5, 16 layers, gin 1024) + conv_out
struct RedW {
    size_t emb_p = 0, emb_c[2] = {0, 0};
    ConvW cond, wn_in[16], wn_rs[16], conv_out;
    int hidden = 512, layers = 16;
};
struct QuantW {
    VqW vq[6];
    ConvW spec0, spec3, glu[2], cq, ck, cv, co, fc, timbre_linear;
    ConvW mel_lin, wn_in[8], wn_rs[8], mel_lin2;
    ConvW dft; size_t fb = 0;
    ConvW dft_tc;      // same basis as a K=1 GEMM over gathered frames: Cin = 1200, Cout padded to 2176 (17 x 128)
};

struct DevFree { void operator()(void* p) const { cudaFree(p); } };
template <typename E> using DevBuf = std::unique_ptr<E, DevFree>;   // owned device memory
using DevMem = DevBuf<char>;

// One fac_rvq_create set and the arena its offsets point into.
struct RvqSet { int nq; VqW vq[8]; DevBuf<float> arena; };

// One CNNLSTM predictor head (modules/quantize.py:106-125): 3 ResidualUnits (alias-free SnakeBeta, k7 conv dilation
// 1/2/3 with zero padding, alias-free SnakeBeta, 1x1 conv, +x), a final alias-free SnakeBeta, nheads Linear layers.
// Packed with the codec's conv packers; weights live in their own arena.
struct HeadSet {
    int indim = 0, outdim = 0, nheads = 0, global_pred = 0;
    struct Unit { size_t a1, b1, a2, b2; ConvW c7, c1; int dil; } unit[3];
    size_t af, bf;                  // final activation exp(alpha), exp(beta)
    ConvW lin[8];
    TensorMap staged;
    DevBuf<float> arena;
    bool ready = false;
};

// One JDCNet(num_class=1) in eval mode (modules/JDC/model.py:102-137).  Every 3x3 conv that a BatchNorm follows carries it
// folded into its weights and bias; the BatchNorms before a max-pool are per-channel scale / shift pairs.
struct JdcSet {
    struct Bn { size_t sc = 0, sh = 0; };
    size_t conv_in_w = 0, conv_in_b = 0;       // conv_block.0 + .1: [9][64], [64]
    ConvW c0b;                                 // conv_block.3 (64 -> 64, no BN after it)
    struct Block { Bn pre; ConvW c1, c2, c11; int F = 0; } blk[3];    // res_block1..3: F = input frequency columns
    Bn pool;                                   // pool_block.0
    ConvW ih[2];                               // bilstm_classifier input GEMMs (forward, reverse): 512 -> 1024
    size_t whh2[2] = {0, 0};                   // their recurrent weights, lstm2_pack(pass3 = 1)
    int U = 0, G = 0;
    size_t cls_w = 0, cls_b = 0;               // classifier: [512], [1]
    TensorMap staged;
    DevBuf<float> arena;
    bool ready = false;
};

struct LstmState { uint32_t* h[2] = {nullptr, nullptr}; float* c[2] = {nullptr, nullptr}; };

// Streaming state of one batch of utterances: the encoder and the decoder are causal (README.md:105-107), so a chunk's
// outputs depend on the past only through (a) a bounded window of earlier samples / frames of every FIR-like conv stack
// and (b) the LSTM states.  Histories are kept on the device; chunks are computed on [history | chunk] windows with the
// ordinary kernels and the history part of the output is dropped.  The encoder and decoder halves are independent: a
// B-row fac_stream_* stream owns one of each; a pool keeps B = 1 views of one kind in its slots and B = 32 in its lanes.
// The LSTM state is state tiles (a stream, a pool's lanes), or in a pool slot [2 layers][carry_words] in lstm2_lane_map
// order.  Device pointers are views into memory owned elsewhere (Stream::mem, Pool::mem), except the mel rows.
struct EncHalf {
    // Compression to codes (fac_stream_encode_codes / fac_stream_finish_codes).  Mel frame t reads samples up to 300 t + 600,
    // so the last frame seen is final only at the end of the stream: codes run one frame behind the encoder.
    enum Mode { kNone, kLatents, kCodes, kFinished };
    int B = 0;
    int mode = kNone;                                       // which call feeds the encoder half
    int n_c = 0;                                            // content codebooks of the codes calls
    long long samples = 0;                                  // samples encoded
    long long emitted = 0;                                  // frames of codes written so far
    float* x_hist = nullptr; int x_hist_len = 0;            // [B][kEncCtx] last samples
    float* ey_hist = nullptr; int ey_hist_len = 0;          // [B][2][1024] last encoder-LSTM output frames (conv_out, k = 3)
    float* z_held = nullptr;                                // [B][1024] latent frame `emitted`, quantized by the next call
    LstmState lstm; uint32_t* carry = nullptr;
    DevBuf<float> mel; int mel_cap = 0;                     // [B][mel_cap][80] every mel80 row so far: the timbre pools them all
    long long mel_base = 0;                                 // frame of mel row 0 (a pool's batch holds only the prosody window)
};
struct DecHalf {
    int B = 0;
    long long frames = 0;                                   // frames decoded
    float* z_hist = nullptr;                                // [B][6][1024] last latent frames (decoder conv0, k = 7)
    float* dy_hist = nullptr;                               // [B][kDecCtx][1536] last decoder-LSTM output frames
    LstmState lstm; uint32_t* carry = nullptr;
    float* gb = nullptr;                                    // a decode-pool slot's timbre_linear(timbre), [2048]
};
struct Stream { EncHalf enc; DecHalf dec; DevMem mem; };

// Streaming voice conversion: the redecoder and its decoder are non-causal but carry no LSTM, so a chunk's outputs depend
// only on bounded windows of codes and latents on both sides (kVcRedCtx / kVcDecCtx frames, fac_vc_stream_lookahead).
// Frames [0, Zf) of z and [0, Yf) of the output are final; the device keeps the channels-last z [max(0, Yf - kVcDecCtx), Zf)
// the decoder's windows still need, and the codes [max(0, Yf - kVcDecCtx - kVcRedCtx), N) from which that z can be
// recomputed under a new timbre (set_timbre; the redecoder's own windows need only [max(0, Zf - kVcRedCtx), N)).
struct VcStream {
    int B = 0, use_p = 0, use_c = 0, n_c = 0;
    bool finished = false;
    bool stale = false;                     // g changed since z was computed: the next step recomputes the z history
    long long N = 0, Zf = 0, Yf = 0;        // code frames received, z frames final, output frames emitted
    float* g = nullptr;                     // [B][2 * 512 * 16] cond_layer(timbre), computed at begin and set_timbre
    int64_t* codes = nullptr;               // [B][3][kVcCodesHist]: row 0 prosody, rows 1..2 content; frame t of the last
                                            // kVcCodesHist at column t - N + kVcCodesHist (right-aligned at N)
    float* z = nullptr;                     // [B][kVcZHist][1024]
    DevMem mem;                             // a fac_vc_stream_* stream's own state (null in a pool)
};

// A stream pool: `cap` slots of session state, each a B = 1 view, and the B = 32 lanes a batch runs in.
template <typename S>
struct Pool {
    int cap = 0;
    std::vector<S> slot;
    std::vector<char> used;
    S lanes;                                // a codes pool's n_c, a vc pool's options: those of the lanes and every slot
    DevMem mem;
};
using CodesPool = Pool<EncHalf>;
using VcPool = Pool<VcStream>;
using DecPool = Pool<DecHalf>;

}  // namespace

struct fac_handle {
    int device = 0;
    std::string err;
    TensorMap host[FAC_NUM_MODULES];
    bool have[FAC_NUM_MODULES] = {false, false, false, false, false};
    bool finalized = false;
    uint64_t fp[FAC_NUM_MODULES] = {0, 0, 0, 0, 0};   // weight fingerprints of the modules, taken at fac_finalize (session state)
    DevBuf<float> warena;           // the codec's weights: the offsets in enc, dec, qw, red and dec2 point into it
    EncW enc; DecW dec; QuantW qw;
    RedW red; DecW dec2;            // voice-conversion model: Redecoder + its non-causal, LSTM-free decoder
    // weight sets, streams and pools by id; a destroyed set, an ended stream or a destroyed pool leaves a null entry, so ids
    // are never reused
    std::vector<std::unique_ptr<RvqSet>> rvqs;              // residual VQ sets (fac_rvq_*)
    std::vector<std::unique_ptr<HeadSet>> heads;            // modules/quantize.py:106-125 CNNLSTM instances (fac_head_*)
    std::vector<std::unique_ptr<JdcSet>> jdcs;              // modules/JDC/model.py JDCNet instances, eval mode (fac_jdc_*)
    std::vector<std::unique_ptr<Stream>> streams;           // chunked encoder / decoder (fac_stream_*)
    std::vector<std::unique_ptr<VcStream>> vc_streams;      // chunked voice conversion through the redecoder (fac_vc_stream_*)
    std::vector<std::unique_ptr<CodesPool>> codes_pools;    // many B = 1 compression streams (fac_codes_pool_*)
    std::vector<std::unique_ptr<VcPool>> vc_pools;          // many B = 1 voice-conversion streams (fac_vc_pool_*)
    std::vector<std::unique_ptr<DecPool>> dec_pools;        // many B = 1 decode-from-codes streams (fac_dec_pool_*)
    fac::RsHost* rs = nullptr;      // resampler filter tables and session pools (fac_resample*, fac_rs_pool_*), made on use
    DevMem ws; size_t ws_bytes = 0;
    int launches = 0;
    // tensor-core path (fac_set_option "tensor_cores"): 0 = never, 1 = layers downstream of the VQ only
    // (decoder, timbre branch), 2 = every eligible layer (default; promoted accumulation upstream of the VQ)
    int use_tc = 2;
    int fuse_res = 1;               // fused ResidualUnit launches (fac_set_option "fuse_resunit"): the decoder's, and the
                                    // encoder's C = 64 and 128 units in the promoted fp16 hi + scaled-lo class (bit-identical
                                    // to their two launches); 2 = only where the fused tile still allows two CTAs per SM
                                    // (C <= 128)
    int lstm_v2 = 1;                // fac_set_option "lstm_v2": resident-W fp16 recurrence kernel (lstm2.cu); 0 = round-1 kernel
    int dec_lstm_fp16 = 1;          // fac_set_option "decoder_lstm_fp16": downstream LSTMs run ONE fp16 pass (0 = bf16 hi/lo 3-pass)
    int attn_stream = 0;            // fac_set_option "attention_stream": 1 forces the recomputing attention kernel (test aid)
    int dec_c7_f16 = 1;             // fac_set_option "decoder_conv7_fp16": k = 7 convs downstream of the VQ take ONE fp16 pass (0 = bf16 hi/lo 3-pass)
    int enc_f16 = 1;                // fac_set_option "encoder_f16x2": promoted layers use the fp16 hi + scaled-lo split (0 = 3xTF32)
    int enc_tt = 0;                 // fac_set_option "encoder_tt": those layers use the transposed formulation (time = wgmma N)
    int tc_occ2 = 0;                // fac_set_option "tc_occ2_maxn": tiles with N <= this are planned for two CTAs per SM (0 = off)
    bool dec_bf16 = true;           // decoder-side layers use the bf16x3 split (fac_set_option "decoder_bf16")
    // second stream for the waveform-only half of the quantizer (fac_set_option "overlap_front")
    int overlap_front = 1; cudaStream_t side = nullptr; cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    DevBuf<float> aa_filter;
    // dataset-side mel (meldataset.py:29-47: MelSpectrogram with its default sample_rate 16000): own constants, built lazily
    DevBuf<float> mel16_arena; ConvW mel16_dft, mel16_dft_tc; size_t mel16_fb = 0;
    // losses.py:65-89 reconstruction_loss: per scale s = 64 << i the window-folded DFT basis [s][ld] (+ tensor-core blobs)
    // and the 64-band HTK filterbank [n_fft/2 + 1][64]; built on first use
    struct LossScale { ConvW dft; size_t fb = 0; int s = 0, nfft = 0, nb = 0, ld = 0; };
    DevBuf<float> loss_arena; LossScale loss_scale[6];
    // dac/nn/loss.py MultiScaleSTFTLoss / MelSpectrogramLoss: one cached configuration (rebuilt when the arguments change);
    // dftT is the same basis transposed ([ld][w]: the gradient GEMM dframes = dspec basis^T)
    struct SpecScale { ConvW dft, dftT; size_t fb = 0; int w = 0, nb = 0, ld = 0, n_out = 0; bool mel = false; };
    DevBuf<float> spec_arena; std::vector<SpecScale> spec_scales; std::vector<double> spec_key;
    // optional per-kernel-family timing (fac_profile_*): CUDA events around every launch
    bool profiling = false;
    struct ProfRec { std::string name; cudaEvent_t a, b; double flops, bytes; };
    std::vector<ProfRec> prof;
    struct ProfAgg { double ms = 0, flops = 0, bytes = 0; long launches = 0; };
    std::map<std::string, ProfAgg> prof_agg;
    // debug taps: named intermediates copied out during a forward (fac_debug_tap)
    std::map<std::string, std::pair<float*, size_t>> taps;
};

namespace {

// ------------------------------------------------------------------------------------------
// packing helpers (host)
// ------------------------------------------------------------------------------------------
// Host staging of one weight arena: every tensor starts on a 64-float boundary.
struct Packer {
    std::vector<float> pack;
    size_t alloc(size_t n) {
        size_t off = (pack.size() + 63) / 64 * 64;
        pack.resize(off + n, 0.f);
        return off;
    }
};

const HostTensor* find(const TensorMap& ts, const std::string& k) {
    auto it = ts.find(k);
    return it == ts.end() ? nullptr : &it->second;
}

struct PackError { std::string msg; };
const HostTensor& need(const TensorMap& ts, const std::string& k) {
    const HostTensor* t = find(ts, k);
    if (!t) throw PackError{"missing tensor '" + k + "'"};
    return *t;
}

// Folded conv weight in PyTorch layout [d0][d1][K] (weight-norm over dims != 0, encodec.py:42-51).
std::vector<float> folded_weight(const TensorMap& ts, const std::string& prefix, std::vector<int64_t>& shape) {
    if (const HostTensor* w = find(ts, prefix + ".weight")) {
        shape = w->shape;
        return w->data;
    }
    const HostTensor& v = need(ts, prefix + ".weight_v");
    const HostTensor& g = need(ts, prefix + ".weight_g");
    shape = v.shape;
    size_t d0 = (size_t)v.shape[0], inner = v.numel() / d0;
    if (g.numel() != d0) throw PackError{"weight_g shape mismatch at " + prefix};
    std::vector<float> w(v.numel());
    for (size_t i = 0; i < d0; ++i) {
        double s = 0.0;
        for (size_t j = 0; j < inner; ++j) { double x = v.data[i * inner + j]; s += x * x; }
        float scale = g.data[i] / (float)std::sqrt(s);
        for (size_t j = 0; j < inner; ++j) w[i * inner + j] = v.data[i * inner + j] * scale;
    }
    return w;
}

// Builds the tensor-core weight blob for a packed conv (stride-1 in rows; `stride` > 1 means the
// kernel-2*stride down-conv viewed as a 2-tap conv over rows of `stride` samples).
void attach_tc(Packer& P, ConvW& c, int stride, bool promoted) {
    TcConvParams tp;
    tp.Cin = c.Cin; tp.Cout = c.Cout; tp.dil = 1; tp.promoted = promoted ? 1 : 0;
    if (stride == 1) { tp.vf = 1; tp.Kr = c.K; }
    else if (c.K == 2 * stride) { tp.vf = stride; tp.Kr = 2; }
    else return;
    if (!tc_conv_plan(tp)) return;
    c.vf = tp.vf; c.Kr = tp.Kr; c.promoted = promoted; c.tcN = tp.N;
    size_t n = tc_blob_floats(tp);
    c.tcw = P.alloc(n);
    tc_pack_blob(tp, P.pack.data() + c.w, c.ldw, P.pack.data() + c.tcw);
    c.tc = true;
    if (promoted) {
        TcConvParams t16 = tp;
        t16.f16x2 = 1;
        if (tc_conv_plan(t16)) {
            c.tcw16 = P.alloc(tc_blob_floats(t16));
            tc_pack_blob(t16, P.pack.data() + c.w, c.ldw, P.pack.data() + c.tcw16);
            c.has16 = true;
        }
    } else {
        TcConvParams t16 = tp;
        t16.bf16 = 1;
        if (tc_conv_plan(t16)) {
            c.tcw16 = P.alloc(tc_blob_floats(t16));
            tc_pack_blob(t16, P.pack.data() + c.w, c.ldw, P.pack.data() + c.tcw16);
            c.has16 = true;
        }
    }
}

// hi-only fp16 blob of a stride-1 layer downstream of the VQ (conv_tc_kernel's one-pass class; the dilated k = 7 convs of
// the ResidualUnits: 7/8 of a unit's MACs, 1.4e-5 RMS on the waveform, scripts/cpu_decoder_precision.py)
void attach_f16_single(Packer& P, ConvW& c) {
    if (!c.tc || c.promoted || !c.has16 || c.vf != 1) return;
    TcConvParams t1;
    t1.Cin = c.Cin; t1.Cout = c.Cout; t1.dil = 1; t1.vf = 1; t1.Kr = c.K; t1.bf16 = 1; t1.g1f16 = 1;
    if (!tc_conv_plan(t1)) return;
    c.tcw_f16s = P.alloc(tc_blob_floats(t1));
    tc_pack_blob(t1, P.pack.data() + c.w, c.ldw, P.pack.data() + c.tcw_f16s);
    c.has_f16s = true;
}

// nn.Conv1d [Cout][Cin][K] -> packed [K*Cin][ldw]
ConvW pack_conv(Packer& P, const TensorMap& ts, const std::string& prefix, int stride = 1, bool promoted = false) {
    std::vector<int64_t> shp;
    std::vector<float> w = folded_weight(ts, prefix, shp);
    if (shp.size() == 2) shp.push_back(1);
    if (shp.size() != 3) throw PackError{"conv weight rank at " + prefix};
    ConvW c;
    c.Cout = (int)shp[0]; c.Cin = (int)shp[1]; c.K = (int)shp[2];
    c.ldw = (c.Cout + 3) / 4 * 4;
    c.w = P.alloc((size_t)c.K * c.Cin * c.ldw);
    for (int co = 0; co < c.Cout; ++co)
        for (int ci = 0; ci < c.Cin; ++ci)
            for (int k = 0; k < c.K; ++k)
                P.pack[c.w + ((size_t)k * c.Cin + ci) * c.ldw + co] = w[((size_t)co * c.Cin + ci) * c.K + k];
    const HostTensor& b = need(ts, prefix + ".bias");
    c.b = P.alloc(c.Cout);
    for (int co = 0; co < c.Cout; ++co) P.pack[c.b + co] = b.data[co];
    attach_tc(P, c, stride, promoted);
    return c;
}

// nn.ConvTranspose1d [Cin][Cout][2s] stride s + right trim (encodec.py:248-270) -> K=2 conv with
// Cout*s phase-major output channels: tap0 (x[t-1]) = w[..][r+s], tap1 (x[t]) = w[..][r].
ConvW pack_convtr(Packer& P, const TensorMap& ts, const std::string& prefix, int stride, bool promoted = false) {
    std::vector<int64_t> shp;
    std::vector<float> w = folded_weight(ts, prefix, shp);
    if (shp.size() != 3 || shp[2] != 2 * stride) throw PackError{"convtr kernel != 2*stride at " + prefix};
    int Cin = (int)shp[0], Cout = (int)shp[1], K = (int)shp[2];
    ConvW c;
    c.Cin = Cin; c.Cout = Cout * stride; c.K = 2; c.ldw = (c.Cout + 3) / 4 * 4;
    c.w = P.alloc((size_t)2 * Cin * c.ldw);
    for (int ci = 0; ci < Cin; ++ci)
        for (int co = 0; co < Cout; ++co)
            for (int r = 0; r < stride; ++r) {
                P.pack[c.w + ((size_t)0 * Cin + ci) * c.ldw + r * Cout + co] = w[((size_t)ci * Cout + co) * K + r + stride];
                P.pack[c.w + ((size_t)1 * Cin + ci) * c.ldw + r * Cout + co] = w[((size_t)ci * Cout + co) * K + r];
            }
    const HostTensor& b = need(ts, prefix + ".bias");
    c.b = P.alloc(c.Cout);
    for (int r = 0; r < stride; ++r)
        for (int co = 0; co < Cout; ++co) P.pack[c.b + r * Cout + co] = b.data[co];
    attach_tc(P, c, 1, promoted);
    return c;
}

// Non-causal variant (encodec.py:264-269: trim padding_total - padding_total/2 on the left, padding_total/2 on the right):
// output sample n = t*s + r reads full[n + pl], pl = s - s/2, i.e. x[t-1]*w[a+s] (a < s) + x[t]*w[a] + x[t+1]*w[a-s] (a >= s)
// with a = r + pl: a 3-tap conv over (x[t-1], x[t], x[t+1]), zero padding 1 | 1, s*Cout phase-major channels.
ConvW pack_convtr_noncausal(Packer& P, const TensorMap& ts, const std::string& prefix, int stride, bool promoted = false) {
    std::vector<int64_t> shp;
    std::vector<float> w = folded_weight(ts, prefix, shp);
    if (shp.size() != 3 || shp[2] != 2 * stride) throw PackError{"convtr kernel != 2*stride at " + prefix};
    int Cin = (int)shp[0], Cout = (int)shp[1], K = (int)shp[2];
    const int pl = stride - stride / 2;
    ConvW c;
    c.Cin = Cin; c.Cout = Cout * stride; c.K = 3; c.ldw = (c.Cout + 3) / 4 * 4;
    c.w = P.alloc((size_t)3 * Cin * c.ldw);
    for (int ci = 0; ci < Cin; ++ci)
        for (int co = 0; co < Cout; ++co)
            for (int r = 0; r < stride; ++r) {
                const int a = r + pl;
                const float* wk = &w[((size_t)ci * Cout + co) * K];
                P.pack[c.w + ((size_t)0 * Cin + ci) * c.ldw + r * Cout + co] = a < stride ? wk[a + stride] : 0.f;
                P.pack[c.w + ((size_t)1 * Cin + ci) * c.ldw + r * Cout + co] = wk[a];
                P.pack[c.w + ((size_t)2 * Cin + ci) * c.ldw + r * Cout + co] = a >= stride ? wk[a - stride] : 0.f;
            }
    const HostTensor& b = need(ts, prefix + ".bias");
    c.b = P.alloc(c.Cout);
    for (int r = 0; r < stride; ++r)
        for (int co = 0; co < Cout; ++co) P.pack[c.b + r * Cout + co] = b.data[co];
    attach_tc(P, c, 1, promoted);
    return c;
}

SnakeW pack_snake(Packer& P, const TensorMap& ts, const std::string& key) {
    const HostTensor& a = need(ts, key);
    SnakeW s;
    s.C = (int)a.numel();
    s.a = P.alloc(s.C);
    s.ia = P.alloc(s.C);
    for (int i = 0; i < s.C; ++i) {
        P.pack[s.a + i] = a.data[i];
        P.pack[s.ia + i] = 1.0f / (a.data[i] + 1e-9f);   // (alpha + 1e-9).reciprocal(), fp32
    }
    return s;
}

ResW pack_res(Packer& P, const TensorMap& ts, const std::string& prefix, int dil, bool promoted = false) {
    ResW r;
    r.dil = dil;
    r.s1 = pack_snake(P, ts, prefix + ".block.0.alpha");
    r.c7 = pack_conv(P, ts, prefix + ".block.1.conv.conv", 1, promoted);
    if (!promoted) attach_f16_single(P, r.c7);
    r.s2 = pack_snake(P, ts, prefix + ".block.2.alpha");
    r.c1 = pack_conv(P, ts, prefix + ".block.3.conv.conv", 1, promoted);
    return r;
}

LstmW pack_lstm(Packer& P, const TensorMap& ts, const std::string& prefix, bool promoted = false) {
    LstmW L;
    const HostTensor& w0 = need(ts, prefix + ".weight_hh_l0");
    L.H = (int)w0.shape[1];
    L.U = lstm_units_per_cta(L.H);
    if (L.U == 0) throw PackError{"unsupported LSTM width " + std::to_string(L.H)};
    L.G = L.H / L.U;
    const int H = L.H, U = L.U, R = 4 * U;
    for (int l = 0; l < 2; ++l) {
        std::string sfx = "_l" + std::to_string(l);
        const HostTensor& wih = need(ts, prefix + ".weight_ih" + sfx);
        const HostTensor& whh = need(ts, prefix + ".weight_hh" + sfx);
        const HostTensor& bih = need(ts, prefix + ".bias_ih" + sfx);
        const HostTensor& bhh = need(ts, prefix + ".bias_hh" + sfx);
        ConvW c;
        c.Cin = H; c.Cout = 4 * H; c.K = 1; c.ldw = 4 * H;
        c.w = P.alloc((size_t)H * c.ldw);
        for (int row = 0; row < 4 * H; ++row)
            for (int k = 0; k < H; ++k) P.pack[c.w + (size_t)k * c.ldw + row] = wih.data[(size_t)row * H + k];
        c.b = P.alloc(4 * H);
        for (int row = 0; row < 4 * H; ++row) P.pack[c.b + row] = bih.data[row] + bhh.data[row];
        attach_tc(P, c, 1, promoted);
        L.ih[l] = c;
        L.whh[l] = P.alloc((size_t)L.G * H * R);
        for (int cta = 0; cta < L.G; ++cta)
            for (int k = 0; k < H; ++k)
                for (int g = 0; g < 4; ++g)
                    for (int u = 0; u < U; ++u)
                        P.pack[L.whh[l] + ((size_t)cta * H + k) * R + g * U + u] =
                            whh.data[((size_t)g * H + cta * U + u) * H + k];
        for (int p3 = 0; p3 < 2; ++p3) {
            // second-generation kernel: promoted (upstream) layers use the 3-pass pack, the others the one-pass pack; the
            // 3-pass pack of a downstream layer backs fac_set_option("decoder_bf16", 0)
            if (p3 == 0 && promoted) continue;
            if ((H / 16) % 8 != 0 || lstm2_smem_bytes(H, U, p3) > 227 * 1024) continue;
            const size_t nw = lstm2_pack_words(H, U, p3);
            L.whh2[l][p3] = P.alloc(nw);
            lstm2_pack(whh.data.data(), H, U, p3, reinterpret_cast<uint32_t*>(P.pack.data() + L.whh2[l][p3]));
            L.has2[p3] = true;
        }
        if (!promoted) {
            // bf16 hi/lo words for the recurrence downstream of the VQ: [cta][H/16][hi|lo][8 k-pairs][R]
            auto bf16_rn = [](float f) { uint32_t u; memcpy(&u, &f, 4); u += 0x7FFFu + ((u >> 16) & 1u); return (uint32_t)(u >> 16); };
            auto bf16_f = [](uint32_t b) { uint32_t u = b << 16; float f; memcpy(&f, &u, 4); return f; };
            L.whh16[l] = P.alloc((size_t)L.G * H * R);
            for (int cta = 0; cta < L.G; ++cta)
                for (int sub = 0; sub < H / 16; ++sub)
                    for (int k2 = 0; k2 < 8; ++k2)
                        for (int r = 0; r < R; ++r) {
                            const int g = r / U, u = r % U;
                            const float* wrow = &whh.data[((size_t)g * H + cta * U + u) * H + sub * 16 + 2 * k2];
                            uint32_t h0 = bf16_rn(wrow[0]), h1 = bf16_rn(wrow[1]);
                            uint32_t l0 = bf16_rn(wrow[0] - bf16_f(h0)), l1 = bf16_rn(wrow[1] - bf16_f(h1));
                            uint32_t hw = h0 | (h1 << 16), lw = l0 | (l1 << 16);
                            size_t base = L.whh16[l] + ((size_t)cta * (H / 16) + sub) * 16 * R;
                            memcpy(&P.pack[base + (size_t)k2 * R + r], &hw, 4);
                            memcpy(&P.pack[base + (size_t)(8 + k2) * R + r], &lw, 4);
                        }
            L.has16 = true;
        }
    }
    return L;
}

VqW pack_vq_raw(Packer& P, const float* in_w, const float* in_b, const float* out_w, const float* out_b, const float* codebook) {
    VqW v;
    v.w_in = P.alloc(8 * 1024);
    for (int i = 0; i < 8 * 1024; ++i) P.pack[v.w_in + i] = in_w[i];
    v.b_in = P.alloc(8);
    for (int i = 0; i < 8; ++i) P.pack[v.b_in + i] = in_b[i];
    v.cb = P.alloc(1024 * 8);
    v.cbn = P.alloc(1024 * 8);
    v.cbn2 = P.alloc(1024);
    for (int j = 0; j < 1024; ++j) {
        float n2 = 0.f;
        for (int k = 0; k < 8; ++k) n2 = fmaf(codebook[j * 8 + k], codebook[j * 8 + k], n2);
        float nrm = fmaxf(sqrtf(n2), 1e-12f);
        float c2 = 0.f;
        for (int k = 0; k < 8; ++k) {
            float cn = codebook[j * 8 + k] / nrm;
            P.pack[v.cb + j * 8 + k] = codebook[j * 8 + k];
            P.pack[v.cbn + j * 8 + k] = cn;
            c2 = fmaf(cn, cn, c2);
        }
        P.pack[v.cbn2 + j] = c2;
    }
    v.w_out = P.alloc(8 * 1024);   // transposed [k][c]
    for (int c = 0; c < 1024; ++c)
        for (int k = 0; k < 8; ++k) P.pack[v.w_out + (size_t)k * 1024 + c] = out_w[c * 8 + k];
    v.b_out = P.alloc(1024);
    for (int c = 0; c < 1024; ++c) P.pack[v.b_out + c] = out_b[c];
    return v;
}

VqW pack_vq(Packer& P, const TensorMap& ts, const std::string& prefix) {
    std::vector<int64_t> s1, s2;
    std::vector<float> win = folded_weight(ts, prefix + ".in_proj", s1);
    std::vector<float> wout = folded_weight(ts, prefix + ".out_proj", s2);
    if (s1[0] != 8 || s1[1] != 1024 || s2[0] != 1024 || s2[1] != 8) throw PackError{"VQ shape at " + prefix};
    const HostTensor& bi = need(ts, prefix + ".in_proj.bias");
    const HostTensor& bo = need(ts, prefix + ".out_proj.bias");
    const HostTensor& cb = need(ts, prefix + ".codebook.weight");
    if (cb.shape[0] != 1024 || cb.shape[1] != 8) throw PackError{"codebook shape at " + prefix};
    return pack_vq_raw(P, win.data(), bi.data.data(), wout.data(), bo.data.data(), cb.data.data());
}

void pack_encoder(Packer& P, const TensorMap& ts, EncW& e) {
    const int rates[4] = {2, 5, 5, 6};
    e.conv0 = pack_conv(P, ts, "block.0.conv.conv");
    for (int i = 0; i < 4; ++i) {
        std::string p = "block." + std::to_string(i + 1);
        const int dils[3] = {1, 3, 9};
        for (int j = 0; j < 3; ++j) e.blk[i].res[j] = pack_res(P, ts, p + ".block." + std::to_string(j), dils[j], true);
        e.blk[i].snake = pack_snake(P, ts, p + ".block.3.alpha");
        e.blk[i].down = pack_conv(P, ts, p + ".block.4.conv.conv", rates[i], true);
        e.blk[i].stride = rates[i];
        if (e.blk[i].down.K != 2 * rates[i]) throw PackError{"encoder stride/kernel mismatch"};
    }
    e.lstm = pack_lstm(P, ts, "block.5.lstm", true);
    e.snake = pack_snake(P, ts, "block.6.alpha");
    e.conv_out = pack_conv(P, ts, "block.7.conv.conv", 1, true);
}

void pack_decoder(Packer& P, const TensorMap& ts, DecW& d, bool lstm, bool causal) {
    const int rates[4] = {6, 5, 5, 2};
    d.causal = causal; d.has_lstm = lstm;
    // The two layers with the longest chains outside the ResidualUnits (conv0: 1024 x 7 products per output, block 1's
    // up-conv: 1536 x 2) take the promoted packing: on conv_tc_kernel's bf16 hi/lo class the truncating tensor-core
    // accumulation over such a chain reaches 2.4-6x the error of the class's operand rounding
    // (tests/test_gpu_codec_stages.py).  Later up-convs (<= 768 x 2) stay within it; the units keep their classes.
    d.conv0 = pack_conv(P, ts, "model.0.conv.conv", 1, true);
    int base = 1;
    if (lstm) { d.lstm = pack_lstm(P, ts, "model.1.lstm"); base = 2; }
    for (int i = 0; i < 4; ++i) {
        std::string p = "model." + std::to_string(i + base);
        d.blk[i].snake = pack_snake(P, ts, p + ".block.0.alpha");
        const bool long_chain = i == 0;
        d.blk[i].up = causal ? pack_convtr(P, ts, p + ".block.1.convtr.convtr", rates[i], long_chain)
                             : pack_convtr_noncausal(P, ts, p + ".block.1.convtr.convtr", rates[i], long_chain);
        d.blk[i].stride = rates[i];
        d.blk[i].cout = d.blk[i].up.Cout / rates[i];
        const int dils[3] = {1, 3, 9};
        for (int j = 0; j < 3; ++j) d.blk[i].res[j] = pack_res(P, ts, p + ".block." + std::to_string(j + 2), dils[j]);
    }
    d.snake = pack_snake(P, ts, "model." + std::to_string(4 + base) + ".alpha");
    d.conv_out = pack_conv(P, ts, "model." + std::to_string(5 + base) + ".conv.conv");
}

// modules/redecoder.py:5-21 (encoder_type "wavenet"); key names of modules/wavenet.py:103-136 under "encoder."
void pack_redecoder(Packer& P, const TensorMap& ts, RedW& r) {
    auto emb = [&](const std::string& key) {
        const HostTensor& t = need(ts, key);
        if (t.shape.size() != 2 || t.shape[0] != 1024 || t.shape[1] != r.hidden) throw PackError{"embedding shape at " + key};
        size_t off = P.alloc(t.numel());
        for (size_t i = 0; i < t.numel(); ++i) P.pack[off + i] = t.data[i];
        return off;
    };
    r.emb_p = emb("prosody_embed.0.weight");
    r.emb_c[0] = emb("content_embed.0.weight");
    r.emb_c[1] = emb("content_embed.1.weight");
    r.cond = pack_conv(P, ts, "encoder.cond_layer.conv.conv");
    for (int i = 0; i < r.layers; ++i) {
        r.wn_in[i] = pack_conv(P, ts, "encoder.in_layers." + std::to_string(i) + ".conv.conv");
        r.wn_rs[i] = pack_conv(P, ts, "encoder.res_skip_layers." + std::to_string(i) + ".conv.conv");
    }
    r.conv_out = pack_conv(P, ts, "conv_out");
    if (r.cond.Cin != LATENT || r.cond.Cout != 2 * r.hidden * r.layers || r.wn_in[0].K != 5 || r.conv_out.Cout != LATENT)
        throw PackError{"redecoder geometry (expects WN(512, kernel 5, 16 layers, gin 1024))"};
}

// Periodic Hann window of n samples (torch.hann_window, scipy.signal.get_window("hann")), fp64.
std::vector<double> periodic_hann(int n) {
    std::vector<double> w(n);
    for (int i = 0; i < n; ++i) w[i] = 0.5 - 0.5 * std::cos(2.0 * M_PI * (double)i / (double)n);
    return w;
}

// Window-folded real DFT basis: row n of dst (stride ld) holds win[n] (cos, -sin)(2 pi k (n + left) / n_fft) for k < nb,
// interleaved (fp64, rounded once to fp32).
void dft_basis(float* dst, size_t ld, const std::vector<double>& win, int n_fft, int nb, int left) {
    for (int n = 0; n < (int)win.size(); ++n)
        for (int k = 0; k < nb; ++k) {
            // reduce the phase index mod n_fft in integers so the fp64 angle stays small
            const long long ph = ((long long)k * (n + left)) % n_fft;
            const double ang = 2.0 * M_PI * (double)ph / (double)n_fft;
            dst[(size_t)n * ld + 2 * k] = (float)(win[n] * std::cos(ang));
            dst[(size_t)n * ld + 2 * k + 1] = (float)(-win[n] * std::sin(ang));
        }
}

// torchaudio.functional.melscale_fbanks(n_bins, f_min = 0, f_max, n_mels, sample_rate = 2 f_max, norm = None, "htk"):
// [n_bins][n_mels]
std::vector<float> htk_fbank(double f_max, int n_bins, int n_mels) {
    auto hz2mel = [](double f) { return 2595.0 * std::log10(1.0 + f / 700.0); };
    auto mel2hz = [](double m) { return 700.0 * (std::pow(10.0, m / 2595.0) - 1.0); };
    std::vector<double> fpts(n_mels + 2);
    for (int i = 0; i < n_mels + 2; ++i) fpts[i] = mel2hz(hz2mel(0.0) + (hz2mel(f_max) - hz2mel(0.0)) * i / (n_mels + 1));
    std::vector<float> fb((size_t)n_bins * n_mels);
    for (int k = 0; k < n_bins; ++k) {
        const double f = f_max * k / (n_bins - 1);
        for (int m = 0; m < n_mels; ++m) {
            const double down = (f - fpts[m]) / (fpts[m + 1] - fpts[m]), up = (fpts[m + 2] - f) / (fpts[m + 2] - fpts[m + 1]);
            fb[(size_t)k * n_mels + m] = (float)std::max(0.0, std::min(down, up));
        }
    }
    return fb;
}

// The mel front-end's constants: [1200][2*1025] windowed DFT basis (fp64 -> fp32), its tensor-core variant, the filterbank.
void pack_mel_frontend(Packer& P, ConvW& dft, ConvW& dft_tc, size_t& fb_off, const float* win, const float* fb) {
    dft.Cin = 1; dft.Cout = 2 * N_BINS; dft.K = WIN; dft.ldw = SPEC_LD;
    dft.w = P.alloc((size_t)WIN * SPEC_LD);
    dft.b = 0;
    dft_basis(P.pack.data() + dft.w, SPEC_LD, std::vector<double>(win, win + WIN), N_FFT, N_BINS, (N_FFT - WIN) / 2);
    // tensor-core variant: [1200][2176] with zero columns beyond 2*1025, zero bias
    dft_tc.Cin = WIN; dft_tc.Cout = SPEC_TC_LD; dft_tc.K = 1; dft_tc.ldw = SPEC_TC_LD;
    dft_tc.w = P.alloc((size_t)WIN * SPEC_TC_LD);
    for (int n = 0; n < WIN; ++n)
        for (int k = 0; k < 2 * N_BINS; ++k) P.pack[dft_tc.w + (size_t)n * SPEC_TC_LD + k] = P.pack[dft.w + (size_t)n * SPEC_LD + k];
    dft_tc.b = P.alloc(SPEC_TC_LD);
    attach_tc(P, dft_tc, 1, true);
    fb_off = P.alloc((size_t)N_BINS * N_MELS);
    for (size_t i = 0; i < (size_t)N_BINS * N_MELS; ++i) P.pack[fb_off + i] = fb[i];
}

void pack_quantizer(Packer& P, const TensorMap& ts, QuantW& q) {
    q.vq[0] = pack_vq(P, ts, "prosody_quantizer.quantizers.0");
    q.vq[1] = pack_vq(P, ts, "content_quantizer.quantizers.0");
    q.vq[2] = pack_vq(P, ts, "content_quantizer.quantizers.1");
    for (int i = 0; i < 3; ++i) q.vq[3 + i] = pack_vq(P, ts, "residual_quantizer.quantizers." + std::to_string(i));
    q.spec0 = pack_conv(P, ts, "timbre_encoder.spectral.0", 1, true);
    q.spec3 = pack_conv(P, ts, "timbre_encoder.spectral.3", 1, true);
    q.glu[0] = pack_conv(P, ts, "timbre_encoder.temporal.0.conv1", 1, true);
    q.glu[1] = pack_conv(P, ts, "timbre_encoder.temporal.1.conv1", 1, true);
    q.cq = pack_conv(P, ts, "timbre_encoder.slf_attn.conv_q", 1, true);
    q.ck = pack_conv(P, ts, "timbre_encoder.slf_attn.conv_k", 1, true);
    q.cv = pack_conv(P, ts, "timbre_encoder.slf_attn.conv_v", 1, true);
    q.co = pack_conv(P, ts, "timbre_encoder.slf_attn.conv_o", 1, true);
    q.fc = pack_conv(P, ts, "timbre_encoder.fc", 1, true);
    q.timbre_linear = pack_conv(P, ts, "timbre_linear", 1, true);
    q.mel_lin = pack_conv(P, ts, "melspec_linear.conv.conv");
    for (int i = 0; i < 8; ++i) {
        q.wn_in[i] = pack_conv(P, ts, "melspec_encoder.in_layers." + std::to_string(i) + ".conv.conv", 1, true);
        q.wn_rs[i] = pack_conv(P, ts, "melspec_encoder.res_skip_layers." + std::to_string(i) + ".conv.conv", 1, true);
    }
    q.mel_lin2 = pack_conv(P, ts, "melspec_linear2.conv.conv", 1, true);
    // STFT basis with the Hann window folded in: frame sample n+424 of the zero-padded window
    const HostTensor& win = need(ts, "to_mel.spectrogram.window");
    const HostTensor& fb = need(ts, "to_mel.mel_scale.fb");
    if ((int)win.numel() != WIN || fb.shape[0] != N_BINS || fb.shape[1] != N_MELS) throw PackError{"mel buffers shape"};
    pack_mel_frontend(P, q.dft, q.dft_tc, q.fb, win.data.data(), fb.data.data());
}

// ------------------------------------------------------------------------------------------
// forward context: bump allocator over the handle's workspace + launch helpers
// ------------------------------------------------------------------------------------------
struct Ctx {
    fac_handle* h;
    cudaStream_t st;
    bool dry;          // size pass: allocate only
    const float* wbase = nullptr;   // the weight arena W() reads
    bool vq_critical = false;   // inside the encoder / prosody branch: feeds the bit-exact VQ argmin
    size_t off = 0;
    cudaError_t cerr = cudaSuccess;
    const char* where = "";

    template <typename T>
    T* alloc(size_t n) {
        size_t bytes = (n * sizeof(T) + 255) / 256 * 256;
        char* p = h->ws ? h->ws.get() + off : nullptr;
        off += bytes;
        return reinterpret_cast<T*>(p);
    }
    const float* W(size_t o) const { return wbase + o; }
    bool ok() const { return cerr == cudaSuccess; }
    void check(cudaError_t e, const char* w) {     // a kernel launch
        if (!dry) h->launches++;
        if (e != cudaSuccess && cerr == cudaSuccess) { cerr = e; where = w; }
    }
    void check_nk(cudaError_t e, const char* w) {  // memset / memcpy: not a kernel
        if (e != cudaSuccess && cerr == cudaSuccess) { cerr = e; where = w; }
    }
    void tap(const char* name, const float* src, size_t n) {
        if (dry || h->taps.empty()) return;
        auto it = h->taps.find(name);
        if (it == h->taps.end()) return;
        size_t m = n < it->second.second ? n : it->second.second;
        check_nk(cudaMemcpyAsync(it->second.first, src, m * sizeof(float), cudaMemcpyDeviceToDevice, st), "tap");
    }
    // profiling: begin()/end() bracket one launch with events on the launching stream
    void begin(const char* fam, double flops, double bytes, const char* detail = nullptr) {
        if (dry || !h->profiling) return;
        fac_handle::ProfRec r;
        r.name = fam; r.flops = flops; r.bytes = bytes;
        if (detail) { r.name += ":"; r.name += detail; }
        cudaEventCreate(&r.a); cudaEventCreate(&r.b);
        cudaEventRecord(r.a, st);
        h->prof.push_back(r);
    }
    void end() {
        if (dry || !h->profiling) return;
        cudaEventRecord(h->prof.back().b, st);
    }
};

struct ConvOpts {
    int dil = 1, stride = 1, pad_left = 0, pad_right = 0, reflect = 0;
    const SnakeW* in_snake = nullptr;
    const SnakeW* out_snake = nullptr;
    int act = ACT_NONE;
    const float* res = nullptr;
    const int* valid_len = nullptr;
    const int* lane_len = nullptr;   // [B] device: each lane's own input rows (a ragged batch), or null
    int transposed = 0;
    int ldx = 0;            // input row stride (0 = Cin)
    int ldy = 0;            // output row stride (0 = Cout)
    bool no_bias = false;
};

// SConv1d padding rule (encodec.py:212-228): causal => (k_eff - stride) on the left (reflect),
// plus "extra" on the right so the last window is full (encodec.py:71-78).
int conv_out_len(int T, int k_eff, int stride) {
    int padding_total = k_eff - stride;
    double n_frames = (double)(T - k_eff + padding_total) / stride + 1.0;
    int ideal = ((int)std::ceil(n_frames) - 1) * stride + (k_eff - padding_total);
    int extra = ideal - T;
    return (T + padding_total + extra - k_eff) / stride + 1;
}
int conv_extra_pad(int T, int k_eff, int stride) {
    int padding_total = k_eff - stride;
    double n_frames = (double)(T - k_eff + padding_total) / stride + 1.0;
    int ideal = ((int)std::ceil(n_frames) - 1) * stride + (k_eff - padding_total);
    return ideal - T;
}

void run_conv(Ctx& c, const ConvW& w, const float* x, float* y, int B, int Tin, int Tout, const ConvOpts& o,
              const char* name) {
    if (c.dry) return;
    if (c.h->use_tc >= (c.vq_critical ? 2 : 1) && w.tc && !o.transposed && !o.valid_len && (o.ldx == 0 || o.ldx == w.Cin) &&
        (o.ldy == 0 || o.ldy == w.Cout) && o.stride == w.vf && (w.vf == 1 || o.dil == 1) && !o.no_bias) {
        TcConvParams tp;
        tp.Cin = w.Cin; tp.Cout = w.Cout; tp.vf = w.vf; tp.Kr = w.Kr; tp.promoted = w.promoted ? 1 : 0;
        // Every promoted layer runs the promoted kernel, the short 1x1 convs of the 64- and 128-channel encoder stages
        // included: on conv_tc_kernel they would take its 3xTF32 class, whose units measure 2.4x the rms error of the fp32
        // kernels against 0.07-0.10 of the bf16 hi/lo error (tests/test_gpu_codec_stages.py), and they feed the VQ argmin.
        tp.dil = w.vf == 1 ? o.dil : 1;
        tp.bf16 = (c.h->dec_bf16 && w.has16 && !w.promoted && !c.vq_critical) ? 1 : 0;
        tp.g1f16 = (tp.bf16 && w.has_f16s && c.h->dec_c7_f16) ? 1 : 0;
        tp.f16x2 = (tp.promoted && c.h->enc_f16 && w.has16) ? 1 : 0;
        tp.occ2_maxn = c.h->tc_occ2;
        tp.Tout = Tout;
        if (tp.f16x2 && c.h->enc_tt) {
            TcConvParams t2 = tp;
            t2.tt = 1;
            if (tc_conv_plan(t2)) tp = t2;
        }
        if (tc_conv_plan(tp)) {
            tp.x = x; tp.y = y; tp.wblob = c.W(tp.g1f16 ? w.tcw_f16s : ((tp.bf16 || tp.f16x2) ? w.tcw16 : w.tcw)); tp.bias = c.W(w.b);
            if (o.in_snake) { tp.in_alpha = c.W(o.in_snake->a); tp.in_inv_alpha = c.W(o.in_snake->ia); }
            tp.out_act = o.act;
            if (o.out_snake) { tp.out_act = ACT_SNAKE; tp.out_alpha = c.W(o.out_snake->a); tp.out_inv_alpha = c.W(o.out_snake->ia); }
            tp.res = o.res;
            tp.B = B; tp.Tin = Tin; tp.ldx = w.Cin;
            tp.PLr = o.pad_left / w.vf;
            tp.pad_left_s = o.pad_left; tp.pad_right_s = o.pad_right; tp.reflect = o.reflect; tp.lane_len = o.lane_len;
            tp.Tout = Tout; tp.ldy = w.Cout;
            tp.x_bstride = (size_t)Tin * w.Cin; tp.y_bstride = (size_t)Tout * w.Cout;
            double flops = 2.0 * B * Tout * (double)w.Cout * w.K * w.Cin;
            double bytes = 4.0 * ((double)B * Tin * w.Cin + (double)B * Tout * w.Cout * (o.res ? 2 : 1) + (double)w.K * w.Cin * w.Cout);
            char det[96];
            snprintf(det, sizeof det, "%s Cin%d Cout%d K%d d%d T%d", name, w.Cin, w.Cout, w.K, o.dil, Tout);
            c.begin(tp.promoted ? "conv_tcp" : "conv_tc", flops, bytes, det);
            c.check(launch_conv_tc(tp, c.st), name);
            c.end();
            return;
        }
    }
    ConvParams p;
    p.x = x; p.y = y;
    p.w = c.W(w.w);
    p.bias = o.no_bias ? nullptr : c.W(w.b);
    if (o.in_snake) { p.in_alpha = c.W(o.in_snake->a); p.in_inv_alpha = c.W(o.in_snake->ia); }
    p.out_act = o.act;
    if (o.out_snake) { p.out_act = ACT_SNAKE; p.out_alpha = c.W(o.out_snake->a); p.out_inv_alpha = c.W(o.out_snake->ia); }
    p.res = o.res; p.valid_len = o.valid_len; p.lane_len = o.lane_len;
    p.B = B; p.Tin = Tin; p.Cin = w.Cin; p.Tout = Tout; p.Cout = w.Cout;
    p.K = w.K; p.dil = o.dil; p.stride = o.stride;
    p.pad_left = o.pad_left; p.pad_right = o.pad_right; p.pad_reflect = o.reflect;
    p.ldw = w.ldw; p.ldy = o.ldy ? o.ldy : w.Cout; p.ldx = o.ldx ? o.ldx : w.Cin;
    p.y_transposed = o.transposed;
    p.x_bstride = (size_t)Tin * p.ldx;
    p.y_bstride = (size_t)Tout * p.ldy;
    // algorithmic work of this launch: 2*MACs; bytes = input + output (+ residual) + weights once
    double flops = 2.0 * B * Tout * (double)w.Cout * w.K * w.Cin;
    double bytes = 4.0 * ((double)B * Tin * w.Cin + (double)B * Tout * w.Cout * (o.res ? 2 : 1) + (double)w.K * w.Cin * w.Cout);
    char det[96];
    snprintf(det, sizeof det, "%s Cin%d Cout%d K%d d%d T%d", name, w.Cin, w.Cout, w.K, o.dil, Tout);
    c.begin("conv", flops, bytes, det);
    c.check(launch_conv(p, c.st), name);
    c.end();
}

// SConv1d with reflect padding (encodec.py:212-228): causal = everything on the left, else padding_total - padding_total/2
// on the left and padding_total/2 (+ extra) on the right; returns output length
int sconv(Ctx& c, const ConvW& w, const float* x, float* y, int B, int T, int dil, int stride, ConvOpts o,
          const char* name, bool causal = true) {
    int k_eff = (w.K - 1) * dil + 1;
    o.dil = dil; o.stride = stride;
    const int total = k_eff - stride, extra = conv_extra_pad(T, k_eff, stride);
    o.pad_left = causal ? total : total - total / 2;
    o.pad_right = (causal ? 0 : total / 2) + extra;
    o.reflect = 1;
    int Tout = conv_out_len(T, k_eff, stride);
    run_conv(c, w, x, y, B, T, Tout, o, name);
    return Tout;
}

// Whole ResidualUnit in one tensor-core launch (conv_tc_kernel<true>) when every channel fits one CTA tile.  Upstream of
// the VQ only where the two launches would run the promoted fp16 hi + scaled-lo class (the fused launch is bit-identical
// to them there); every other route upstream keeps its two launches.
bool residual_unit_fused(Ctx& c, const ResW& r, const float* x, float* y, int B, int T, bool causal, const int* lane_len) {
    const bool promoted = r.c7.promoted && r.c1.promoted;
    if (!c.h->fuse_res || !r.c7.tc || !r.c1.tc || r.c7.promoted != r.c1.promoted || r.c7.Cin != r.c7.Cout ||
        r.c1.K != 1 || r.c7.vf != 1)
        return false;
    if (c.vq_critical ? (!promoted || c.h->use_tc < 2 || !c.h->enc_f16 || c.h->enc_tt || !r.c7.has16 || !r.c1.has16)
                      : (promoted || c.h->use_tc < 1))
        return false;
    TcConvParams tp;
    tp.Cin = r.c7.Cin; tp.Cout = r.c7.Cout; tp.vf = 1; tp.Kr = r.c7.K; tp.dil = r.dil; tp.fused = 1;
    tp.promoted = promoted ? 1 : 0;
    tp.f16x2 = tp.promoted;
    tp.bf16 = (!promoted && c.h->dec_bf16 && r.c7.has16 && r.c1.has16) ? 1 : 0;
    tp.g1f16 = (tp.bf16 && r.c7.has_f16s && c.h->dec_c7_f16) ? 1 : 0;
    tp.occ2_maxn = c.h->tc_occ2;
    tp.Tout = T;
    if (c.h->fuse_res == 2 && r.c7.Cout > 128) return false;
    if (!tc_conv_plan(tp)) return false;
    // the unit's weight blobs were laid out by the unfused plans of the same split classes: their tile must be N = C too
    TcConvParams q7 = tp, q1 = tp;
    q7.fused = 0; q1.fused = 0; q1.Kr = 1; q1.g1f16 = 0;
    if (!tc_conv_plan(q7) || !tc_conv_plan(q1) || q7.N != tp.N || q1.N != tp.N) return false;
    if (c.dry) return true;
    const int k_eff = (r.c7.K - 1) * r.dil + 1;
    tp.x = x; tp.y = y; tp.res = x;
    tp.wblob = c.W(tp.g1f16 ? r.c7.tcw_f16s : ((tp.bf16 || tp.f16x2) ? r.c7.tcw16 : r.c7.tcw)); tp.bias = c.W(r.c7.b);
    tp.wblob2 = c.W((tp.bf16 || tp.f16x2) ? r.c1.tcw16 : r.c1.tcw); tp.bias2 = c.W(r.c1.b);
    tp.in_alpha = c.W(r.s1.a); tp.in_inv_alpha = c.W(r.s1.ia);
    tp.out_act = ACT_SNAKE; tp.out_alpha = c.W(r.s2.a); tp.out_inv_alpha = c.W(r.s2.ia);
    tp.B = B; tp.Tin = T; tp.ldx = r.c7.Cin;
    const int pl = causal ? k_eff - 1 : (k_eff - 1) - (k_eff - 1) / 2;
    tp.PLr = pl; tp.pad_left_s = pl; tp.pad_right_s = k_eff - 1 - pl; tp.reflect = 1; tp.lane_len = lane_len;
    tp.Tout = T; tp.ldy = r.c7.Cout;
    tp.x_bstride = (size_t)T * r.c7.Cin; tp.y_bstride = (size_t)T * r.c7.Cout;
    double flops = 2.0 * B * T * (double)r.c7.Cout * r.c7.Cin * (r.c7.K + 1);
    double bytes = 4.0 * ((double)B * T * r.c7.Cin * 2 + (double)B * T * r.c7.Cout + (double)(r.c7.K + 1) * r.c7.Cin * r.c7.Cout);
    char det[96];
    snprintf(det, sizeof det, "res.fused C%d K%d d%d T%d", r.c7.Cin, r.c7.K, r.dil, T);
    c.begin(tp.promoted ? "conv_tcp" : "conv_tc", flops, bytes, det);
    c.check(launch_conv_tc(tp, c.st), "res.fused");
    c.end();
    return true;
}

// ResidualUnit (dac.py:25-42): y = x + conv1(snake2(conv7_d(snake1(x)))); lane_len as ConvOpts::lane_len
void residual_unit(Ctx& c, const ResW& r, const float* x, float* tmp, float* y, int B, int T, bool causal = true,
                   const int* lane_len = nullptr) {
    if (residual_unit_fused(c, r, x, y, B, T, causal, lane_len)) return;
    ConvOpts o1;
    o1.in_snake = &r.s1;
    o1.out_snake = &r.s2;
    o1.lane_len = lane_len;
    sconv(c, r.c7, x, tmp, B, T, r.dil, 1, o1, "res.conv7", causal);
    ConvOpts o2;
    o2.res = x;
    sconv(c, r.c1, tmp, y, B, T, 1, 1, o2, "res.conv1", causal);
}

// Carried state of one 2-layer SLSTM (streaming): h in the kernel's published fp16 layout, c per CTA.
// Precision class of slstm's recurrence: 3-pass fp32-faithful upstream of the VQ (and when "decoder_bf16" is off), one fp16
// pass downstream.
int lstm_pass3(const Ctx& c) { return (c.vq_critical || !c.h->dec_bf16) ? 1 : 0; }
// Whether slstm runs the resident-W kernel (lstm2.cu), the only one that can carry a stream's state.
bool lstm_resident(const Ctx& c, const LstmW& L) {
    const int pass3 = lstm_pass3(c);
    return c.h->lstm_v2 && L.has2[pass3] && (pass3 || c.h->dec_lstm_fp16);
}

// SLSTM (encodec.py:272-288) on channels-last x [B][T][H]; y = lstm2(lstm1(x)) + x.  st (streaming, B <= 32, resident-W
// kernel only): initial state read from / final state written to st.  lens (HOST, B entries, with st): row b runs lens[b]
// steps, and st receives the state after them (rows of y past lens[b] are finite don't-cares).
void slstm(Ctx& c, const LstmW& L, const float* x, float* y, int B, int T, LstmState* st = nullptr, const int* lens = nullptr) {
    const int H = L.H;
    float* xg = c.alloc<float>((size_t)B * T * 4 * H);
    float* h1 = c.alloc<float>((size_t)B * T * H);
    float* hT = c.alloc<float>((size_t)2 * H * 32);
    uint32_t* h16 = c.alloc<uint32_t>((size_t)2 * 2 * (H / 2) * 32);
    unsigned int* bar = c.alloc<unsigned int>(64);
    for (int l = 0; l < 2; ++l) {
        const float* in = l == 0 ? x : h1;
        ConvOpts o;
        run_conv(c, L.ih[l], in, xg, 1, B * T, B * T, o, "lstm.ih");
        if (c.dry) continue;
        const int pass3 = lstm_pass3(c);
        const bool v2 = lstm_resident(c, L);
        for (int b0 = 0; b0 < B; b0 += 32) {
            int nb = B - b0 < 32 ? B - b0 : 32;
            LstmParams p;
            p.xg = xg + (size_t)b0 * T * 4 * H;
            p.whh_p = c.W(L.whh[l]);
            if (c.h->dec_bf16 && L.has16 && !c.vq_critical) { p.bf16 = 1; p.whh_p16 = c.W(L.whh16[l]); }
            p.skip = l == 1 ? x + (size_t)b0 * T * H : nullptr;
            p.y = (l == 0 ? h1 : y) + (size_t)b0 * T * H;
            p.hT = hT; p.bar = bar;
            p.B = nb; p.T = T; p.H = H; p.U = L.U; p.G = L.G;
            c.begin("lstm_rec", 2.0 * nb * T * 4.0 * H * H, 4.0 * ((double)nb * T * 5 * H + 4.0 * H * H));
            if ((st || lens) && (!v2 || B > 32 || !st)) {
                c.check(cudaErrorNotSupported, "lstm.stream (needs the resident-W kernel and B <= 32)"); c.end(); continue;
            }
            if (v2) {
                p.whh_p2 = reinterpret_cast<const uint32_t*>(c.W(L.whh2[l][pass3]));
                p.h16 = h16; p.pass3 = pass3;
                if (st) { p.state_h = st->h[l]; p.state_c = st->c[l]; }
                LstmLaneLens ll = {};
                for (int b = 0; lens && b < nb; ++b) ll.len[b] = lens[b];
                c.check(launch_lstm2_layer(p, c.st, lens ? &ll : nullptr), "lstm.rec2");
            } else {
                c.check(launch_lstm_layer(p, c.st), "lstm.rec");
            }
            c.end();
        }
    }
}

// Per-lane lengths of a ragged encode / forward: device rows of B ints (in the workspace) and their host copy.  Rows
// kEncRows[0..4]: the encoder's input samples and the rows after each down-sampling block (the conv_out_len chain, the
// last = latent frames); kTmRow: mel frames (samples / 300); kTqRow: code frames, min(mel, latent); kDecRow..+4: lane_rows()
// of the decoder from the code frames.  A null Lanes* is a batch whose lanes all have its own length.
constexpr int kTmRow = 5, kTqRow = 6, kDecRow = 7, kLaneRows = 12;
struct Lanes {
    const int* d = nullptr;
    std::vector<int> h;
    int B = 0;
    const int* at(int row) const { return d ? d + (size_t)row * B : nullptr; }
    const int* host(int row) const { return h.data() + (size_t)row * B; }
};
const int* lane_at(const Lanes* ln, int row) { return ln ? ln->at(row) : nullptr; }

size_t enc_stage_floats(int B, int T) {
    // largest activation of the encoder: [B][T][64] (== [B][T/2][128])
    return (size_t)B * ((size_t)T + 16) * 64;
}

// Encoder.forward (dac.py:69-104): x [B][T][1] -> z channels-last [B][Tz][1024] (or NCT when z_nct)
// Encoder front: conv0 + the four EncoderBlocks (a causal FIR stack) -> features [B][ceil(T/300)][1024] in workspace.
float* encoder_front(Ctx& c, const float* x, int B, int T, int* frames, const Lanes* ln = nullptr) {
    const EncW& e = c.h->enc;
    size_t stage = enc_stage_floats(B, T);
    float* buf[3] = {c.alloc<float>(stage), c.alloc<float>(stage), c.alloc<float>(stage)};
    int cur = 0;
    ConvOpts o0;
    o0.lane_len = lane_at(ln, 0);
    int t = sconv(c, e.conv0, x, buf[0], B, T, 1, 1, o0, "enc.conv0");
    c.tap("enc_conv0", buf[0], (size_t)B * t * 64);
    static const char* blk_names[4] = {"enc_block1", "enc_block2", "enc_block3", "enc_block4"};
    static const char* res_names[4][3] = {{"enc_block1.res0", "enc_block1.res1", "enc_block1.res2"},
                                          {"enc_block2.res0", "enc_block2.res1", "enc_block2.res2"},
                                          {"enc_block3.res0", "enc_block3.res1", "enc_block3.res2"},
                                          {"enc_block4.res0", "enc_block4.res1", "enc_block4.res2"}};
    for (int i = 0; i < 4; ++i) {
        for (int j = 0; j < 3; ++j) {
            int tmp = (cur + 1) % 3, nxt = (cur + 2) % 3;
            residual_unit(c, e.blk[i].res[j], buf[cur], buf[tmp], buf[nxt], B, t, true, lane_at(ln, i));
            cur = nxt;
            c.tap(res_names[i][j], buf[cur], (size_t)B * t * e.blk[i].res[j].c1.Cout);
        }
        ConvOpts o;
        o.in_snake = &e.blk[i].snake;
        o.lane_len = lane_at(ln, i);    // a down-sampling conv reflects about the lane's own end (its "extra" follows from it)
        int nxt = (cur + 1) % 3;
        t = sconv(c, e.blk[i].down, buf[cur], buf[nxt], B, t, 1, e.blk[i].stride, o, "enc.down");
        cur = nxt;
        c.tap(blk_names[i], buf[cur], (size_t)B * t * e.blk[i].down.Cout);
    }
    *frames = t;
    return buf[cur];
}

// Encoder.forward (dac.py:69-104): x [B][T][1] -> z channels-last [B][Tz][1024] (or NCT when z_nct)
int encoder_forward(Ctx& c, const float* x, int B, int T, float* z_out, bool z_nct, const Lanes* ln = nullptr) {
    const EncW& e = c.h->enc;
    c.vq_critical = true;
    int t = 0;
    float* feats = encoder_front(c, x, B, T, &t, ln);
    float* ylstm = c.alloc<float>((size_t)B * t * LATENT);
    slstm(c, e.lstm, feats, ylstm, B, t);
    c.tap("enc_lstm", ylstm, (size_t)B * t * 1024);
    ConvOpts o;
    o.in_snake = &e.snake;
    o.lane_len = lane_at(ln, 4);
    if (z_nct) {
        // same kernel as the channels-last path (bit-identical z), then a [B][T][C] -> [B][C][T] transpose
        float* zcl = c.alloc<float>((size_t)B * t * LATENT);
        sconv(c, e.conv_out, ylstm, zcl, B, t, 1, 1, o, "enc.conv_out");
        if (!c.dry) c.check(launch_transpose(zcl, z_out, B, t, LATENT, c.st), "enc.z_T");
    } else {
        sconv(c, e.conv_out, ylstm, z_out, B, t, 1, 1, o, "enc.conv_out");
    }
    c.vq_critical = false;
    return t;
}

// Decoder.forward (dac.py:131-165): z channels-last [B][Tf][1024] -> y [B][300 Tf][1].  d = the codec's decoder (causal,
// SLSTM) or the redecoder's (non-causal, no SLSTM).
// The upsampling stack after the (optional) SLSTM: 4 DecoderBlocks, Snake, final conv, tanh.  in [B][Tf][1536] -> y [B][300 Tf].
// buf[0..2]: three stage buffers of decoder_stage_floats(B, Tf) each; `in` may be one of them (index in_idx) or external (-1).
size_t decoder_stage_floats(int B, int Tf) {
    size_t stage = (size_t)B * (size_t)Tf * 28800 + 1024;   // largest: [B][Tf*150][192] == [B][Tf*300][96]
    size_t first = (size_t)B * Tf * 1536;
    return first > stage ? first : stage;
}
// lens (a ragged batch): [5][B] device, lane_rows() of d; null when every lane has Tf frames.
void decoder_stack(Ctx& c, const DecW& d, const float* in, int in_idx, float* const* buf, int B, int Tf, float* y,
                   const int* lens = nullptr) {
    int t = Tf;
    const float* cur_p = in;
    int cur = in_idx;
    static const char* dblk_names[4] = {"dec_block1", "dec_block2", "dec_block3", "dec_block4"};
    static const char* up_names[4] = {"dec_block1.up", "dec_block2.up", "dec_block3.up", "dec_block4.up"};
    static const char* res_names[4][3] = {{"dec_block1.res0", "dec_block1.res1", "dec_block1.res2"},
                                          {"dec_block2.res0", "dec_block2.res1", "dec_block2.res2"},
                                          {"dec_block3.res0", "dec_block3.res1", "dec_block3.res2"},
                                          {"dec_block4.res0", "dec_block4.res1", "dec_block4.res2"}};
    for (int i = 0; i < 4; ++i) {
        // Snake -> SConvTranspose1d(k=2s, stride s) as a zero-padded conv with s*Cout phase-major channels:
        // causal = 2 taps (x[t-1], x[t]), non-causal = 3 taps (x[t-1], x[t], x[t+1])
        ConvOpts o;
        o.in_snake = &d.blk[i].snake;
        o.pad_left = 1; o.pad_right = d.causal ? 0 : 1; o.reflect = 0;
        o.lane_len = lens ? lens + (size_t)i * B : nullptr;
        int nxt = cur < 0 ? 0 : (cur + 1) % 3;
        run_conv(c, d.blk[i].up, cur_p, buf[nxt], B, t, t, o, "dec.up");
        cur = nxt; cur_p = buf[cur];
        t *= d.blk[i].stride;
        c.tap(up_names[i], buf[cur], (size_t)B * t * d.blk[i].cout);
        for (int j = 0; j < 3; ++j) {
            int tmp = (cur + 1) % 3, nx2 = (cur + 2) % 3;
            residual_unit(c, d.blk[i].res[j], buf[cur], buf[tmp], buf[nx2], B, t, d.causal, lens ? lens + (size_t)(i + 1) * B : nullptr);
            cur = nx2; cur_p = buf[cur];
            c.tap(res_names[i][j], buf[cur], (size_t)B * t * d.blk[i].cout);
        }
        c.tap(dblk_names[i], buf[cur], (size_t)B * t * d.blk[i].cout);
    }
    ConvOpts o;
    o.in_snake = &d.snake;
    o.act = ACT_TANH;
    o.lane_len = lens ? lens + (size_t)4 * B : nullptr;
    sconv(c, d.conv_out, buf[cur], y, B, t, 1, 1, o, "dec.conv_out", d.causal);
}

// Rows of each lane of a ragged batch at every stage of decoder d: [5][B], row 0 the lanes' frames, row i + 1 the rows
// after DecoderBlock i's up-sampling (300 frames in row 4).  Each conv of the stack pads a lane about its own end.
std::vector<int> lane_rows(const DecW& d, const int* frames, int B) {
    std::vector<int> rows((size_t)5 * B);
    for (int b = 0; b < B; ++b) {
        rows[b] = frames[b];
        for (int i = 0; i < 4; ++i) rows[(size_t)(i + 1) * B + b] = rows[(size_t)i * B + b] * d.blk[i].stride;
    }
    return rows;
}

// Host ints -> workspace (null when v is empty).  The copy is queued on the call's stream, ahead of its kernels.
const int* upload_ints(Ctx& c, const std::vector<int>& v) {
    if (v.empty()) return nullptr;
    int* d = c.alloc<int>(v.size());
    if (!c.dry) c.check_nk(cudaMemcpyAsync(d, v.data(), sizeof(int) * v.size(), cudaMemcpyHostToDevice, c.st), "lanes.h2d");
    return d;
}

// y [B][T]: samples [lens[b], T) of lane b set to 0, the output past a ragged lane's end.
__global__ void zero_tails_kernel(float* __restrict__ y, const int* __restrict__ lens, int T) {
    float* yb = y + (size_t)blockIdx.y * T;
    for (int t = lens[blockIdx.y] + blockIdx.x * blockDim.x + threadIdx.x; t < T; t += gridDim.x * blockDim.x) yb[t] = 0.f;
}
void zero_tails(Ctx& c, float* y, const int* lens, int B, int T) {
    if (c.dry || !lens) return;
    const int blocks = std::min((T + 255) / 256, 64);
    zero_tails_kernel<<<dim3(blocks, B), 256, 0, c.st>>>(y, lens, T);
    c.check(cudaGetLastError(), "zero_tails");
}

void decoder_forward(Ctx& c, const DecW& d, const float* z, int B, int Tf, float* y, const int* lens = nullptr) {
    const size_t stage = decoder_stage_floats(B, Tf);
    float* buf[3] = {c.alloc<float>(stage), c.alloc<float>(stage), c.alloc<float>(stage)};
    int cur = 0;
    ConvOpts o0;
    o0.lane_len = lens;
    int t = sconv(c, d.conv0, z, buf[0], B, Tf, 1, 1, o0, "dec.conv0", d.causal);
    c.tap("dec_conv0", buf[0], (size_t)B * t * 1536);
    if (d.has_lstm) {
        slstm(c, d.lstm, buf[0], buf[1], B, t);
        cur = 1;
        c.tap("dec_lstm", buf[1], (size_t)B * t * 1536);
    }
    decoder_stack(c, d, buf[cur], cur, buf, B, t, y, lens);
}

constexpr int kRedCodes = 1024;   // rows of each embedding table (pack_redecoder)

__global__ void embed_sum_kernel(const int64_t* __restrict__ codes_p, int cp_stride, const int64_t* __restrict__ codes_c,
                                 int cc_stride, const float* __restrict__ ep, const float* __restrict__ ec0,
                                 const float* __restrict__ ec1, float* __restrict__ out, int T, int hidden, int use_p, int n_c,
                                 const int* __restrict__ frames, const int* __restrict__ lane_mode) {
    // one CTA per (b, t): out[b][t][:] = [use_p] E_p[codes_p[b,0,t]] + sum_{i < n_c} E_c[i][codes_c[b,i,t]]  (redecoder.py:36-46)
    // codes_p / codes_c rows of utterance b start at b * cp_stride / b * cc_stride; content row i at + i * T.
    // A code outside [0, kRedCodes) reads nothing and makes the frame's embedding NaN.  frames (null: T each): frames
    // t >= frames[b] of a ragged batch read no code and are 0.  lane_mode (null: use_p and n_c for every b): [B][2] each
    // row's own use_p and n_c, so a row computes what a launch of its own mode computes.
    const int bt = blockIdx.x, b = bt / T, t = bt - b * T;
    if (frames && t >= frames[b]) {
        for (int c = threadIdx.x; c < hidden; c += blockDim.x) out[(size_t)bt * hidden + c] = 0.f;
        return;
    }
    if (lane_mode) { use_p = lane_mode[2 * b]; n_c = lane_mode[2 * b + 1]; }
    const long long ip = use_p ? codes_p[(size_t)b * cp_stride + t] : 0;
    const long long i0 = n_c > 0 ? codes_c[(size_t)b * cc_stride + t] : 0;
    const long long i1 = n_c > 1 ? codes_c[(size_t)b * cc_stride + T + t] : 0;
    const bool bad = ip < 0 || ip >= kRedCodes || i0 < 0 || i0 >= kRedCodes || i1 < 0 || i1 >= kRedCodes;
    for (int c = threadIdx.x; c < hidden; c += blockDim.x) {
        float v = __int_as_float(0x7fc00000);
        if (!bad) {
            float pe = 0.f, ce = 0.f;             // the reference sums the prosody and the content embeddings apart
            if (use_p) pe += ep[(size_t)ip * hidden + c];
            if (n_c > 0) ce += ec0[(size_t)i0 * hidden + c];
            if (n_c > 1) ce += ec1[(size_t)i1 * hidden + c];
            v = pe + ce;
        }
        out[(size_t)bt * hidden + c] = v;
    }
}

// cond_layer(timbre) of the redecoder's WN (modules/wavenet.py:143-151): timbre [B][1024] -> g [B][2 * 512 * 16], every
// layer's slice of the per-utterance conditioning (a Linear per utterance).
void redecoder_cond(Ctx& c, const float* timbre, int B, float* g) {
    run_conv(c, c.h->red.cond, timbre, g, 1, B, B, ConvOpts(), "red.cond");
}
size_t redecoder_cond_floats(const fac_handle* h, int B) { return (size_t)B * 2 * h->red.hidden * h->red.layers; }

// Redecoder.forward (modules/redecoder.py:35-48) after the cond layer: codes -> embeddings -> WN conditioned on g
// (redecoder_cond) -> conv_out.  codes_p row b at codes_p + b * cp_stride, codes_c rows at codes_c + b * cc_stride + i * T
// (int64, device); returns channels-last z [B][T][1024] in workspace.  frames (a ragged batch): [B] device, each lane's own
// frames, or null.  lane_mode (a pool batch of mixed modes): [B][2] device, each lane's use_p and effective n_c, or null.
float* redecoder_body(Ctx& c, const int64_t* codes_p, int cp_stride, const int64_t* codes_c, int cc_stride, const float* g,
                      int B, int T, int use_p, int use_c, int n_c, const int* frames = nullptr, const int* lane_mode = nullptr) {
    const RedW& r = c.h->red;
    const int Hd = r.hidden;
    float* x = c.alloc<float>((size_t)B * T * Hd);
    float* pin = c.alloc<float>((size_t)B * T * 2 * Hd);
    float* acts = c.alloc<float>((size_t)B * T * Hd);
    float* rs = c.alloc<float>((size_t)B * T * 2 * Hd);
    float* skip = c.alloc<float>((size_t)B * T * Hd);
    float* z = c.alloc<float>((size_t)B * T * LATENT);
    if (!c.dry) {
        embed_sum_kernel<<<B * T, 128, 0, c.st>>>(codes_p, cp_stride, codes_c, cc_stride, c.W(r.emb_p), c.W(r.emb_c[0]),
                                                  c.W(r.emb_c[1]), x, T, Hd, use_p ? 1 : 0, use_c ? n_c : 0, frames,
                                                  lane_mode);
        c.check(cudaGetLastError(), "red.embed");
    }
    if (!c.dry) c.check_nk(cudaMemsetAsync(skip, 0, sizeof(float) * (size_t)B * T * Hd, c.st), "red.zero");
    ConvOpts o;
    o.lane_len = frames;
    for (int i = 0; i < r.layers; ++i) {
        sconv(c, r.wn_in[i], x, pin, B, T, 1, 1, o, "red.in", false);
        if (!c.dry) c.check(launch_wn_gate(pin, acts, (size_t)B * T, Hd, c.st, g + (size_t)i * 2 * Hd, (size_t)T, (size_t)2 * Hd * r.layers), "red.gate");
        sconv(c, r.wn_rs[i], acts, rs, B, T, 1, 1, o, "red.rs", false);
        if (!c.dry) c.check(launch_wn_update(rs, x, skip, (size_t)B * T, Hd, i == r.layers - 1, c.st), "red.upd");
    }
    run_conv(c, r.conv_out, skip, z, B, T, T, ConvOpts(), "red.conv_out");
    return z;
}

// Redecoder.forward (modules/redecoder.py:35-48): codes_p [B][1][T], codes_c [B][ncc][T] int64 (device), timbre [B][1024];
// returns channels-last z [B][T][1024] in workspace.
float* redecoder_forward(Ctx& c, const int64_t* codes_p, const int64_t* codes_c, int ncc, const float* timbre, int B, int T,
                         int use_p, int use_c, int n_c, const int* frames = nullptr) {
    float* g = c.alloc<float>(redecoder_cond_floats(c.h, B));
    redecoder_cond(c, timbre, B, g);
    return redecoder_body(c, codes_p, T, codes_c, ncc * T, g, B, T, use_p, use_c, n_c, frames);
}

// mel [B][Tm][80] from wave [B][T] (Tm = T/300), preprocess modules/quantize.py:239-242
struct MelW { const ConvW* dft; const ConvW* dft_tc; size_t fb; };
// The tensor-core path: mel frames [f_first, f_first + F) of wave [B][T] (reflected at both ends of the T samples) ->
// [B][F][80].  Frames gather + K=1 GEMM on the promoted tensor-core kernel (the mel feeds the prosody VQ: fp32-grade sums).
float* mel_frames_tc(Ctx& c, const MelW& q, const float* wave, int B, int T, int f_first, int F, const int* lane_len = nullptr) {
    float* frames = c.alloc<float>((size_t)B * F * WIN);
    float* spec = c.alloc<float>((size_t)B * F * SPEC_TC_LD);
    float* mel = c.alloc<float>((size_t)B * F * N_MELS);
    if (!c.dry) c.check(launch_stft_frames(wave, frames, B, T, F, HOP, WIN, N_FFT / 2 - (N_FFT - WIN) / 2, c.st, f_first, lane_len), "mel.frames");
    run_conv(c, *q.dft_tc, frames, spec, 1, B * F, B * F, ConvOpts(), "mel.dft");
    if (!c.dry) c.check(launch_mel_from_spec(spec, SPEC_TC_LD, c.W(q.fb), mel, B, F, F, c.st), "mel.fb");
    return mel;
}
MelW quantizer_mel(const fac_handle* h) { return MelW{&h->qw.dft, &h->qw.dft_tc, h->qw.fb}; }
// lane_len (a ragged batch, device [B]): each lane's samples, reflected about their own ends
float* mel_forward(Ctx& c, const float* wave, int B, int T, int Tm, const MelW* mw = nullptr, const int* lane_len = nullptr) {
    const MelW q = mw ? *mw : quantizer_mel(c.h);
    if (c.h->use_tc >= 2 && q.dft_tc->tc) {
        float* mel = mel_frames_tc(c, q, wave, B, T, 0, Tm, lane_len);
        c.tap("mel80", mel, (size_t)B * Tm * N_MELS);
        return mel;
    }
    float* spec = c.alloc<float>((size_t)B * Tm * SPEC_LD);
    float* mel = c.alloc<float>((size_t)B * Tm * N_MELS);
    ConvOpts o;
    o.stride = HOP;
    o.pad_left = N_FFT / 2 - (N_FFT - WIN) / 2;   // 1024 - 424 = 600
    o.pad_right = 600;
    o.reflect = 1;
    o.no_bias = true;
    o.ldy = SPEC_LD;
    o.lane_len = lane_len;
    run_conv(c, *q.dft, wave, spec, B, T, Tm, o, "mel.dft");
    if (!c.dry) c.check(launch_mel_from_spec(spec, SPEC_LD, c.W(q.fb), mel, B, Tm, Tm, c.st), "mel.fb");
    c.tap("mel80", mel, (size_t)B * Tm * N_MELS);
    return mel;
}

// StyleEncoder.forward (modules/style_encoder.py:63-81): mel80 [B][Tm][80] -> timbre [B][1024]
// ln (a ragged batch): lane b is the StyleEncoder of its own ln mel frames -- GLU convs zero-padded at its end, attention
// over its own frames in the variant its own call takes, the mean over its own frames.
void style_encoder(Ctx& c, const float* mel, int B, int Tm, const int* vlen, float* timbre, const Lanes* ln = nullptr) {
    const QuantW& q = c.h->qw;
    float* a = c.alloc<float>((size_t)B * Tm * 512);
    float* x = c.alloc<float>((size_t)B * Tm * 512);
    float* y2 = c.alloc<float>((size_t)B * Tm * 1024);
    float* qb = c.alloc<float>((size_t)B * Tm * 512);
    float* kb = c.alloc<float>((size_t)B * Tm * 512);
    float* vb = c.alloc<float>((size_t)B * Tm * 512);
    float* ob = c.alloc<float>((size_t)B * Tm * 512);
    ConvOpts o;
    o.act = ACT_MISH;
    run_conv(c, q.spec0, mel, a, B, Tm, Tm, o, "se.spec0");
    o.valid_len = vlen;
    run_conv(c, q.spec3, a, x, B, Tm, Tm, o, "se.spec3");
    for (int i = 0; i < 2; ++i) {
        ConvOpts g;
        g.pad_left = 2; g.pad_right = 2; g.reflect = 0;
        g.lane_len = lane_at(ln, kTmRow);
        run_conv(c, q.glu[i], x, y2, B, Tm, Tm, g, "se.glu");
        if (!c.dry) c.check(launch_glu_res(y2, x, B, Tm, 512, i == 1 ? vlen : nullptr, c.st), "se.glu_res");
    }
    ConvOpts p;
    run_conv(c, q.cq, x, qb, B, Tm, Tm, p, "se.q");
    run_conv(c, q.ck, x, kb, B, Tm, Tm, p, "se.k");
    run_conv(c, q.cv, x, vb, B, Tm, Tm, p, "se.v");
    if (!c.dry)
        c.check(launch_attention(qb, kb, vb, ob, B, Tm, 2, 256, vlen, c.st, c.h->attn_stream, lane_at(ln, kTmRow),
                                 ln ? ln->host(kTmRow) : nullptr), "se.attn");
    ConvOpts r;
    r.res = x;
    run_conv(c, q.co, ob, a, B, Tm, Tm, r, "se.o");          // a = x + conv_o(attn)
    run_conv(c, q.fc, a, y2, B, Tm, Tm, ConvOpts(), "se.fc");
    if (!c.dry) c.check(launch_mean_pool(y2, timbre, B, Tm, 1024, vlen, c.st, lane_at(ln, kTmRow)), "se.pool");
}

__global__ void lens_to_frames_kernel(const int64_t* lens, int* out, int B, int hop, int maxf) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < B) {
        long long f = lens[i] / hop;
        out[i] = (int)(f < maxf ? f : maxf);
    }
}

struct QuantOut {
    float* outs_cl; float* zp_cl; float* zc_cl; float* zr_cl; int Tq;
};

// FAquantizer.forward_v2, the part that depends on the waveform only (modules/quantize.py:378-404): timbre (mel ->
// StyleEncoder -> timbre_linear) and the prosody features (mel[:, :20] -> melspec_linear -> WN -> melspec_linear2).  Nothing
// here reads the encoder's latents, so fac_codec_forward runs it on a second stream beside the encoder.
struct QuantFront { float* gb; float* f0; int Tm; };

// gamma | beta = timbre_linear(timbre) (modules/quantize.py:444-445): [B][2048] in workspace.  Run with the promoted
// quantizer-side kernel, so that decoding from codes sees the same gamma / beta as the forward.
float* timbre_gamma_beta(Ctx& c, const float* timbre, int B) {
    const bool was_critical = c.vq_critical;
    c.vq_critical = true;
    float* gb = c.alloc<float>((size_t)B * 2048);
    run_conv(c, c.h->qw.timbre_linear, timbre, gb, 1, B, B, ConvOpts(), "timbre_linear");
    c.tap("gamma_beta", gb, (size_t)B * 2048);
    c.vq_critical = was_critical;
    return gb;
}

// The prosody branch (modules/quantize.py:399-404): mel[:, :20] -> melspec_linear -> WN (8 causal k = 5 layers) ->
// melspec_linear2.  mel [B][Tm][80] -> f0 [B][Tm][1024] in workspace; run with c.vq_critical set.
float* prosody_forward(Ctx& c, const float* mel, int B, int Tm, const int* lane_len = nullptr) {
    const QuantW& q = c.h->qw;
    float* px = c.alloc<float>((size_t)B * Tm * 256);
    float* pin = c.alloc<float>((size_t)B * Tm * 512);
    float* acts = c.alloc<float>((size_t)B * Tm * 256);
    float* rs = c.alloc<float>((size_t)B * Tm * 512);
    float* skip = c.alloc<float>((size_t)B * Tm * 256);
    float* f0 = c.alloc<float>((size_t)B * Tm * 1024);
    ConvW lin = q.mel_lin;
    ConvOpts o;
    o.ldx = N_MELS;
    run_conv(c, lin, mel, px, B, Tm, Tm, o, "melspec_linear");
    if (!c.dry) c.check_nk(cudaMemsetAsync(skip, 0, sizeof(float) * (size_t)B * Tm * 256, c.st), "wn.zero");
    ConvOpts ow;
    ow.lane_len = lane_len;
    for (int i = 0; i < 8; ++i) {
        sconv(c, q.wn_in[i], px, pin, B, Tm, 1, 1, ow, "wn.in");
        if (!c.dry) c.check(launch_wn_gate(pin, acts, (size_t)B * Tm, 256, c.st), "wn.gate");
        sconv(c, q.wn_rs[i], acts, rs, B, Tm, 1, 1, ow, "wn.rs");
        if (!c.dry) c.check(launch_wn_update(rs, px, skip, (size_t)B * Tm, 256, i == 7, c.st), "wn.upd");
    }
    sconv(c, q.mel_lin2, skip, f0, B, Tm, 1, 1, ConvOpts(), "melspec_linear2");
    return f0;
}

QuantFront quantizer_front(Ctx& c, const float* wave, int B, int T, const float* full_waves, int T_full, const int64_t* wave_lens,
                           float* timbre, const Lanes* ln = nullptr) {
    const int Tm = T / HOP;
    const bool was_critical = c.vq_critical;
    c.vq_critical = true;      // quantizer-side layers are tiny: all of them use the promoted kernel
    // --- timbre ---
    float* mel = mel_forward(c, wave, B, T, Tm, nullptr, lane_at(ln, 0));
    float* timbre_ws = c.alloc<float>((size_t)B * 1024);
    if (!timbre) timbre = timbre_ws;
    if (full_waves) {
        int Tmf = T_full / HOP;
        float* melf = mel_forward(c, full_waves, B, T_full, Tmf);
        int* vlen = c.alloc<int>(B);
        if (!c.dry) {
            lens_to_frames_kernel<<<(B + 127) / 128, 128, 0, c.st>>>(wave_lens, vlen, B, HOP, Tmf);
            c.check(cudaGetLastError(), "lens");
        }
        style_encoder(c, melf, B, Tmf, vlen, timbre);
    } else {
        style_encoder(c, mel, B, Tm, nullptr, timbre, ln);
    }
    float* gb = timbre_gamma_beta(c, timbre, B);
    float* f0 = prosody_forward(c, mel, B, Tm, lane_at(ln, kTmRow));
    c.tap("f0_input", f0, (size_t)B * Tm * 1024);
    c.vq_critical = was_critical;
    QuantFront fr;
    fr.gb = gb; fr.f0 = f0; fr.Tm = Tm;
    return fr;
}

// FAquantizer.forward_v2 on channels-last z; returns channels-last outputs in workspace
QuantOut quantizer_forward(Ctx& c, const float* z_cl, const float* wave, int B, int T, int Tz, int n_c,
                           const float* full_waves, int T_full, const int64_t* wave_lens, float* losses2,
                           float* timbre, int64_t* codes_p, int64_t* codes_c, int64_t* codes_r, bool want_parts,
                           const QuantFront* pre = nullptr, const Lanes* ln = nullptr) {
    const QuantW& q = c.h->qw;
    const int Tm = T / HOP;
    const int Tq = Tm < Tz ? Tm : Tz;
    c.vq_critical = true;
    QuantFront fr = pre ? *pre : quantizer_front(c, wave, B, T, full_waves, T_full, wave_lens, timbre, ln);
    float* gb = fr.gb;
    float* f0 = fr.f0;
    // --- fused per-frame VQ + AdaLN ---
    QuantOut out;
    out.Tq = Tq;
    out.outs_cl = c.alloc<float>((size_t)B * Tq * 1024);
    out.zp_cl = want_parts ? c.alloc<float>((size_t)B * Tq * 1024) : nullptr;
    out.zc_cl = want_parts ? c.alloc<float>((size_t)B * Tq * 1024) : nullptr;
    out.zr_cl = want_parts ? c.alloc<float>((size_t)B * Tq * 1024) : nullptr;
    float* sqerr = c.alloc<float>((size_t)6 * B * Tq);
    int64_t* cp = c.alloc<int64_t>((size_t)B * Tq);
    int64_t* cc = c.alloc<int64_t>((size_t)B * 2 * Tq);
    int64_t* cr = c.alloc<int64_t>((size_t)B * 3 * Tq);
    float* loss_ws = c.alloc<float>(2);
    c.vq_critical = false;
    if (c.dry) return out;
    FaqParams fp;
    fp.f0 = f0; fp.z = z_cl;
    for (int i = 0; i < 6; ++i) {
        const VqW& v = q.vq[i];
        fp.vq[i] = VqWeights{c.W(v.w_in), c.W(v.b_in), c.W(v.cb), c.W(v.cbn), c.W(v.cbn2), c.W(v.w_out), c.W(v.b_out)};
    }
    fp.n_c = n_c;
    fp.gamma_beta = gb;
    fp.outs = out.outs_cl; fp.zp = out.zp_cl; fp.zc = out.zc_cl; fp.zr = out.zr_cl;
    fp.codes_p = codes_p ? codes_p : cp;
    fp.codes_c = codes_c ? codes_c : cc;
    fp.codes_r = codes_r ? codes_r : cr;
    fp.sqerr = sqerr;
    fp.B = B; fp.Tq = Tq; fp.Tz = Tz; fp.Tf0 = Tm;
    c.begin("fa_quantize", 2.0 * B * Tq * (3 + n_c + 1) * (8.0 * 1024 * 3), 4.0 * (double)B * Tq * 1024 * (3 + (want_parts ? 3 : 0)));
    c.check(launch_fa_quantize(fp, c.st), "fa_quantize");
    c.end();
    c.check(launch_vq_loss_reduce(sqerr, 6, B, Tq, losses2 ? losses2 : loss_ws, c.st), "vq_loss");
    return out;
}

// FAquantizer from codes (the composition of ResidualVectorQuantize.from_codes, dac/nn/quantize.py:200-220, per RVQ and
// the AdaLN of modules/quantize.py:444-449): codes_p [B][1][T], codes_c [B][n_c][T], codes_r [B][n_r][T] int64 (device),
// timbre [B][1024] -> channels-last outs [B][T][1024] in workspace; the parts too when want_parts.
QuantOut dequantize_forward(Ctx& c, const int64_t* codes_p, const int64_t* codes_c, int n_c, const int64_t* codes_r, int n_r,
                            const float* timbre, int B, int T, bool want_parts) {
    const QuantW& q = c.h->qw;
    float* gb = timbre_gamma_beta(c, timbre, B);
    QuantOut out;
    out.Tq = T;
    out.outs_cl = c.alloc<float>((size_t)B * T * 1024);
    out.zp_cl = want_parts ? c.alloc<float>((size_t)B * T * 1024) : nullptr;
    out.zc_cl = want_parts ? c.alloc<float>((size_t)B * T * 1024) : nullptr;
    out.zr_cl = want_parts ? c.alloc<float>((size_t)B * T * 1024) : nullptr;
    if (c.dry) return out;
    DeqParams dp;
    dp.codes_p = codes_p; dp.codes_c = codes_c; dp.codes_r = codes_r;
    dp.n_c = n_c; dp.n_r = n_r;
    for (int i = 0; i < 6; ++i) {
        const VqW& v = q.vq[i];
        dp.vq[i] = VqWeights{c.W(v.w_in), c.W(v.b_in), c.W(v.cb), c.W(v.cbn), c.W(v.cbn2), c.W(v.w_out), c.W(v.b_out)};
    }
    dp.gamma_beta = gb;
    dp.outs = out.outs_cl; dp.zp = out.zp_cl; dp.zc = out.zc_cl; dp.zr = out.zr_cl;
    dp.B = B; dp.T = T;
    // codes in + outs out; the 6 x 32 KB of out_proj weights and the gathered codebook rows stay cache-resident
    const double frames = (double)B * T, ncodes = 1 + n_c + n_r;
    c.begin("dequantize", 2.0 * frames * ncodes * 8.0 * 1024, frames * (8.0 * ncodes + 4.0 * 1024 * (want_parts ? 4 : 1)));
    c.check(launch_dequantize(dp, c.st), "dequantize");
    c.end();
    return out;
}

// dequantize_forward for a ragged batch (no parts): lane b reads frames [0, frames[b]) of its codes (rows T apart; host
// frames) and its frames past them are 0.  Each frame is dequantize_kernel's, bit for bit, in launches of <= 32 lanes.
QuantOut dequantize_lanes_forward(Ctx& c, const int64_t* codes_p, const int64_t* codes_c, int n_c, const int64_t* codes_r,
                                  int n_r, const float* timbre, int B, int T, const int* frames) {
    const QuantW& q = c.h->qw;
    float* gb = timbre_gamma_beta(c, timbre, B);
    QuantOut out = {};
    out.Tq = T;
    out.outs_cl = c.alloc<float>((size_t)B * T * 1024);
    if (c.dry) return out;
    DeqLaneParams dp;
    for (int i = 0; i < 6; ++i) {
        const VqW& v = q.vq[i];
        dp.vq[i] = VqWeights{c.W(v.w_in), c.W(v.b_in), c.W(v.cb), c.W(v.cbn), c.W(v.cbn2), c.W(v.w_out), c.W(v.b_out)};
    }
    dp.Fmax = T; dp.ld = T;
    for (int b0 = 0; b0 < B; b0 += kLaneMax) {
        dp.n = std::min(B - b0, kLaneMax);
        double codes = 0;
        for (int j = 0; j < dp.n; ++j) {
            const size_t b = (size_t)(b0 + j);
            dp.codes_p[j] = codes_p + b * T; dp.codes_c[j] = codes_c + b * n_c * T;
            dp.codes_r[j] = n_r ? codes_r + b * n_r * T : nullptr;
            dp.n_c[j] = n_c; dp.n_r[j] = n_r; dp.F[j] = frames[b];
            dp.gamma_beta[j] = gb + b * 2048;
            codes += (double)frames[b] * (1 + n_c + n_r);
        }
        dp.outs = out.outs_cl + (size_t)b0 * T * 1024;
        c.begin("dequantize", 2.0 * codes * 8.0 * 1024, 8.0 * codes + 4.0 * 1024 * dp.n * T);
        c.check(launch_dequantize_lanes(dp, c.st), "dequantize_lanes");
        c.end();
    }
    return out;
}

// Runs the waveform-only half of the quantizer on the handle's side stream, forked after whatever the main stream has
// queued so far (the input copy) and joined by the caller with join_front() before fa_quantize.
bool fork_front(Ctx& c, QuantFront& fr, const float* wave, int B, int T, float* timbre, const Lanes* ln = nullptr) {
    fac_handle* h = c.h;
    if (!h->overlap_front || h->profiling) { return false; }
    if (c.dry) { fr = quantizer_front(c, wave, B, T, nullptr, 0, nullptr, timbre, ln); return true; }
    if (!h->side) {
        if (cudaStreamCreateWithFlags(&h->side, cudaStreamNonBlocking) != cudaSuccess ||
            cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming) != cudaSuccess) {
            cudaGetLastError();
            h->overlap_front = 0;
            return false;
        }
    }
    cudaStream_t main_st = c.st;
    c.check_nk(cudaEventRecord(h->ev_fork, main_st), "front.fork");
    c.check_nk(cudaStreamWaitEvent(h->side, h->ev_fork, 0), "front.fork_wait");
    c.st = h->side;
    fr = quantizer_front(c, wave, B, T, nullptr, 0, nullptr, timbre, ln);
    c.check_nk(cudaEventRecord(h->ev_join, h->side), "front.join");
    c.st = main_st;
    return true;
}
void join_front(Ctx& c) {
    if (!c.dry) c.check_nk(cudaStreamWaitEvent(c.st, c.h->ev_join, 0), "front.join_wait");
}

int ensure_ws(fac_handle* h, size_t bytes) {
    if (bytes <= h->ws_bytes) return FAC_OK;
    if (h->ws) { cudaDeviceSynchronize(); h->ws.reset(); h->ws_bytes = 0; }
    size_t want = bytes + (bytes >> 4) + (1 << 20);
    char* p = nullptr;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) {
        h->err = std::string("workspace cudaMalloc failed: ") + cudaGetErrorString(e);
        cudaGetLastError();
        return FAC_ERR_CUDA;
    }
    h->ws.reset(p);
    h->ws_bytes = want;
    return FAC_OK;
}

// Copies `host` to a new device buffer that replaces `dst` (`slack` more elements allocated past the end, left unset).  A
// previous buffer is dropped only once the device is idle: kernels in flight may still read it.  On failure dst is empty.
template <typename T>
int upload(fac_handle* h, const std::vector<T>& host, DevBuf<T>& dst, const char* who, size_t slack = 0) {
    cudaError_t e = cudaSetDevice(h->device);
    if (e == cudaSuccess && dst) { cudaDeviceSynchronize(); dst.reset(); }
    T* p = nullptr;
    if (e == cudaSuccess) e = cudaMalloc(&p, (host.size() + slack) * sizeof(T));
    if (e == cudaSuccess) dst.reset(p);
    if (e == cudaSuccess) e = cudaMemcpy(p, host.data(), host.size() * sizeof(T), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        dst.reset();
        h->err = std::string(who) + ": " + cudaGetErrorString(e);
        cudaGetLastError();
        return FAC_ERR_CUDA;
    }
    return FAC_OK;
}

// A weight arena: the packed floats and 64 floats of slack.
int upload_weights(fac_handle* h, const Packer& P, DevBuf<float>& dst, const char* who) { return upload(h, P.pack, dst, who, 64); }

int finish(fac_handle* h, Ctx& c) {
    if (c.cerr != cudaSuccess) {
        h->err = std::string("CUDA error at ") + c.where + ": " + cudaGetErrorString(c.cerr);
        return FAC_ERR_CUDA;
    }
    return FAC_OK;
}

// Stages one C-ABI tensor (HOST data, 0 <= ndim <= 4 non-negative dimensions) as ts[key].
int stage_tensor(TensorMap& ts, const char* key, const float* data, const int64_t* shape, int ndim) {
    if (!key || !data || ndim < 0 || ndim > 4) return FAC_ERR_INVALID;
    HostTensor t;
    for (int i = 0; i < ndim; ++i) { if (shape[i] < 0) return FAC_ERR_INVALID; t.shape.push_back(shape[i]); }
    t.data.assign(data, data + t.numel());
    ts[key] = std::move(t);
    return FAC_OK;
}

// FNV-1a 64 of n bytes, continuing from h.
uint64_t fnv1a(const void* p, size_t n, uint64_t h = 14695981039346656037ull) {
    const unsigned char* b = static_cast<const unsigned char*>(p);
    for (size_t i = 0; i < n; ++i) { h ^= b[i]; h *= 1099511628211ull; }
    return h;
}

// A module's weight fingerprint: every key, shape and float of its host tensors in key order, the floats as raw words over
// four interleaved FNV-style lanes (a byte-wise hash of ~100 M floats would add seconds to fac_finalize).  Not a secure hash:
// it tells apart weights, not adversaries.
uint64_t weights_fingerprint(const TensorMap& m) {
    uint64_t h = fnv1a("facodec_b200 weights", 20);
    for (const auto& kv : m) {
        h = fnv1a(kv.first.c_str(), kv.first.size() + 1, h);
        h = fnv1a(kv.second.shape.data(), kv.second.shape.size() * sizeof(int64_t), h);
        uint64_t l[4] = {h, h + 1, h + 2, h + 3};
        const float* f = kv.second.data.data();
        const size_t n = kv.second.data.size();
        size_t i = 0;
        for (; i + 4 <= n; i += 4)
            for (int k = 0; k < 4; ++k) {
                uint32_t w;
                std::memcpy(&w, f + i + k, 4);
                l[k] = (l[k] ^ w) * 1099511628211ull;
            }
        for (; i < n; ++i) { uint32_t w; std::memcpy(&w, f + i, 4); l[0] = (l[0] ^ w) * 1099511628211ull; }
        h = fnv1a(l, sizeof l, h);
    }
    return h;
}

// run `body` twice: size pass, then for real, reading the weights of arena `weights`
template <typename F>
int two_pass(fac_handle* h, cudaStream_t st, const float* weights, F body) {
    cudaError_t e = cudaSetDevice(h->device);
    if (e != cudaSuccess) { h->err = cudaGetErrorString(e); return FAC_ERR_CUDA; }
    Ctx dry{h, st, true, weights};
    body(dry);
    int rc = ensure_ws(h, dry.off);
    if (rc != FAC_OK) return rc;
    h->launches = 0;
    Ctx c{h, st, false, weights};
    body(c);
    return finish(h, c);
}
// ... with the codec's own weights
template <typename F>
int two_pass(fac_handle* h, cudaStream_t st, F body) { return two_pass(h, st, h->warena.get(), body); }

}  // namespace

// ==========================================================================================
// C-ABI
// ==========================================================================================
extern "C" {

int fac_abi_version(void) { return 2; }

int fac_create(fac_handle** out, int device) {
    if (!out) return FAC_ERR_INVALID;
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || device < 0 || device >= n) { cudaGetLastError(); return FAC_ERR_CUDA; }
    fac_handle* h = new fac_handle();
    h->device = device;
    *out = h;
    return FAC_OK;
}

int fac_destroy(fac_handle* h) {
    if (!h) return FAC_OK;
    cudaSetDevice(h->device);
    cudaDeviceSynchronize();
    if (h->side) cudaStreamDestroy(h->side);
    if (h->ev_fork) cudaEventDestroy(h->ev_fork);
    if (h->ev_join) cudaEventDestroy(h->ev_join);
    fac::rs_host_free(h->rs);
    delete h;   // and with it every arena, the workspace, the weight sets' and the streams' and pools' device state
    return FAC_OK;
}

const char* fac_last_error(const fac_handle* h) { return h ? h->err.c_str() : "null handle"; }

int fac_load_tensor(fac_handle* h, int module, const char* key, const float* data_host, const int64_t* shape, int ndim) {
    if (!h || module < 0 || module >= FAC_NUM_MODULES) return FAC_ERR_INVALID;
    const int rc = stage_tensor(h->host[module], key, data_host, shape, ndim);
    if (rc == FAC_OK) { h->have[module] = true; h->finalized = false; }
    return rc;
}

int fac_finalize(fac_handle* h) {
    if (!h) return FAC_ERR_INVALID;
    Packer P;
    P.pack.reserve(160u << 20);
    try {
        if (h->have[FAC_ENCODER]) pack_encoder(P, h->host[FAC_ENCODER], h->enc);
        if (h->have[FAC_QUANTIZER]) pack_quantizer(P, h->host[FAC_QUANTIZER], h->qw);
        if (h->have[FAC_DECODER]) pack_decoder(P, h->host[FAC_DECODER], h->dec, true, true);
        if (h->have[FAC_REDECODER]) pack_redecoder(P, h->host[FAC_REDECODER], h->red);
        if (h->have[FAC_REDECODER_DECODER]) pack_decoder(P, h->host[FAC_REDECODER_DECODER], h->dec2, false, false);
    } catch (const PackError& e) {
        h->err = e.msg;
        return FAC_ERR_STATE;
    }
    const int rc = upload_weights(h, P, h->warena, "weight upload");
    if (rc != FAC_OK) return rc;
    for (int m = 0; m < FAC_NUM_MODULES; ++m) h->fp[m] = h->have[m] ? weights_fingerprint(h->host[m]) : 0;
    for (int m = 0; m < FAC_NUM_MODULES; ++m) h->host[m].clear();
    h->finalized = true;
    return FAC_OK;
}

int fac_encode_frames(int T) {
    const int rates[4] = {2, 5, 5, 6};
    int t = T;
    for (int i = 0; i < 4; ++i) t = conv_out_len(t, 2 * rates[i], rates[i]);
    return t;
}

static int check_ready(fac_handle* h, std::initializer_list<int> modules) {
    if (!h) return FAC_ERR_INVALID;
    for (int m : modules)
        if (!h->finalized || !h->have[m]) { h->err = "module weights not loaded/finalized"; return FAC_ERR_STATE; }
    return FAC_OK;
}

int fac_encode(fac_handle* h, const float* x, int B, int T, float* z, void* stream) {
    int rc = check_ready(h, {FAC_ENCODER});
    if (rc) return rc;
    if (!x || !z || B <= 0 || T <= 0) { h->err = "fac_encode: bad arguments"; return FAC_ERR_INVALID; }
    return two_pass(h, (cudaStream_t)stream, [&](Ctx& c) { encoder_forward(c, x, B, T, z, true); });
}

int fac_decode(fac_handle* h, const float* z, int B, int Tf, float* y, void* stream) {
    int rc = check_ready(h, {FAC_DECODER});
    if (rc) return rc;
    if (!z || !y || B <= 0 || Tf <= 0) { h->err = "fac_decode: bad arguments"; return FAC_ERR_INVALID; }
    return two_pass(h, (cudaStream_t)stream, [&](Ctx& c) {
        float* zcl = c.alloc<float>((size_t)B * Tf * LATENT);
        if (!c.dry) c.check(launch_transpose(z, zcl, B, LATENT, Tf, c.st), "dec.z_transpose");
        decoder_forward(c, h->dec, zcl, B, Tf, y);
    });
}

int fac_quantize(fac_handle* h, const float* z, const float* wave, int B, int T, int Tz, int n_c,
                 const float* full_waves, int T_full, const int64_t* wave_lens, float* outs, float* zp, float* zc,
                 float* zr, float* losses2, float* timbre, int64_t* codes_p, int64_t* codes_c, int64_t* codes_r,
                 void* stream) {
    int rc = check_ready(h, {FAC_QUANTIZER});
    if (rc) return rc;
    if (!z || !wave || !outs || B <= 0 || Tz <= 0 || n_c < 1 || n_c > 2) { h->err = "fac_quantize: bad arguments"; return FAC_ERR_INVALID; }
    if (T <= N_FFT / 2 || (full_waves && (T_full <= N_FFT / 2 || !wave_lens))) {
        h->err = "fac_quantize: wave shorter than the STFT reflect padding (1024), as torch.stft";
        return FAC_ERR_INVALID;
    }
    return two_pass(h, (cudaStream_t)stream, [&](Ctx& c) {
        float* zcl = c.alloc<float>((size_t)B * Tz * LATENT);
        if (!c.dry) c.check(launch_transpose(z, zcl, B, LATENT, Tz, c.st), "q.z_transpose");
        QuantOut o = quantizer_forward(c, zcl, wave, B, T, Tz, n_c, full_waves, T_full, wave_lens, losses2, timbre,
                                       codes_p, codes_c, codes_r, zp || zc || zr);
        if (c.dry) return;
        c.check(launch_transpose(o.outs_cl, outs, B, o.Tq, LATENT, c.st), "q.outs_T");
        if (zp) c.check(launch_transpose(o.zp_cl, zp, B, o.Tq, LATENT, c.st), "q.zp_T");
        if (zc) c.check(launch_transpose(o.zc_cl, zc, B, o.Tq, LATENT, c.st), "q.zc_T");
        if (zr) c.check(launch_transpose(o.zr_cl, zr, B, o.Tq, LATENT, c.st), "q.zr_T");
    });
}

}  // extern "C"

namespace {
// The compress half of reconstruct.py:56-61: encoder -> quantizer(n_c), with the waveform-only quantizer front forked
// beside the encoder.  Returns the channels-last AdaLN output the decoder reads.
// ln: a ragged batch (null: every lane has T samples).
QuantOut codec_encode(Ctx& c, const float* x, int B, int T, int n_c, int64_t* codes_p, int64_t* codes_c, int64_t* codes_r,
                      float* timbre, const Lanes* ln = nullptr) {
    int Tz = fac_encode_frames(T);
    float* zcl = c.alloc<float>((size_t)B * Tz * LATENT);
    float* timbre_buf = timbre ? timbre : c.alloc<float>((size_t)B * 1024);
    QuantFront fr;
    const bool forked = fork_front(c, fr, x, B, T, timbre_buf, ln);
    encoder_forward(c, x, B, T, zcl, false, ln);
    if (forked) join_front(c);
    return quantizer_forward(c, zcl, x, B, T, Tz, n_c, nullptr, 0, nullptr, nullptr, timbre_buf, codes_p, codes_c, codes_r,
                             false, forked ? &fr : nullptr, ln);
}

// The timbre of codec_encode alone: the launches quantizer_front runs for it (mel80 -> StyleEncoder, promoted class, the
// same lanes), and no encoder, prosody or VQ launch.  timbre [B][1024].
void codec_timbre(Ctx& c, const float* x, int B, int T, float* timbre, const Lanes* ln = nullptr) {
    const bool was_critical = c.vq_critical;
    c.vq_critical = true;
    const int Tm = T / HOP;
    const float* mel = mel_forward(c, x, B, T, Tm, nullptr, lane_at(ln, 0));
    style_encoder(c, mel, B, Tm, nullptr, timbre, ln);
    c.vq_critical = was_critical;
}

// The lanes of a ragged encode of B lanes of lens[b] samples (kLaneRows rows, see Lanes), uploaded by the caller's Ctx.
std::vector<int> encode_lane_rows(const DecW& d, const int* lens, int B) {
    static const int rates[4] = {2, 5, 5, 6};
    std::vector<int> rows((size_t)kLaneRows * B);
    std::vector<int> tq(B);
    for (int b = 0; b < B; ++b) {
        rows[b] = lens[b];
        for (int i = 0; i < 4; ++i) rows[(size_t)(i + 1) * B + b] = conv_out_len(rows[(size_t)i * B + b], 2 * rates[i], rates[i]);
        rows[(size_t)kTmRow * B + b] = lens[b] / HOP;
        tq[b] = std::min(lens[b] / HOP, rows[(size_t)4 * B + b]);
        rows[(size_t)kTqRow * B + b] = tq[b];
    }
    const std::vector<int> dec = lane_rows(d, tq.data(), B);
    std::copy(dec.begin(), dec.end(), rows.begin() + (size_t)kDecRow * B);
    return rows;
}
Lanes upload_lanes(Ctx& c, const std::vector<int>& rows, int B) {
    Lanes l;
    l.h = rows; l.B = B;
    l.d = upload_ints(c, rows);
    return l;
}

// codes [B][rows][T]: codes t >= frames[b] of lane b set to -1 (past a ragged lane's end)
__global__ void code_tails_kernel(int64_t* __restrict__ codes, const int* __restrict__ frames, int rows, int T) {
    const int b = blockIdx.y;
    int64_t* cb = codes + (size_t)b * rows * T;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < rows * T; i += gridDim.x * blockDim.x)
        if (i % T >= frames[b]) cb[i] = -1;
}
void code_tails(Ctx& c, int64_t* codes, const int* frames, int B, int rows, int T) {
    if (c.dry || !frames || !codes) return;
    code_tails_kernel<<<dim3(std::min((rows * T + 255) / 256, 64), B), 256, 0, c.st>>>(codes, frames, rows, T);
    c.check(cudaGetLastError(), "code_tails");
}

// Per-lane counts of a ragged call (host, B entries): each must lie in [lo, hi].  A batch whose every lane has hi is the
// call without counts, launch for launch, so `counts` is cleared for it.
int lane_counts(fac_handle* h, const int*& counts, int B, int lo, int hi, const char* who) {
    if (!counts) return FAC_OK;
    bool full = true;
    for (int b = 0; b < B; ++b) {
        if (counts[b] < lo || counts[b] > hi) {
            h->err = std::string(who) + ": lane " + std::to_string(b) + " has " + std::to_string(counts[b]) + ", outside [" +
                     std::to_string(lo) + ", " + std::to_string(hi) + "]";
            return FAC_ERR_INVALID;
        }
        full = full && counts[b] == hi;
    }
    if (full) counts = nullptr;
    return FAC_OK;
}

// Arguments of the decode-from-codes entry points: 1 prosody row, 1..2 content rows, 0..3 residual rows (codes_r unread
// when there are none), timbre [B][1024].
bool bad_codes_args(const int64_t* codes_p, const int64_t* codes_c, int n_c_rows, const int64_t* codes_r, int n_r_rows,
                    const float* timbre, int B, int T) {
    return !codes_p || !codes_c || !timbre || n_c_rows < 1 || n_c_rows > 2 || n_r_rows < 0 || n_r_rows > 3 ||
           (n_r_rows > 0 && !codes_r) || B <= 0 || T <= 0;
}
}  // namespace

extern "C" {

int fac_codec_forward_lens(fac_handle* h, const float* x, int B, int T, const int* lengths, int n_c, float* y, int64_t* codes_p,
                           int64_t* codes_c, int64_t* codes_r, float* timbre, void* stream) {
    if (int rc = check_ready(h, {FAC_ENCODER, FAC_QUANTIZER, FAC_DECODER})) return rc;
    if (!x || !y || B <= 0 || T <= N_FFT / 2 || n_c < 1 || n_c > 2) { h->err = "fac_codec_forward: bad arguments"; return FAC_ERR_INVALID; }
    if (int rc = lane_counts(h, lengths, B, N_FFT / 2 + 1, T, "fac_codec_forward_lens: lengths")) return rc;
    const std::vector<int> rows = lengths ? encode_lane_rows(h->dec, lengths, B) : std::vector<int>();
    return two_pass(h, (cudaStream_t)stream, [&](Ctx& c) {
        const Lanes ln = upload_lanes(c, rows, B);
        const Lanes* lp = lengths ? &ln : nullptr;
        QuantOut o = codec_encode(c, x, B, T, n_c, codes_p, codes_c, codes_r, timbre, lp);
        decoder_forward(c, h->dec, o.outs_cl, B, o.Tq, y, lane_at(lp, kDecRow));
        zero_tails(c, y, lane_at(lp, kDecRow + 4), B, o.Tq * HOP);
        code_tails(c, codes_p, lane_at(lp, kTqRow), B, 1, o.Tq);
        code_tails(c, codes_c, lane_at(lp, kTqRow), B, n_c, o.Tq);
        code_tails(c, codes_r, lane_at(lp, kTqRow), B, 3, o.Tq);
    });
}

int fac_codec_forward(fac_handle* h, const float* x, int B, int T, int n_c, float* y, int64_t* codes_p,
                      int64_t* codes_c, int64_t* codes_r, float* timbre, void* stream) {
    return fac_codec_forward_lens(h, x, B, T, nullptr, n_c, y, codes_p, codes_c, codes_r, timbre, stream);
}

int fac_codec_encode_lens(fac_handle* h, const float* x, int B, int T, const int* lengths, int n_c, int64_t* codes_p,
                          int64_t* codes_c, int64_t* codes_r, float* timbre, void* stream) {
    if (int rc = check_ready(h, {FAC_ENCODER, FAC_QUANTIZER})) return rc;
    if (!x || !codes_p || !codes_c || !codes_r || B <= 0 || T <= N_FFT / 2 || n_c < 1 || n_c > 2) {
        h->err = "fac_codec_encode: bad arguments";
        return FAC_ERR_INVALID;
    }
    if (int rc = lane_counts(h, lengths, B, N_FFT / 2 + 1, T, "fac_codec_encode_lens: lengths")) return rc;
    const std::vector<int> rows = lengths ? encode_lane_rows(h->dec, lengths, B) : std::vector<int>();
    return two_pass(h, (cudaStream_t)stream, [&](Ctx& c) {
        const Lanes ln = upload_lanes(c, rows, B);
        const Lanes* lp = lengths ? &ln : nullptr;
        QuantOut o = codec_encode(c, x, B, T, n_c, codes_p, codes_c, codes_r, timbre, lp);
        code_tails(c, codes_p, lane_at(lp, kTqRow), B, 1, o.Tq);
        code_tails(c, codes_c, lane_at(lp, kTqRow), B, n_c, o.Tq);
        code_tails(c, codes_r, lane_at(lp, kTqRow), B, 3, o.Tq);
    });
}

int fac_codec_encode(fac_handle* h, const float* x, int B, int T, int n_c, int64_t* codes_p, int64_t* codes_c,
                     int64_t* codes_r, float* timbre, void* stream) {
    return fac_codec_encode_lens(h, x, B, T, nullptr, n_c, codes_p, codes_c, codes_r, timbre, stream);
}

int fac_codec_timbre_lens(fac_handle* h, const float* x, int B, int T, const int* lengths, float* timbre, void* stream) {
    if (int rc = check_ready(h, {FAC_QUANTIZER})) return rc;
    if (!x || !timbre || B <= 0 || T <= N_FFT / 2) { h->err = "fac_codec_timbre: bad arguments"; return FAC_ERR_INVALID; }
    if (int rc = lane_counts(h, lengths, B, N_FFT / 2 + 1, T, "fac_codec_timbre_lens: lengths")) return rc;
    const std::vector<int> rows = lengths ? encode_lane_rows(h->dec, lengths, B) : std::vector<int>();
    return two_pass(h, (cudaStream_t)stream, [&](Ctx& c) {
        const Lanes ln = upload_lanes(c, rows, B);
        codec_timbre(c, x, B, T, timbre, lengths ? &ln : nullptr);
    });
}

int fac_dequantize(fac_handle* h, const int64_t* codes_p, const int64_t* codes_c, int n_c_rows, const int64_t* codes_r,
                   int n_r_rows, const float* timbre, int B, int T, float* outs, float* zp, float* zc, float* zr, void* stream) {
    int rc = check_ready(h, {FAC_QUANTIZER});
    if (rc) return rc;
    if (!outs || bad_codes_args(codes_p, codes_c, n_c_rows, codes_r, n_r_rows, timbre, B, T)) {
        h->err = "fac_dequantize: bad arguments (1 <= content rows <= 2, 0 <= residual rows <= 3)";
        return FAC_ERR_INVALID;
    }
    return two_pass(h, (cudaStream_t)stream, [&](Ctx& c) {
        QuantOut o = dequantize_forward(c, codes_p, codes_c, n_c_rows, codes_r, n_r_rows, timbre, B, T, zp || zc || zr);
        if (c.dry) return;
        c.check(launch_transpose(o.outs_cl, outs, B, T, LATENT, c.st), "deq.outs_T");
        if (zp) c.check(launch_transpose(o.zp_cl, zp, B, T, LATENT, c.st), "deq.zp_T");
        if (zc) c.check(launch_transpose(o.zc_cl, zc, B, T, LATENT, c.st), "deq.zc_T");
        if (zr) c.check(launch_transpose(o.zr_cl, zr, B, T, LATENT, c.st), "deq.zr_T");
    });
}

int fac_codes_decode_lens(fac_handle* h, const int64_t* codes_p, const int64_t* codes_c, int n_c_rows, const int64_t* codes_r,
                          int n_r_rows, const float* timbre, int B, int T, const int* frames, float* y, void* stream) {
    int rc = check_ready(h, {FAC_QUANTIZER, FAC_DECODER});
    if (rc) return rc;
    if (!y || bad_codes_args(codes_p, codes_c, n_c_rows, codes_r, n_r_rows, timbre, B, T)) {
        h->err = "fac_codes_decode: bad arguments (1 <= content rows <= 2, 0 <= residual rows <= 3)";
        return FAC_ERR_INVALID;
    }
    if ((rc = lane_counts(h, frames, B, 1, T, "fac_codes_decode_lens: frames"))) return rc;
    const std::vector<int> rows = frames ? lane_rows(h->dec, frames, B) : std::vector<int>();
    return two_pass(h, (cudaStream_t)stream, [&](Ctx& c) {
        const int* lens = upload_ints(c, rows);
        QuantOut o = frames ? dequantize_lanes_forward(c, codes_p, codes_c, n_c_rows, codes_r, n_r_rows, timbre, B, T, frames)
                            : dequantize_forward(c, codes_p, codes_c, n_c_rows, codes_r, n_r_rows, timbre, B, T, false);
        decoder_forward(c, h->dec, o.outs_cl, B, T, y, lens);
        zero_tails(c, y, lens ? lens + (size_t)4 * B : nullptr, B, T * HOP);
    });
}

int fac_codes_decode(fac_handle* h, const int64_t* codes_p, const int64_t* codes_c, int n_c_rows, const int64_t* codes_r,
                     int n_r_rows, const float* timbre, int B, int T, float* y, void* stream) {
    return fac_codes_decode_lens(h, codes_p, codes_c, n_c_rows, codes_r, n_r_rows, timbre, B, T, nullptr, y, stream);
}

int fac_codec_forward_host(fac_handle* h, const float* x_host, int B, int T, int n_c, float* y_host,
                           int64_t* codes_p_host, int64_t* codes_c_host, int64_t* codes_r_host, void* stream) {
    if (int rc = check_ready(h, {FAC_ENCODER, FAC_QUANTIZER, FAC_DECODER})) return rc;
    if (!x_host || !y_host || B <= 0 || T <= N_FFT / 2 || n_c < 1 || n_c > 2) { h->err = "fac_codec_forward_host: bad arguments"; return FAC_ERR_INVALID; }
    cudaStream_t st = (cudaStream_t)stream;
    int Tq = 0;
    int rc = two_pass(h, st, [&](Ctx& c) {
        int Tz = fac_encode_frames(T);
        int Tm = T / HOP;
        Tq = Tm < Tz ? Tm : Tz;
        float* xd = c.alloc<float>((size_t)B * T);
        float* yd = c.alloc<float>((size_t)B * Tq * HOP);
        int64_t* cp = c.alloc<int64_t>((size_t)B * Tq);
        int64_t* cc = c.alloc<int64_t>((size_t)B * 2 * Tq);
        int64_t* cr = c.alloc<int64_t>((size_t)B * 3 * Tq);
        float* zcl = c.alloc<float>((size_t)B * Tz * LATENT);
        if (!c.dry) c.check_nk(cudaMemcpyAsync(xd, x_host, sizeof(float) * (size_t)B * T, cudaMemcpyHostToDevice, c.st), "h2d");
        float* timbre_buf = c.alloc<float>((size_t)B * 1024);
        QuantFront fr;
        const bool forked = fork_front(c, fr, xd, B, T, timbre_buf);
        encoder_forward(c, xd, B, T, zcl, false);
        if (forked) join_front(c);
        QuantOut o = quantizer_forward(c, zcl, xd, B, T, Tz, n_c, nullptr, 0, nullptr, nullptr, timbre_buf, cp, cc, cr, false,
                                       forked ? &fr : nullptr);
        decoder_forward(c, h->dec, o.outs_cl, B, o.Tq, yd);
        if (c.dry) return;
        c.check_nk(cudaMemcpyAsync(y_host, yd, sizeof(float) * (size_t)B * Tq * HOP, cudaMemcpyDeviceToHost, c.st), "d2h.y");
        if (codes_p_host) c.check_nk(cudaMemcpyAsync(codes_p_host, cp, sizeof(int64_t) * (size_t)B * Tq, cudaMemcpyDeviceToHost, c.st), "d2h.cp");
        if (codes_c_host) c.check_nk(cudaMemcpyAsync(codes_c_host, cc, sizeof(int64_t) * (size_t)B * n_c * Tq, cudaMemcpyDeviceToHost, c.st), "d2h.cc");
        if (codes_r_host) c.check_nk(cudaMemcpyAsync(codes_r_host, cr, sizeof(int64_t) * (size_t)B * 3 * Tq, cudaMemcpyDeviceToHost, c.st), "d2h.cr");
    });
    if (rc) return rc;
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { h->err = std::string("stream sync: ") + cudaGetErrorString(e); return FAC_ERR_CUDA; }
    return FAC_OK;
}

int fac_redecode(fac_handle* h, const int64_t* codes_p, const int64_t* codes_c, int n_c_rows, const float* timbre, int B, int T,
                 int use_p_code, int use_c_code, int n_c, float* z, void* stream) {
    int rc = check_ready(h, {FAC_REDECODER});
    if (rc) return rc;
    if (!codes_p || !codes_c || !timbre || !z || B <= 0 || T <= 0 || n_c < 0 || n_c > 2 || n_c > n_c_rows) {
        h->err = "fac_redecode: bad arguments (n_c <= rows of codes_c <= 2)";
        return FAC_ERR_INVALID;
    }
    return two_pass(h, (cudaStream_t)stream, [&](Ctx& c) {
        float* zcl = redecoder_forward(c, codes_p, codes_c, n_c_rows, timbre, B, T, use_p_code, use_c_code, n_c);
        if (!c.dry) c.check(launch_transpose(zcl, z, B, T, LATENT, c.st), "red.z_T");
    });
}

int fac_redecoder_decode(fac_handle* h, const float* z, int B, int Tf, float* y, void* stream) {
    int rc = check_ready(h, {FAC_REDECODER_DECODER});
    if (rc) return rc;
    if (!z || !y || B <= 0 || Tf <= 0) { h->err = "fac_redecoder_decode: bad arguments"; return FAC_ERR_INVALID; }
    return two_pass(h, (cudaStream_t)stream, [&](Ctx& c) {
        float* zcl = c.alloc<float>((size_t)B * Tf * LATENT);
        if (!c.dry) c.check(launch_transpose(z, zcl, B, LATENT, Tf, c.st), "red.dec.z_transpose");
        decoder_forward(c, h->dec2, zcl, B, Tf, y);
    });
}

int fac_voice_convert_lens(fac_handle* h, const int64_t* codes_p, const int64_t* codes_c, int n_c_rows, const float* timbre,
                           int B, int T, int use_p_code, int use_c_code, int n_c, const int* frames, float* y, void* stream) {
    int rc = check_ready(h, {FAC_REDECODER, FAC_REDECODER_DECODER});
    if (rc) return rc;
    if (!codes_p || !codes_c || !timbre || !y || B <= 0 || T <= 0 || n_c < 0 || n_c > 2 || n_c > n_c_rows) {
        h->err = "fac_voice_convert: bad arguments";
        return FAC_ERR_INVALID;
    }
    if ((rc = lane_counts(h, frames, B, 1, T, "fac_voice_convert_lens: frames"))) return rc;
    const std::vector<int> rows = frames ? lane_rows(h->dec2, frames, B) : std::vector<int>();
    return two_pass(h, (cudaStream_t)stream, [&](Ctx& c) {
        const int* lens = upload_ints(c, rows);
        float* zcl = redecoder_forward(c, codes_p, codes_c, n_c_rows, timbre, B, T, use_p_code, use_c_code, n_c, lens);
        decoder_forward(c, h->dec2, zcl, B, T, y, lens);
        zero_tails(c, y, lens ? lens + (size_t)4 * B : nullptr, B, T * HOP);
    });
}

int fac_voice_convert(fac_handle* h, const int64_t* codes_p, const int64_t* codes_c, int n_c_rows, const float* timbre, int B,
                      int T, int use_p_code, int use_c_code, int n_c, float* y, void* stream) {
    return fac_voice_convert_lens(h, codes_p, codes_c, n_c_rows, timbre, B, T, use_p_code, use_c_code, n_c, nullptr, y, stream);
}

// ---- streaming (SURVEY.md 8f rank 4): chunked encoder / decoder with LSTM-state carry and conv halos ----
// Left context of the encoder's conv stack: 5581 samples (conv0 6 + stage 1 78 + down 3 + stage 2 156 + down 18 + stage 3 780
// + down 90 + stage 4 3900 + down 550) -> 6000 (20 frames); of the decoder's stack after the LSTM: < 18 latent frames -> 20.
constexpr int kEncCtx = 6000, kDecCtx = 20, kStreamMinFirst = 10;
constexpr int kWnCtx = 32;   // mel frames of prosody-net history a codes window recomputes over (stream_codes)

}  // extern "C"

namespace {
// Zeroed device memory laid out by `layout(Carve&)`, which runs twice: to size the block, then to hand out its pieces.
struct Carve {
    char* base = nullptr;
    size_t off = 0;
    template <typename E>
    E* take(size_t n) {
        E* p = base ? reinterpret_cast<E*>(base + off) : nullptr;
        off += (n * sizeof(E) + 255) / 256 * 256;
        return p;
    }
};

template <typename F>
int dev_block(fac_handle* h, DevMem& mem, const char* who, F layout) {
    Carve size;
    layout(size);
    char* p = nullptr;
    cudaError_t e = cudaSetDevice(h->device);
    if (e == cudaSuccess) e = cudaMalloc(&p, size.off);
    mem.reset(p);
    if (e == cudaSuccess) e = cudaMemset(p, 0, size.off);
    if (e != cudaSuccess) {
        h->err = std::string(who) + ": " + cudaGetErrorString(e);
        cudaGetLastError();
        mem.reset();
        return FAC_ERR_CUDA;
    }
    Carve at{p};
    layout(at);
    return FAC_OK;
}

// One LSTM layer of one lane in lstm2_lane_map order: hi | lo h planes (pass3) or one fp16 h plane, then c.
constexpr int carry_words(int H, int pass3) { return (pass3 ? 2 : 1) * (H / 2) + H; }

// The LSTM state tiles of a stream or a pool's lanes: the encoder's LSTM (H = 1024) runs the 3-pass recurrence, the
// decoder's (H = 1536) one fp16 pass.
void take_lstm(Carve& m, LstmState& st, int H, int pass3) {
    size_t hw, cf;
    lstm2_state_sizes(H, lstm_units_per_cta(H), pass3, &hw, &cf);
    for (int l = 0; l < 2; ++l) { st.h[l] = m.take<uint32_t>(hw); st.c[l] = m.take<float>(cf); }
}

// B rows of encoder-half state; a pool slot (B = 1) keeps its LSTM carry in lane-map order instead of state tiles.
void take_enc(Carve& m, EncHalf& s, int B, bool slot) {
    s.B = B;
    s.x_hist = m.take<float>((size_t)B * kEncCtx);
    s.ey_hist = m.take<float>((size_t)B * 2 * LATENT);
    s.z_held = m.take<float>((size_t)B * LATENT);
    if (slot) s.carry = m.take<uint32_t>(2 * carry_words(LATENT, 1));
    else take_lstm(m, s.lstm, LATENT, 1);
}

// ... of decoder-half state; a decode-pool slot also holds its session's gamma | beta.
void take_dec(Carve& m, DecHalf& s, int B, bool slot) {
    s.B = B;
    s.z_hist = m.take<float>((size_t)B * 6 * LATENT);
    s.dy_hist = m.take<float>((size_t)B * kDecCtx * 1536);
    if (slot) { s.carry = m.take<uint32_t>(2 * carry_words(1536, 0)); s.gb = m.take<float>(2048); }
    else take_lstm(m, s.lstm, 1536, 0);
}

// The handle's streams and pools of one kind, by id.
template <typename T>
using List = std::vector<std::unique_ptr<T>> fac_handle::*;

template <typename T>
T* by_id(fac_handle* h, List<T> list, int id) {
    return h && id >= 0 && id < (int)(h->*list).size() ? (h->*list)[id].get() : nullptr;
}

// Frees live entry `id` once the device is idle; its id stays unused.
template <typename T>
int free_by_id(fac_handle* h, List<T> list, int id) {
    if (!by_id(h, list, id)) return FAC_ERR_INVALID;
    cudaSetDevice(h->device);
    cudaDeviceSynchronize();
    (h->*list)[id].reset();
    return FAC_OK;
}
}  // namespace

extern "C" {

int fac_stream_begin(fac_handle* h, int B) {
    if (!h || B < 1 || B > 32) { if (h) h->err = "fac_stream_begin: 1 <= B <= 32"; return FAC_ERR_INVALID; }
    if (!h->finalized) { h->err = "module weights not loaded/finalized"; return FAC_ERR_STATE; }
    auto s = std::make_unique<Stream>();
    int rc = dev_block(h, s->mem, "fac_stream_begin", [&](Carve& m) { take_enc(m, s->enc, B, false); take_dec(m, s->dec, B, false); });
    if (rc) return rc;
    h->streams.push_back(std::move(s));
    return (int)h->streams.size() - 1;
}

int fac_stream_end(fac_handle* h, int stream_id) {
    if (!h || stream_id < 0 || stream_id >= (int)h->streams.size()) return FAC_ERR_INVALID;
    return h->streams[stream_id] ? free_by_id(h, &fac_handle::streams, stream_id) : FAC_OK;
}

}  // extern "C"

namespace {
// dst[b][0..n) = src[b][off..off+n) for rows of `w` elements each (row pitches in rows)
template <typename E>
void copy_rows(Ctx& c, E* dst, int dst_pitch_rows, const E* src, int src_pitch_rows, int off_rows, int n_rows, int w, int B,
               const char* what) {
    if (c.dry || n_rows <= 0) return;
    c.check_nk(cudaMemcpy2DAsync(dst, sizeof(E) * (size_t)dst_pitch_rows * w, src + (size_t)off_rows * w,
                                 sizeof(E) * (size_t)src_pitch_rows * w, sizeof(E) * (size_t)n_rows * w, B,
                                 cudaMemcpyDeviceToDevice, c.st), what);
}

// Inside a launch sequence: lane b of n <= N copies `words` (a count, or a function of b) 32-bit words from src(b) to dst(b)
// (launch_lane_copy).
template <int N = kLaneMax, typename W, typename S, typename D>
void lane_copy(Ctx& c, int n, W words, S src, D dst, const char* what) {
    if (c.dry) return;
    LaneCopyParamsN<N> p;
    p.n = n;
    for (int b = 0; b < n; ++b) {
        p.src[b] = (const uint32_t*)src(b); p.dst[b] = (uint32_t*)dst(b);
        if constexpr (std::is_invocable_v<W, int>) p.words[b] = words(b);
        else p.words[b] = words;
    }
    c.check(launch_lane_copy(p, c.st), what);
}

// Inside a launch sequence: moves the 2-layer LSTM carries (H, pass3) of lanes [0, n) between the state tiles `st` and
// per-lane carries carry(b) ([2 layers][carry_words]; to_lanes = 1: carry -> lane, 0: lane -> carry).
template <typename P>
void lane_carry(Ctx& c, const LstmState& st, int H, int pass3, int n, P carry, int to_lanes) {
    if (c.dry) return;
    for (int l = 0; l < 2; ++l) {
        LaneCarryParams p;
        p.n = n; p.H = H; p.U = lstm_units_per_cta(H); p.pass3 = pass3; p.to_lanes = to_lanes;
        p.state_h = st.h[l]; p.state_c = st.c[l];
        for (int b = 0; b < n; ++b) p.slot[b] = carry(b) + (size_t)l * carry_words(H, pass3);
        c.check(launch_lstm2_lane_carry(p, c.st), "pool.carry");
    }
}

// The chunk rules and the encoder-half state of fac_stream_encode (mode kLatents) / fac_stream_encode_codes (kCodes).
int stream_encode_check(fac_handle* h, const EncHalf& s, int T, int mode, const char* who) {
    if (T <= 0 || T % HOP != 0 || (s.samples == 0 && T < kStreamMinFirst * HOP)) {
        h->err = std::string(who) + ": chunks must be multiples of 300 samples, the first one at least 3000";
        return FAC_ERR_INVALID;
    }
    if (s.mode == EncHalf::kFinished) {
        h->err = std::string(who) + ": the stream's encoder was closed by fac_stream_finish_codes";
        return FAC_ERR_STATE;
    }
    if (s.mode != EncHalf::kNone && s.mode != mode) {
        h->err = std::string(who) + (mode == EncHalf::kCodes ? ": the stream is already fed by fac_stream_encode (latents)"
                                                             : ": the stream is already fed by fac_stream_encode_codes");
        return FAC_ERR_STATE;
    }
    if (!h->lstm_v2 || !h->enc.lstm.has2[1]) { h->err = std::string(who) + ": needs the resident-W LSTM kernel"; return FAC_ERR_UNSUPPORTED; }
    return FAC_OK;
}

// Every integer the launch sequence of an encoder-half chunk depends on, for a half at (samples, hist, yh, emitted = E) fed T
// samples, and the histories it leaves.  Codes of frames [E, E + Fout) are final: frame N - 1 reads 300 samples past what
// has arrived (reflected only at the true end).  Halves with equal keys share one pool batch.
struct EncPlan {
    int T, hist, yh;            // chunk, sample history, encoder-LSTM output history
    int first, f_first, Fout;   // first chunk; frame E within the [x_hist | chunk] window; frames of codes
    int win, Fw;                // the prosody window [lo, E + Fout): E - lo and its length
    long long lo;
    int hist1, yh1;             // the histories after the chunk
    std::vector<long long> key() const { return {T, hist, yh, first, f_first, Fout, win, Fw}; }
};

EncPlan enc_plan(long long samples, int hist, int yh, long long E, int T) {
    const long long N = (samples + T) / HOP, lo = E > kWnCtx ? E - kWnCtx : 0;
    EncPlan p;
    p.T = T; p.hist = hist; p.yh = yh;
    p.first = samples == 0; p.f_first = (int)(E - (samples - hist) / HOP); p.Fout = (int)(N - 1 - E);
    p.win = (int)(E - lo); p.Fw = p.win + p.Fout; p.lo = lo;
    p.hist1 = std::min(hist + T, kEncCtx); p.yh1 = std::min(yh + T / HOP, 2);
    return p;
}
EncPlan enc_plan(const EncHalf& s, int T) { return enc_plan(s.samples, s.x_hist_len, s.ey_hist_len, s.emitted, T); }

// The counters of s after chunk p fed in `mode` (kLatents or kCodes).
void enc_commit(EncHalf& s, const EncPlan& p, int mode) {
    s.samples += p.T; s.x_hist_len = p.hist1; s.ey_hist_len = p.yh1; s.mode = mode;
    if (mode == EncHalf::kCodes) s.emitted += p.Fout;
}

// The encoder half of chunk p on the rows of s: hands the [x_hist | chunk] window xw [B][hist + T] (global samples
// [samples - hist, samples + T)) and the chunk's channels-last latents znew [B][T/300][1024], both in workspace, to
// `tail(xw, znew)`, then keeps the new histories.
template <typename F>
void stream_encode(Ctx& c, EncHalf& s, const EncPlan& p, const float* x, F tail) {
    const EncW& e = c.h->enc;
    const int B = s.B, T = p.T, hist = p.hist, yh = p.yh, Tw = hist + T, Fc = T / HOP, Fh = hist / HOP;
    c.vq_critical = true;
    float* xw = c.alloc<float>((size_t)B * Tw);
    copy_rows(c, xw, Tw, s.x_hist, kEncCtx, 0, hist, 1, B, "stream.xh");
    copy_rows(c, xw + hist, Tw, x, T, 0, T, 1, B, "stream.xc");
    int Fw = 0;
    float* feats = encoder_front(c, xw, B, Tw, &Fw);                    // [B][Fw][1024], Fw == Fh + Fc
    float* fnew = c.alloc<float>((size_t)B * Fc * LATENT);
    copy_rows(c, fnew, Fc, feats, Fw, Fh, Fc, LATENT, B, "stream.fnew");
    float* yw = c.alloc<float>((size_t)B * (yh + Fc) * LATENT);        // [hist | new] LSTM outputs
    float* ynew = c.alloc<float>((size_t)B * Fc * LATENT);
    LstmState st = s.lstm;
    slstm(c, e.lstm, fnew, ynew, B, Fc, &st);
    copy_rows(c, yw, yh + Fc, s.ey_hist, 2, 0, yh, LATENT, B, "stream.yh");
    copy_rows(c, yw + (size_t)yh * LATENT, yh + Fc, ynew, Fc, 0, Fc, LATENT, B, "stream.yc");
    float* zw = c.alloc<float>((size_t)B * (yh + Fc) * LATENT);
    float* znew = c.alloc<float>((size_t)B * Fc * LATENT);
    ConvOpts o;
    o.in_snake = &e.snake;
    sconv(c, e.conv_out, yw, zw, B, yh + Fc, 1, 1, o, "enc.conv_out");
    copy_rows(c, znew, Fc, zw, yh + Fc, yh, Fc, LATENT, B, "stream.znew");
    tail(xw, znew);
    // new histories: the last kEncCtx samples / 2 LSTM-output frames of what has been seen so far
    float* tmpx = c.alloc<float>((size_t)B * kEncCtx);
    copy_rows(c, tmpx, kEncCtx, xw, Tw, Tw - p.hist1, p.hist1, 1, B, "stream.xh2");
    copy_rows(c, s.x_hist, kEncCtx, tmpx, kEncCtx, 0, p.hist1, 1, B, "stream.xh3");
    copy_rows(c, s.ey_hist, 2, yw, yh + Fc, yh + Fc - p.yh1, p.yh1, LATENT, B, "stream.yh2");
    c.vq_critical = false;
}

// Codes of Fq frames from E = the window's frame win (the kCodesOnly VQ kernel): the prosody net recomputed over the mel
// rows [m0, m0 + win + Fq) of s, i.e. frames [max(0, E - 32), E + Fq) -- each of the WN's 8 causal k = 5 convs reflect-pads
// 4 frames at the window's left edge, so the first 32 frames of a window are not those of the whole utterance unless the
// window starts at frame 0 -- and the latents zq [B][Fq][1024] (row pitch zpitch frames).  Runs with c.vq_critical set, as
// the offline quantizer.
void stream_codes(Ctx& c, const EncHalf& s, int m0, int win, int Fq, const float* zq, int zpitch, int64_t* codes_p,
                  int64_t* codes_c, int64_t* codes_r) {
    const int B = s.B, Fw = win + Fq;
    float* melw = c.alloc<float>((size_t)B * Fw * N_MELS);
    copy_rows(c, melw, Fw, s.mel.get(), s.mel_cap, m0, Fw, N_MELS, B, "stream.melw");
    const float* f0 = prosody_forward(c, melw, B, Fw);
    if (c.dry) return;
    FaqParams fp;
    fp.f0 = f0 + (size_t)win * LATENT; fp.Tf0 = Fw;
    fp.z = zq; fp.Tz = zpitch;
    for (int i = 0; i < 6; ++i) {
        const VqW& v = c.h->qw.vq[i];
        fp.vq[i] = VqWeights{c.W(v.w_in), c.W(v.b_in), c.W(v.cb), c.W(v.cbn), c.W(v.cbn2), c.W(v.w_out), c.W(v.b_out)};
    }
    fp.n_c = s.n_c;
    fp.codes_p = codes_p; fp.codes_c = codes_c; fp.codes_r = codes_r;
    fp.B = B; fp.Tq = Fq;
    c.check(launch_fa_codes(fp, c.st), "fa_codes");
}

// Grow-only (doubling) capacity of s.mel for B rows of `rows` frames; the first `keep` rows of each move along.
int grow_mel(fac_handle* h, EncHalf& s, int B, long long keep, int rows, cudaStream_t st) {
    if (rows <= s.mel_cap) return FAC_OK;
    int cap = s.mel_cap > 0 ? s.mel_cap : 64;
    while (cap < rows) cap *= 2;
    cudaError_t e = cudaSetDevice(h->device);
    float* p = nullptr;
    if (e == cudaSuccess) e = cudaMalloc(&p, sizeof(float) * (size_t)B * cap * N_MELS);
    DevBuf<float> grown(p);
    if (e == cudaSuccess && s.mel) {
        e = cudaMemcpy2DAsync(p, sizeof(float) * (size_t)cap * N_MELS, s.mel.get(), sizeof(float) * (size_t)s.mel_cap * N_MELS,
                              sizeof(float) * (size_t)keep * N_MELS, B, cudaMemcpyDeviceToDevice, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    }
    if (e != cudaSuccess) {
        h->err = std::string("stream mel buffer: ") + cudaGetErrorString(e);
        cudaGetLastError();
        return FAC_ERR_CUDA;
    }
    s.mel = std::move(grown); s.mel_cap = cap;
    return FAC_OK;
}

// The compressor needs the mel frames cut explicitly (stft_frames, tensor_cores = 2): the FMA path's strided DFT conv
// reflects at whatever window edge it is given.
int stream_codes_supported(fac_handle* h, const char* who) {
    if (h->use_tc >= 2 && h->qw.dft_tc.tc) return FAC_OK;
    h->err = std::string(who) + ": needs tensor_cores = 2 (the mel path that frames the wave explicitly)";
    return FAC_ERR_UNSUPPORTED;
}

// The argument-independent rules of fac_stream_encode_codes on half s (pointers and the stream id checked by the caller).
int stream_encode_codes_check(fac_handle* h, const EncHalf& s, int T, int n_c, const char* who) {
    int rc = stream_encode_check(h, s, T, EncHalf::kCodes, who);
    if (rc) return rc;
    if (s.mode == EncHalf::kCodes && n_c != s.n_c) {
        h->err = std::string(who) + ": n_c changed mid-stream (" + std::to_string(s.n_c) + " -> " + std::to_string(n_c) + ")";
        return FAC_ERR_INVALID;
    }
    return stream_codes_supported(h, who);
}

// The launch sequence of a codes chunk p on a checked half whose mel rows reach frame E + Fout - 1 (frame f at row
// f - s.mel_base).
void stream_encode_codes(Ctx& c, EncHalf& s, const EncPlan& p, const float* x, int64_t* codes_p, int64_t* codes_c,
                         int64_t* codes_r) {
    const int B = s.B, Fc = p.T / HOP, Fout = p.Fout, m0 = (int)(p.lo - s.mel_base);
    stream_encode(c, s, p, x, [&](const float* xw, const float* znew) {
        c.vq_critical = true;
        const float* mel = mel_frames_tc(c, quantizer_mel(c.h), xw, B, p.hist + p.T, p.f_first, Fout);
        copy_rows(c, s.mel.get() + (size_t)(m0 + p.win) * N_MELS, s.mel_cap, mel, Fout, 0, Fout, N_MELS, B, "stream.mel");
        // latents of frames [E, N - 1): the held frame (after the first chunk) then all but the chunk's last frame
        const float* zq = znew;
        if (!p.first) {
            float* zcat = c.alloc<float>((size_t)B * Fout * LATENT);
            copy_rows(c, zcat, Fout, s.z_held, 1, 0, 1, LATENT, B, "stream.zheld");
            copy_rows(c, zcat + LATENT, Fout, znew, Fc, 0, Fc - 1, LATENT, B, "stream.zcat");
            zq = zcat;
        }
        stream_codes(c, s, m0, p.win, Fout, zq, p.first ? Fc : Fout, codes_p, codes_c, codes_r);
        copy_rows(c, s.z_held, 1, znew, Fc, Fc - 1, 1, LATENT, B, "stream.zhold");
    });
}

int stream_finish_codes_check(fac_handle* h, const EncHalf& s, const char* who) {
    if (s.mode != EncHalf::kCodes) {
        h->err = std::string(who) + (s.mode == EncHalf::kFinished ? ": the stream's encoder is already finished"
                                                                   : ": nothing was encoded with fac_stream_encode_codes");
        return FAC_ERR_STATE;
    }
    return stream_codes_supported(h, who);
}

// Mel row N - 1 (N = samples / 300) of a half fed by fac_stream_encode_codes, as if the utterance ended now: cut from
// the last `hist` samples [B][hist] (x_hist rows) reflected at their end, where the row sits at hist / 300 - 1.
// [B][1][80] in workspace.
const float* last_mel_row(Ctx& c, const float* xw, int B, int hist) {
    return mel_frames_tc(c, quantizer_mel(c.h), xw, B, hist, hist / HOP - 1, 1);
}

// fac_stream_finish_codes on a checked half whose mel rows start at frame 0 (a stream, or a pool session's B = 1 slot,
// which keeps all of its mel rows): returns the frames written (1) or a negative status.
int finish_codes(fac_handle* h, EncHalf& s, int64_t* codes_p, int64_t* codes_c, int64_t* codes_r, float* timbre,
                 void* stream) {
    const int B = s.B, hist = s.x_hist_len, N = (int)(s.samples / HOP);
    const long long E = s.emitted;   // == N - 1
    const int win = (int)(E > kWnCtx ? kWnCtx : E);
    int rc = two_pass(h, (cudaStream_t)stream, [&](Ctx& c) {
        c.vq_critical = true;
        // frame N - 1 from the last `hist` samples, reflected at the utterance's true end
        float* xw = c.alloc<float>((size_t)B * hist);
        copy_rows(c, xw, hist, s.x_hist, kEncCtx, 0, hist, 1, B, "stream.xfin");
        const float* mel = last_mel_row(c, xw, B, hist);
        copy_rows(c, s.mel.get() + (size_t)E * N_MELS, s.mel_cap, mel, 1, 0, 1, N_MELS, B, "stream.mel");
        stream_codes(c, s, (int)E - win, win, 1, s.z_held, 1, codes_p, codes_c, codes_r);
        if (timbre) {
            // the offline StyleEncoder input: every mel80 row of the utterance
            float* melall = c.alloc<float>((size_t)B * N * N_MELS);
            copy_rows(c, melall, N, s.mel.get(), s.mel_cap, 0, N, N_MELS, B, "stream.melall");
            style_encoder(c, melall, B, N, nullptr, timbre);
        }
        c.vq_critical = false;
    });
    if (rc != FAC_OK) return rc;
    s.emitted = N;
    s.mode = EncHalf::kFinished;
    return 1;
}

// The timbre finish_codes would return if the utterance ended now, for a checked half whose mel rows start at frame 0:
// the StyleEncoder over its N mel rows, the kept N - 1 and the last cut by last_mel_row, gathered in workspace.  s is
// not changed.
int stream_timbre(fac_handle* h, const EncHalf& s, float* timbre, void* stream) {
    const int B = s.B, hist = s.x_hist_len, N = (int)(s.samples / HOP);
    return two_pass(h, (cudaStream_t)stream, [&](Ctx& c) {
        c.vq_critical = true;
        float* melall = c.alloc<float>((size_t)B * N * N_MELS);
        copy_rows(c, melall, N, s.mel.get(), s.mel_cap, 0, N - 1, N_MELS, B, "stream.melall");
        float* xw = c.alloc<float>((size_t)B * hist);
        copy_rows(c, xw, hist, s.x_hist, kEncCtx, 0, hist, 1, B, "stream.xfin");
        copy_rows(c, melall + (size_t)(N - 1) * N_MELS, N, last_mel_row(c, xw, B, hist), 1, 0, 1, N_MELS, B, "stream.mel_last");
        style_encoder(c, melall, B, N, nullptr, timbre);
        c.vq_critical = false;
    });
}
}  // namespace

extern "C" {

int fac_stream_encode(fac_handle* h, int stream_id, const float* x, int T, float* z, void* stream) {
    int rc = check_ready(h, {FAC_ENCODER});
    if (rc) return rc;
    Stream* st = by_id(h, &fac_handle::streams, stream_id);
    if (!st || !x || !z) { h->err = "fac_stream_encode: bad arguments"; return FAC_ERR_INVALID; }
    EncHalf& s = st->enc;
    if ((rc = stream_encode_check(h, s, T, EncHalf::kLatents, "fac_stream_encode"))) return rc;
    const EncPlan p = enc_plan(s, T);
    rc = two_pass(h, (cudaStream_t)stream, [&](Ctx& c) {
        stream_encode(c, s, p, x, [&](const float*, const float* znew) {
            if (!c.dry) c.check(launch_transpose(znew, z, s.B, T / HOP, LATENT, c.st), "enc.z_T");
        });
    });
    if (rc == FAC_OK) enc_commit(s, p, EncHalf::kLatents);
    return rc;
}

int fac_stream_encode_codes(fac_handle* h, int stream_id, const float* x, int T, int n_c, int64_t* codes_p, int64_t* codes_c,
                            int64_t* codes_r, void* stream) {
    int rc = check_ready(h, {FAC_ENCODER, FAC_QUANTIZER});
    if (rc) return rc;
    const char* who = "fac_stream_encode_codes";
    Stream* st = by_id(h, &fac_handle::streams, stream_id);
    if (!st || !x || !codes_p || !codes_c || !codes_r || n_c < 1 || n_c > 2) {
        h->err = "fac_stream_encode_codes: bad arguments (1 <= n_c <= 2)";
        return FAC_ERR_INVALID;
    }
    EncHalf& s = st->enc;
    if ((rc = stream_encode_codes_check(h, s, T, n_c, who))) return rc;
    if ((rc = grow_mel(h, s, s.B, s.emitted, (int)((s.samples + T) / HOP), (cudaStream_t)stream))) return rc;
    const EncPlan p = enc_plan(s, T);
    s.n_c = n_c;
    rc = two_pass(h, (cudaStream_t)stream, [&](Ctx& c) { stream_encode_codes(c, s, p, x, codes_p, codes_c, codes_r); });
    if (rc) return rc;
    enc_commit(s, p, EncHalf::kCodes);
    return p.Fout;
}

int fac_stream_finish_codes(fac_handle* h, int stream_id, int64_t* codes_p, int64_t* codes_c, int64_t* codes_r, float* timbre,
                            void* stream) {
    int rc = check_ready(h, {FAC_ENCODER, FAC_QUANTIZER});
    if (rc) return rc;
    Stream* st = by_id(h, &fac_handle::streams, stream_id);
    if (!st || !codes_p || !codes_c || !codes_r) { h->err = "fac_stream_finish_codes: bad arguments"; return FAC_ERR_INVALID; }
    if ((rc = stream_finish_codes_check(h, st->enc, "fac_stream_finish_codes"))) return rc;
    return finish_codes(h, st->enc, codes_p, codes_c, codes_r, timbre, stream);
}

int fac_stream_timbre(fac_handle* h, int stream_id, float* timbre, void* stream) {
    int rc = check_ready(h, {FAC_ENCODER, FAC_QUANTIZER});
    if (rc) return rc;
    Stream* st = by_id(h, &fac_handle::streams, stream_id);
    if (!st || !timbre) { h->err = "fac_stream_timbre: bad arguments"; return FAC_ERR_INVALID; }
    if ((rc = stream_finish_codes_check(h, st->enc, "fac_stream_timbre"))) return rc;
    return stream_timbre(h, st->enc, timbre, stream);
}

}  // extern "C"

namespace {
// The chunk rules and the decoder support of fac_stream_decode / fac_stream_decode_codes, for a stream row that has decoded
// `frames` frames and is fed Fc more.
int stream_decode_check(fac_handle* h, long long frames, int Fc, const char* who) {
    if (Fc <= 0 || (frames == 0 && Fc < kStreamMinFirst)) { h->err = std::string(who) + ": the first chunk needs at least 10 frames"; return FAC_ERR_INVALID; }
    if (!h->lstm_v2 || !h->dec_bf16 || !h->dec_lstm_fp16 || !h->dec.lstm.has2[0]) { h->err = std::string(who) + ": needs the resident-W LSTM kernel"; return FAC_ERR_UNSUPPORTED; }
    return FAC_OK;
}

// The decoder half's launch sequence depends only on its history depth: zh = min(frames, 6) latent and dh = min(frames, 20)
// LSTM-output frames (a first chunk has >= 10 frames, so dh fixes zh).  The chunk lengths of its rows may differ.
struct DecPlan {
    int zh, dh;
    std::vector<long long> key() const { return {zh, dh}; }
};
DecPlan dec_plan(long long frames) { return {(int)std::min(frames, 6LL), (int)std::min(frames, (long long)kDecCtx)}; }

// The decoder half of a chunk on the rows of s (plan p): row b takes F[b] new frames (HOST, s.B entries), whose channels-last
// latents `latents(c, B)` returns as [B][Fmax][1024] (Fmax = the largest F[b]; transposed from the caller's z, or
// dequantized from codes).  y receives [B][300 Fmax], row b valid for its first 300 F[b] samples.  With equal F this is one
// stream chunk.  With unequal F (a decode pool's batch) each row runs on a window padded past its own end: the decoder after
// the LSTM is causal (left reflect padding, no right padding, transposed convs trimmed on the right), so no sample before a
// row's end reads the padding; the LSTM stops each row at its own end, and the histories are cut at each row's own end.
template <typename L>
void stream_decode(Ctx& c, DecHalf& s, const DecPlan& p, const int* F, float* y, L latents) {
    const DecW& d = c.h->dec;
    const int B = s.B, zh = p.zh, dh = p.dh;
    int Fc = 0;
    bool mixed = false;
    for (int b = 0; b < B; ++b) { Fc = F[b] > Fc ? F[b] : Fc; mixed = mixed || F[b] != F[0]; }
    const float* znew = latents(c, B);
    float* zw = c.alloc<float>((size_t)B * (zh + Fc) * LATENT);
    copy_rows(c, zw, zh + Fc, s.z_hist, 6, 0, zh, LATENT, B, "stream.zh");
    copy_rows(c, zw + (size_t)zh * LATENT, zh + Fc, znew, Fc, 0, Fc, LATENT, B, "stream.zc");
    float* c0w = c.alloc<float>((size_t)B * (zh + Fc) * 1536);
    sconv(c, d.conv0, zw, c0w, B, zh + Fc, 1, 1, ConvOpts(), "dec.conv0");
    float* c0new = c.alloc<float>((size_t)B * Fc * 1536);
    copy_rows(c, c0new, Fc, c0w, zh + Fc, zh, Fc, 1536, B, "stream.c0new");
    float* ynew = c.alloc<float>((size_t)B * Fc * 1536);
    LstmState st = s.lstm;
    slstm(c, d.lstm, c0new, ynew, B, Fc, &st, mixed ? F : nullptr);
    const int Fw = dh + Fc;
    const size_t stage = decoder_stage_floats(B, Fw);
    float* buf[3] = {c.alloc<float>(stage), c.alloc<float>(stage), c.alloc<float>(stage)};
    float* yw_in = c.alloc<float>((size_t)B * Fw * 1536);
    copy_rows(c, yw_in, Fw, s.dy_hist, kDecCtx, 0, dh, 1536, B, "stream.dh");
    copy_rows(c, yw_in + (size_t)dh * 1536, Fw, ynew, Fc, 0, Fc, 1536, B, "stream.dc");
    float* yw = c.alloc<float>((size_t)B * Fw * HOP);
    decoder_stack(c, d, yw_in, -1, buf, B, Fw, yw);
    copy_rows(c, y, Fc * HOP, yw, Fw * HOP, dh * HOP, Fc * HOP, 1, B, "stream.ynew");
    if (mixed) {
        auto nz = [&](int b) { return zh + F[b] < 6 ? zh + F[b] : 6; };
        auto nd = [&](int b) { return dh + F[b] < kDecCtx ? dh + F[b] : kDecCtx; };
        lane_copy(c, B, [&](int b) { return (long long)nz(b) * LATENT; },
                  [&](int b) { return zw + ((size_t)b * (zh + Fc) + zh + F[b] - nz(b)) * LATENT; },
                  [&](int b) { return s.z_hist + (size_t)b * 6 * LATENT; }, "stream.zh_lanes");
        lane_copy(c, B, [&](int b) { return (long long)nd(b) * 1536; },
                  [&](int b) { return yw_in + ((size_t)b * Fw + dh + F[b] - nd(b)) * 1536; },
                  [&](int b) { return s.dy_hist + (size_t)b * kDecCtx * 1536; }, "stream.dh_lanes");
        return;
    }
    const int nzh = zh + Fc < 6 ? zh + Fc : 6, ndh = Fw < kDecCtx ? Fw : kDecCtx;
    float* tz = c.alloc<float>((size_t)B * 6 * LATENT);
    float* td = c.alloc<float>((size_t)B * kDecCtx * 1536);
    copy_rows(c, tz, 6, zw, zh + Fc, zh + Fc - nzh, nzh, LATENT, B, "stream.zh2");
    copy_rows(c, s.z_hist, 6, tz, 6, 0, nzh, LATENT, B, "stream.zh3");
    copy_rows(c, td, kDecCtx, yw_in, Fw, Fw - ndh, ndh, 1536, B, "stream.dh2");
    copy_rows(c, s.dy_hist, kDecCtx, td, kDecCtx, 0, ndh, 1536, B, "stream.dh3");
}

// fac_stream_decode / fac_stream_decode_codes on a live stream: the checks, then one chunk of Fc frames on every row.
template <typename L>
int stream_decode_chunk(fac_handle* h, Stream& st, int Fc, float* y, void* stream, const char* who, L latents) {
    DecHalf& s = st.dec;
    int rc = stream_decode_check(h, s.frames, Fc, who);
    if (rc) return rc;
    const std::vector<int> F(s.B, Fc);
    rc = two_pass(h, (cudaStream_t)stream, [&](Ctx& c) { stream_decode(c, s, dec_plan(s.frames), F.data(), y, latents); });
    if (rc == FAC_OK) s.frames += Fc;
    return rc;
}
}  // namespace

extern "C" {

int fac_stream_decode(fac_handle* h, int stream_id, const float* z, int Fc, float* y, void* stream) {
    int rc = check_ready(h, {FAC_DECODER});
    if (rc) return rc;
    Stream* st = by_id(h, &fac_handle::streams, stream_id);
    if (!st || !z || !y) { h->err = "fac_stream_decode: bad arguments"; return FAC_ERR_INVALID; }
    return stream_decode_chunk(h, *st, Fc, y, stream, "fac_stream_decode", [&](Ctx& c, int B) {
        float* znew = c.alloc<float>((size_t)B * Fc * LATENT);
        if (!c.dry) c.check(launch_transpose(z, znew, B, LATENT, Fc, c.st), "dec.z_transpose");
        return znew;
    });
}

int fac_stream_decode_codes(fac_handle* h, int stream_id, const int64_t* codes_p, const int64_t* codes_c, int n_c_rows,
                            const int64_t* codes_r, int n_r_rows, const float* timbre, int Fc, float* y, void* stream) {
    int rc = check_ready(h, {FAC_QUANTIZER, FAC_DECODER});
    if (rc) return rc;
    Stream* st = by_id(h, &fac_handle::streams, stream_id);
    if (!st || !y || bad_codes_args(codes_p, codes_c, n_c_rows, codes_r, n_r_rows, timbre, st->dec.B, Fc)) {
        h->err = "fac_stream_decode_codes: bad arguments (1 <= content rows <= 2, 0 <= residual rows <= 3)";
        return FAC_ERR_INVALID;
    }
    return stream_decode_chunk(h, *st, Fc, y, stream, "fac_stream_decode_codes", [&](Ctx& c, int B) {
        return (const float*)dequantize_forward(c, codes_p, codes_c, n_c_rows, codes_r, n_r_rows, timbre, B, Fc, false).outs_cl;
    });
}

}  // extern "C"

// ---- streaming voice conversion (fac_vc_stream_*): codes -> redecoder -> non-causal decoder on windows ----
namespace {
// Reach of the redecoder in code frames: its 16 WN layers are non-causal k = 5 SConv1ds, each reflect-padding (5 - 1) / 2 = 2
// frames on both sides; the embeddings, the 1x1 res/skip convs and conv_out are per frame.  So z frame t reads codes
// [t - 32, t + 32], and a window edge that is not the utterance's own corrupts the 32 z frames next to it.
constexpr int kVcRedCtx = 16 * (5 - 1) / 2;

// Reach of the non-causal decoder in z frames.  z frame f reaches output samples [300 f + lo, 300 f + hi]: conv0 (k 7) reaches
// +-3 frames; each DecoderBlock of stride s takes input position u through its 3-tap transposed conv (pack_convtr_noncausal:
// phases r < s/2 also read x[t-1], phases r >= s/2 also read x[t+1]) to outputs [s u - s + s/2, s u + s + s/2 - 1], and its
// ResidualUnits (k 7, dilations 1, 3, 9) add +-39; conv_out (k 7) adds +-3.  That gives [300 f - 3547, 300 f + 3834]: output
// frame t (samples [300 t, 300 t + 300)) reads z frames [t - 12, t + 12], and a window edge corrupts the 12 frames next to it.
constexpr int vc_decoder_reach() {
    const int rates[4] = {6, 5, 5, 2};
    int lo = -3, hi = 3;
    for (int s : rates) { lo = s * lo - s + s / 2 - 39; hi = s * hi + s + s / 2 - 1 + 39; }
    lo -= 3; hi += 3;
    const int ahead = (HOP - 1 - lo) / HOP, behind = hi / HOP;
    return ahead > behind ? ahead : behind;
}
constexpr int kVcDecCtx = vc_decoder_reach();
// Stream state capacities.  z history: at most 2 * kVcDecCtx frames after every call.  Codes history: the last
// kVcCodesHist frames.  A step after set_timbre reads codes from max(0, Yf - kVcDecCtx - kVcRedCtx), and since Yf trails N by
// at most the look-ahead kVcRedCtx + kVcDecCtx, that start lies at most 2 * (kVcRedCtx + kVcDecCtx) frames back.
constexpr int kVcCodesHist = 2 * (kVcRedCtx + kVcDecCtx), kVcZHist = 2 * kVcDecCtx;

// B rows of voice-conversion state.
void take_vc(Carve& m, VcStream& s, int B, size_t gfl) {
    s.B = B;
    s.g = m.take<float>((size_t)B * gfl);
    s.codes = m.take<int64_t>((size_t)B * 3 * kVcCodesHist);
    s.z = m.take<float>((size_t)B * kVcZHist * LATENT);
}

// Every integer of a voice-conversion step on a stream at (N, Zf, Yf) fed F code frames (F = 0 at finish, which makes every
// frame final), and the counters it leaves.  The step runs on the codes window [hc0, N1) (Tw frames, hist of them history)
// and the z window [zh0, Zf1) (Tz frames, zhist of them history).  It makes z final up to Zf1 and the output up to Yf1:
// both stages reach kVcRedCtx / kVcDecCtx frames past the rows they keep, so those rows never see a window edge except the
// utterance's own (frame 0, and frame N at finish).  Streams with equal keys share one pool batch.
// A stale step (the timbre changed since the z history [zh0, Zf) was computed) recomputes it: its codes window starts at
// hc0 = max(0, zh0 - kVcRedCtx) and every row of the z window comes from it (zhist = 0, zoff = zh0 - hc0).  The same
// argument holds: z row t in [zh0, Zf1) reads codes [t - kVcRedCtx, t + kVcRedCtx], which lie inside [hc0, N1) except where
// hc0 = 0 or N1 is the utterance's end -- the edges an offline run reflects at too -- so the rows equal the offline z under
// the new timbre, bit for bit.  A step whose z history is empty is never stale: the plain step computes every row anew.
struct VcPlan {
    int F, Tw, hist, Tz, zhist;
    int zoff, znew;             // z rows [Zf or zh0 (stale), Zf1) in the codes window
    int k, yoff;                // output frames [Yf, Yf1) and Yf in the z window
    int zkeep_at, zkeep;        // z history kept: [zh1, Zf1) in the z window
    int stale;                  // 1: the z history is recomputed from the codes (set_timbre)
    long long N1, Zf1, Yf1;
    std::vector<long long> key() const { return {F, Tw, hist, Tz, zhist, zoff, znew, k, yoff, zkeep_at, zkeep, stale}; }
};

VcPlan vc_plan(long long N, long long Zf, long long Yf, int F, bool finish, bool stale = false) {
    auto floor0 = [](long long v) { return v > 0 ? v : 0; };
    VcPlan p;
    p.N1 = N + F;
    p.Zf1 = finish ? p.N1 : std::max(p.N1 - kVcRedCtx, Zf);
    p.Yf1 = finish ? p.N1 : std::max(p.Zf1 - kVcDecCtx, Yf);
    const long long zh0 = floor0(Yf - kVcDecCtx), zh1 = floor0(p.Yf1 - kVcDecCtx);
    p.stale = stale && Zf > zh0 ? 1 : 0;
    const long long hc0 = p.stale ? floor0(zh0 - kVcRedCtx) : floor0(Zf - kVcRedCtx), z0 = p.stale ? zh0 : Zf;
    p.F = F; p.Tw = (int)(p.N1 - hc0); p.hist = (int)(N - hc0); p.Tz = (int)(p.Zf1 - zh0); p.zhist = (int)(z0 - zh0);
    p.zoff = (int)(z0 - hc0); p.znew = (int)(p.Zf1 - z0); p.k = (int)(p.Yf1 - Yf); p.yoff = (int)(Yf - zh0);
    p.zkeep_at = (int)(zh1 - zh0); p.zkeep = (int)(p.Zf1 - zh1);
    return p;
}
VcPlan vc_plan(const VcStream& s, int F, bool finish) { return vc_plan(s.N, s.Zf, s.Yf, F, finish, s.stale); }

// The conversion mode of a step's rows: one for all (a stream, or a pool batch of one mode), or per lane.
struct VcMode {
    int use_p = 0, use_c = 0, n_c = 0;      // n_c: the content rows copied into the codes window
    const int* lanes = nullptr;             // [B][2] device: each row's use_p and effective n_c (use_c ? n_c : 0), or null
};
VcMode vc_mode(const VcStream& s) { return VcMode{s.use_p, s.use_c, s.n_c, nullptr}; }

// The launch sequence of step p on the rows of s: appends F code frames (codes_p [B][1][F], codes_c [B][n_c_rows][F]) and
// writes output frames [Yf, Yf1) to y as [B][1][300 k].
void vc_step(Ctx& c, VcStream& s, const VcPlan& p, const VcMode& m, const int64_t* codes_p, const int64_t* codes_c,
             int n_c_rows, float* y) {
    const int B = s.B, F = p.F, Tw = p.Tw, hist = p.hist, Tz = p.Tz, H = kVcCodesHist;
    // codes [hc0, N1) as [B][3][Tw]: the history, then the new frames
    int64_t* cw = c.alloc<int64_t>((size_t)B * 3 * Tw);
    copy_rows(c, cw, Tw, s.codes, H, H - hist, hist, 1, 3 * B, "vc.codes_hist");
    copy_rows(c, cw + hist, 3 * Tw, codes_p, F, 0, F, 1, B, "vc.codes_p");
    for (int i = 0; i < m.n_c; ++i)
        copy_rows(c, cw + (size_t)(1 + i) * Tw + hist, 3 * Tw, codes_c + (size_t)i * F, n_c_rows * F, 0, F, 1, B, "vc.codes_c");
    if (p.znew > 0) {
        // z over the codes window, of which rows [Zf, Zf1) are final; the decoder's window is z [zh0, Zf1)
        float* zc = redecoder_body(c, cw, 3 * Tw, cw + Tw, 3 * Tw, s.g, B, Tw, m.use_p, m.use_c, m.n_c, nullptr, m.lanes);
        float* zw = c.alloc<float>((size_t)B * Tz * LATENT);
        copy_rows(c, zw, Tz, s.z, kVcZHist, 0, p.zhist, LATENT, B, "vc.z_hist");
        copy_rows(c, zw + (size_t)p.zhist * LATENT, Tz, zc, Tw, p.zoff, p.znew, LATENT, B, "vc.z_new");
        if (p.k > 0) {
            float* yw = c.alloc<float>((size_t)B * Tz * HOP);
            decoder_forward(c, c.h->dec2, zw, B, Tz, yw);
            copy_rows(c, y, p.k * HOP, yw, Tz * HOP, p.yoff * HOP, p.k * HOP, 1, B, "vc.y");
        }
        copy_rows(c, s.z, kVcZHist, zw, Tz, p.zkeep_at, p.zkeep, LATENT, B, "vc.z_keep");
    }
    // codes [N1 - H, N1), right-aligned: the frames before the window from the old history (columns [F, H - hist)), the
    // rest from the window, assembled in workspace (the two ranges of s.codes may overlap)
    const int fresh = std::min(Tw, H);
    int64_t* ck = c.alloc<int64_t>((size_t)B * 3 * H);
    copy_rows(c, ck, H, s.codes, H, F, H - Tw, 1, 3 * B, "vc.codes_old");
    copy_rows(c, ck + (H - fresh), H, cw, Tw, Tw - fresh, fresh, 1, 3 * B, "vc.codes_new");
    copy_rows(c, s.codes, H, ck, H, 0, H, 1, 3 * B, "vc.codes_keep");
}

void vc_commit(VcStream& s, const VcPlan& p) { s.N = p.N1; s.Zf = p.Zf1; s.Yf = p.Yf1; s.stale = false; }

// Step p of a voice-conversion stream (or a pool session's B = 1 slot) in its own launch sequence: returns the output frames
// written or a negative status.
int vc_run(fac_handle* h, VcStream& s, const VcPlan& p, const int64_t* codes_p, const int64_t* codes_c, int n_c_rows, float* y,
           void* stream) {
    int rc = two_pass(h, (cudaStream_t)stream, [&](Ctx& c) { vc_step(c, s, p, vc_mode(s), codes_p, codes_c, n_c_rows, y); });
    if (rc) return rc;
    vc_commit(s, p);
    return p.k;
}

// The target voice of B rows of s from timbre [B][1024]: the cond layer into workspace, then into s.g (nothing of s changes
// unless the launch sequence is queued); the next step recomputes the z history under it.
int vc_set_timbre(fac_handle* h, VcStream& s, const float* timbre, void* stream) {
    const size_t gfl = redecoder_cond_floats(h, s.B);
    int rc = two_pass(h, (cudaStream_t)stream, [&](Ctx& c) {
        float* g = c.alloc<float>(gfl);
        redecoder_cond(c, timbre, s.B, g);
        if (!c.dry) c.check_nk(cudaMemcpyAsync(s.g, g, sizeof(float) * gfl, cudaMemcpyDeviceToDevice, c.st), "vc.g");
    });
    if (rc == FAC_OK) s.stale = true;
    return rc;
}
}  // namespace

extern "C" {

int fac_vc_stream_lookahead(void) { return kVcRedCtx + kVcDecCtx; }

int fac_vc_stream_begin(fac_handle* h, int B, const float* timbre, int use_p_code, int use_c_code, int n_c, void* stream) {
    int rc = check_ready(h, {FAC_REDECODER, FAC_REDECODER_DECODER});
    if (rc) return rc;
    if (!timbre || B < 1 || B > 32 || n_c < 0 || n_c > 2) {
        h->err = "fac_vc_stream_begin: bad arguments (1 <= B <= 32, 0 <= n_c <= 2)";
        return FAC_ERR_INVALID;
    }
    auto s = std::make_unique<VcStream>();
    s->use_p = use_p_code ? 1 : 0; s->use_c = use_c_code ? 1 : 0; s->n_c = n_c;
    rc = dev_block(h, s->mem, "fac_vc_stream_begin", [&](Carve& m) { take_vc(m, *s, B, redecoder_cond_floats(h, 1)); });
    if (rc == FAC_OK) rc = two_pass(h, (cudaStream_t)stream, [&](Ctx& c) { redecoder_cond(c, timbre, B, s->g); });
    if (rc != FAC_OK) return rc;
    h->vc_streams.push_back(std::move(s));
    return (int)h->vc_streams.size() - 1;
}

int fac_vc_stream_convert(fac_handle* h, int stream_id, const int64_t* codes_p, const int64_t* codes_c, int n_c_rows, int F,
                          float* y, void* stream) {
    int rc = check_ready(h, {FAC_REDECODER, FAC_REDECODER_DECODER});
    if (rc) return rc;
    VcStream* s = by_id(h, &fac_handle::vc_streams, stream_id);
    if (!s || !codes_p || !codes_c || !y || F <= 0 || n_c_rows < s->n_c || n_c_rows > 2) {
        h->err = "fac_vc_stream_convert: bad arguments (F >= 1, n_c <= rows of codes_c <= 2)";
        return FAC_ERR_INVALID;
    }
    if (s->finished) { h->err = "fac_vc_stream_convert: the stream was finished"; return FAC_ERR_STATE; }
    return vc_run(h, *s, vc_plan(*s, F, false), codes_p, codes_c, n_c_rows, y, stream);
}

int fac_vc_stream_finish(fac_handle* h, int stream_id, float* y, void* stream) {
    int rc = check_ready(h, {FAC_REDECODER, FAC_REDECODER_DECODER});
    if (rc) return rc;
    VcStream* s = by_id(h, &fac_handle::vc_streams, stream_id);
    if (!s || !y) { h->err = "fac_vc_stream_finish: bad arguments"; return FAC_ERR_INVALID; }
    if (s->finished || s->N == 0) {
        h->err = s->finished ? "fac_vc_stream_finish: the stream was finished" : "fac_vc_stream_finish: no codes were received";
        return FAC_ERR_STATE;
    }
    rc = vc_run(h, *s, vc_plan(*s, 0, true), nullptr, nullptr, 0, y, stream);
    if (rc >= 0) s->finished = true;
    return rc;
}

int fac_vc_stream_set_timbre(fac_handle* h, int stream_id, const float* timbre, void* stream) {
    int rc = check_ready(h, {FAC_REDECODER, FAC_REDECODER_DECODER});
    if (rc) return rc;
    VcStream* s = by_id(h, &fac_handle::vc_streams, stream_id);
    if (!s || !timbre) { h->err = "fac_vc_stream_set_timbre: bad arguments"; return FAC_ERR_INVALID; }
    if (s->finished) { h->err = "fac_vc_stream_set_timbre: the stream was finished"; return FAC_ERR_STATE; }
    return vc_set_timbre(h, *s, timbre, stream);
}

int fac_vc_stream_end(fac_handle* h, int stream_id) {
    if (!h || stream_id < 0 || stream_id >= (int)h->vc_streams.size()) return FAC_ERR_INVALID;
    return h->vc_streams[stream_id] ? free_by_id(h, &fac_handle::vc_streams, stream_id) : FAC_OK;
}

}  // extern "C"

// ---- stream pools (fac_codes_pool_*, fac_vc_pool_*, fac_dec_pool_*): many B = 1 streams stepped in shared batches ----
// A session's state lives in a slot: a B = 1 view of the state its step advances (an encoder half, a VcStream, a decoder
// half), on which finishes run directly.  A step groups its sessions by their plans' keys (every integer the launch
// sequence depends on), and runs each batch of <= 32 as one launch sequence: gather the sessions' state into the lanes of a
// B = 32 state (pool.cu, lstm2.cu), run the stream body on them, scatter the state back.  Every lane of the batched kernels
// computes as a B = 1 launch does (batch invariance), so a session's bits do not depend on who shares its launch.
namespace {
// Batches of one pool step: sessions with equal keys form a group (groups in order of first appearance, members in input
// order), each group cut into batches of at most kLaneMax.  group[i] / batch[i] (optional) receive input i's.
std::vector<std::vector<int>> pool_plan(const std::vector<std::vector<long long>>& keys, int* group, int* batch) {
    std::map<std::vector<long long>, int> index;
    std::vector<std::vector<int>> groups, batches;
    for (int i = 0; i < (int)keys.size(); ++i) {
        auto it = index.find(keys[i]);
        int g = it != index.end() ? it->second : (index[keys[i]] = (int)groups.size());
        if (g == (int)groups.size()) groups.emplace_back();
        groups[g].push_back(i);
        if (group) group[i] = g;
    }
    for (const auto& g : groups)
        for (size_t o = 0; o < g.size(); o += kLaneMax) {
            batches.emplace_back(g.begin() + o, g.begin() + (o + kLaneMax < g.size() ? o + kLaneMax : g.size()));
            if (batch) for (int i : batches.back()) batch[i] = (int)batches.size() - 1;
        }
    return batches;
}

// A pool of `capacity` slots: take(m, state, B, slot) lays out the B = 32 lanes and each B = 1 slot.
template <typename S, typename T>
int pool_create(fac_handle* h, List<Pool<S>> pools, int capacity, const char* who, T take) {
    auto P = std::make_unique<Pool<S>>();
    P->cap = capacity;
    P->slot.resize(capacity);
    P->used.assign(capacity, 0);
    int rc = dev_block(h, P->mem, who, [&](Carve& m) {
        take(m, P->lanes, kLaneMax, false);
        for (S& s : P->slot) take(m, s, 1, true);
    });
    if (rc) return rc;
    (h->*pools).push_back(std::move(P));
    return (int)(h->*pools).size() - 1;
}

// Opens the first free slot after init(slot) succeeds; returns the session id or a status.
template <typename S, typename I>
int pool_open(fac_handle* h, List<Pool<S>> pools, int id, const char* who, I init) {
    Pool<S>* P = by_id(h, pools, id);
    if (!P) { if (h) h->err = std::string(who) + ": no such pool"; return FAC_ERR_INVALID; }
    int i = 0;
    while (i < P->cap && P->used[i]) ++i;
    if (i == P->cap) { h->err = std::string(who) + ": the pool is full (capacity " + std::to_string(P->cap) + ")"; return FAC_ERR_STATE; }
    int rc = init(P->slot[i]);
    if (rc) return rc;
    P->used[i] = 1;
    return i;
}

template <typename S>
int pool_close(fac_handle* h, List<Pool<S>> pools, int id, int session, const char* who) {
    Pool<S>* P = by_id(h, pools, id);
    if (!P || session < 0 || session >= P->cap || !P->used[session]) {
        if (h) h->err = std::string(who) + ": session " + std::to_string(session) + " is not open";
        return FAC_ERR_INVALID;
    }
    P->used[session] = 0;
    return FAC_OK;
}

// The sessions of one step: each open and named once.
template <typename S>
int check_sessions(fac_handle* h, const Pool<S>& pool, int n, const int* sessions, const char* who) {
    std::vector<char> seen(pool.cap, 0);
    for (int i = 0; i < n; ++i) {
        const int sid = sessions[i];
        if (sid < 0 || sid >= pool.cap || !pool.used[sid]) {
            h->err = std::string(who) + ": session " + std::to_string(sid) + " is not open";
            return FAC_ERR_INVALID;
        }
        if (seen[sid]++) {
            h->err = std::string(who) + ": session " + std::to_string(sid) + " is named twice";
            return FAC_ERR_INVALID;
        }
    }
    return FAC_OK;
}

// One batch of a codes-pool step: inputs b (equal plan keys) of the step's sessions, fed T samples each from x.  The lanes'
// mel rows hold the batch's prosody windows, from frame lo.
int codes_pool_batch(fac_handle* h, CodesPool& P, const std::vector<int>& b, const int* sessions, const std::vector<EncPlan>& plan,
                     const float* const* x, int64_t* const* codes_p, int64_t* const* codes_c, int64_t* const* codes_r,
                     cudaStream_t st) {
    EncHalf& L = P.lanes;
    const EncPlan& p = plan[b[0]];
    const int nb = (int)b.size(), n_c = L.n_c, T = p.T, Fout = p.Fout, win = p.win;
    auto sl = [&](int j) -> EncHalf& { return P.slot[sessions[b[j]]]; };
    const size_t pitch = (size_t)L.mel_cap * N_MELS;
    L.B = nb; L.mel_base = p.lo;
    int rc = two_pass(h, st, [&](Ctx& c) {
        float* xin = c.alloc<float>((size_t)nb * T);
        int64_t* cp = c.alloc<int64_t>((size_t)nb * Fout);
        int64_t* cc = c.alloc<int64_t>((size_t)nb * n_c * Fout);
        int64_t* cr = c.alloc<int64_t>((size_t)nb * 3 * Fout);
        lane_copy(c, nb, T, [&](int j) { return x[b[j]]; }, [&](int j) { return xin + (size_t)j * T; }, "pool.x");
        lane_copy(c, nb, p.hist, [&](int j) { return sl(j).x_hist; }, [&](int j) { return L.x_hist + (size_t)j * kEncCtx; },
                  "pool.x_hist");
        lane_copy(c, nb, (long long)p.yh * LATENT, [&](int j) { return sl(j).ey_hist; },
                  [&](int j) { return L.ey_hist + (size_t)j * 2 * LATENT; }, "pool.ey_hist");
        if (!p.first)
            lane_copy(c, nb, LATENT, [&](int j) { return sl(j).z_held; }, [&](int j) { return L.z_held + (size_t)j * LATENT; },
                      "pool.z_held");
        lane_copy(c, nb, (long long)win * N_MELS, [&](int j) { return sl(j).mel.get() + (size_t)(sl(j).emitted - win) * N_MELS; },
                  [&](int j) { return L.mel.get() + j * pitch; }, "pool.mel");
        lane_carry(c, L.lstm, LATENT, 1, nb, [&](int j) { return sl(j).carry; }, 1);
        stream_encode_codes(c, L, p, xin, cp, cc, cr);
        lane_copy(c, nb, p.hist1, [&](int j) { return L.x_hist + (size_t)j * kEncCtx; }, [&](int j) { return sl(j).x_hist; },
                  "pool.x_hist");
        lane_copy(c, nb, (long long)p.yh1 * LATENT, [&](int j) { return L.ey_hist + (size_t)j * 2 * LATENT; },
                  [&](int j) { return sl(j).ey_hist; }, "pool.ey_hist");
        lane_copy(c, nb, LATENT, [&](int j) { return L.z_held + (size_t)j * LATENT; }, [&](int j) { return sl(j).z_held; },
                  "pool.z_held");
        lane_copy(c, nb, (long long)Fout * N_MELS, [&](int j) { return L.mel.get() + j * pitch + (size_t)win * N_MELS; },
                  [&](int j) { return sl(j).mel.get() + (size_t)sl(j).emitted * N_MELS; }, "pool.mel");
        lane_carry(c, L.lstm, LATENT, 1, nb, [&](int j) { return sl(j).carry; }, 0);
        lane_copy(c, nb, 2LL * Fout, [&](int j) { return cp + (size_t)j * Fout; }, [&](int j) { return codes_p[b[j]]; },
                  "pool.codes_p");
        lane_copy(c, nb, 2LL * n_c * Fout, [&](int j) { return cc + (size_t)j * n_c * Fout; },
                  [&](int j) { return codes_c[b[j]]; }, "pool.codes_c");
        lane_copy(c, nb, 6LL * Fout, [&](int j) { return cr + (size_t)j * 3 * Fout; }, [&](int j) { return codes_r[b[j]]; },
                  "pool.codes_r");
    });
    if (rc) return rc;
    for (int j = 0; j < nb; ++j) enc_commit(sl(j), plan[b[j]], EncHalf::kCodes);
    return FAC_OK;
}

// Lanes x longest lane of one codes-pool timbre batch stay within this many mel frames (~16 KB of StyleEncoder workspace
// each: ~0.5 GB), so an hour-long session does not grow the workspace by the batch's width; a longer session runs alone.
constexpr long long kTimbreFrameBudget = 1 << 15;

// Batches of a codes-pool timbre call over sessions of N[i] mel frames: by N (stable), each batch as many sessions as
// fit kLaneMax lanes and kTimbreFrameBudget frames.
std::vector<std::vector<int>> timbre_plan(const std::vector<int>& N) {
    std::vector<int> order(N.size());
    for (size_t i = 0; i < order.size(); ++i) order[i] = (int)i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return N[a] < N[b]; });
    std::vector<std::vector<int>> batches;
    for (int i : order) {
        if (batches.empty() || (int)batches.back().size() == kLaneMax ||
            (long long)(batches.back().size() + 1) * N[i] > kTimbreFrameBudget)
            batches.emplace_back();
        batches.back().push_back(i);
    }
    return batches;
}

// One batch of a codes-pool timbre call: inputs b of the step's sessions, each the StyleEncoder lane of its own N mel
// rows -- the N - 1 its slot keeps and the last one cut by last_mel_row (lanes with equal sample histories share that
// launch) -- in one ragged StyleEncoder; each lane is the session's B = 1 stream_timbre, bit for bit.
int codes_pool_timbre_batch(fac_handle* h, CodesPool& P, const std::vector<int>& b, const int* sessions,
                            float* const* timbre, cudaStream_t st) {
    const int nb = (int)b.size();
    auto sl = [&](int j) -> const EncHalf& { return P.slot[sessions[b[j]]]; };
    std::vector<int> rows((size_t)kLaneRows * nb, 0), N(nb);
    std::map<int, std::vector<int>> by_hist;     // lanes by sample history
    int Tm = 0;
    for (int j = 0; j < nb; ++j) {
        N[j] = (int)(sl(j).samples / HOP);
        rows[(size_t)kTmRow * nb + j] = N[j];
        Tm = std::max(Tm, N[j]);
        by_hist[sl(j).x_hist_len].push_back(j);
    }
    return two_pass(h, st, [&](Ctx& c) {
        c.vq_critical = true;
        const Lanes ln = upload_lanes(c, rows, nb);
        const size_t pitch = (size_t)Tm * N_MELS;
        float* mel = c.alloc<float>((size_t)nb * pitch);
        if (!c.dry) c.check_nk(cudaMemsetAsync(mel, 0, sizeof(float) * nb * pitch, c.st), "pool.mel_zero");
        lane_copy(c, nb, [&](int j) { return (long long)(N[j] - 1) * N_MELS; }, [&](int j) { return sl(j).mel.get(); },
                  [&](int j) { return mel + j * pitch; }, "pool.mel");
        for (const auto& kv : by_hist) {
            const int hist = kv.first, ng = (int)kv.second.size();
            const std::vector<int>& g = kv.second;
            float* xw = c.alloc<float>((size_t)ng * hist);
            lane_copy(c, ng, hist, [&](int k) { return sl(g[k]).x_hist; }, [&](int k) { return xw + (size_t)k * hist; },
                      "pool.x_hist");
            const float* last = last_mel_row(c, xw, ng, hist);
            lane_copy(c, ng, N_MELS, [&](int k) { return last + (size_t)k * N_MELS; },
                      [&](int k) { return mel + g[k] * pitch + (size_t)(N[g[k]] - 1) * N_MELS; }, "pool.mel_last");
        }
        float* tv = c.alloc<float>((size_t)nb * 1024);
        style_encoder(c, mel, nb, Tm, nullptr, tv, &ln);
        lane_copy(c, nb, 1024, [&](int j) { return tv + (size_t)j * 1024; }, [&](int j) { return timbre[b[j]]; }, "pool.timbre");
        c.vq_critical = false;
    });
}

// One batch of a vc-pool step: inputs b (equal plan keys) of the step's sessions.  Their modes may differ: a batch of one
// mode runs the launches of a stream of that mode, a mixed one the same launches with each lane's mode uploaded.
int vc_pool_batch(fac_handle* h, VcPool& P, const std::vector<int>& b, const int* sessions, const std::vector<VcPlan>& plan,
                  const int64_t* const* codes_p, const int64_t* const* codes_c, float* const* y, cudaStream_t st) {
    VcStream& L = P.lanes;
    const VcPlan& p = plan[b[0]];
    const int nb = (int)b.size(), F = p.F;
    auto sl = [&](int j) -> VcStream& { return P.slot[sessions[b[j]]]; };
    const size_t gfl = redecoder_cond_floats(h, 1), cpl = 3 * kVcCodesHist, zpl = (size_t)kVcZHist * LATENT;
    VcMode m = vc_mode(sl(0));
    std::vector<int> lane_mode(2 * nb);
    bool mixed = false;
    for (int j = 0; j < nb; ++j) {
        const VcStream& s = sl(j);
        lane_mode[2 * j] = s.use_p; lane_mode[2 * j + 1] = s.use_c ? s.n_c : 0;
        mixed |= s.use_p != m.use_p || s.use_c != m.use_c || s.n_c != m.n_c;
        m.n_c = std::max(m.n_c, s.n_c);
    }
    const int rows = m.n_c > 0 ? m.n_c : 1;
    L.B = nb;
    int rc = two_pass(h, st, [&](Ctx& c) {
        int64_t* cp = c.alloc<int64_t>((size_t)nb * F);
        int64_t* cc = c.alloc<int64_t>((size_t)nb * rows * F);
        float* yout = c.alloc<float>((size_t)nb * p.k * HOP);
        VcMode mc = m;
        if (mixed) mc.lanes = upload_ints(c, lane_mode);
        lane_copy(c, nb, (long long)gfl, [&](int j) { return sl(j).g; }, [&](int j) { return L.g + j * gfl; }, "pool.g");
        lane_copy(c, nb, 2LL * cpl, [&](int j) { return sl(j).codes; }, [&](int j) { return L.codes + j * cpl; }, "pool.codes");
        lane_copy(c, nb, (long long)p.zhist * LATENT, [&](int j) { return sl(j).z; }, [&](int j) { return L.z + j * zpl; }, "pool.z");
        lane_copy(c, nb, 2LL * F, [&](int j) { return codes_p[b[j]]; }, [&](int j) { return cp + (size_t)j * F; }, "pool.codes_p");
        lane_copy(c, nb, [&](int j) { return 2LL * sl(j).n_c * F; }, [&](int j) { return codes_c[b[j]]; },
                  [&](int j) { return cc + (size_t)j * rows * F; }, "pool.codes_c");
        vc_step(c, L, p, mc, cp, cc, rows, yout);
        lane_copy(c, nb, 2LL * cpl, [&](int j) { return L.codes + j * cpl; }, [&](int j) { return sl(j).codes; }, "pool.codes");
        if (p.znew > 0)
            lane_copy(c, nb, (long long)p.zkeep * LATENT, [&](int j) { return L.z + j * zpl; }, [&](int j) { return sl(j).z; },
                      "pool.z");
        lane_copy(c, nb, (long long)p.k * HOP, [&](int j) { return yout + (size_t)j * p.k * HOP; }, [&](int j) { return y[b[j]]; },
                  "pool.y");
    });
    if (rc) return rc;
    for (int j = 0; j < nb; ++j) vc_commit(sl(j), plan[b[j]]);
    return FAC_OK;
}

// One batch of a decode-pool step: inputs b (equal plan keys) of the step's sessions, fed F frames each, their codes and
// rows per lane.
int dec_pool_batch(fac_handle* h, DecPool& P, const std::vector<int>& b, const int* sessions, const int* F_in,
                   const int64_t* const* codes_p, const int64_t* const* codes_c, const int* n_c, const int64_t* const* codes_r,
                   const int* n_r, float* const* y, cudaStream_t st) {
    DecHalf& L = P.lanes;
    const int nb = (int)b.size();
    auto sl = [&](int j) -> DecHalf& { return P.slot[sessions[b[j]]]; };
    const DecPlan p = dec_plan(sl(0).frames);
    std::vector<int> F(nb);
    for (int j = 0; j < nb; ++j) F[j] = F_in[b[j]];
    const int Fmax = *std::max_element(F.begin(), F.end());
    const size_t zpl = (size_t)6 * LATENT, dpl = (size_t)kDecCtx * 1536;
    L.B = nb;
    int rc = two_pass(h, st, [&](Ctx& c) {
        float* yout = c.alloc<float>((size_t)nb * Fmax * HOP);
        lane_copy(c, nb, (long long)p.zh * LATENT, [&](int j) { return sl(j).z_hist; }, [&](int j) { return L.z_hist + j * zpl; },
                  "pool.z_hist");
        lane_copy(c, nb, (long long)p.dh * 1536, [&](int j) { return sl(j).dy_hist; }, [&](int j) { return L.dy_hist + j * dpl; },
                  "pool.dy_hist");
        lane_carry(c, L.lstm, 1536, 0, nb, [&](int j) { return sl(j).carry; }, 1);
        stream_decode(c, L, p, F.data(), yout, [&](Ctx& c, int B) {
            float* z = c.alloc<float>((size_t)B * Fmax * LATENT);
            if (c.dry) return (const float*)z;
            DeqLaneParams dp;
            for (int i = 0; i < 6; ++i) {
                const VqW& v = h->qw.vq[i];
                dp.vq[i] = VqWeights{c.W(v.w_in), c.W(v.b_in), c.W(v.cb), c.W(v.cbn), c.W(v.cbn2), c.W(v.w_out), c.W(v.b_out)};
            }
            double codes = 0;
            for (int j = 0; j < B; ++j) {
                const int i = b[j];
                dp.codes_p[j] = codes_p[i]; dp.codes_c[j] = codes_c[i]; dp.codes_r[j] = codes_r[i];
                dp.n_c[j] = n_c[i]; dp.n_r[j] = n_r[i]; dp.F[j] = F[j];
                dp.gamma_beta[j] = sl(j).gb;
                codes += (double)F[j] * (1 + n_c[i] + n_r[i]);
            }
            dp.outs = z; dp.n = B; dp.Fmax = Fmax;
            c.begin("dequantize", 2.0 * codes * 8.0 * 1024, 8.0 * codes + 4.0 * 1024 * B * Fmax);
            c.check(launch_dequantize_lanes(dp, c.st), "dequantize_lanes");
            c.end();
            c.tap("dec_pool.latents", z, (size_t)B * Fmax * LATENT);
            return (const float*)z;
        });
        lane_copy(c, nb, [&](int j) { return (long long)std::min(p.zh + F[j], 6) * LATENT; },
                  [&](int j) { return L.z_hist + j * zpl; }, [&](int j) { return sl(j).z_hist; }, "pool.z_hist");
        lane_copy(c, nb, [&](int j) { return (long long)std::min(p.dh + F[j], kDecCtx) * 1536; },
                  [&](int j) { return L.dy_hist + j * dpl; }, [&](int j) { return sl(j).dy_hist; }, "pool.dy_hist");
        lane_carry(c, L.lstm, 1536, 0, nb, [&](int j) { return sl(j).carry; }, 0);
        lane_copy(c, nb, [&](int j) { return (long long)F[j] * HOP; }, [&](int j) { return yout + (size_t)j * Fmax * HOP; },
                  [&](int j) { return y[b[j]]; }, "pool.y");
    });
    if (rc) return rc;
    for (int j = 0; j < nb; ++j) sl(j).frames += F[j];
    return FAC_OK;
}

// A decode-pool slot's gamma | beta from timbre [1][1024], by the B = 1 launch a stream's decode_codes runs on every
// chunk, so the bits are the same.
void dec_slot_gamma_beta(Ctx& c, DecHalf& s, const float* timbre) {
    const float* gb = timbre_gamma_beta(c, timbre, 1);
    if (!c.dry) c.check_nk(cudaMemcpyAsync(s.gb, gb, sizeof(float) * 2048, cudaMemcpyDeviceToDevice, c.st), "pool.gb");
}
}  // namespace

extern "C" {

int fac_codes_pool_create(fac_handle* h, int capacity, int n_c) {
    int rc = check_ready(h, {FAC_ENCODER, FAC_QUANTIZER});
    if (rc) return rc;
    if (capacity < 1 || n_c < 1 || n_c > 2) { h->err = "fac_codes_pool_create: bad arguments (capacity >= 1, 1 <= n_c <= 2)"; return FAC_ERR_INVALID; }
    return pool_create(h, &fac_handle::codes_pools, capacity, "fac_codes_pool_create", [&](Carve& m, EncHalf& s, int B, bool slot) {
        take_enc(m, s, B, slot);
        s.n_c = n_c;
    });
}

int fac_codes_pool_open(fac_handle* h, int pool_id, void* stream) {
    return pool_open(h, &fac_handle::codes_pools, pool_id, "fac_codes_pool_open", [&](EncHalf& s) {
        cudaSetDevice(h->device);
        cudaError_t e = cudaMemsetAsync(s.carry, 0, sizeof(uint32_t) * 2 * carry_words(LATENT, 1), (cudaStream_t)stream);
        if (e != cudaSuccess) { h->err = std::string("fac_codes_pool_open: ") + cudaGetErrorString(e); cudaGetLastError(); return FAC_ERR_CUDA; }
        s.samples = 0; s.x_hist_len = 0; s.ey_hist_len = 0; s.emitted = 0;
        s.mode = EncHalf::kNone;
        return FAC_OK;
    });
}

int fac_codes_pool_encode_codes(fac_handle* h, int pool_id, int n, const int* sessions, const int* T, const float* const* x,
                                int64_t* const* codes_p, int64_t* const* codes_c, int64_t* const* codes_r, int* frames,
                                void* stream) {
    int rc = check_ready(h, {FAC_ENCODER, FAC_QUANTIZER});
    if (rc) return rc;
    const char* who = "fac_codes_pool_encode_codes";
    CodesPool* P = by_id(h, &fac_handle::codes_pools, pool_id);
    if (!P || n < 0 || (n > 0 && (!sessions || !T || !x || !codes_p || !codes_c || !codes_r || !frames))) {
        h->err = "fac_codes_pool_encode_codes: bad arguments";
        return FAC_ERR_INVALID;
    }
    if ((rc = check_sessions(h, *P, n, sessions, who))) return rc;
    std::vector<EncPlan> plan(n);
    std::vector<std::vector<long long>> keys(n);
    int maxWin = 0;
    for (int i = 0; i < n; ++i) {
        const EncHalf& s = P->slot[sessions[i]];
        if (!x[i] || !codes_p[i] || !codes_c[i] || !codes_r[i]) {
            h->err = "fac_codes_pool_encode_codes: null buffer of session " + std::to_string(sessions[i]);
            return FAC_ERR_INVALID;
        }
        if ((rc = stream_encode_codes_check(h, s, T[i], P->lanes.n_c, who))) return rc;
        plan[i] = enc_plan(s, T[i]);
        keys[i] = plan[i].key();
        maxWin = std::max(maxWin, plan[i].Fw);
    }
    if (n == 0) return FAC_OK;
    // capacities: no session changes before every one of these has succeeded
    cudaStream_t st = (cudaStream_t)stream;
    for (int i = 0; i < n; ++i) {
        EncHalf& s = P->slot[sessions[i]];
        if ((rc = grow_mel(h, s, 1, s.emitted, (int)((s.samples + T[i]) / HOP), st))) return rc;
    }
    if ((rc = grow_mel(h, P->lanes, kLaneMax, 0, maxWin, st))) return rc;
    for (const auto& b : pool_plan(keys, nullptr, nullptr))
        if ((rc = codes_pool_batch(h, *P, b, sessions, plan, x, codes_p, codes_c, codes_r, st))) return rc;
    for (int i = 0; i < n; ++i) frames[i] = plan[i].Fout;
    return FAC_OK;
}

int fac_codes_pool_finish_codes(fac_handle* h, int pool_id, int n, const int* sessions, int64_t* const* codes_p,
                                int64_t* const* codes_c, int64_t* const* codes_r, float* const* timbre, void* stream) {
    int rc = check_ready(h, {FAC_ENCODER, FAC_QUANTIZER});
    if (rc) return rc;
    const char* who = "fac_codes_pool_finish_codes";
    CodesPool* P = by_id(h, &fac_handle::codes_pools, pool_id);
    if (!P || n < 0 || (n > 0 && (!sessions || !codes_p || !codes_c || !codes_r))) {
        h->err = "fac_codes_pool_finish_codes: bad arguments";
        return FAC_ERR_INVALID;
    }
    if ((rc = check_sessions(h, *P, n, sessions, who))) return rc;
    for (int i = 0; i < n; ++i) {
        if (!codes_p[i] || !codes_c[i] || !codes_r[i]) {
            h->err = "fac_codes_pool_finish_codes: null buffer of session " + std::to_string(sessions[i]);
            return FAC_ERR_INVALID;
        }
        if ((rc = stream_finish_codes_check(h, P->slot[sessions[i]], who))) return rc;
    }
    for (int i = 0; i < n; ++i) {
        rc = finish_codes(h, P->slot[sessions[i]], codes_p[i], codes_c[i], codes_r[i], timbre ? timbre[i] : nullptr, stream);
        if (rc < 0) return rc;
    }
    return FAC_OK;
}

int fac_codes_pool_timbre(fac_handle* h, int pool_id, int n, const int* sessions, float* const* timbre, void* stream) {
    int rc = check_ready(h, {FAC_ENCODER, FAC_QUANTIZER});
    if (rc) return rc;
    const char* who = "fac_codes_pool_timbre";
    CodesPool* P = by_id(h, &fac_handle::codes_pools, pool_id);
    if (!P || n < 0 || (n > 0 && (!sessions || !timbre))) { h->err = "fac_codes_pool_timbre: bad arguments"; return FAC_ERR_INVALID; }
    if ((rc = check_sessions(h, *P, n, sessions, who))) return rc;
    std::vector<int> N(n);
    for (int i = 0; i < n; ++i) {
        const EncHalf& s = P->slot[sessions[i]];
        if (!timbre[i]) { h->err = "fac_codes_pool_timbre: null output of session " + std::to_string(sessions[i]); return FAC_ERR_INVALID; }
        if ((rc = stream_finish_codes_check(h, s, who))) return rc;
        N[i] = (int)(s.samples / HOP);
    }
    int launches = 0;
    for (const auto& b : timbre_plan(N)) {
        if ((rc = codes_pool_timbre_batch(h, *P, b, sessions, timbre, (cudaStream_t)stream))) return rc;
        launches += h->launches;
    }
    h->launches = launches;
    return FAC_OK;
}

int fac_codes_pool_close(fac_handle* h, int pool_id, int session) {
    return pool_close(h, &fac_handle::codes_pools, pool_id, session, "fac_codes_pool_close");
}

int fac_codes_pool_destroy(fac_handle* h, int pool_id) { return free_by_id(h, &fac_handle::codes_pools, pool_id); }

int fac_vc_pool_create(fac_handle* h, int capacity, int use_p_code, int use_c_code, int n_c) {
    int rc = check_ready(h, {FAC_REDECODER, FAC_REDECODER_DECODER});
    if (rc) return rc;
    if (capacity < 1 || n_c < 0 || n_c > 2) { h->err = "fac_vc_pool_create: bad arguments (capacity >= 1, 0 <= n_c <= 2)"; return FAC_ERR_INVALID; }
    const size_t gfl = redecoder_cond_floats(h, 1);
    return pool_create(h, &fac_handle::vc_pools, capacity, "fac_vc_pool_create", [&](Carve& m, VcStream& s, int B, bool) {
        take_vc(m, s, B, gfl);
        s.use_p = use_p_code ? 1 : 0; s.use_c = use_c_code ? 1 : 0; s.n_c = n_c;
    });
}

int fac_vc_pool_open_mode(fac_handle* h, int pool_id, const float* timbre, int use_p_code, int use_c_code, int n_c,
                          void* stream) {
    int rc = check_ready(h, {FAC_REDECODER, FAC_REDECODER_DECODER});
    if (rc) return rc;
    if (!timbre || n_c < 0 || n_c > 2) { h->err = "fac_vc_pool_open: bad arguments (0 <= n_c <= 2)"; return FAC_ERR_INVALID; }
    return pool_open(h, &fac_handle::vc_pools, pool_id, "fac_vc_pool_open", [&](VcStream& s) {
        s.N = s.Zf = s.Yf = 0;
        s.finished = false;
        s.stale = false;
        s.use_p = use_p_code ? 1 : 0; s.use_c = use_c_code ? 1 : 0; s.n_c = n_c;
        return two_pass(h, (cudaStream_t)stream, [&](Ctx& c) { redecoder_cond(c, timbre, 1, s.g); });
    });
}

int fac_vc_pool_open(fac_handle* h, int pool_id, const float* timbre, void* stream) {
    const VcPool* P = h ? by_id(h, &fac_handle::vc_pools, pool_id) : nullptr;
    if (!P) { if (h) h->err = "fac_vc_pool_open: no such pool"; return FAC_ERR_INVALID; }
    const VcStream& d = P->lanes;       // the pool's options
    return fac_vc_pool_open_mode(h, pool_id, timbre, d.use_p, d.use_c, d.n_c, stream);
}

int fac_vc_pool_set_timbre(fac_handle* h, int pool_id, int session, const float* timbre, void* stream) {
    int rc = check_ready(h, {FAC_REDECODER, FAC_REDECODER_DECODER});
    if (rc) return rc;
    VcPool* P = by_id(h, &fac_handle::vc_pools, pool_id);
    if (!P || !timbre) { h->err = "fac_vc_pool_set_timbre: bad arguments"; return FAC_ERR_INVALID; }
    if (session < 0 || session >= P->cap || !P->used[session]) {
        h->err = "fac_vc_pool_set_timbre: session " + std::to_string(session) + " is not open";
        return FAC_ERR_INVALID;
    }
    VcStream& s = P->slot[session];
    if (s.finished) { h->err = "fac_vc_pool_set_timbre: session " + std::to_string(session) + " was finished"; return FAC_ERR_STATE; }
    return vc_set_timbre(h, s, timbre, stream);
}

int fac_vc_pool_convert(fac_handle* h, int pool_id, int n, const int* sessions, const int* F, const int64_t* const* codes_p,
                        const int64_t* const* codes_c, const int* n_c_rows, float* const* y, int* frames, void* stream) {
    int rc = check_ready(h, {FAC_REDECODER, FAC_REDECODER_DECODER});
    if (rc) return rc;
    const char* who = "fac_vc_pool_convert";
    VcPool* P = by_id(h, &fac_handle::vc_pools, pool_id);
    if (!P || n < 0 || (n > 0 && (!sessions || !F || !codes_p || !codes_c || !n_c_rows || !y || !frames))) {
        h->err = "fac_vc_pool_convert: bad arguments";
        return FAC_ERR_INVALID;
    }
    if ((rc = check_sessions(h, *P, n, sessions, who))) return rc;
    std::vector<VcPlan> plan(n);
    std::vector<std::vector<long long>> keys(n);
    for (int i = 0; i < n; ++i) {
        const VcStream& s = P->slot[sessions[i]];
        if (!codes_p[i] || !codes_c[i] || !y[i] || F[i] <= 0 || n_c_rows[i] < s.n_c || n_c_rows[i] > 2) {
            h->err = "fac_vc_pool_convert: bad arguments of session " + std::to_string(sessions[i]) +
                     " (F >= 1, n_c <= rows of codes_c <= 2)";
            return FAC_ERR_INVALID;
        }
        if (s.finished) { h->err = "fac_vc_pool_convert: session " + std::to_string(sessions[i]) + " was finished"; return FAC_ERR_STATE; }
        plan[i] = vc_plan(s, F[i], false);
        keys[i] = plan[i].key();
    }
    int launches = 0;
    for (const auto& b : pool_plan(keys, nullptr, nullptr)) {
        if ((rc = vc_pool_batch(h, *P, b, sessions, plan, codes_p, codes_c, y, (cudaStream_t)stream))) return rc;
        launches += h->launches;
    }
    h->launches = launches;
    for (int i = 0; i < n; ++i) frames[i] = plan[i].k;
    return FAC_OK;
}

int fac_vc_pool_finish(fac_handle* h, int pool_id, int n, const int* sessions, float* const* y, int* frames, void* stream) {
    int rc = check_ready(h, {FAC_REDECODER, FAC_REDECODER_DECODER});
    if (rc) return rc;
    const char* who = "fac_vc_pool_finish";
    VcPool* P = by_id(h, &fac_handle::vc_pools, pool_id);
    if (!P || n < 0 || (n > 0 && (!sessions || !y || !frames))) { h->err = "fac_vc_pool_finish: bad arguments"; return FAC_ERR_INVALID; }
    if ((rc = check_sessions(h, *P, n, sessions, who))) return rc;
    for (int i = 0; i < n; ++i) {
        const VcStream& s = P->slot[sessions[i]];
        if (!y[i]) { h->err = "fac_vc_pool_finish: null output of session " + std::to_string(sessions[i]); return FAC_ERR_INVALID; }
        if (s.finished || s.N == 0) {
            h->err = "fac_vc_pool_finish: session " + std::to_string(sessions[i]) + (s.finished ? " was finished" : " received no codes");
            return FAC_ERR_STATE;
        }
    }
    for (int i = 0; i < n; ++i) {
        VcStream& s = P->slot[sessions[i]];
        if ((rc = vc_run(h, s, vc_plan(s, 0, true), nullptr, nullptr, 0, y[i], stream)) < 0) return rc;
        frames[i] = rc;
        s.finished = true;
    }
    return FAC_OK;
}

int fac_vc_pool_close(fac_handle* h, int pool_id, int session) {
    return pool_close(h, &fac_handle::vc_pools, pool_id, session, "fac_vc_pool_close");
}

int fac_vc_pool_destroy(fac_handle* h, int pool_id) { return free_by_id(h, &fac_handle::vc_pools, pool_id); }

int fac_dec_pool_create(fac_handle* h, int capacity) {
    int rc = check_ready(h, {FAC_QUANTIZER, FAC_DECODER});
    if (rc) return rc;
    if (capacity < 1) { h->err = "fac_dec_pool_create: bad arguments (capacity >= 1)"; return FAC_ERR_INVALID; }
    return pool_create(h, &fac_handle::dec_pools, capacity, "fac_dec_pool_create", take_dec);
}

int fac_dec_pool_open(fac_handle* h, int pool_id, const float* timbre, void* stream) {
    int rc = check_ready(h, {FAC_QUANTIZER, FAC_DECODER});
    if (rc) return rc;
    if (!timbre) { h->err = "fac_dec_pool_open: bad arguments"; return FAC_ERR_INVALID; }
    return pool_open(h, &fac_handle::dec_pools, pool_id, "fac_dec_pool_open", [&](DecHalf& s) {
        s.frames = 0;
        return two_pass(h, (cudaStream_t)stream, [&](Ctx& c) {
            dec_slot_gamma_beta(c, s, timbre);
            if (!c.dry) c.check_nk(cudaMemsetAsync(s.carry, 0, sizeof(uint32_t) * 2 * carry_words(1536, 0), c.st), "pool.carry");
        });
    });
}

int fac_dec_pool_set_timbre(fac_handle* h, int pool_id, int session, const float* timbre, void* stream) {
    int rc = check_ready(h, {FAC_QUANTIZER, FAC_DECODER});
    if (rc) return rc;
    DecPool* P = by_id(h, &fac_handle::dec_pools, pool_id);
    if (!P || !timbre) { h->err = "fac_dec_pool_set_timbre: bad arguments"; return FAC_ERR_INVALID; }
    if (session < 0 || session >= P->cap || !P->used[session]) {
        h->err = "fac_dec_pool_set_timbre: session " + std::to_string(session) + " is not open";
        return FAC_ERR_INVALID;
    }
    DecHalf& s = P->slot[session];
    return two_pass(h, (cudaStream_t)stream, [&](Ctx& c) { dec_slot_gamma_beta(c, s, timbre); });
}

int fac_dec_pool_decode_codes(fac_handle* h, int pool_id, int n, const int* sessions, const int* F, const int64_t* const* codes_p,
                              const int64_t* const* codes_c, const int* n_c_rows, const int64_t* const* codes_r,
                              const int* n_r_rows, float* const* y, void* stream) {
    int rc = check_ready(h, {FAC_QUANTIZER, FAC_DECODER});
    if (rc) return rc;
    const char* who = "fac_dec_pool_decode_codes";
    DecPool* P = by_id(h, &fac_handle::dec_pools, pool_id);
    if (!P || n < 0 || (n > 0 && (!sessions || !F || !codes_p || !codes_c || !n_c_rows || !codes_r || !n_r_rows || !y))) {
        h->err = "fac_dec_pool_decode_codes: bad arguments";
        return FAC_ERR_INVALID;
    }
    if ((rc = check_sessions(h, *P, n, sessions, who))) return rc;
    std::vector<std::vector<long long>> keys(n);
    for (int i = 0; i < n; ++i) {
        if (!codes_p[i] || !codes_c[i] || !y[i] || (n_r_rows[i] > 0 && !codes_r[i]) || n_c_rows[i] < 1 || n_c_rows[i] > 2 ||
            n_r_rows[i] < 0 || n_r_rows[i] > 3) {
            h->err = "fac_dec_pool_decode_codes: bad arguments of session " + std::to_string(sessions[i]) +
                     " (null buffer, or not 1 <= content rows <= 2, 0 <= residual rows <= 3)";
            return FAC_ERR_INVALID;
        }
        const long long frames = P->slot[sessions[i]].frames;
        if ((rc = stream_decode_check(h, frames, F[i], who))) return rc;
        keys[i] = dec_plan(frames).key();
    }
    for (const auto& b : pool_plan(keys, nullptr, nullptr))
        if ((rc = dec_pool_batch(h, *P, b, sessions, F, codes_p, codes_c, n_c_rows, codes_r, n_r_rows, y, (cudaStream_t)stream)))
            return rc;
    return FAC_OK;
}

int fac_dec_pool_close(fac_handle* h, int pool_id, int session) {
    return pool_close(h, &fac_handle::dec_pools, pool_id, session, "fac_dec_pool_close");
}

int fac_dec_pool_destroy(fac_handle* h, int pool_id) { return free_by_id(h, &fac_handle::dec_pools, pool_id); }

// Sinc resampling (resample.cu): the handle lends the resampler its device, error text, launch counter and state.
static fac::RsEnv rs_env(fac_handle* h) { return fac::RsEnv{h->device, h->err, h->launches, h->rs}; }

int fac_resample_geometry(int orig, int new_rate, int* out4) { return fac::rs_geometry(orig, new_rate, out4); }
long long fac_resample_out_len(int orig, int new_rate, long long n) { return fac::rs_out_len(orig, new_rate, n); }
long long fac_resample_ready(int orig, int new_rate, int quantum, long long seen, long long emitted) {
    return fac::rs_ready(orig, new_rate, quantum, seen, emitted);
}

int fac_resample_table(fac_handle* h, int orig, int new_rate, const float* table_host) {
    return h ? fac::rs_table(rs_env(h), orig, new_rate, table_host) : FAC_ERR_INVALID;
}

int fac_resample(fac_handle* h, const float* x, int B, int T, const int* lengths, int orig, int new_rate, float* y, void* stream) {
    return h ? fac::rs_resample(rs_env(h), x, B, T, lengths, orig, new_rate, y, (cudaStream_t)stream) : FAC_ERR_INVALID;
}

int fac_rs_pool_create(fac_handle* h, int capacity, int quantum) {
    return h ? fac::rs_pool_create(rs_env(h), capacity, quantum) : FAC_ERR_INVALID;
}

int fac_rs_pool_open(fac_handle* h, int pool_id, int orig, int new_rate) {
    return h ? fac::rs_pool_open(rs_env(h), pool_id, orig, new_rate) : FAC_ERR_INVALID;
}

int fac_rs_pool_push(fac_handle* h, int pool_id, int n, const int* sessions, const int* T, const float* const* x, float* const* y,
                     int* counts, void* stream) {
    return h ? fac::rs_pool_step(rs_env(h), pool_id, n, sessions, T, x, y, counts, false, (cudaStream_t)stream) : FAC_ERR_INVALID;
}

int fac_rs_pool_finish(fac_handle* h, int pool_id, int n, const int* sessions, const int* T, const float* const* x,
                       float* const* y, int* counts, void* stream) {
    return h ? fac::rs_pool_step(rs_env(h), pool_id, n, sessions, T, x, y, counts, true, (cudaStream_t)stream) : FAC_ERR_INVALID;
}

int fac_rs_pool_undo(fac_handle* h, int pool_id, int n, const int* sessions) {
    return h ? fac::rs_pool_undo(rs_env(h), pool_id, n, sessions) : FAC_ERR_INVALID;
}

int fac_rs_pool_close(fac_handle* h, int pool_id, int session) {
    return h ? fac::rs_pool_close(rs_env(h), pool_id, session) : FAC_ERR_INVALID;
}

int fac_rs_pool_destroy(fac_handle* h, int pool_id) { return h ? fac::rs_pool_destroy(rs_env(h), pool_id) : FAC_ERR_INVALID; }

}  // extern "C"

// ---- session state (fac_*_pool_export / _import; layout in include/facodec_b200.h) ----
// A kind adapter binds to one pool and knows its slots: read(session) gives an open session's counters and regions;
// place(state) checks an imported state's counters and region sizes against the pool, readies a free slot (growing its
// buffers if need be) and points the state's regions at it, returning the slot; commit(slot, state) opens that slot.  The
// templates below do the rest, alike for every kind: the header, the checks, and one lane_copy launch per region.
namespace {
using fac::SlotState;
constexpr int kStateOptions = 11;

uint64_t kind_fingerprint(int kind, uint64_t a, uint64_t b) {
    const uint64_t v[3] = {(uint64_t)kind, a, b};
    return fnv1a(v, sizeof v);
}

void state_options(const fac_handle* h, int64_t* o) {
    const int64_t v[kStateOptions] = {h->use_tc, h->fuse_res, h->lstm_v2, h->dec_lstm_fp16, h->attn_stream, h->dec_c7_f16,
                                      h->enc_f16, h->enc_tt, h->tc_occ2, h->dec_bf16, h->overlap_front};
    std::copy(v, v + kStateOptions, o);
}

uint64_t header_checksum(const fac_state_header& hd) { return fnv1a(&hd, offsetof(fac_state_header, checksum)); }

bool on_device(const void* p, int device) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) && a.device == device;
}

int state_error(fac_handle* h, const char* who, const std::string& what, int rc) {
    h->err = std::string(who) + ": " + what;
    return rc;
}

void set_regions(SlotState& st, std::initializer_list<std::pair<void*, long long>> r) {
    st.nreg = 0;
    for (const auto& x : r) { st.region[st.nreg] = x.first; st.bytes[st.nreg] = x.second; ++st.nreg; }
}

// Export reads open sessions; import takes the first free slot.
template <typename S>
int check_open(fac_handle* h, const Pool<S>& P, int session, const char* who) {
    if (session < 0 || session >= P.cap || !P.used[session])
        return state_error(h, who, "session " + std::to_string(session) + " is not open", FAC_ERR_INVALID);
    return FAC_OK;
}
template <typename S>
int free_slot(fac_handle* h, const Pool<S>& P, const char* who) {
    int i = 0;
    while (i < P.cap && P.used[i]) ++i;
    if (i == P.cap) return state_error(h, who, "the pool is full (capacity " + std::to_string(P.cap) + ")", FAC_ERR_STATE);
    return i;
}

// Points an imported state at the regions `want` of its readied slot; their sizes must be the header's.
int adopt(fac_handle* h, const SlotState& want, SlotState& st, const char* who) {
    if (!std::equal(want.bytes, want.bytes + FAC_STATE_REGIONS, st.bytes))
        return state_error(h, who, "the region sizes disagree with the counters", FAC_ERR_INVALID);
    std::copy(want.region, want.region + FAC_STATE_REGIONS, st.region);
    st.nreg = want.nreg;
    return FAC_OK;
}

// counters {n_c, mode, samples, emitted, x_hist_len, ey_hist_len}; regions {x_hist, ey_hist, z_held, carry, mel rows}
struct CodesKind {
    static constexpr int kind = FAC_STATE_CODES;
    fac_handle* h = nullptr; CodesPool* P = nullptr;
    int bind(fac_handle* hh, int id, const char* who) {
        h = hh;
        if (int rc = check_ready(h, {FAC_ENCODER, FAC_QUANTIZER})) return rc;
        P = by_id(h, &fac_handle::codes_pools, id);
        return P ? FAC_OK : state_error(h, who, "no such pool", FAC_ERR_INVALID);
    }
    uint64_t fingerprint() const { return kind_fingerprint(kind, h->fp[FAC_ENCODER], h->fp[FAC_QUANTIZER]); }
    static void regions(const EncHalf& s, long long rows, SlotState& st) {
        set_regions(st, {{s.x_hist, 4LL * kEncCtx}, {s.ey_hist, 4LL * 2 * LATENT}, {s.z_held, 4LL * LATENT},
                         {s.carry, 4LL * 2 * carry_words(LATENT, 1)}, {s.mel.get(), 4LL * N_MELS * rows}});
    }
    int read(int sid, SlotState& st, const char* who) {
        if (int rc = check_open(h, *P, sid, who)) return rc;
        const EncHalf& s = P->slot[sid];
        if (s.mode == EncHalf::kFinished)
            return state_error(h, who, "session " + std::to_string(sid) + " was finished by finish_codes", FAC_ERR_STATE);
        const long long c[6] = {P->lanes.n_c, s.mode, s.samples, s.emitted, s.x_hist_len, s.ey_hist_len};
        std::copy(c, c + 6, st.counters);
        regions(s, s.emitted, st);
        return FAC_OK;
    }
    int place(SlotState& st, const char* who, cudaStream_t stream) {
        const long long* c = st.counters;
        if (c[0] != P->lanes.n_c)
            return state_error(h, who, "the state's n_c " + std::to_string(c[0]) + " is not the pool's " + std::to_string(P->lanes.n_c),
                               FAC_ERR_STATE);
        const long long S = c[2], frames = S / HOP;
        if (!((c[1] == EncHalf::kNone && S == 0) || (c[1] == EncHalf::kCodes && S >= kStreamMinFirst * HOP)) || S % HOP ||
            c[3] != (S ? frames - 1 : 0) || c[4] != std::min<long long>(S, kEncCtx) || c[5] != std::min<long long>(frames, 2) ||
            frames > (1LL << 30))
            return state_error(h, who, "the encoder counters are inconsistent", FAC_ERR_INVALID);
        int i = free_slot(h, *P, who);
        if (i < 0) return i;
        EncHalf& s = P->slot[i];
        if (int rc = grow_mel(h, s, 1, 0, (int)c[3], stream)) return rc;
        SlotState want;
        regions(s, c[3], want);
        return adopt(h, want, st, who) ? FAC_ERR_INVALID : i;
    }
    void commit(int i, const SlotState& st) {
        EncHalf& s = P->slot[i];
        s.mode = (int)st.counters[1]; s.samples = st.counters[2]; s.emitted = st.counters[3];
        s.x_hist_len = (int)st.counters[4]; s.ey_hist_len = (int)st.counters[5];
        P->used[i] = 1;
    }
};

// counters {use_p, use_c, n_c, stale, N, Zf, Yf}; regions {g, codes, z}
struct VcKind {
    static constexpr int kind = FAC_STATE_VC;
    fac_handle* h = nullptr; VcPool* P = nullptr;
    int bind(fac_handle* hh, int id, const char* who) {
        h = hh;
        if (int rc = check_ready(h, {FAC_REDECODER, FAC_REDECODER_DECODER})) return rc;
        P = by_id(h, &fac_handle::vc_pools, id);
        return P ? FAC_OK : state_error(h, who, "no such pool", FAC_ERR_INVALID);
    }
    uint64_t fingerprint() const { return kind_fingerprint(kind, h->fp[FAC_REDECODER], h->fp[FAC_REDECODER_DECODER]); }
    void regions(const VcStream& s, SlotState& st) const {
        set_regions(st, {{s.g, 4LL * (long long)redecoder_cond_floats(h, 1)}, {s.codes, 8LL * 3 * kVcCodesHist},
                         {s.z, 4LL * kVcZHist * LATENT}});
    }
    int read(int sid, SlotState& st, const char* who) {
        if (int rc = check_open(h, *P, sid, who)) return rc;
        const VcStream& s = P->slot[sid];
        if (s.finished) return state_error(h, who, "session " + std::to_string(sid) + " was finished", FAC_ERR_STATE);
        const long long c[7] = {s.use_p, s.use_c, s.n_c, s.stale, s.N, s.Zf, s.Yf};
        std::copy(c, c + 7, st.counters);
        regions(s, st);
        return FAC_OK;
    }
    int place(SlotState& st, const char* who, cudaStream_t) {
        const long long* c = st.counters;
        if (c[0] < 0 || c[0] > 1 || c[1] < 0 || c[1] > 1 || c[2] < 0 || c[2] > 2 || c[3] < 0 || c[3] > 1 || c[6] < 0 ||
            c[6] > c[5] || c[5] > c[4])
            return state_error(h, who, "the conversion counters are inconsistent", FAC_ERR_INVALID);
        int i = free_slot(h, *P, who);
        if (i < 0) return i;
        SlotState want;
        regions(P->slot[i], want);
        return adopt(h, want, st, who) ? FAC_ERR_INVALID : i;
    }
    void commit(int i, const SlotState& st) {
        VcStream& s = P->slot[i];
        const long long* c = st.counters;
        s.use_p = (int)c[0]; s.use_c = (int)c[1]; s.n_c = (int)c[2]; s.stale = c[3] != 0; s.N = c[4]; s.Zf = c[5]; s.Yf = c[6];
        s.finished = false;
        P->used[i] = 1;
    }
};

// counters {frames}; regions {z_hist, dy_hist, carry, gamma | beta}
struct DecKind {
    static constexpr int kind = FAC_STATE_DEC;
    fac_handle* h = nullptr; DecPool* P = nullptr;
    int bind(fac_handle* hh, int id, const char* who) {
        h = hh;
        if (int rc = check_ready(h, {FAC_QUANTIZER, FAC_DECODER})) return rc;
        P = by_id(h, &fac_handle::dec_pools, id);
        return P ? FAC_OK : state_error(h, who, "no such pool", FAC_ERR_INVALID);
    }
    uint64_t fingerprint() const { return kind_fingerprint(kind, h->fp[FAC_QUANTIZER], h->fp[FAC_DECODER]); }
    static void regions(const DecHalf& s, SlotState& st) {
        set_regions(st, {{s.z_hist, 4LL * 6 * LATENT}, {s.dy_hist, 4LL * kDecCtx * 1536}, {s.carry, 4LL * 2 * carry_words(1536, 0)},
                         {s.gb, 4LL * 2048}});
    }
    int read(int sid, SlotState& st, const char* who) {
        if (int rc = check_open(h, *P, sid, who)) return rc;
        st.counters[0] = P->slot[sid].frames;
        regions(P->slot[sid], st);
        return FAC_OK;
    }
    int place(SlotState& st, const char* who, cudaStream_t) {
        if (st.counters[0] < 0) return state_error(h, who, "the decoder counters are inconsistent", FAC_ERR_INVALID);
        int i = free_slot(h, *P, who);
        if (i < 0) return i;
        SlotState want;
        regions(P->slot[i], want);
        return adopt(h, want, st, who) ? FAC_ERR_INVALID : i;
    }
    void commit(int i, const SlotState& st) {
        P->slot[i].frames = st.counters[0];
        P->used[i] = 1;
    }
};

// resample.cu keeps the slots; see fac::rs_slot_read / _place / _commit
struct RsKind {
    static constexpr int kind = FAC_STATE_RS;
    fac_handle* h = nullptr; int id = -1;
    int bind(fac_handle* hh, int pid, const char*) {     // read and place check the pool id
        h = hh; id = pid;
        return FAC_OK;
    }
    uint64_t fingerprint() const { return 0; }
    int read(int sid, SlotState& st, const char* who) { return fac::rs_slot_read(rs_env(h), id, sid, st, who); }
    int place(SlotState& st, const char* who, cudaStream_t) { return fac::rs_slot_place(rs_env(h), id, st, who); }
    void commit(int i, const SlotState& st) { fac::rs_slot_commit(rs_env(h), id, i, st); }
};

// Moves region r of n states: src(i, r) -> dst(i, r), one launch per region for up to kMoveLanes states.
template <typename Src, typename Dst>
int move_regions(fac_handle* h, int n, int nreg, const std::vector<SlotState>& st, Src src, Dst dst, cudaStream_t stream) {
    return two_pass(h, stream, [&](Ctx& c) {
        for (int r = 0; r < nreg; ++r)
            for (int o = 0; o < n; o += kMoveLanes)
                lane_copy<kMoveLanes>(c, std::min(n - o, kMoveLanes), [&](int b) { return st[o + b].bytes[r] / 4; },
                                      [&](int b) { return src(o + b, r); }, [&](int b) { return dst(o + b, r); }, "state.region");
    });
}

long long payload_offset(const SlotState& st, int r) {
    long long off = 0;
    for (int k = 0; k < r; ++k) off += st.bytes[k];
    return off;
}

template <typename K>
int state_size(fac_handle* h, int pool_id, int session, size_t* header_bytes, size_t* payload_bytes, const char* who) {
    if (!h) return FAC_ERR_INVALID;
    K k;
    if (int rc = k.bind(h, pool_id, who)) return rc;
    if (!header_bytes || !payload_bytes) return state_error(h, who, "null output", FAC_ERR_INVALID);
    SlotState st;
    if (int rc = k.read(session, st, who)) return rc;
    *header_bytes = sizeof(fac_state_header);
    *payload_bytes = (size_t)payload_offset(st, st.nreg);
    return FAC_OK;
}

template <typename K>
int state_export(fac_handle* h, int pool_id, int n, const int* sessions, void* const* headers, void* const* payloads, void* stream,
                 const char* who) {
    if (!h) return FAC_ERR_INVALID;
    K k;
    if (int rc = k.bind(h, pool_id, who)) return rc;
    if (n < 0 || (n > 0 && (!sessions || !headers || !payloads))) return state_error(h, who, "bad arguments", FAC_ERR_INVALID);
    std::vector<SlotState> st(n);
    std::vector<int> seen;
    for (int i = 0; i < n; ++i) {
        if (int rc = k.read(sessions[i], st[i], who)) return rc;
        if (std::find(seen.begin(), seen.end(), sessions[i]) != seen.end())
            return state_error(h, who, "session " + std::to_string(sessions[i]) + " is named twice", FAC_ERR_INVALID);
        seen.push_back(sessions[i]);
        if (!headers[i] || (payload_offset(st[i], st[i].nreg) > 0 &&
                            (!payloads[i] || (uintptr_t)payloads[i] % 4 || !on_device(payloads[i], h->device))))
            return state_error(h, who, "session " + std::to_string(sessions[i]) +
                                       ": a null header, or a payload that is not 4-byte aligned memory of the handle's device",
                               FAC_ERR_INVALID);
    }
    const uint64_t fp = k.fingerprint();
    for (int i = 0; i < n; ++i) {
        fac_state_header hd;
        std::memset(&hd, 0, sizeof hd);
        hd.magic = FAC_STATE_MAGIC; hd.version = FAC_STATE_VERSION; hd.kind = K::kind; hd.header_bytes = sizeof hd;
        hd.fingerprint = fp;
        state_options(h, hd.options);
        std::copy(st[i].counters, st[i].counters + FAC_STATE_COUNTERS, hd.counters);
        std::copy(st[i].bytes, st[i].bytes + st[i].nreg, hd.region_bytes);
        hd.payload_bytes = (uint64_t)payload_offset(st[i], st[i].nreg);
        hd.checksum = header_checksum(hd);
        std::memcpy(headers[i], &hd, sizeof hd);
    }
    if (n == 0) { h->launches = 0; return FAC_OK; }
    return move_regions(h, n, st[0].nreg, st, [&](int i, int r) { return st[i].region[r]; },
                        [&](int i, int r) { return (char*)payloads[i] + payload_offset(st[i], r); }, (cudaStream_t)stream);
}

// The header checks of an import into a pool of `kind` whose weights give `fp` and whose handle has options `opts`: on
// success st holds the header's counters and region sizes.  Host only (fac_debug_state_header).
int check_header(const void* header, size_t header_bytes, int kind, uint64_t fp, const int64_t* opts, size_t payload_bytes,
                 SlotState& st, std::string& err) {
    fac_state_header hd;
    auto fail = [&](const std::string& what, int rc) { err = what; return rc; };
    if (!header || header_bytes < sizeof hd) return fail("the header is missing or truncated", FAC_ERR_INVALID);
    std::memcpy(&hd, header, sizeof hd);
    if (hd.magic != FAC_STATE_MAGIC || hd.header_bytes != sizeof hd || header_bytes != sizeof hd)
        return fail("not a session-state header", FAC_ERR_INVALID);
    if (hd.checksum != header_checksum(hd)) return fail("the header is corrupt (checksum)", FAC_ERR_INVALID);
    if (hd.version != FAC_STATE_VERSION)
        return fail("state format version " + std::to_string(hd.version) + ", this library reads " + std::to_string(FAC_STATE_VERSION),
                    FAC_ERR_STATE);
    if (hd.kind != (uint32_t)kind)
        return fail("a state of pool kind " + std::to_string(hd.kind) + ", this pool is kind " + std::to_string(kind), FAC_ERR_INVALID);
    if (hd.fingerprint != fp) return fail("the state comes from other weights", FAC_ERR_STATE);
    if (!std::equal(opts, opts + FAC_STATE_OPTIONS, hd.options))
        return fail("the state comes from a handle with other fac_set_option values", FAC_ERR_STATE);
    std::copy(hd.counters, hd.counters + FAC_STATE_COUNTERS, st.counters);
    unsigned long long total = 0;
    for (int r = 0; r < FAC_STATE_REGIONS; ++r) {
        if (hd.region_bytes[r] < 0 || hd.region_bytes[r] % 4 || hd.region_bytes[r] > (1LL << 40)) return fail("a bad region size", FAC_ERR_INVALID);
        st.bytes[r] = hd.region_bytes[r];
        total += (unsigned long long)hd.region_bytes[r];
    }
    if (total != hd.payload_bytes || payload_bytes != hd.payload_bytes)
        return fail("the payload size disagrees with the header", FAC_ERR_INVALID);
    return FAC_OK;
}

template <typename K>
int state_import(fac_handle* h, int pool_id, const void* header, size_t header_bytes, const void* payload, size_t payload_bytes,
                 void* stream, const char* who) {
    if (!h) return FAC_ERR_INVALID;
    K k;
    if (int rc = k.bind(h, pool_id, who)) return rc;
    int64_t opts[FAC_STATE_OPTIONS] = {};
    state_options(h, opts);
    SlotState st;
    std::string why;
    if (int rc = check_header(header, header_bytes, K::kind, k.fingerprint(), opts, payload_bytes, st, why))
        return state_error(h, who, why, rc);
    if (payload_bytes > 0 && (!payload || (uintptr_t)payload % 4 || !on_device(payload, h->device)))
        return state_error(h, who, "the payload is not 4-byte aligned memory of the handle's device (cuda:" +
                                   std::to_string(h->device) + ")", FAC_ERR_INVALID);
    const int slot = k.place(st, who, (cudaStream_t)stream);
    if (slot < 0) return slot;
    std::vector<SlotState> one{st};
    int rc = move_regions(h, 1, st.nreg, one, [&](int, int r) { return (const char*)payload + payload_offset(st, r); },
                          [&](int, int r) { return st.region[r]; }, (cudaStream_t)stream);
    if (rc) return rc;
    k.commit(slot, st);
    return slot;
}
}  // namespace

extern "C" {

int fac_codes_pool_export_size(fac_handle* h, int pool_id, int session, size_t* header_bytes, size_t* payload_bytes) {
    return state_size<CodesKind>(h, pool_id, session, header_bytes, payload_bytes, "fac_codes_pool_export_size");
}
int fac_codes_pool_export(fac_handle* h, int pool_id, int n, const int* sessions, void* const* headers, void* const* payloads,
                          void* stream) {
    return state_export<CodesKind>(h, pool_id, n, sessions, headers, payloads, stream, "fac_codes_pool_export");
}
int fac_codes_pool_import(fac_handle* h, int pool_id, const void* header, size_t header_bytes, const void* payload,
                          size_t payload_bytes, void* stream) {
    return state_import<CodesKind>(h, pool_id, header, header_bytes, payload, payload_bytes, stream, "fac_codes_pool_import");
}
int fac_vc_pool_export_size(fac_handle* h, int pool_id, int session, size_t* header_bytes, size_t* payload_bytes) {
    return state_size<VcKind>(h, pool_id, session, header_bytes, payload_bytes, "fac_vc_pool_export_size");
}
int fac_vc_pool_export(fac_handle* h, int pool_id, int n, const int* sessions, void* const* headers, void* const* payloads,
                       void* stream) {
    return state_export<VcKind>(h, pool_id, n, sessions, headers, payloads, stream, "fac_vc_pool_export");
}
int fac_vc_pool_import(fac_handle* h, int pool_id, const void* header, size_t header_bytes, const void* payload,
                       size_t payload_bytes, void* stream) {
    return state_import<VcKind>(h, pool_id, header, header_bytes, payload, payload_bytes, stream, "fac_vc_pool_import");
}
int fac_dec_pool_export_size(fac_handle* h, int pool_id, int session, size_t* header_bytes, size_t* payload_bytes) {
    return state_size<DecKind>(h, pool_id, session, header_bytes, payload_bytes, "fac_dec_pool_export_size");
}
int fac_dec_pool_export(fac_handle* h, int pool_id, int n, const int* sessions, void* const* headers, void* const* payloads,
                        void* stream) {
    return state_export<DecKind>(h, pool_id, n, sessions, headers, payloads, stream, "fac_dec_pool_export");
}
int fac_dec_pool_import(fac_handle* h, int pool_id, const void* header, size_t header_bytes, const void* payload,
                        size_t payload_bytes, void* stream) {
    return state_import<DecKind>(h, pool_id, header, header_bytes, payload, payload_bytes, stream, "fac_dec_pool_import");
}
int fac_rs_pool_export_size(fac_handle* h, int pool_id, int session, size_t* header_bytes, size_t* payload_bytes) {
    return state_size<RsKind>(h, pool_id, session, header_bytes, payload_bytes, "fac_rs_pool_export_size");
}
int fac_rs_pool_export(fac_handle* h, int pool_id, int n, const int* sessions, void* const* headers, void* const* payloads,
                       void* stream) {
    return state_export<RsKind>(h, pool_id, n, sessions, headers, payloads, stream, "fac_rs_pool_export");
}
int fac_rs_pool_import(fac_handle* h, int pool_id, const void* header, size_t header_bytes, const void* payload,
                       size_t payload_bytes, void* stream) {
    return state_import<RsKind>(h, pool_id, header, header_bytes, payload, payload_bytes, stream, "fac_rs_pool_import");
}

int fac_debug_pool_plan(int kind, int n, const long long* counters, const int* lengths, int* group, int* batch) {
    if (n < 0 || (n > 0 && (!counters || !lengths || !group || !batch)) || kind < 0 || kind > 3) return FAC_ERR_INVALID;
    std::vector<std::vector<long long>> keys(n);
    for (int i = 0; i < n; ++i) {
        const long long* c = counters + (size_t)i * (kind == 0 ? 4 : kind == 1 ? 3 : kind == 2 ? 1 : 4);
        keys[i] = kind == 0 ? enc_plan(c[0], (int)c[1], (int)c[2], c[3], lengths[i]).key()
                : kind == 1 ? vc_plan(c[0], c[1], c[2], lengths[i], false).key()
                : kind == 2 ? dec_plan(c[0]).key() : vc_plan(c[0], c[1], c[2], lengths[i], false, c[3] != 0).key();
    }
    return (int)pool_plan(keys, group, batch).size();
}

int fac_debug_state_header(const void* header, size_t header_bytes, int kind, uint64_t fingerprint, const int64_t* options,
                           size_t payload_bytes, long long* counters_out) {
    if (!options) return FAC_ERR_INVALID;
    SlotState st;
    std::string why;
    int rc = check_header(header, header_bytes, kind, fingerprint, options, payload_bytes, st, why);
    if (rc == FAC_OK && counters_out) std::copy(st.counters, st.counters + FAC_STATE_COUNTERS, counters_out);
    return rc;
}

int fac_debug_vc_plan(long long N, long long Zf, long long Yf, int F, int finish, int stale, long long* out16) {
    if (!out16 || F < 0 || (F == 0) != (finish != 0)) return FAC_ERR_INVALID;
    const VcPlan p = vc_plan(N, Zf, Yf, F, finish != 0, stale != 0);
    const long long v[16] = {p.F, p.Tw, p.hist, p.Tz, p.zhist, p.zoff, p.znew, p.k, p.yoff, p.zkeep_at, p.zkeep, p.stale,
                             p.N1, p.Zf1, p.Yf1, kVcCodesHist};
    std::copy(v, v + 16, out16);
    return 16;
}

int fac_debug_timbre_plan(int n, const int* frames, int* batch) {
    if (n < 0 || (n > 0 && (!frames || !batch))) return FAC_ERR_INVALID;
    const auto batches = timbre_plan(std::vector<int>(frames, frames + n));
    for (size_t k = 0; k < batches.size(); ++k)
        for (int i : batches[k]) batch[i] = (int)k;
    return (int)batches.size();
}

long long fac_debug_lstm_lane_map(int H, int pass3, int lane, long long* pos, long long capacity) {
    const int U = lstm_units_per_cta(H);
    if (U == 0 || lane < 0 || lane >= kLaneMax) return FAC_ERR_INVALID;
    const long long words = carry_words(H, pass3);
    if (pos && capacity >= words) lstm2_lane_map(H, U, pass3 ? 1 : 0, lane, pos);
    return words;
}

// meldataset.py:37-47 preprocess: torchaudio MelSpectrogram(n_mels=80, n_fft=2048, win_length=1200, hop_length=300) with
// its DEFAULT sample_rate = 16000 (HTK filterbank over [0, 8000] Hz -- not the quantizer's 24 kHz one), centre = True
// (T/300 + 1 frames), then (log(1e-5 + mel) + 4) / 4.
int fac_dataset_mel(fac_handle* h, const float* wave, int B, int T, float* mel, void* stream) {
    if (!h || !wave || !mel || B <= 0) return FAC_ERR_INVALID;
    if (T <= N_FFT / 2) { h->err = "fac_dataset_mel: wave shorter than the STFT reflect padding (1024), as torch.stft"; return FAC_ERR_INVALID; }
    if (!h->mel16_arena) {
        const std::vector<double> hann = periodic_hann(WIN);
        const std::vector<float> win(hann.begin(), hann.end());
        Packer P;
        pack_mel_frontend(P, h->mel16_dft, h->mel16_dft_tc, h->mel16_fb, win.data(), htk_fbank(8000.0, N_BINS, N_MELS).data());
        const int rc = upload_weights(h, P, h->mel16_arena, "fac_dataset_mel");
        if (rc != FAC_OK) return rc;
    }
    const int F = T / HOP + 1;
    return two_pass(h, (cudaStream_t)stream, h->mel16_arena.get(), [&](Ctx& c) {
        MelW mw{&h->mel16_dft, &h->mel16_dft_tc, h->mel16_fb};
        c.vq_critical = true;                        // fp32-faithful DFT (the promoted tensor-core kernel)
        float* mel_cl = mel_forward(c, wave, B, T, F, &mw);
        c.vq_critical = false;
        if (!c.dry) c.check(launch_transpose(mel_cl, mel, B, F, N_MELS, c.st), "mel16.T");
    });
}

// ---- losses.py:65-89 reconstruction_loss (SURVEY.md 8f rank 3: the loss forward of the training step) ----
// L = 100 * mse(x, G_x) + sum_{s = 64..2048} (l1_s + sqrt(s/2) * l2_s) over 64-band mel spectrograms
// (torchaudio MelSpectrogram(sample_rate=16000, n_fft=max(s,512), win_length=s, hop_length=s/4, n_mels=64): periodic Hann
// window of s samples centred in the n_fft frame, centre = True reflect padding, power 2, HTK bands over [0, 8000] Hz).
// Per scale: frame gather of both signals -> one GEMM against the window-folded DFT basis (fp32-faithful tensor-core class)
// -> mel_loss_terms_kernel -> fp64 sums in a fixed order.
int fac_reconstruction_loss(fac_handle* h, const float* x, const float* gx, int B, int T, float* loss, float* terms, void* stream) {
    if (!h || !x || !gx || !loss || B <= 0 || T <= 0) return FAC_ERR_INVALID;
    if (T <= 1024) { h->err = "fac_reconstruction_loss: signals must be longer than the largest STFT reflect padding (1024), as torch.stft"; return FAC_ERR_INVALID; }
    if (B > 32767) { h->err = "fac_reconstruction_loss: B > 32767"; return FAC_ERR_UNSUPPORTED; }
    if (!h->loss_arena) {
        Packer P;
        for (int i = 0; i < 6; ++i) {
            fac_handle::LossScale& L = h->loss_scale[i];
            L.s = 64 << i; L.nfft = L.s < 512 ? 512 : L.s; L.nb = L.nfft / 2 + 1;
            L.ld = (2 * L.nb + 127) / 128 * 128;            // zero columns beyond 2 * nb: whole 128-channel MMA tiles
            ConvW& d = L.dft;
            d = ConvW();
            d.Cin = L.s; d.Cout = L.ld; d.K = 1; d.ldw = L.ld;
            d.w = P.alloc((size_t)L.s * L.ld);
            d.b = P.alloc(L.ld);
            dft_basis(P.pack.data() + d.w, L.ld, periodic_hann(L.s), L.nfft, L.nb, (L.nfft - L.s) / 2);
            attach_tc(P, d, 1, true);
            const std::vector<float> fb = htk_fbank(8000.0, L.nb, 64);
            L.fb = P.alloc(fb.size());
            std::copy(fb.begin(), fb.end(), P.pack.begin() + L.fb);
        }
        const int rc = upload_weights(h, P, h->loss_arena, "fac_reconstruction_loss");
        if (rc != FAC_OK) return rc;
    }
    return two_pass(h, (cudaStream_t)stream, h->loss_arena.get(), [&](Ctx& c) {
        double* sums = c.alloc<double>(16);
        const int nblk = 1024;
        float* part = c.alloc<float>(nblk);
        if (!c.dry) {
            c.check(launch_sqdiff_partial(x, gx, (long long)B * T, part, nblk, c.st), "loss.mse");
            c.check(launch_strided_sum(part, nblk, 1, 1.0 / ((double)B * T), sums, c.st), "loss.mse.sum");
        }
        const size_t mark = c.off;                                   // the scales run one after another on one stream:
        size_t peak = c.off;                                         // they share the scratch above this mark
        c.vq_critical = true;                                        // fp32-faithful DFT (promoted tensor-core class)
        for (int i = 0; i < 6; ++i) {
            c.off = mark;
            const fac_handle::LossScale& L = c.h->loss_scale[i];
            const int hop = L.s / 4, F = T / hop + 1;
            const size_t rows = (size_t)2 * B * F;
            float* frames = c.alloc<float>(rows * L.s);
            float* spec = c.alloc<float>(rows * L.ld);
            float* tr = c.alloc<float>((size_t)B * F * 2);
            if (!c.dry) {
                c.check(launch_stft_frames(x, frames, B, T, F, hop, L.s, L.s / 2, c.st), "loss.frames");
                c.check(launch_stft_frames(gx, frames + (size_t)B * F * L.s, B, T, F, hop, L.s, L.s / 2, c.st), "loss.frames");
            }
            run_conv(c, L.dft, frames, spec, 1, (int)rows, (int)rows, ConvOpts(), "loss.dft");
            if (!c.dry) {
                c.check(launch_mel_loss_terms(spec, L.ld, L.nb, c.W(L.fb), B, F, 1e-7f, tr, c.st), "loss.mel");
                c.check(launch_strided_sum(tr, (long long)B * F, 2, 1.0 / ((double)B * F * 64.0), sums + 1 + 2 * i, c.st), "loss.l1");
                c.check(launch_strided_sum(tr + 1, (long long)B * F, 2, 1.0 / ((double)B * F), sums + 2 + 2 * i, c.st), "loss.l2");
            }
            // before the next scale reuses the scratch (the tap copies are ordered on c.st)
            const std::string si = std::to_string(i);
            c.tap(("recon.dft." + si).c_str(), spec, rows * L.ld);
            c.tap(("recon.terms." + si).c_str(), tr, (size_t)B * F * 2);
            c.tap(("recon.fb." + si).c_str(), c.W(L.fb), (size_t)L.nb * 64);
            if (c.off > peak) peak = c.off;
        }
        c.vq_critical = false;
        c.off = peak;
        if (!c.dry) c.check(launch_loss_combine(sums, loss, terms, c.st), "loss.combine");
    });
}

// ---- dac/nn/loss.py:142-327 MultiScaleSTFTLoss / MelSpectrogramLoss, :11-47 L1Loss (forward values) ----
// The reference computes them on audiotools AudioSignal objects (AudioSignal.stft / .magnitude / .mel_spectrogram; the
// package is not vendored: SURVEY.md 8c, parity unpinned).  Restated semantics: torch.stft(n_fft = window_length, hop =
// window_length / 4, periodic Hann window (scipy.signal.get_window("hann")), centre = True, reflect padding), magnitude =
// |stft|; mel_spectrogram = magnitude @ librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax)^T (Slaney scale, Slaney area
// normalisation).  loss = sum over scales of log_weight * L1(log10(clamp(v, eps)^pow)) + mag_weight * L1(v).
namespace {
void slaney_mel_fb(double sr, int n_fft, int n_mels, double fmin, double fmax, std::vector<float>& fb /* [nb][n_mels] */) {
    const int nb = n_fft / 2 + 1;
    const double f_sp = 200.0 / 3.0, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = std::log(6.4) / 27.0;
    auto hz2mel = [&](double f) { return f >= min_log_hz ? min_log_mel + std::log(f / min_log_hz) / logstep : f / f_sp; };
    auto mel2hz = [&](double m) { return m >= min_log_mel ? min_log_hz * std::exp(logstep * (m - min_log_mel)) : f_sp * m; };
    std::vector<double> mf(n_mels + 2);
    const double m0 = hz2mel(fmin), m1 = hz2mel(fmax);
    for (int i = 0; i < n_mels + 2; ++i) mf[i] = mel2hz(m0 + (m1 - m0) * i / (n_mels + 1));
    fb.assign((size_t)nb * n_mels, 0.f);
    for (int k = 0; k < nb; ++k) {
        const double f = (sr / 2.0) * k / (nb - 1);
        for (int m = 0; m < n_mels; ++m) {
            const double lower = (f - mf[m]) / (mf[m + 1] - mf[m]), upper = (mf[m + 2] - f) / (mf[m + 2] - mf[m + 1]);
            const double w = std::max(0.0, std::min(lower, upper)) * (2.0 / (mf[m + 2] - mf[m]));
            fb[(size_t)k * n_mels + m] = (float)w;
        }
    }
}
}  // namespace

// dx / dy (either may be null): dL/dx, dL/dy [B][T].  Per scale, after the loss terms: spec_loss_grad_kernel turns the spec
// rows of the requested signals into dL/d(Re, Im) in place, the transposed DFT GEMM (same fp32-faithful class) maps them to
// dL/dframes over the frames buffer, and the overlap-add gather folds those into dx / dy (the first scale writes, the later
// ones add, on one stream: bit-reproducible).  With both null this is the forward call, launch for launch.
static int spectral_loss(fac_handle* h, const float* x, const float* y, int B, int T, int sample_rate, int n_scales, const int* window_lengths,
                         const int* n_mels, const float* mel_fmin, const float* mel_fmax, float clamp_eps, float mag_weight, float log_weight,
                         float pw, float* loss, float* dx, float* dy, void* stream) {
    if (!h || !x || !y || !loss || !window_lengths || B <= 0 || T <= 0 || n_scales < 1 || n_scales > 16 || sample_rate <= 0) return FAC_ERR_INVALID;
    if (B > 32767) { h->err = "fac_spectral_loss: B > 32767"; return FAC_ERR_UNSUPPORTED; }
    std::vector<double> key{(double)sample_rate, (double)n_scales};
    for (int i = 0; i < n_scales; ++i) {
        const int w = window_lengths[i];
        if (w < 16 || w > 4096 || (w & (w - 1)) != 0) { h->err = "fac_spectral_loss: window lengths must be powers of two in [16, 4096]"; return FAC_ERR_UNSUPPORTED; }
        if (T <= w / 2) { h->err = "fac_spectral_loss: signals must be longer than half the largest window (reflect padding), as torch.stft"; return FAC_ERR_INVALID; }
        const int nm = n_mels ? n_mels[i] : 0;
        if (nm < 0 || nm > 1024) return FAC_ERR_INVALID;
        const double f0 = (n_mels && mel_fmin) ? mel_fmin[i] : 0.0;
        const double f1 = (n_mels && mel_fmax && mel_fmax[i] > 0.f) ? mel_fmax[i] : sample_rate / 2.0;
        key.push_back(w); key.push_back(nm); key.push_back(f0); key.push_back(f1);
    }
    if (!h->spec_arena || h->spec_key != key) {
        Packer P;
        std::vector<fac_handle::SpecScale> scales(n_scales);
        for (int i = 0; i < n_scales; ++i) {
            fac_handle::SpecScale& L = scales[i];
            L.w = window_lengths[i]; L.nb = L.w / 2 + 1; L.ld = (2 * L.nb + 127) / 128 * 128;
            const int nm = (int)key[2 + 4 * i + 1];
            L.mel = nm > 0; L.n_out = L.mel ? nm : L.nb;
            ConvW& d = L.dft;
            d = ConvW();
            d.Cin = L.w; d.Cout = L.ld; d.K = 1; d.ldw = L.ld;
            d.w = P.alloc((size_t)L.w * L.ld);
            d.b = P.alloc(L.ld);
            dft_basis(P.pack.data() + d.w, L.ld, periodic_hann(L.w), L.w, L.nb, 0);
            attach_tc(P, d, 1, true);
            ConvW& dt = L.dftT;
            dt = ConvW();
            dt.Cin = L.ld; dt.Cout = L.w; dt.K = 1; dt.ldw = L.w;
            dt.w = P.alloc((size_t)L.ld * L.w);
            dt.b = P.alloc(L.w);
            for (int n = 0; n < L.w; ++n)
                for (int col = 0; col < 2 * L.nb; ++col) P.pack[dt.w + (size_t)col * L.w + n] = P.pack[d.w + (size_t)n * L.ld + col];
            attach_tc(P, dt, 1, true);
            if (L.mel) {
                std::vector<float> fb;
                slaney_mel_fb((double)sample_rate, L.w, nm, key[2 + 4 * i + 2], key[2 + 4 * i + 3], fb);
                L.fb = P.alloc(fb.size());
                std::copy(fb.begin(), fb.end(), P.pack.begin() + L.fb);
            }
        }
        const int rc = upload_weights(h, P, h->spec_arena, "fac_spectral_loss");
        if (rc != FAC_OK) return rc;
        h->spec_scales = scales;
        h->spec_key = key;
    }
    return two_pass(h, (cudaStream_t)stream, h->spec_arena.get(), [&](Ctx& c) {
        double* sums = c.alloc<double>(2 * 16 + 2);
        const size_t mark = c.off;
        size_t peak = c.off;
        c.vq_critical = true;                                        // fp32-faithful DFT (promoted tensor-core class)
        for (int i = 0; i < n_scales; ++i) {
            c.off = mark;
            const fac_handle::SpecScale& L = c.h->spec_scales[i];
            const int hop = L.w / 4, F = T / hop + 1;
            const size_t rows = (size_t)2 * B * F;
            float* frames = c.alloc<float>(rows * L.w);
            float* spec = c.alloc<float>(rows * L.ld);
            float* tr = c.alloc<float>((size_t)B * F * 2);
            if (!c.dry) {
                c.check(launch_stft_frames(x, frames, B, T, F, hop, L.w, L.w / 2, c.st), "spec.frames");
                c.check(launch_stft_frames(y, frames + (size_t)B * F * L.w, B, T, F, hop, L.w, L.w / 2, c.st), "spec.frames");
            }
            run_conv(c, L.dft, frames, spec, 1, (int)rows, (int)rows, ConvOpts(), "spec.dft");
            if (!c.dry) {
                const double inv = 1.0 / ((double)B * F * L.n_out);
                c.check(launch_spec_loss_terms(spec, L.ld, L.nb, L.mel ? c.W(L.fb) : nullptr, L.n_out, B, F, clamp_eps, pw, tr, c.st), "spec.terms");
                c.check(launch_strided_sum(tr, (long long)B * F, 2, inv, sums + 2 * i, c.st), "spec.mag");
                c.check(launch_strided_sum(tr + 1, (long long)B * F, 2, inv, sums + 2 * i + 1, c.st), "spec.log");
            }
            // before the next scale reuses the scratch (the tap copies are ordered on c.st)
            const std::string si = std::to_string(i);
            c.tap(("spec.dft." + si).c_str(), spec, rows * L.ld);
            c.tap(("spec.terms." + si).c_str(), tr, (size_t)B * F * 2);
            if (L.mel) c.tap(("spec.fb." + si).c_str(), c.W(L.fb), (size_t)L.nb * L.n_out);
            if (dx || dy) {
                // rows of the signals whose gradient is asked for: [0, B*F) x, [B*F, 2*B*F) y
                const size_t r0 = dx ? 0 : (size_t)B * F, nr = (dx && dy) ? rows : (size_t)B * F;
                float* inv = c.alloc<float>(rows);                   // per-row inverse scales of the gradient rows
                if (!c.dry) {
                    const double n_el = (double)B * F * L.n_out;
                    c.check(launch_spec_loss_grad(spec, L.ld, L.nb, L.mel ? c.W(L.fb) : nullptr, L.n_out, B, F, clamp_eps, pw,
                                                  (float)(mag_weight / n_el), (float)(log_weight / n_el), dx != nullptr, dy != nullptr, inv,
                                                  c.st),
                            "spec.grad");
                }
                run_conv(c, L.dftT, spec + r0 * L.ld, frames + r0 * L.w, 1, (int)nr, (int)nr, ConvOpts(), "spec.dftT");
                if (!c.dry) {
                    if (dx) c.check(launch_stft_overlap_add_grad(frames, inv, dx, B, T, F, hop, L.w, L.w / 2, i > 0, c.st), "spec.ola");
                    if (dy) c.check(launch_stft_overlap_add_grad(frames + (size_t)B * F * L.w, inv + (size_t)B * F, dy, B, T, F, hop, L.w,
                                                                 L.w / 2, i > 0, c.st),
                                    "spec.ola");
                }
                c.tap(("spec.dframes." + si).c_str(), frames, rows * L.w);
                c.tap(("spec.dscale." + si).c_str(), inv, rows);
            }
            if (c.off > peak) peak = c.off;
        }
        c.vq_critical = false;
        c.off = peak;
        if (!c.dry) c.check(launch_spec_loss_combine(sums, n_scales, mag_weight, log_weight, loss, c.st), "spec.combine");
    });
}

int fac_spectral_loss(fac_handle* h, const float* x, const float* y, int B, int T, int sample_rate, int n_scales, const int* window_lengths,
                      const int* n_mels, const float* mel_fmin, const float* mel_fmax, float clamp_eps, float mag_weight, float log_weight,
                      float pw, float* loss, void* stream) {
    return spectral_loss(h, x, y, B, T, sample_rate, n_scales, window_lengths, n_mels, mel_fmin, mel_fmax, clamp_eps, mag_weight,
                         log_weight, pw, loss, nullptr, nullptr, stream);
}

int fac_spectral_loss_grad(fac_handle* h, const float* x, const float* y, int B, int T, int sample_rate, int n_scales,
                           const int* window_lengths, const int* n_mels, const float* mel_fmin, const float* mel_fmax, float clamp_eps,
                           float mag_weight, float log_weight, float pw, float* loss, float* dx, float* dy, void* stream) {
    return spectral_loss(h, x, y, B, T, sample_rate, n_scales, window_lengths, n_mels, mel_fmin, mel_fmax, clamp_eps, mag_weight,
                         log_weight, pw, loss, dx, dy, stream);
}

// dac/nn/loss.py:11-47 L1Loss on the waveforms: mean |x - y| over n floats
// (dx / dy: null, or dL/dx = sgn(x - y) / n and dL/dy = -dL/dx)
static int l1_loss(fac_handle* h, const float* x, const float* y, long long n, float* loss, float* dx, float* dy, void* stream) {
    if (!h || !x || !y || !loss || n <= 0) return FAC_ERR_INVALID;
    cudaSetDevice(h->device);
    return two_pass(h, (cudaStream_t)stream, [&](Ctx& c) {
        double* sum = c.alloc<double>(2);
        const int nblk = 1024;
        float* part = c.alloc<float>(nblk);
        if (!c.dry) {
            c.check(launch_absdiff_partial(x, y, n, part, nblk, c.st), "l1.partial");
            c.check(launch_strided_sum(part, nblk, 1, 1.0 / (double)n, sum, c.st), "l1.sum");
            c.check(launch_spec_loss_combine(sum, 0, 0.f, 0.f, loss, c.st), "l1.out");
            if (dx || dy) c.check(launch_l1_grad(x, y, n, (float)(1.0 / (double)n), dx, dy, c.st), "l1.grad");
        }
    });
}
int fac_l1_loss(fac_handle* h, const float* x, const float* y, long long n, float* loss, void* stream) {
    return l1_loss(h, x, y, n, loss, nullptr, nullptr, stream);
}
int fac_l1_loss_grad(fac_handle* h, const float* x, const float* y, long long n, float* loss, float* dx, float* dy, void* stream) {
    return l1_loss(h, x, y, n, loss, dx, dy, stream);
}

// ---- predictor heads (SURVEY.md 8f rank 1; training-side in the reference, forward only here) ----
int fac_head_begin(fac_handle* h) {
    if (!h) return FAC_ERR_INVALID;
    h->heads.push_back(std::make_unique<HeadSet>());
    return (int)h->heads.size() - 1;
}

int fac_head_tensor(fac_handle* h, int head_id, const char* key, const float* data_host, const int64_t* shape, int ndim) {
    HeadSet* hs = by_id(h, &fac_handle::heads, head_id);
    if (!hs) return FAC_ERR_INVALID;
    const int rc = stage_tensor(hs->staged, key, data_host, shape, ndim);
    if (rc == FAC_OK) hs->ready = false;
    return rc;
}

int fac_head_finalize(fac_handle* h, int head_id, int indim, int outdim, int nheads, int global_pred) {
    HeadSet* set = by_id(h, &fac_handle::heads, head_id);
    if (!set || indim <= 0 || outdim <= 0 || nheads < 1 || nheads > 8) return FAC_ERR_INVALID;
    if (indim % 16 != 0) { h->err = "fac_head_finalize: indim must be a multiple of 16"; return FAC_ERR_UNSUPPORTED; }
    HeadSet& hs = *set;
    const TensorMap& ts = hs.staged;
    Packer P;
    hs.indim = indim; hs.outdim = outdim; hs.nheads = nheads; hs.global_pred = global_pred;
    try {
        if (global_pred == 2) {
            // kind "linear": a plain nn.Linear(indim, outdim) staged as linear.weight [outdim][indim] / linear.bias
            // (FApredictors.timbre_predictor under timbre_norm, modules/quantize.py:470-473)
            if (nheads != 1) throw PackError{"a linear head has exactly one output"};
            hs.lin[0] = pack_conv(P, ts, "linear");
            if (hs.lin[0].Cin != indim || hs.lin[0].Cout != outdim) throw PackError{"Linear geometry"};
        } else {
        auto expv = [&](const std::string& key) {
            const HostTensor& t = need(ts, key);
            if ((int)t.numel() != indim) throw PackError{"shape of " + key};
            size_t off = P.alloc(indim);
            for (int i = 0; i < indim; ++i) P.pack[off + i] = expf(t.data[i]);     // alpha_logscale=True: exp() of the parameter
            return off;
        };
        const int dils[3] = {1, 2, 3};
        for (int j = 0; j < 3; ++j) {
            const std::string p = "model." + std::to_string(j);
            auto& u = hs.unit[j];
            u.dil = dils[j];
            u.a1 = expv(p + ".block.0.act.alpha"); u.b1 = expv(p + ".block.0.act.beta");
            u.c7 = pack_conv(P, ts, p + ".block.1");
            u.a2 = expv(p + ".block.2.act.alpha"); u.b2 = expv(p + ".block.2.act.beta");
            u.c1 = pack_conv(P, ts, p + ".block.3");
            if (u.c7.Cin != indim || u.c7.Cout != indim || u.c7.K != 7 || u.c1.K != 1) throw PackError{"head ResidualUnit geometry"};
        }
        hs.af = expv("model.3.act.alpha"); hs.bf = expv("model.3.act.beta");
        for (int i = 0; i < nheads; ++i) {
            hs.lin[i] = pack_conv(P, ts, "heads." + std::to_string(i));
            if (hs.lin[i].Cin != indim || hs.lin[i].Cout != outdim) throw PackError{"head Linear geometry"};
        }
        }
    } catch (const PackError& e) {
        h->err = e.msg;
        return FAC_ERR_STATE;
    }
    const int rc = upload_weights(h, P, hs.arena, "fac_head_finalize");
    if (rc != FAC_OK) return rc;
    hs.staged.clear();
    hs.ready = true;
    return FAC_OK;
}

static int ensure_aa_filter(fac_handle* h);

int fac_head_forward(fac_handle* h, int head_id, const float* x, int B, int T, float* const* outs, void* stream) {
    const HeadSet* set = by_id(h, &fac_handle::heads, head_id);
    if (!set || !x || !outs || B <= 0 || T <= 0) return FAC_ERR_INVALID;
    const HeadSet& hs = *set;
    if (!hs.ready) { h->err = "fac_head_forward: head not finalized"; return FAC_ERR_STATE; }
    int rc = ensure_aa_filter(h);
    if (rc) return rc;
    const int C = hs.indim;
    if (hs.global_pred == 2) {
        // kind "linear": x [B*T rows][indim] -> outs[0] [B*T][outdim]
        return two_pass(h, (cudaStream_t)stream, hs.arena.get(), [&](Ctx& c) {
            run_conv(c, hs.lin[0], x, outs[0], 1, B * T, B * T, ConvOpts(), "head.linear");
        });
    }
    return two_pass(h, (cudaStream_t)stream, hs.arena.get(), [&](Ctx& c) {
        const size_t n = (size_t)B * T * C;
        float* a_nct = c.alloc<float>(n);
        float* a_cl = c.alloc<float>(n);
        float* c7_cl = c.alloc<float>(n);
        float* c7_nct = c.alloc<float>(n);
        float* x_cl[2] = {c.alloc<float>(n), c.alloc<float>(n)};
        float* x_nct = c.alloc<float>(n);
        float* pooled = c.alloc<float>((size_t)B * C);
        auto act = [&](const float* src, float* dst, size_t al, size_t be, const char* nm) {
            if (!c.dry) c.check(launch_alias_free_act(src, dst, B, C, T, h->aa_filter.get(), c.W(al), c.W(be), c.st), nm);
        };
        auto tr = [&](const float* src, float* dst, int R, int Cc, const char* nm) {     // [B][R][Cc] -> [B][Cc][R]
            if (!c.dry) c.check(launch_transpose(src, dst, B, R, Cc, c.st), nm);
        };
        tr(x, x_cl[0], C, T, "head.x_T");                                              // NCT -> channels-last
        const float* cur_nct = x;
        int cur = 0;
        for (int j = 0; j < 3; ++j) {
            const auto& u = hs.unit[j];
            act(cur_nct, a_nct, u.a1, u.b1, "head.act1");
            tr(a_nct, a_cl, C, T, "head.a_T");
            ConvOpts o7;
            o7.dil = u.dil; o7.pad_left = 3 * u.dil; o7.pad_right = 3 * u.dil; o7.reflect = 0;     // padding = ((7-1)*d)//2, zeros
            run_conv(c, u.c7, a_cl, c7_cl, B, T, T, o7, "head.conv7");
            tr(c7_cl, c7_nct, T, C, "head.c7_T");
            act(c7_nct, a_nct, u.a2, u.b2, "head.act2");
            tr(a_nct, a_cl, C, T, "head.b_T");
            ConvOpts o1;
            o1.res = x_cl[cur];
            run_conv(c, u.c1, a_cl, x_cl[cur ^ 1], B, T, T, o1, "head.conv1");
            cur ^= 1;
            tr(x_cl[cur], x_nct, T, C, "head.y_T");
            cur_nct = x_nct;
        }
        act(cur_nct, a_nct, hs.af, hs.bf, "head.act_final");
        tr(a_nct, a_cl, C, T, "head.f_T");                                             // Rearrange("b c t -> b t c")
        for (int i = 0; i < hs.nheads; ++i) {
            if (hs.global_pred) {
                if (!c.dry) c.check(launch_mean_pool(a_cl, pooled, B, T, C, nullptr, c.st), "head.mean");
                run_conv(c, hs.lin[i], pooled, outs[i], 1, B, B, ConvOpts(), "head.linear");
            } else {
                run_conv(c, hs.lin[i], a_cl, outs[i], 1, B * T, B * T, ConvOpts(), "head.linear");
            }
        }
    });
}

// ---- JDCNet pitch extractor (modules/JDC/model.py, eval mode) ----
int fac_jdc_begin(fac_handle* h) {
    if (!h) return FAC_ERR_INVALID;
    h->jdcs.push_back(std::make_unique<JdcSet>());
    return (int)h->jdcs.size() - 1;
}

int fac_jdc_tensor(fac_handle* h, int jdc_id, const char* key, const float* data_host, const int64_t* shape, int ndim) {
    JdcSet* js = by_id(h, &fac_handle::jdcs, jdc_id);
    if (!js) return FAC_ERR_INVALID;
    const int rc = stage_tensor(js->staged, key, data_host, shape, ndim);
    if (rc == FAC_OK) js->ready = false;
    return rc;
}

namespace {
// BatchNorm2d (eval) at `prefix` as y = x * sc + sh, in fp64 then rounded
void jdc_bn(const TensorMap& ts, const std::string& prefix, int C, std::vector<double>& sc, std::vector<double>& sh) {
    const HostTensor& g = need(ts, prefix + ".weight");
    const HostTensor& b = need(ts, prefix + ".bias");
    const HostTensor& m = need(ts, prefix + ".running_mean");
    const HostTensor& v = need(ts, prefix + ".running_var");
    if ((int)g.numel() != C || (int)b.numel() != C || (int)m.numel() != C || (int)v.numel() != C) throw PackError{"BatchNorm shape at " + prefix};
    sc.resize(C); sh.resize(C);
    for (int c = 0; c < C; ++c) {
        sc[c] = (double)g.data[c] / std::sqrt((double)v.data[c] + 1e-5);
        sh[c] = (double)b.data[c] - (double)m.data[c] * sc[c];
    }
}
JdcSet::Bn jdc_pack_bn(Packer& P, const TensorMap& ts, const std::string& prefix, int C) {
    std::vector<double> sc, sh;
    jdc_bn(ts, prefix, C, sc, sh);
    JdcSet::Bn r;
    r.sc = P.alloc(C); r.sh = P.alloc(C);
    for (int c = 0; c < C; ++c) { P.pack[r.sc + c] = (float)sc[c]; P.pack[r.sh + c] = (float)sh[c]; }
    return r;
}
// nn.Conv2d(Cin, Cout, k, bias=False) at `prefix` (k = 3: 9 row-offset taps tap = kh * 3 + kw; k = 1: one tap), with the
// BatchNorm at `bn` (or none) folded in, packed [taps * Cin][ldw] with its promoted fp16 hi + scaled-lo blob (conv_tc.cu)
ConvW jdc_pack_conv(Packer& P, const TensorMap& ts, const std::string& prefix, int Cin, int Cout, int k, const char* bn) {
    const HostTensor& w = need(ts, prefix + ".weight");
    if (w.shape.size() != 4 || w.shape[0] != Cout || w.shape[1] != Cin || w.shape[2] != k || w.shape[3] != k)
        throw PackError{"Conv2d shape at " + prefix};
    std::vector<double> sc(Cout, 1.0), sh(Cout, 0.0);
    if (bn) jdc_bn(ts, bn, Cout, sc, sh);
    ConvW c;
    c.Cin = Cin; c.Cout = Cout; c.K = k * k; c.ldw = (Cout + 3) / 4 * 4;
    c.w = P.alloc((size_t)c.K * Cin * c.ldw);
    for (int co = 0; co < Cout; ++co)
        for (int ci = 0; ci < Cin; ++ci)
            for (int tap = 0; tap < c.K; ++tap)
                P.pack[c.w + ((size_t)tap * Cin + ci) * c.ldw + co] = (float)(w.data[((size_t)co * Cin + ci) * c.K + tap] * sc[co]);
    c.b = P.alloc(Cout);
    for (int co = 0; co < Cout; ++co) P.pack[c.b + co] = (float)sh[co];
    TcConvParams tp;
    tp.Cin = Cin; tp.Cout = Cout; tp.Kr = c.K; tp.vf = 1; tp.dil = 1; tp.promoted = 1; tp.f16x2 = 1; tp.row2d = k == 3 ? 82 : 0;
    if (!tc_conv_plan(tp)) throw PackError{"no tensor-core plan for " + prefix};
    c.Kr = c.K; c.promoted = true; c.tcN = tp.N; c.tc = true; c.has16 = true;
    c.tcw16 = P.alloc(tc_blob_floats(tp));
    tc_pack_blob(tp, P.pack.data() + c.w, c.ldw, P.pack.data() + c.tcw16);
    return c;
}

// 3x3 conv over [B][T][F + 2][Cin] maps (conv2d_tc_kernel): rows = frames x (F + 2), per-lane rows in rows_len
void jdc_conv3(Ctx& c, const ConvW& w, const float* x, float* y, int B, int T, int F, const int* rows_len, int act,
               const float* res, const char* name) {
    if (c.dry) return;
    TcConvParams tp;
    tp.Cin = w.Cin; tp.Cout = w.Cout; tp.vf = 1; tp.Kr = 9; tp.dil = 1; tp.promoted = 1; tp.f16x2 = 1; tp.row2d = F + 2;
    const int rows = T * (F + 2);
    tp.Tout = rows;
    if (!tc_conv_plan(tp) || tp.N != w.tcN) { c.check(cudaErrorInvalidValue, name); return; }
    tp.x = x; tp.y = y; tp.wblob = c.W(w.tcw16); tp.bias = c.W(w.b); tp.res = res; tp.out_act = act;
    tp.B = B; tp.Tin = rows; tp.ldx = w.Cin; tp.PLr = F + 3; tp.pad_left_s = F + 3; tp.pad_right_s = F + 3; tp.reflect = 0;
    tp.lane_len = rows_len; tp.ldy = w.Cout;
    tp.x_bstride = (size_t)rows * w.Cin; tp.y_bstride = (size_t)rows * w.Cout;
    char det[96];
    snprintf(det, sizeof det, "%s Cin%d Cout%d F%d T%d", name, w.Cin, w.Cout, F, T);
    c.begin("conv2d_tc", 2.0 * B * T * F * 9.0 * w.Cin * w.Cout, 4.0 * ((double)B * rows * (w.Cin + w.Cout) + 9.0 * w.Cin * w.Cout), det);
    c.check(launch_conv_tc(tp, c.st), name);
    c.end();
}
}  // namespace

int fac_jdc_finalize(fac_handle* h, int jdc_id) {
    JdcSet* set = by_id(h, &fac_handle::jdcs, jdc_id);
    if (!set) return FAC_ERR_INVALID;
    JdcSet& js = *set;
    const TensorMap& ts = js.staged;
    Packer P;
    try {
        {   // conv_block.0 (1 -> 64) with conv_block.1 folded: SIMT, [9][64]
            const HostTensor& w = need(ts, "conv_block.0.weight");
            if (w.shape.size() != 4 || w.shape[0] != 64 || w.shape[1] != 1 || w.shape[2] != 3 || w.shape[3] != 3)
                throw PackError{"Conv2d shape at conv_block.0"};
            std::vector<double> sc, sh;
            jdc_bn(ts, "conv_block.1", 64, sc, sh);
            js.conv_in_w = P.alloc(9 * 64);
            js.conv_in_b = P.alloc(64);
            for (int co = 0; co < 64; ++co) {
                for (int k = 0; k < 9; ++k) P.pack[js.conv_in_w + k * 64 + co] = (float)(w.data[co * 9 + k] * sc[co]);
                P.pack[js.conv_in_b + co] = (float)sh[co];
            }
        }
        js.c0b = jdc_pack_conv(P, ts, "conv_block.3", 64, 64, 3, nullptr);
        const int cin[3] = {64, 128, 192}, cout[3] = {128, 192, 256}, F[3] = {80, 40, 20};
        for (int i = 0; i < 3; ++i) {
            const std::string p = "res_block" + std::to_string(i + 1);
            auto& b = js.blk[i];
            b.F = F[i];
            b.pre = jdc_pack_bn(P, ts, p + ".pre_conv.0", cin[i]);
            b.c1 = jdc_pack_conv(P, ts, p + ".conv.0", cin[i], cout[i], 3, (p + ".conv.1").c_str());
            b.c2 = jdc_pack_conv(P, ts, p + ".conv.3", cout[i], cout[i], 3, nullptr);
            b.c11 = jdc_pack_conv(P, ts, p + ".conv1by1", cin[i], cout[i], 1, nullptr);
        }
        js.pool = jdc_pack_bn(P, ts, "pool_block.0", 256);
        const int H = 256;
        js.U = lstm_units_per_cta(H);
        js.G = H / js.U;
        for (int d = 0; d < 2; ++d) {
            const std::string sfx = d ? "_l0_reverse" : "_l0";
            const HostTensor& wih = need(ts, "bilstm_classifier.weight_ih" + sfx);
            const HostTensor& whh = need(ts, "bilstm_classifier.weight_hh" + sfx);
            const HostTensor& bih = need(ts, "bilstm_classifier.bias_ih" + sfx);
            const HostTensor& bhh = need(ts, "bilstm_classifier.bias_hh" + sfx);
            if (wih.numel() != (size_t)4 * H * 512 || whh.numel() != (size_t)4 * H * H || bih.numel() != 4 * H || bhh.numel() != 4 * H)
                throw PackError{"bilstm_classifier shape"};
            ConvW c;
            c.Cin = 512; c.Cout = 4 * H; c.K = 1; c.ldw = 4 * H;
            c.w = P.alloc((size_t)512 * c.ldw);
            for (int row = 0; row < 4 * H; ++row)
                for (int k = 0; k < 512; ++k) P.pack[c.w + (size_t)k * c.ldw + row] = wih.data[(size_t)row * 512 + k];
            c.b = P.alloc(4 * H);
            for (int row = 0; row < 4 * H; ++row) P.pack[c.b + row] = bih.data[row] + bhh.data[row];
            attach_tc(P, c, 1, true);
            if (!c.tc || !c.has16) throw PackError{"no tensor-core plan for the BiLSTM input GEMM"};
            js.ih[d] = c;
            js.whh2[d] = P.alloc(lstm2_pack_words(H, js.U, 1));
            lstm2_pack(whh.data.data(), H, js.U, 1, reinterpret_cast<uint32_t*>(P.pack.data() + js.whh2[d]));
        }
        const HostTensor& cw = need(ts, "classifier.weight");
        const HostTensor& cb = need(ts, "classifier.bias");
        if (cw.numel() != 512 || cb.numel() != 1) throw PackError{"classifier shape (num_class must be 1)"};
        js.cls_w = P.alloc(512);
        for (int k = 0; k < 512; ++k) P.pack[js.cls_w + k] = cw.data[k];
        js.cls_b = P.alloc(1);
        P.pack[js.cls_b] = cb.data[0];
    } catch (const PackError& e) {
        h->err = e.msg;
        return FAC_ERR_STATE;
    }
    const int rc = upload_weights(h, P, js.arena, "fac_jdc_finalize");
    if (rc != FAC_OK) return rc;
    js.staged.clear();
    js.ready = true;
    return FAC_OK;
}

int fac_jdc_forward(fac_handle* h, int jdc_id, const float* mel, int B, int T, const int* lengths, float* f0, float* gan_feature,
                    float* pool_out, void* stream) {
    const JdcSet* set = by_id(h, &fac_handle::jdcs, jdc_id);
    if (!set || !mel || !f0 || !gan_feature || !pool_out || B <= 0 || T <= 0) return FAC_ERR_INVALID;
    const JdcSet& js = *set;
    if (!js.ready) { h->err = "fac_jdc_forward: JDCNet not finalized"; return FAC_ERR_STATE; }
    std::vector<int> lens(B, T);
    if (lengths)
        for (int b = 0; b < B; ++b) {
            if (lengths[b] < 1 || lengths[b] > T) { h->err = "fac_jdc_forward: lengths must be in [1, T]"; return FAC_ERR_INVALID; }
            lens[b] = lengths[b];
        }
    if (B > 65535) { h->err = "fac_jdc_forward: B > 65535"; return FAC_ERR_UNSUPPORTED; }
    const int H = 256;
    return two_pass(h, (cudaStream_t)stream, js.arena.get(), [&](Ctx& c) {
        // per-lane frames, then rows of each map width (F + 2 = 82, 42, 22, 12)
        int* dl = lengths ? c.alloc<int>((size_t)5 * B) : nullptr;
        const int Fs[4] = {80, 40, 20, 10};
        if (!c.dry && lengths) {
            std::vector<int> hl((size_t)5 * B);
            for (int b = 0; b < B; ++b) {
                hl[b] = lens[b];
                for (int i = 0; i < 4; ++i) hl[(size_t)(i + 1) * B + b] = lens[b] * (Fs[i] + 2);
            }
            // ordered before the launches that read it on the same stream; a copy from pageable memory has taken the
            // host data by the time it returns, so hl may go out of scope without a synchronize
            c.check_nk(cudaMemcpyAsync(dl, hl.data(), hl.size() * sizeof(int), cudaMemcpyHostToDevice, c.st), "jdc.lens");
        }
        const int* len_d = lengths ? dl : nullptr;
        auto rows_of = [&](int i) { return lengths ? dl + (size_t)(i + 1) * B : nullptr; };
        const size_t big = (size_t)B * T * 42 * 128;      // the largest map: [B][T][42][128] (> [82][64], [22][192], [12][256])
        float* m0 = c.alloc<float>(big);
        float* m1 = c.alloc<float>(big);
        float* m2 = c.alloc<float>(big);
        float* m3 = c.alloc<float>(big);
        float* lstm_in = c.alloc<float>((size_t)B * T * 512);
        float* xg = c.alloc<float>((size_t)B * T * 4 * H);
        float* yd[2] = {c.alloc<float>((size_t)B * T * H), c.alloc<float>((size_t)B * T * H)};
        uint32_t* h16 = c.alloc<uint32_t>((size_t)2 * 2 * (H / 2) * 32);
        unsigned int* bar = c.alloc<unsigned int>(64);
        if (!c.dry) c.check(launch_jdc_conv_in(mel, c.W(js.conv_in_w), c.W(js.conv_in_b), m0, B, T, len_d, c.st), "jdc.conv_in");
        c.tap("jdc.conv_in", m0, (size_t)B * T * 82 * 64);
        jdc_conv3(c, js.c0b, m0, m1, B, T, 80, rows_of(0), ACT_NONE, nullptr, "jdc.conv_block");
        c.tap("jdc.conv_block", m1, (size_t)B * T * 82 * 64);
        float* cur = m1;
        int Cc = 64;
        for (int i = 0; i < 3; ++i) {
            const auto& bk = js.blk[i];
            const int Fo = bk.F / 2;
            float* xin = cur == m1 ? m0 : m1;         // pre_conv output
            float* hmid = m2;
            float* r11 = m3;
            float* out = cur;                         // cur is dead once pre_conv has read it
            if (!c.dry) c.check(launch_jdc_pre_pool(cur, c.W(bk.pre.sc), c.W(bk.pre.sh), xin, B, T, bk.F, Cc, c.st), "jdc.pre_conv");
            const std::string si = std::to_string(i + 1);
            c.tap(("jdc.res" + si + ".pre").c_str(), xin, (size_t)B * T * (Fo + 2) * Cc);
            // conv1by1 as a 1-tap row GEMM over the same map: its rows at the pad columns are zeroed by conv2's epilogue
            if (!c.dry) {
                TcConvParams tp;
                tp.Cin = Cc; tp.Cout = bk.c11.Cout; tp.vf = 1; tp.Kr = 1; tp.dil = 1; tp.promoted = 1; tp.f16x2 = 1;
                const int rows = T * (Fo + 2);
                tp.Tout = rows;
                if (!tc_conv_plan(tp) || tp.N != bk.c11.tcN) c.check(cudaErrorInvalidValue, "jdc.conv1by1");
                else {
                    tp.x = xin; tp.y = r11; tp.wblob = c.W(bk.c11.tcw16); tp.bias = c.W(bk.c11.b);
                    tp.B = B; tp.Tin = rows; tp.ldx = Cc; tp.lane_len = rows_of(i + 1); tp.ldy = bk.c11.Cout;
                    tp.x_bstride = (size_t)rows * Cc; tp.y_bstride = (size_t)rows * bk.c11.Cout;
                    c.begin("conv_tcp", 2.0 * B * rows * Cc * bk.c11.Cout, 4.0 * ((double)B * rows * (Cc + bk.c11.Cout)), "jdc.conv1by1");
                    c.check(launch_conv_tc(tp, c.st), "jdc.conv1by1");
                    c.end();
                }
            }
            jdc_conv3(c, bk.c1, xin, hmid, B, T, Fo, rows_of(i + 1), ACT_LRELU, nullptr, "jdc.conv1");
            c.tap(("jdc.res" + si + ".conv1").c_str(), hmid, (size_t)B * T * (Fo + 2) * bk.c1.Cout);
            jdc_conv3(c, bk.c2, hmid, out, B, T, Fo, rows_of(i + 1), ACT_NONE, r11, "jdc.conv2");
            c.tap(("jdc.res" + si).c_str(), out, (size_t)B * T * (Fo + 2) * bk.c2.Cout);
            Cc = bk.c2.Cout;
        }
        if (!c.dry)
            c.check(launch_jdc_pool_block(cur, c.W(js.pool.sc), c.W(js.pool.sh), gan_feature, pool_out, lstm_in, B, T, len_d, c.st),
                    "jdc.pool_block");
        c.tap("jdc.lstm_in", lstm_in, (size_t)B * T * 512);
        for (int d = 0; d < 2; ++d) {
            run_conv(c, js.ih[d], lstm_in, xg, 1, B * T, B * T, ConvOpts(), "jdc.lstm.ih");
            c.tap(d ? "jdc.lstm.xg_rev" : "jdc.lstm.xg_fwd", xg, (size_t)B * T * 4 * H);
            if (c.dry) continue;
            for (int b0 = 0; b0 < B; b0 += 32) {
                const int nb = B - b0 < 32 ? B - b0 : 32;
                LstmParams p;
                p.xg = xg + (size_t)b0 * T * 4 * H;
                p.whh_p2 = reinterpret_cast<const uint32_t*>(c.W(js.whh2[d]));
                p.h16 = h16; p.pass3 = 1; p.hT = nullptr; p.bar = bar;
                p.y = yd[d] + (size_t)b0 * T * H;
                p.B = nb; p.T = T; p.H = H; p.U = js.U; p.G = js.G;
                LstmLaneLens ll = {};
                for (int b = 0; b < nb; ++b) ll.len[b] = lens[b0 + b];
                c.begin("lstm_rec", 2.0 * nb * T * 4.0 * H * H, 4.0 * ((double)nb * T * 5 * H + 4.0 * H * H));
                c.check(launch_lstm2_layer(p, c.st, d ? &ll : nullptr, d == 1), d ? "jdc.lstm.rev" : "jdc.lstm.fwd");
                c.end();
            }
        }
        c.tap("jdc.lstm.fwd", yd[0], (size_t)B * T * H);
        c.tap("jdc.lstm.rev", yd[1], (size_t)B * T * H);
        if (!c.dry) c.check(launch_jdc_head(yd[0], yd[1], c.W(js.cls_w), c.W(js.cls_b), f0, B, T, len_d, c.st), "jdc.head");
    });
}

int fac_f0_targets(fac_handle* h, const float* f0, int B, int T, const int* lengths, float* targets, float* glob_f0, void* stream) {
    if (!h || !f0 || !targets || !glob_f0 || B <= 0 || T <= 0) return FAC_ERR_INVALID;
    std::vector<int> hl;
    if (lengths) {
        hl.assign(lengths, lengths + B);
        for (int b = 0; b < B; ++b)
            if (hl[b] < 0 || hl[b] > T) { h->err = "fac_f0_targets: lengths must be in [0, T]"; return FAC_ERR_INVALID; }
    }
    return two_pass(h, (cudaStream_t)stream, [&](Ctx& c) {
        int* dl = lengths ? c.alloc<int>(B) : nullptr;
        if (c.dry) return;
        if (dl) {
            c.check_nk(cudaMemcpyAsync(dl, hl.data(), (size_t)B * sizeof(int), cudaMemcpyHostToDevice, c.st), "f0_targets.lens");
        }
        c.check(launch_f0_targets(f0, dl, B, T, targets, glob_f0, c.st), "f0_targets");
    });
}

int fac_log_norm(fac_handle* h, const float* mel, int B, int T, float* out, void* stream) {
    if (!h || !mel || !out || B <= 0 || T <= 0) return FAC_ERR_INVALID;
    cudaSetDevice(h->device);
    cudaError_t e = launch_log_norm(mel, B, T, out, (cudaStream_t)stream);
    if (e != cudaSuccess) { h->err = std::string("CUDA error at log_norm: ") + cudaGetErrorString(e); return FAC_ERR_CUDA; }
    h->launches = 1;
    return FAC_OK;
}

// out = a + b (+ c): the latent sums FApredictors.forward_v2 feeds its reversal heads (modules/quantize.py:571-586), in the
// reference's left-to-right order
int fac_add3(fac_handle* h, const float* a, const float* b, const float* c3, long long n, float* out, void* stream) {
    if (!h || !a || !b || !out || n <= 0) return FAC_ERR_INVALID;
    cudaSetDevice(h->device);
    cudaError_t e = launch_add3(a, b, c3, n, out, (cudaStream_t)stream);
    if (e != cudaSuccess) { h->err = std::string("CUDA error at add3: ") + cudaGetErrorString(e); return FAC_ERR_CUDA; }
    return FAC_OK;
}

int fac_rvq_create(fac_handle* h, int nq, const float* const* in_w, const float* const* in_b, const float* const* out_w,
                   const float* const* out_b, const float* const* codebook) {
    if (!h || nq < 1 || nq > 8) return FAC_ERR_INVALID;
    auto s = std::make_unique<RvqSet>();
    s->nq = nq;
    Packer P;
    for (int q = 0; q < nq; ++q) s->vq[q] = pack_vq_raw(P, in_w[q], in_b[q], out_w[q], out_b[q], codebook[q]);
    const int rc = upload_weights(h, P, s->arena, "fac_rvq_create");
    if (rc != FAC_OK) return rc;
    h->rvqs.push_back(std::move(s));
    return (int)h->rvqs.size() - 1;
}

// Frees the device arena of one fac_rvq_create set (ids of other sets stay valid; the id is not reused; destroying a set
// twice is a no-op).
int fac_rvq_destroy(fac_handle* h, int rvq_id) {
    if (!h || rvq_id < 0 || rvq_id >= (int)h->rvqs.size()) return FAC_ERR_INVALID;
    return h->rvqs[rvq_id] ? free_by_id(h, &fac_handle::rvqs, rvq_id) : FAC_OK;
}

int fac_rvq_forward(fac_handle* h, int rvq_id, const float* x, int B, int T, int x_channels_last, float* quantized_out,
                    int64_t* indices, float* all_quantized, void* stream) {
    if (!h || rvq_id < 0 || rvq_id >= (int)h->rvqs.size() || !x || !quantized_out || !indices || B <= 0 || T <= 0) return FAC_ERR_INVALID;
    const RvqSet* set = by_id(h, &fac_handle::rvqs, rvq_id);
    if (!set) { h->err = "fac_rvq_forward: set was destroyed"; return FAC_ERR_STATE; }
    const RvqSet& s = *set;
    return two_pass(h, (cudaStream_t)stream, s.arena.get(), [&](Ctx& c) {
        size_t n = (size_t)B * T * 1024;
        float* xcl = x_channels_last ? nullptr : c.alloc<float>(n);
        float* qcl = x_channels_last ? nullptr : c.alloc<float>(n);
        float* acl = (x_channels_last || !all_quantized) ? nullptr : c.alloc<float>(n * s.nq);
        if (c.dry) return;
        RvqParams p;
        if (!x_channels_last) c.check(launch_transpose(x, xcl, B, 1024, T, c.st), "rvq.xT");
        p.x = x_channels_last ? x : xcl;
        p.qout = x_channels_last ? quantized_out : qcl;
        p.allq = all_quantized ? (x_channels_last ? all_quantized : acl) : nullptr;
        p.idx = indices;
        p.nq = s.nq; p.B = B; p.T = T;
        for (int q = 0; q < s.nq; ++q) {
            const VqW& v = s.vq[q];
            p.vq[q] = VqWeights{c.W(v.w_in), c.W(v.b_in), c.W(v.cb), c.W(v.cbn), c.W(v.cbn2), c.W(v.w_out), c.W(v.b_out)};
        }
        c.check(launch_rvq(p, c.st), "rvq");
        if (!x_channels_last) {
            c.check(launch_transpose(qcl, quantized_out, B, T, 1024, c.st), "rvq.qT");
            if (all_quantized) c.check(launch_transpose(acl, all_quantized, B * s.nq, T, 1024, c.st), "rvq.aT");
        }
    });
}

static int ensure_aa_filter(fac_handle* h) {
    cudaSetDevice(h->device);
    if (!h->aa_filter) {
        // kaiser_sinc_filter1d(cutoff=0.25, half_width=0.3, kernel_size=12), alias_free_torch/filter.py:27-58
        const int ks = 12, half = 6;
        const double cutoff = 0.25, half_width = 0.3;
        double delta_f = 4 * half_width;
        double A = 2.285 * (half - 1) * M_PI * delta_f + 7.95;
        double beta_k = A > 50.0 ? 0.1102 * (A - 8.7) : (A >= 21.0 ? 0.5842 * std::pow(A - 21, 0.4) + 0.07886 * (A - 21.0) : 0.0);
        auto i0 = [](double v) { double s = 1, t = 1; for (int k = 1; k < 60; ++k) { t *= (v / (2 * k)) * (v / (2 * k)); s += t; } return s; };
        std::vector<float> f(ks);
        double sum = 0;
        double tmp[12];
        for (int i = 0; i < ks; ++i) {
            double r = 2.0 * i / (ks - 1) - 1.0;                       // torch.kaiser_window(periodic=False)
            double w = i0(beta_k * std::sqrt(std::max(0.0, 1 - r * r))) / i0(beta_k);
            double tm = (i - half) + 0.5;
            double xx = 2 * cutoff * tm;
            double sinc = xx == 0 ? 1.0 : std::sin(M_PI * xx) / (M_PI * xx);
            tmp[i] = 2 * cutoff * w * sinc;
            sum += tmp[i];
        }
        for (int i = 0; i < ks; ++i) f[i] = (float)(tmp[i] / sum);
        return upload(h, f, h->aa_filter, "anti-alias filter");
    }
    return FAC_OK;
}

int fac_alias_free_act(fac_handle* h, const float* x, int B, int C, int T, int act, const float* alpha,
                       const float* beta, float* y, void* stream) {
    if (!h || !x || !y || B <= 0 || C <= 0 || T <= 0 || (act == 1 && (!alpha || !beta))) return FAC_ERR_INVALID;
    int rc0 = ensure_aa_filter(h);
    if (rc0) return rc0;
    cudaError_t e = launch_alias_free_act(x, y, B, C, T, h->aa_filter.get(), act == 1 ? alpha : nullptr, act == 1 ? beta : nullptr,
                                          (cudaStream_t)stream);
    if (e != cudaSuccess) { h->err = cudaGetErrorString(e); return FAC_ERR_CUDA; }
    return FAC_OK;
}

}  // extern "C"

namespace {
// The per-lane lengths of a debug conv hook (HOST, B entries, or null) checked and copied to the device: dev receives
// the device copy (empty when lane_len_host is null).  Nothing is launched when a length lies outside [1, Tin].
int debug_upload_lanes(fac_handle* h, const char* who, const int* lane_len_host, int B, int Tin, DevBuf<int>& dev) {
    if (!lane_len_host) return FAC_OK;
    for (int b = 0; b < B; ++b)
        if (lane_len_host[b] < 1 || lane_len_host[b] > Tin) {
            h->err = std::string(who) + ": lane lengths must lie in [1, Tin]";
            return FAC_ERR_INVALID;
        }
    return upload(h, std::vector<int>(lane_len_host, lane_len_host + B), dev, who);
}

// fac_debug_conv, and fac_debug_conv_lanes' path -1: launch_conv (it picks the cin1 / cout1 / generic kernel) on one
// layer; lane_len DEVICE [B] (each lane's own input rows) or null.
int debug_conv(fac_handle* h, const float* x, const float* w_host, const float* bias_host, int B, int Tin, int Cin,
               int Cout, int K, int dil, int stride, int pad_left, int pad_right, int reflect,
               const float* in_alpha_host, const float* out_alpha_host, int act, const float* res, float* y,
               int Tout, const int* lane_len, void* stream) {
    if (!h || !x || !w_host || !y) return FAC_ERR_INVALID;
    cudaSetDevice(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    int ldw = (Cout + 3) / 4 * 4;
    std::vector<float> pk((size_t)K * Cin * ldw + Cout + 2 * Cin + 2 * Cout + 96, 0.f);
    for (int co = 0; co < Cout; ++co)
        for (int ci = 0; ci < Cin; ++ci)
            for (int k = 0; k < K; ++k) pk[((size_t)k * Cin + ci) * ldw + co] = w_host[((size_t)co * Cin + ci) * K + k];
    auto al4 = [](size_t v) { return (v + 3) / 4 * 4; };
    size_t o_b = (size_t)K * Cin * ldw, o_ia = al4(o_b + Cout), o_iia = al4(o_ia + Cin), o_oa = al4(o_iia + Cin), o_oia = al4(o_oa + Cout);
    for (int i = 0; i < Cout; ++i) pk[o_b + i] = bias_host ? bias_host[i] : 0.f;
    for (int i = 0; i < Cin; ++i) { pk[o_ia + i] = in_alpha_host ? in_alpha_host[i] : 1.f; pk[o_iia + i] = 1.0f / (pk[o_ia + i] + 1e-9f); }
    for (int i = 0; i < Cout; ++i) { pk[o_oa + i] = out_alpha_host ? out_alpha_host[i] : 1.f; pk[o_oia + i] = 1.0f / (pk[o_oa + i] + 1e-9f); }
    DevBuf<float> buf;
    const int rc = upload(h, pk, buf, "fac_debug_conv");
    if (rc != FAC_OK) return rc;
    const float* d = buf.get();
    ConvParams p;
    p.x = x; p.y = y; p.w = d; p.bias = bias_host ? d + o_b : nullptr;
    if (in_alpha_host) { p.in_alpha = d + o_ia; p.in_inv_alpha = d + o_iia; }
    p.out_act = act;
    if (out_alpha_host) { p.out_act = ACT_SNAKE; p.out_alpha = d + o_oa; p.out_inv_alpha = d + o_oia; }
    p.res = res; p.lane_len = lane_len;
    p.B = B; p.Tin = Tin; p.Cin = Cin; p.Tout = Tout; p.Cout = Cout; p.K = K; p.dil = dil; p.stride = stride;
    p.pad_left = pad_left; p.pad_right = pad_right; p.pad_reflect = reflect;
    p.ldw = ldw; p.ldy = Cout; p.ldx = Cin;
    p.x_bstride = (size_t)Tin * Cin; p.y_bstride = (size_t)Tout * Cout;
    cudaError_t e = launch_conv(p, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { h->err = std::string("fac_debug_conv: ") + cudaGetErrorString(e); return FAC_ERR_CUDA; }
    return FAC_OK;
}
}  // namespace

extern "C" {

int fac_debug_conv(fac_handle* h, const float* x, const float* w_host, const float* bias_host, int B, int Tin, int Cin,
                   int Cout, int K, int dil, int stride, int pad_left, int pad_right, int reflect,
                   const float* in_alpha_host, const float* out_alpha_host, int act, const float* res, float* y,
                   int Tout, void* stream) {
    return debug_conv(h, x, w_host, bias_host, B, Tin, Cin, Cout, K, dil, stride, pad_left, pad_right, reflect,
                      in_alpha_host, out_alpha_host, act, res, y, Tout, nullptr, stream);
}

}  // extern "C"

namespace {
// fac_debug_slstm, and with `carry` (DEVICE [B][2 layers][lane-map words], read as the initial state and overwritten with
// the final one) fac_debug_slstm_lanes: one pass over T with row b stopped after lens[b] steps (lens null: T).
int debug_slstm(fac_handle* h, const float* x, const float* const* w_host, int B, int T, int H, int upstream,
                const int* chunks, int n_chunks, const int* lens, uint32_t* carry, float* y, void* stream) {
    const bool chunked = chunks && n_chunks > 0;
    if (chunked) {
        long long sum = 0;
        for (int i = 0; i < n_chunks; ++i) {
            if (chunks[i] <= 0) { h->err = "fac_debug_slstm: chunk lengths must be positive"; return FAC_ERR_INVALID; }
            sum += chunks[i];
        }
        if (sum != T) { h->err = "fac_debug_slstm: chunk lengths must sum to T"; return FAC_ERR_INVALID; }
    }
    // a private handle carries the caller's precision options and its own workspace through the slstm code path
    fac_handle tmp;
    tmp.device = h->device;
    tmp.use_tc = h->use_tc; tmp.enc_f16 = h->enc_f16; tmp.enc_tt = h->enc_tt; tmp.tc_occ2 = h->tc_occ2;
    tmp.dec_bf16 = h->dec_bf16; tmp.dec_c7_f16 = h->dec_c7_f16;
    tmp.lstm_v2 = h->lstm_v2; tmp.dec_lstm_fp16 = h->dec_lstm_fp16;
    const char* names[8] = {"weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0", "weight_ih_l1", "weight_hh_l1", "bias_ih_l1", "bias_hh_l1"};
    TensorMap ts;
    for (int i = 0; i < 8; ++i) {
        HostTensor t;
        bool mat = (i % 4) < 2;
        if (mat) t.shape = {4 * H, H}; else t.shape = {4 * H};
        t.data.assign(w_host[i], w_host[i] + t.numel());
        ts[std::string("l.") + names[i]] = std::move(t);
    }
    // upstream: packed and run as the encoder's LSTM (promoted input projection, under vq_critical); else as the decoder's
    Packer P;
    LstmW L;
    try { L = pack_lstm(P, ts, "l", upstream != 0); } catch (const PackError& e) { h->err = e.msg; return FAC_ERR_UNSUPPORTED; }
    cudaStream_t st = (cudaStream_t)stream;
    size_t hw = 0, cf = 0;
    int pass3 = 0;
    if (chunked || carry) {
        Ctx probe{&tmp, st, true};
        probe.vq_critical = upstream != 0;
        if (B > 32 || !lstm_resident(probe, L)) {
            h->err = "fac_debug_slstm: chunks and lanes need B <= 32 and the resident-W LSTM kernel";
            return FAC_ERR_UNSUPPORTED;
        }
        pass3 = lstm_pass3(probe);
        lstm2_state_sizes(H, L.U, pass3, &hw, &cf);
    }
    DevBuf<float> w;
    int rc = upload_weights(h, P, w, "fac_debug_slstm");
    if (rc != FAC_OK) return rc;
    rc = two_pass(&tmp, st, w.get(), [&](Ctx& c) {
        c.vq_critical = upstream != 0;
        if (!chunked && !carry) { slstm(c, L, x, y, B, T); return; }
        // chunk by chunk with the state carried as fac_stream_encode / fac_stream_decode do, from a zero state; or from the
        // caller's per-lane carry, moved as the stream pools move it
        LstmState s;
        for (int l = 0; l < 2; ++l) {
            s.h[l] = c.alloc<uint32_t>(hw);
            s.c[l] = c.alloc<float>(cf);
            if (c.dry) continue;
            c.check_nk(cudaMemsetAsync(s.h[l], 0, sizeof(uint32_t) * hw, c.st), "slstm.state_h");
            c.check_nk(cudaMemsetAsync(s.c[l], 0, sizeof(float) * cf, c.st), "slstm.state_c");
        }
        if (carry) {
            auto lane = [&](int b) { return carry + (size_t)b * 2 * carry_words(H, pass3); };
            lane_carry(c, s, H, pass3, B, lane, 1);
            slstm(c, L, x, y, B, T, &s, lens);
            lane_carry(c, s, H, pass3, B, lane, 0);
            return;
        }
        for (int i = 0, t0 = 0; i < n_chunks; t0 += chunks[i++]) {
            const int n = chunks[i];
            float* xc = c.alloc<float>((size_t)B * n * H);
            float* yc = c.alloc<float>((size_t)B * n * H);
            copy_rows(c, xc, n, x, T, t0, n, H, B, "slstm.xc");
            slstm(c, L, xc, yc, B, n, &s);
            copy_rows(c, y + (size_t)t0 * H, T, yc, n, 0, n, H, B, "slstm.yc");
        }
    });
    cudaStreamSynchronize(st);
    if (rc != FAC_OK) h->err = tmp.err;
    return rc;
}
}  // namespace

extern "C" {

int fac_debug_slstm(fac_handle* h, const float* x, const float* const* w_host, int B, int T, int H, int upstream,
                    const int* chunks, int n_chunks, float* y, void* stream) {
    if (!h || !x || !w_host || !y || B <= 0 || T <= 0 || n_chunks < 0) return FAC_ERR_INVALID;
    return debug_slstm(h, x, w_host, B, T, H, upstream, chunks, n_chunks, nullptr, nullptr, y, stream);
}

int fac_debug_slstm_lanes(fac_handle* h, const float* x, const float* const* w_host, int B, int T, int H, int upstream,
                          const int* lens, uint32_t* carry, float* y, void* stream) {
    if (!h || !x || !w_host || !y || !carry || B <= 0 || T <= 0) return FAC_ERR_INVALID;
    if (lens && upstream) { h->err = "fac_debug_slstm_lanes: per-lane lengths run the decoder's one-pass class only"; return FAC_ERR_UNSUPPORTED; }
    for (int b = 0; lens && b < B; ++b)
        if (lens[b] < 0 || lens[b] > T) { h->err = "fac_debug_slstm_lanes: lane lengths must lie in [0, T]"; return FAC_ERR_INVALID; }
    return debug_slstm(h, x, w_host, B, T, H, upstream, nullptr, 0, lens, carry, y, stream);
}

int fac_debug_fa_quantize(fac_handle* h, const float* f0, const float* z, const float* const vq_host[6][5],
                          const float* gamma_beta, int n_c, int B, int Tq, int Tz, int Tf0, float* outs, float* zp,
                          float* zc, float* zr, int64_t* codes_p, int64_t* codes_c, int64_t* codes_r, float* sqerr,
                          float* losses2, void* stream) {
    if (!h || !f0 || !z || !vq_host || !gamma_beta || !outs || !codes_p || !codes_c || !codes_r || !sqerr || !losses2)
        return FAC_ERR_INVALID;
    if (n_c < 1 || n_c > 2 || B <= 0 || Tq <= 0 || Tz < Tq || Tf0 < Tq) return FAC_ERR_INVALID;
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 5; ++j)
            if (!vq_host[i][j]) return FAC_ERR_INVALID;
    Packer P;
    VqW v[6];
    for (int i = 0; i < 6; ++i) v[i] = pack_vq_raw(P, vq_host[i][0], vq_host[i][1], vq_host[i][2], vq_host[i][3], vq_host[i][4]);
    cudaStream_t st = (cudaStream_t)stream;
    DevBuf<float> buf;
    const int rc = upload(h, P.pack, buf, "fac_debug_fa_quantize");
    if (rc != FAC_OK) return rc;
    const float* d = buf.get();
    FaqParams fp;
    fp.f0 = f0; fp.z = z;
    for (int i = 0; i < 6; ++i)
        fp.vq[i] = VqWeights{d + v[i].w_in, d + v[i].b_in, d + v[i].cb, d + v[i].cbn, d + v[i].cbn2, d + v[i].w_out, d + v[i].b_out};
    fp.n_c = n_c;
    fp.gamma_beta = gamma_beta;
    fp.outs = outs; fp.zp = zp; fp.zc = zc; fp.zr = zr;
    fp.codes_p = codes_p; fp.codes_c = codes_c; fp.codes_r = codes_r;
    fp.sqerr = sqerr;
    fp.B = B; fp.Tq = Tq; fp.Tz = Tz; fp.Tf0 = Tf0;
    cudaError_t e = launch_fa_quantize(fp, st);
    if (e == cudaSuccess) e = launch_vq_loss_reduce(sqerr, 6, B, Tq, losses2, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { h->err = std::string("fac_debug_fa_quantize: ") + cudaGetErrorString(e); return FAC_ERR_CUDA; }
    return FAC_OK;
}

int fac_debug_attention(fac_handle* h, const float* q, const float* k, const float* v, float* o, int B, int T,
                        int heads, const int* valid_len, int force_stream, void* stream) {
    if (!h || !q || !k || !v || !o || B <= 0 || T <= 0 || heads <= 0) return FAC_ERR_INVALID;
    cudaSetDevice(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = launch_attention(q, k, v, o, B, T, heads, 256, valid_len, st, force_stream ? 1 : 0);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { h->err = std::string("fac_debug_attention: ") + cudaGetErrorString(e); return FAC_ERR_CUDA; }
    return FAC_OK;
}

int fac_set_option(fac_handle* h, const char* name, int value) {
    if (!h || !name) return FAC_ERR_INVALID;
    if (std::string(name) == "fuse_resunit") { h->fuse_res = value < 0 ? 0 : (value > 2 ? 2 : value); return FAC_OK; }
    if (std::string(name) == "encoder_f16x2") { h->enc_f16 = value != 0; return FAC_OK; }
    if (std::string(name) == "encoder_tt") { h->enc_tt = value != 0; return FAC_OK; }
    if (std::string(name) == "tc_occ2_maxn") { h->tc_occ2 = value < 0 ? 0 : value; return FAC_OK; }
    if (std::string(name) == "decoder_conv7_fp16") { h->dec_c7_f16 = value != 0; return FAC_OK; }
    if (std::string(name) == "overlap_front") { h->overlap_front = value != 0; return FAC_OK; }
    if (std::string(name) == "lstm_v2") { h->lstm_v2 = value != 0; return FAC_OK; }
    if (std::string(name) == "decoder_lstm_fp16") { h->dec_lstm_fp16 = value != 0; return FAC_OK; }
    if (std::string(name) == "attention_stream") { h->attn_stream = value != 0; return FAC_OK; }
    if (std::string(name) == "decoder_bf16") { h->dec_bf16 = value != 0; return FAC_OK; }
    if (std::string(name) == "tensor_cores") { h->use_tc = value < 0 ? 0 : (value > 2 ? 2 : value); return FAC_OK; }
    h->err = std::string("unknown option ") + name;
    return FAC_ERR_INVALID;
}

static int debug_conv_tc(fac_handle* h, const float* x, const float* w_host, const float* bias_host, int B, int Tin, int Cin,
                         int Cout, int K, int dil, int stride, int pad_left, int pad_right, int reflect,
                         const float* in_alpha_host, const float* out_alpha_host, int act, const float* res, float* y,
                         int Tout, int promoted, void* stream, int* group_out, const int* lane_len) {
    if (!h || !x || !w_host || !y) return FAC_ERR_INVALID;
    cudaSetDevice(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    TcConvParams tp;
    tp.Cin = Cin; tp.Cout = Cout; tp.promoted = (promoted == 1 || promoted == 3 || promoted == 4) ? 1 : 0;
    tp.bf16 = (promoted == 2 || promoted == 5) ? 1 : 0;
    tp.f16x2 = (promoted == 3 || promoted == 4) ? 1 : 0;
    tp.tt = promoted == 4 ? 1 : 0;         // 4 = the transposed formulation of class 3
    tp.g1f16 = promoted == 5 ? 1 : 0;      // 5 = the one-pass fp16 class of conv_tc_kernel
    tp.occ2_maxn = h->tc_occ2;
    tp.Tout = Tout;
    if (stride == 1) { tp.vf = 1; tp.Kr = K; tp.dil = dil; }
    else if (K == 2 * stride && dil == 1) { tp.vf = stride; tp.Kr = 2; tp.dil = 1; }
    else { h->err = "fac_debug_conv_tc: unsupported stride/kernel"; return FAC_ERR_UNSUPPORTED; }
    if (promoted < 0 || promoted > 5 || !tc_conv_plan(tp)) { h->err = "fac_debug_conv_tc: layer not eligible for the tensor-core path"; return FAC_ERR_UNSUPPORTED; }
    if (group_out) {                       // report the plan's chunks per step, run the one-chunk plan
        *group_out = tp.group;
        tp.max_group = 1;
        if (!tc_conv_plan(tp)) { h->err = "fac_debug_conv_tc_group1: no one-chunk plan"; return FAC_ERR_UNSUPPORTED; }
    }
    int ldw = (Cout + 3) / 4 * 4;
    std::vector<float> gen((size_t)K * Cin * ldw, 0.f);
    for (int co = 0; co < Cout; ++co)
        for (int ci = 0; ci < Cin; ++ci)
            for (int k = 0; k < K; ++k) gen[((size_t)k * Cin + ci) * ldw + co] = w_host[((size_t)co * Cin + ci) * K + k];
    size_t nb = tc_blob_floats(tp);
    auto al4 = [](size_t v) { return (v + 3) / 4 * 4; };
    size_t o_b = al4(nb), o_ia = al4(o_b + Cout), o_iia = al4(o_ia + Cin), o_oa = al4(o_iia + Cin), o_oia = al4(o_oa + Cout);
    std::vector<float> pk(o_oia + Cout + 16, 0.f);
    tc_pack_blob(tp, gen.data(), ldw, pk.data());
    for (int i = 0; i < Cout; ++i) pk[o_b + i] = bias_host ? bias_host[i] : 0.f;
    for (int i = 0; i < Cin; ++i) { pk[o_ia + i] = in_alpha_host ? in_alpha_host[i] : 1.f; pk[o_iia + i] = 1.0f / (pk[o_ia + i] + 1e-9f); }
    for (int i = 0; i < Cout; ++i) { pk[o_oa + i] = out_alpha_host ? out_alpha_host[i] : 1.f; pk[o_oia + i] = 1.0f / (pk[o_oa + i] + 1e-9f); }
    DevBuf<float> buf;
    const int rc = upload(h, pk, buf, "fac_debug_conv_tc");
    if (rc != FAC_OK) return rc;
    const float* d = buf.get();
    tp.x = x; tp.y = y; tp.wblob = d; tp.bias = d + o_b;
    if (in_alpha_host) { tp.in_alpha = d + o_ia; tp.in_inv_alpha = d + o_iia; }
    tp.out_act = act;
    if (out_alpha_host) { tp.out_act = ACT_SNAKE; tp.out_alpha = d + o_oa; tp.out_inv_alpha = d + o_oia; }
    tp.res = res;
    tp.B = B; tp.Tin = Tin; tp.ldx = Cin;
    tp.PLr = pad_left / tp.vf;
    tp.pad_left_s = pad_left; tp.pad_right_s = pad_right; tp.reflect = reflect; tp.lane_len = lane_len;
    tp.Tout = Tout; tp.ldy = Cout;
    tp.x_bstride = (size_t)Tin * Cin; tp.y_bstride = (size_t)Tout * Cout;
    cudaError_t e = launch_conv_tc(tp, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { h->err = std::string("fac_debug_conv_tc: ") + cudaGetErrorString(e); return FAC_ERR_CUDA; }
    return FAC_OK;
}

int fac_debug_conv_tc(fac_handle* h, const float* x, const float* w_host, const float* bias_host, int B, int Tin, int Cin,
                      int Cout, int K, int dil, int stride, int pad_left, int pad_right, int reflect,
                      const float* in_alpha_host, const float* out_alpha_host, int act, const float* res, float* y,
                      int Tout, int promoted, void* stream) {
    return debug_conv_tc(h, x, w_host, bias_host, B, Tin, Cin, Cout, K, dil, stride, pad_left, pad_right, reflect,
                         in_alpha_host, out_alpha_host, act, res, y, Tout, promoted, stream, nullptr, nullptr);
}

int fac_debug_conv_tc_group1(fac_handle* h, const float* x, const float* w_host, const float* bias_host, int B, int Tin,
                             int Cin, int Cout, int K, int dil, int stride, int pad_left, int pad_right, int reflect,
                             const float* in_alpha_host, const float* out_alpha_host, int act, const float* res, float* y,
                             int Tout, int promoted, void* stream, int* group) {
    if (!group) return FAC_ERR_INVALID;
    return debug_conv_tc(h, x, w_host, bias_host, B, Tin, Cin, Cout, K, dil, stride, pad_left, pad_right, reflect,
                         in_alpha_host, out_alpha_host, act, res, y, Tout, promoted, stream, group, nullptr);
}

int fac_debug_conv_lanes(fac_handle* h, const float* x, const float* w_host, const float* bias_host, int B, int Tin,
                         int Cin, int Cout, int K, int dil, int stride, int pad_left, int pad_right, int reflect,
                         const float* in_alpha_host, const float* out_alpha_host, int act, const float* res, float* y,
                         int Tout, int path, const int* lane_len_host, void* stream) {
    if (!h || !x || !w_host || !y || B <= 0 || Tin <= 0) return FAC_ERR_INVALID;
    DevBuf<int> lanes;
    int rc = debug_upload_lanes(h, "fac_debug_conv_lanes", lane_len_host, B, Tin, lanes);
    if (rc != FAC_OK) return rc;
    if (path == -1)
        return debug_conv(h, x, w_host, bias_host, B, Tin, Cin, Cout, K, dil, stride, pad_left, pad_right, reflect,
                          in_alpha_host, out_alpha_host, act, res, y, Tout, lanes.get(), stream);
    return debug_conv_tc(h, x, w_host, bias_host, B, Tin, Cin, Cout, K, dil, stride, pad_left, pad_right, reflect,
                         in_alpha_host, out_alpha_host, act, res, y, Tout, path, stream, nullptr, lanes.get());
}

int fac_debug_resunit(fac_handle* h, const float* x, const float* w7_host, const float* b7_host, const float* w1_host,
                      const float* b1_host, const float* alpha1_host, const float* alpha2_host, int B, int T, int C,
                      int dil, int mode, float* y, void* stream) {
    return fac_debug_resunit_lanes(h, x, w7_host, b7_host, w1_host, b1_host, alpha1_host, alpha2_host, B, T, C, dil, mode,
                                   1, nullptr, y, stream);
}

int fac_debug_resunit_lanes(fac_handle* h, const float* x, const float* w7_host, const float* b7_host,
                            const float* w1_host, const float* b1_host, const float* alpha1_host,
                            const float* alpha2_host, int B, int T, int C, int dil, int mode, int causal,
                            const int* lane_len_host, float* y, void* stream) {
    if (!h || !x || !y || !w7_host || !w1_host || B <= 0 || T <= 0) return FAC_ERR_INVALID;
    DevBuf<int> lanes;
    int rc = debug_upload_lanes(h, "fac_debug_resunit_lanes", lane_len_host, B, T, lanes);
    if (rc != FAC_OK) return rc;
    if (mode < 0 || mode > 8) return FAC_ERR_INVALID;
    fac_handle tmp;             // carries this call's precision options
    tmp.device = h->device;
    // 0: fp32 FMA, 1: two tensor-core launches, 2: fused launch; 3/4 = 1/2 with bf16 split; 5/6 = 3/4 with the k = 7 conv
    // in one fp16 pass; 7/8 = 1/2 as an encoder unit (promoted fp16 hi + scaled lo, upstream of the VQ)
    const bool enc = mode >= 7, fused = mode == 2 || mode == 4 || mode == 6 || mode == 8;
    tmp.use_tc = mode == 0 ? 0 : (enc ? 2 : 1);
    tmp.fuse_res = fused ? 1 : 0;
    tmp.dec_bf16 = mode >= 3 && !enc;
    tmp.dec_c7_f16 = mode >= 5 && !enc;
    tmp.tc_occ2 = h->tc_occ2;
    TensorMap ts;
    auto put = [&](const char* key, const float* d, std::vector<int64_t> shp) {
        HostTensor t;
        t.shape = shp;
        t.data.assign(d, d + t.numel());
        ts[key] = std::move(t);
    };
    put("u.block.0.alpha", alpha1_host, {1, C, 1});
    put("u.block.1.conv.conv.weight", w7_host, {C, C, 7});
    put("u.block.1.conv.conv.bias", b7_host, {C});
    put("u.block.2.alpha", alpha2_host, {1, C, 1});
    put("u.block.3.conv.conv.weight", w1_host, {C, C, 1});
    put("u.block.3.conv.conv.bias", b1_host, {C});
    Packer P;
    ResW r;
    try { r = pack_res(P, ts, "u", dil, enc); } catch (const PackError& e) { h->err = e.msg; return FAC_ERR_STATE; }
    DevBuf<float> w;
    rc = upload_weights(h, P, w, "fac_debug_resunit_lanes");
    if (rc != FAC_OK) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    float* p = nullptr;
    cudaError_t e = cudaMalloc(&p, sizeof(float) * (size_t)B * T * C);
    DevBuf<float> scratch(p);
    if (e != cudaSuccess) { h->err = cudaGetErrorString(e); cudaGetLastError(); return FAC_ERR_CUDA; }
    Ctx c{&tmp, st, false, w.get()};
    c.vq_critical = enc;
    residual_unit(c, r, x, scratch.get(), y, B, T, causal != 0, lanes.get());
    rc = finish(&tmp, c);
    cudaError_t e2 = cudaStreamSynchronize(st);
    if (rc == FAC_OK && e2 != cudaSuccess) { tmp.err = cudaGetErrorString(e2); rc = FAC_ERR_CUDA; }
    if (rc == FAC_OK && fused && tmp.launches != 1) { tmp.err = "fused path not taken for this geometry"; rc = FAC_ERR_UNSUPPORTED; }
    if (rc != FAC_OK) h->err = tmp.err;
    return rc;
}

// Host-only: the recurrent-weight packing of lstm_rec_kernel for one nn.LSTM weight_hh [4H][H]:
// bf16 = 0 -> fp32 [G][H][4U] (row r = gate*U + u of CTA g); bf16 = 1 -> [G][H/16][hi|lo][8 k-pairs][4U] 32-bit words.
// Returns the number of 32-bit words (G*H*4U); info3 = {U, G, 4U}.
long long fac_debug_lstm_pack(const float* whh_host, int H, int bf16, float* out, long long capacity_floats, int* info3) {
    if (!whh_host || H <= 0) return FAC_ERR_INVALID;
    const char* names[8] = {"weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0", "weight_ih_l1", "weight_hh_l1", "bias_ih_l1", "bias_hh_l1"};
    TensorMap ts;
    for (int i = 0; i < 8; ++i) {
        HostTensor t;
        const bool mat = (i % 4) < 2;
        if (mat) t.shape = {4 * H, H}; else t.shape = {4 * H};
        if (i == 1) t.data.assign(whh_host, whh_host + (size_t)4 * H * H);
        else t.data.assign(t.numel(), 0.f);
        ts[std::string("l.") + names[i]] = std::move(t);
    }
    Packer P;
    LstmW L;
    try { L = pack_lstm(P, ts, "l"); } catch (const PackError&) { return FAC_ERR_UNSUPPORTED; }
    if (info3) { info3[0] = L.U; info3[1] = L.G; info3[2] = 4 * L.U; }
    if (bf16 == 2 || bf16 == 3) {
        // lstm2.cu layouts: 2 = one fp16 pass [G][H/16][8][4U] words, 3 = fp16 hi + scaled lo [G][H/16][hi|lo][8][4U]
        const int p3 = bf16 == 3;
        const long long n2 = (long long)lstm2_pack_words(H, L.U, p3);
        if (!out || capacity_floats < n2) return n2;
        lstm2_pack(whh_host, H, L.U, p3, reinterpret_cast<uint32_t*>(out));
        return n2;
    }
    const long long n = (long long)L.G * H * 4 * L.U;
    if (bf16 && !L.has16) return FAC_ERR_UNSUPPORTED;
    if (!out || capacity_floats < n) return n;
    memcpy(out, P.pack.data() + (bf16 ? L.whh16[0] : L.whh[0]), sizeof(float) * (size_t)n);
    return n;
}

// Host-only: the conv form of nn.ConvTranspose1d(k = 2s, stride s) weights [Cin][Cout][2s] (HOST, already weight-normed):
// causal != 0 -> 2 taps (x[t-1], x[t]); causal == 0 -> 3 taps (x[t-1], x[t], x[t+1]) (encodec.py:248-270 trims).  out is
// [taps][Cin][s*Cout] (phase-major output channels r*Cout + co); returns the number of floats.
long long fac_debug_convtr_pack(const float* w_host, int Cin, int Cout, int stride, int causal, float* out, long long capacity_floats) {
    if (!w_host || Cin <= 0 || Cout <= 0 || stride <= 0) return FAC_ERR_INVALID;
    HostTensor t, b;
    t.shape = {Cin, Cout, 2 * stride};
    t.data.assign(w_host, w_host + (size_t)Cin * Cout * 2 * stride);
    b.shape = {Cout};
    b.data.assign(Cout, 0.f);
    TensorMap ts;
    ts["c.weight"] = std::move(t);
    ts["c.bias"] = std::move(b);
    Packer P;
    ConvW c;
    try { c = causal ? pack_convtr(P, ts, "c", stride) : pack_convtr_noncausal(P, ts, "c", stride); }
    catch (const PackError&) { return FAC_ERR_UNSUPPORTED; }
    const long long n = (long long)c.K * Cin * c.Cout;
    if (!out || capacity_floats < n) return n;
    for (int k = 0; k < c.K; ++k)
        for (int ci = 0; ci < Cin; ++ci)
            for (int co = 0; co < c.Cout; ++co) out[((size_t)k * Cin + ci) * c.Cout + co] = P.pack[c.w + ((size_t)k * Cin + ci) * c.ldw + co];
    return n;
}

// Host-only: the padding index map every conv kernel uses (common.cuh PadMap): out[i] = source row of padded position
// i - pad_left, or -1 where the padded value is zero.
int fac_debug_pad_map(int L, int pad_left, int pad_right, int reflect, int* out, int n) {
    if (!out || L < 0 || pad_left < 0 || pad_right < 0 || n != pad_left + L + pad_right) return FAC_ERR_INVALID;
    const PadMap pm = PadMap::make(L, pad_left, pad_right, reflect);
    for (int i = 0; i < n; ++i) out[i] = pm.src(i - pad_left);
    return FAC_OK;
}

// Host-only: the same map for every lane of a batch of B lanes with their own lengths, as the conv kernels build it
// (PadMap::lane): out[b * n + i] = source row of padded position i - pad_left of lane b, n = pad_left + Tin + pad_right.
int fac_debug_lane_pad_map(const int* lane_len, int B, int Tin, int pad_left, int pad_right, int reflect, int* out, int n) {
    if (!out || B <= 0 || Tin < 0 || pad_left < 0 || pad_right < 0 || n != pad_left + Tin + pad_right) return FAC_ERR_INVALID;
    for (int b = 0; lane_len && b < B; ++b)
        if (lane_len[b] < 0 || lane_len[b] > Tin) return FAC_ERR_INVALID;
    for (int b = 0; b < B; ++b) {
        const PadMap pm = PadMap::lane(lane_len, b, Tin, pad_left, pad_right, reflect);
        for (int i = 0; i < n; ++i) out[(size_t)b * n + i] = pm.src(i - pad_left);
    }
    return FAC_OK;
}

// Host-only: the tile plan the tensor-core conv kernel would use for a layer geometry (no GPU, no handle).
static int debug_tc_plan(int Cin, int Cout, int K, int dil, int stride, int Tout, int mode, int occ2_maxn, TcConvParams& tp) {
    if (Cin <= 0 || Cout <= 0 || K <= 0 || dil <= 0 || stride <= 0 || mode < 0 || mode > 9) return FAC_ERR_INVALID;
    tp.Cin = Cin; tp.Cout = Cout; tp.Tout = Tout; tp.occ2_maxn = occ2_maxn;
    tp.promoted = (mode == 1 || mode == 3 || mode == 9) ? 1 : 0;
    tp.bf16 = (mode == 2 || mode == 4 || mode == 7 || mode == 8) ? 1 : 0;
    tp.f16x2 = (mode == 3 || mode == 9) ? 1 : 0;
    tp.fused = (mode == 4 || mode == 5 || mode == 8 || mode == 9) ? 1 : 0;     // 9: fused ResidualUnit of mode 3
    tp.g1f16 = (mode == 7 || mode == 8) ? 1 : 0;                     // 7 / 8: one-pass fp16 class, plain / fused
    if (mode == 6) { tp.promoted = 1; tp.f16x2 = 1; tp.tt = 1; }     // 6: transposed formulation of mode 3
    if (stride == 1) { tp.vf = 1; tp.Kr = K; tp.dil = dil; }
    else if (K == 2 * stride && dil == 1) { tp.vf = stride; tp.Kr = 2; tp.dil = 1; }
    else return FAC_ERR_UNSUPPORTED;
    return tc_conv_plan(tp) ? FAC_OK : FAC_ERR_UNSUPPORTED;
}

int fac_debug_tc_plan(int Cin, int Cout, int K, int dil, int stride, int Tout, int mode, int occ2_maxn, int* out8) {
    if (!out8) return FAC_ERR_INVALID;
    TcConvParams tp;
    const int rc = debug_tc_plan(Cin, Cout, K, dil, stride, Tout, mode, occ2_maxn, tp);
    if (rc != FAC_OK) return rc;
    out8[0] = tp.N; out8[1] = tp.MT; out8[2] = tp.nchunk; out8[3] = tp.stagesB; out8[4] = tp.R2pad;
    out8[5] = (int)tp.smem_bytes; out8[6] = tp.Rpad; out8[7] = tp.promote_every;
    return FAC_OK;
}

int fac_debug_tc_plan_group(int Cin, int Cout, int K, int dil, int stride, int Tout, int mode, int occ2_maxn, int* smem2) {
    TcConvParams tp;
    const int rc = debug_tc_plan(Cin, Cout, K, dil, stride, Tout, mode, occ2_maxn, tp);
    if (rc != FAC_OK) return rc;
    if (smem2) {
        TcConvParams t1 = tp;
        t1.max_group = 1;
        if (!tc_conv_plan(t1)) return FAC_ERR_UNSUPPORTED;
        smem2[0] = (int)tp.smem_bytes;
        smem2[1] = (int)t1.smem_bytes;
    }
    return tp.group;
}

// Host-only: the tensor-core weight blob (tc_pack_blob) for nn.Conv1d weights [Cout][Cin][K]; returns the number of
// floats (32-bit words) of the blob, writes it when blob_out has room.
long long fac_debug_tc_pack(const float* w_host, int Cin, int Cout, int K, int stride, int mode, float* blob_out,
                            long long capacity_floats) {
    if (!w_host || Cin <= 0 || Cout <= 0 || K <= 0 || stride <= 0 || mode < 0 || mode > 3) return FAC_ERR_INVALID;
    TcConvParams tp;
    tp.Cin = Cin; tp.Cout = Cout; tp.dil = 1;
    tp.promoted = (mode == 1 || mode == 3) ? 1 : 0; tp.bf16 = mode == 2 ? 1 : 0; tp.f16x2 = mode == 3 ? 1 : 0;
    if (stride == 1) { tp.vf = 1; tp.Kr = K; }
    else if (K == 2 * stride) { tp.vf = stride; tp.Kr = 2; }
    else return FAC_ERR_UNSUPPORTED;
    if (!tc_conv_plan(tp)) return FAC_ERR_UNSUPPORTED;
    const long long n = (long long)tc_blob_floats(tp);
    if (!blob_out || capacity_floats < n) return n;
    const int ldw = (Cout + 3) / 4 * 4;
    std::vector<float> gen((size_t)K * Cin * ldw, 0.f);      // generic packed layout [K*Cin][ldw]
    for (int co = 0; co < Cout; ++co)
        for (int ci = 0; ci < Cin; ++ci)
            for (int k = 0; k < K; ++k) gen[((size_t)k * Cin + ci) * ldw + co] = w_host[((size_t)co * Cin + ci) * K + k];
    tc_pack_blob(tp, gen.data(), ldw, blob_out);
    return n;
}

int fac_debug_tc_phase_clocks(fac_handle* h, long long* out8) {
    if (!h || !out8) return FAC_ERR_INVALID;
    h->err = "fac_debug_tc_phase_clocks: the tensor-core conv kernel records no timing probes";
    return FAC_ERR_UNSUPPORTED;
}

int fac_debug_tc_trace(fac_handle* h, long long* out80) {
    if (!h || !out80) return FAC_ERR_INVALID;
    h->err = "fac_debug_tc_trace: the tensor-core conv kernel records no timing probes";
    return FAC_ERR_UNSUPPORTED;
}

int fac_debug_tc_producer_clocks(fac_handle* h, long long* out4) {
    if (!h || !out4) return FAC_ERR_INVALID;
    h->err = "fac_debug_tc_producer_clocks: the tensor-core conv kernel records no timing probes";
    return FAC_ERR_UNSUPPORTED;
}

int fac_debug_lstm_phase_clocks(fac_handle* h, long long* out4) {
    if (!h || !out4) return FAC_ERR_INVALID;
    cudaSetDevice(h->device);
    cudaDeviceSynchronize();
    cudaError_t e = h->lstm_v2 ? lstm2_read_phase_clocks(out4) : lstm_read_phase_clocks(out4);
    if (e != cudaSuccess) { h->err = cudaGetErrorString(e); return FAC_ERR_CUDA; }
    return FAC_OK;
}

int fac_debug_tap(fac_handle* h, const char* name, float* dst, size_t capacity_floats) {
    if (!h || !name) return FAC_ERR_INVALID;
    if (!dst) h->taps.erase(name);
    else h->taps[name] = std::make_pair(dst, capacity_floats);
    return FAC_OK;
}

int fac_profile_enable(fac_handle* h, int on) {
    if (!h) return FAC_ERR_INVALID;
    h->profiling = on != 0;
    return FAC_OK;
}

// Resolves pending event pairs (synchronises the device) and folds them into per-family totals.
static void profile_collect(fac_handle* h) {
    if (h->prof.empty()) return;
    cudaSetDevice(h->device);
    cudaDeviceSynchronize();
    for (auto& r : h->prof) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, r.a, r.b);
        auto& a = h->prof_agg[r.name];
        a.ms += ms; a.flops += r.flops; a.bytes += r.bytes; a.launches++;
        cudaEventDestroy(r.a); cudaEventDestroy(r.b);
    }
    h->prof.clear();
}

int fac_profile_reset(fac_handle* h) {
    if (!h) return FAC_ERR_INVALID;
    profile_collect(h);
    h->prof_agg.clear();
    return FAC_OK;
}

int fac_profile_get(fac_handle* h, const char* family, double* ms, double* flops, double* bytes, long long* launches) {
    if (!h || !family) return FAC_ERR_INVALID;
    profile_collect(h);
    std::string fam(family);
    fac_handle::ProfAgg t;
    for (auto& kv : h->prof_agg) {
        if (kv.first == fam || (kv.first.size() > fam.size() && kv.first.compare(0, fam.size(), fam) == 0 && kv.first[fam.size()] == ':')) {
            t.ms += kv.second.ms; t.flops += kv.second.flops; t.bytes += kv.second.bytes; t.launches += kv.second.launches;
        }
    }
    if (ms) *ms = t.ms;
    if (flops) *flops = t.flops;
    if (bytes) *bytes = t.bytes;
    if (launches) *launches = t.launches;
    return FAC_OK;
}

// Text dump "key\tms\tgflop\tgbytes\tlaunches\n" of every profiled call site; returns bytes needed.
size_t fac_profile_dump(fac_handle* h, char* buf, size_t cap) {
    if (!h) return 0;
    profile_collect(h);
    std::string out;
    char line[256];
    for (auto& kv : h->prof_agg) {
        snprintf(line, sizeof line, "%s\t%.4f\t%.3f\t%.4f\t%ld\n", kv.first.c_str(), kv.second.ms, kv.second.flops / 1e9,
                 kv.second.bytes / 1e9, kv.second.launches);
        out += line;
    }
    if (buf && cap > 0) {
        size_t n = out.size() < cap - 1 ? out.size() : cap - 1;
        memcpy(buf, out.data(), n);
        buf[n] = 0;
    }
    return out.size() + 1;
}

size_t fac_workspace_bytes(const fac_handle* h) { return h ? h->ws_bytes : 0; }
int fac_last_launch_count(const fac_handle* h) { return h ? h->launches : 0; }

}  // extern "C"
