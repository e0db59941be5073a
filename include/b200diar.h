/* b200diar.h -- C ABI of the H100-native (sm_90a) community-1 diarization hot path.
 *
 * Drop-in boundary for pyannote.audio's sliding-window inference path.  The reference is 100 % Python and has no
 * FFI for this path, so each entry point cites the *Python* interface it replaces (paths relative to
 * /root/reference/src/pyannote/audio).  All functions return 0 on success or a negative b200_status; the message
 * for the calling thread's last failure is available from b200_last_error().  No exceptions cross this boundary,
 * no torch types appear in it: device buffers are raw CUDA pointers owned by the caller, `stream` is a
 * cudaStream_t passed as void*, weights are host fp32 arrays in PyTorch state-dict layout.
 * One ctx per (process, device); a ctx is not thread-safe, use one per stream/thread.
 */
#ifndef B200DIAR_H_
#define B200DIAR_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200_ctx b200_ctx;

enum b200_status {
  B200_STATUS_OK = 0,
  B200_STATUS_INVALID = -1, /* bad argument / unsupported shape            -> ValueError  */
  B200_STATUS_CUDA = -2,    /* CUDA runtime / driver failure               -> RuntimeError */
  B200_STATUS_OOM = -3,     /* cudaErrorMemoryAllocation (inference.py:201-206 maps OOM to MemoryError) */
  B200_STATUS_STATE = -4    /* weights not loaded, ctx misuse                -> RuntimeError */
};

/* fixed geometry of the path */
#define B200_CHUNK_SAMPLES 160000
#define B200_FRAMES_PER_CHUNK 589
#define B200_LOCAL_SPEAKERS 3
#define B200_POWERSET_CLASSES 7
#define B200_EMBED_DIM 256
#define B200_FBANK_FRAMES 998
#define B200_MEL_BINS 80

const char* b200_last_error(void);
int b200_version(void);

/* Model.to(device) / Inference.to(device)  (core/inference.py:169-180) */
int b200_ctx_create(b200_ctx** ctx, int device);
int b200_ctx_destroy(b200_ctx* ctx);
/* Tuning / A-B options (no reference counterpart; results do not depend on the sub-batch sizes):
 *   "seg_max_batch" (2112) / "emb_max_batch" (264): chunks per sub-batch = workspace size (INTEGRATION.md section 4);
 *   "ssl_max_batch" (32): 10 s windows per SSeRiouSS sub-batch, also the longest SSeRiouSS window (32 x 10 s);
 *   "conv_impl" 1 = wgmma tensor-core trunk convs (default), 0 = CUDA-core reference conv; "seg_gemm_impl" 1 = wgmma
 *   split-precision GEMMs, 0 = fp32 CUDA-core twins; "seg_conv_impl" 1 = SincNet sinc / Conv1d layers as split-precision
 *   wgmma implicit GEMMs in persistent kernels, 2 = the same with one CTA per tile (bit-identical), 0 = fp32 CUDA-core twins; "seg_rec_impl" 1 = LSTM recurrence as split-precision wgmma on
 *   2-CTA clusters with two warpgroups per CTA (with "seg_gemm_impl" 1), 2 = the same with one warpgroup per CTA
 *   (bit-identical), 0 = fp32 CUDA-core twin; "fbank_share" 1 = overlapping chunks share their fbank frames;
 *   "profile" 1 = CUDA-event timers around the trunk / the segmentation (b200_ctx_timer); "linkage_grid_min" (32769,
 *   from 2 up to that default): the smallest linkage problem that runs on the whole-GPU path (b200_linkage_centroid).
 *   Unknown keys and values out of range return B200_ERR_INVALID. */
int b200_ctx_set_option(b200_ctx* ctx, const char* key, int64_t value);
/* number of kernels this ctx has launched so far; memcpy and memset operations are not counted */
int64_t b200_ctx_launch_count(const b200_ctx* ctx);
/* with option "profile" = 1 the library brackets the ResNet trunk ("trunk": conv kernels) and the segmentation
 * network ("seg") with CUDA events on the caller's stream; this returns and resets the accumulated device time
 * and the number of units (segments / chunks) processed.  Synchronises the device. */
int b200_ctx_timer(b200_ctx* ctx, const char* name, double* total_ms, int64_t* units);

/* ---- weights: Model.from_pretrained state_dict (core/model.py:497-655) ------------------------------------ */

/* PyanNet (models/segmentation/PyanNet.py:92-161, models/blocks/sincnet.py:41-79). Index of LSTM arrays =
 * layer * 2 + direction (0 = forward, 1 = "_reverse"); PyTorch layouts ([4H][I], [4H][H], [4H]), gate order i,f,g,o. */
typedef struct b200_seg_weights {
  float wav_norm_weight, wav_norm_bias;       /* sincnet.wav_norm1d.{weight,bias}                       */
  const float* sinc_filters;                  /* [80][251] realised ParamSincFB bank (cos 0..39, sin 40..79) */
  const float* norm_weight[3];                /* sincnet.norm1d.{0,1,2}.weight  (80, 60, 60)            */
  const float* norm_bias[3];
  const float* conv_weight[2];                /* sincnet.conv1d.{1,2}.weight  [60][80][5], [60][60][5]  */
  const float* conv_bias[2];
  int32_t lstm_layers;                        /* <= 4 */
  const float* lstm_w_ih[8];
  const float* lstm_w_hh[8];
  const float* lstm_b_ih[8];
  const float* lstm_b_hh[8];
  const float* linear_weight[2];              /* linear.{0,1}.weight [128][256], [128][128]             */
  const float* linear_bias[2];
  const float* classifier_weight;             /* [7][128] */
  const float* classifier_bias;               /* [7]      */
} b200_seg_weights;
/* Model.load_state_dict / Model.from_pretrained (core/model.py:497-655) for PyanNet: host fp32 arrays in PyTorch layouts;
 * fp16 (hi, lo) splits, LSTM shared-memory images and the sinc bank's tensor-core layout are made here, once.
 * b200_seg_load is b200_seg_load_head(ctx, w, 7, B200_SEG_LOGSOFTMAX): the community-1 powerset head. */
int b200_seg_load(b200_ctx* ctx, const b200_seg_weights* w);
/* PyanNet with any classifier head (models/segmentation/PyanNet.py:141-161, core/model.py:271-300):
 * classifier_weight is [num_classes][128], classifier_bias [num_classes], 1 <= num_classes <= 32.
 * B200_SEG_LOGSOFTMAX: mono-label / powerset problems, run with b200_seg_forward_window;
 * B200_SEG_SIGMOID: binary / multi-label problems, run with b200_seg_forward_scores.
 * Other class counts or activations return B200_STATUS_INVALID. */
#define B200_SEG_LOGSOFTMAX 0
#define B200_SEG_SIGMOID 1
#define B200_SEG_MAX_CLASSES 32
int b200_seg_load_head(b200_ctx* ctx, const b200_seg_weights* w, int32_t num_classes, int32_t activation);

/* WeSpeakerResNet34 (models/embedding/wespeaker/resnet.py:84-145, 214-252).  conv weight [Cout][Cin][k][k] fp32,
 * eval-mode BatchNorm2d given by (weight, bias, running_mean, running_var), eps 1e-5; folded by the library. */
typedef struct b200_conv_bn {
  const float* conv_weight;                   /* NULL => layer absent (identity shortcut)               */
  const float* bn_weight;
  const float* bn_bias;
  const float* bn_mean;
  const float* bn_var;
} b200_conv_bn;
typedef struct b200_emb_weights {
  b200_conv_bn stem;                          /* resnet.conv1 / resnet.bn1                               */
  b200_conv_bn block_conv1[16];               /* resnet.layer{1..4}.{i}.conv1/bn1, blocks in order 3+4+6+3 */
  b200_conv_bn block_conv2[16];
  b200_conv_bn block_shortcut[16];            /* resnet.layer{2..4}.0.shortcut.{0,1}                      */
  const float* seg1_weight;                   /* resnet.seg_1.weight [256][5120]                          */
  const float* seg1_bias;                     /* [256]                                                    */
} b200_emb_weights;
/* the same for WeSpeakerResNet34 (models/embedding/wespeaker/__init__.py:324-372): eval-mode BatchNorm is folded into
 * the conv weights / biases, conv weights go to fp16 [tap][c_out][c_in] plus the per-kernel re-layouts. */
int b200_emb_load(b200_ctx* ctx, const b200_emb_weights* w);
/* WeSpeakerResNet152 / 221 / 293 (models/embedding/wespeaker/resnet.py:148-212, 477-508; __init__.py:375-466): the same
 * stem, strides and TSTP pooling with Bottleneck blocks, num_blocks {3, 8, 36, 3}, {6, 16, 48, 3} or {10, 20, 64, 3}
 * (any counts >= 1 are accepted).  The block arrays have sum(num_blocks) entries in block order; block_shortcut[i]
 * has conv_weight == NULL exactly where the block has no shortcut (stride 1 and in_planes == 4 * planes).
 * The trunk outputs C = 1024 channels (256 for ResNet34), the statistics are 20 * C = 20480 wide. */
typedef struct b200_emb_bottleneck_weights {
  int32_t num_blocks[4];
  b200_conv_bn stem;                          /* resnet.conv1 / resnet.bn1                               */
  const b200_conv_bn* block_conv1;            /* resnet.layerL.i.conv1 / bn1 (1x1, in -> p)              */
  const b200_conv_bn* block_conv2;            /* resnet.layerL.i.conv2 / bn2 (3x3, stride, p -> p)       */
  const b200_conv_bn* block_conv3;            /* resnet.layerL.i.conv3 / bn3 (1x1, p -> 4p)              */
  const b200_conv_bn* block_shortcut;         /* resnet.layerL.i.shortcut.{0,1} (1x1, stride, in -> 4p)  */
  const float* seg1_weight;                   /* resnet.seg_1.weight [256][20480]                        */
  const float* seg1_bias;                     /* [256]                                                   */
} b200_emb_bottleneck_weights;
/* Loads a bottleneck trunk into the ctx's one embedding slot (replacing a ResNet34 loaded by b200_emb_load, and the
 * other way round).  BN folding and the fp16 layouts as b200_emb_load.  The embedding entry points below then run
 * this trunk.  Bad arguments or inconsistent shortcuts return B200_STATUS_INVALID. */
int b200_emb_load_bottleneck(b200_ctx* ctx, const b200_emb_bottleneck_weights* w);

/* XVectorSincNet (models/embedding/xvector.py:205-349), the architecture of pyannote/embedding: the SincNet front end
 * of PyanNet (same fields and meaning as in b200_seg_weights), five TDNN layers Conv1d -> LeakyReLU -> BatchNorm1d
 * (eval, eps 1e-5) with (C_out, kernel, dilation) = (512, 5, 1), (512, 3, 2), (512, 3, 3), (512, 1, 1), (1500, 1, 1),
 * StatsPool (mean and std of the 1500 channels) and the Linear 3000 -> dimension. */
typedef struct b200_xvec_weights {
  float wav_norm_weight, wav_norm_bias;       /* sincnet.wav_norm1d.{weight,bias}                       */
  const float* sinc_filters;                  /* [80][251] realised ParamSincFB bank (cos 0..39, sin 40..79) */
  const float* norm_weight[3];                /* sincnet.norm1d.{0,1,2}.weight  (80, 60, 60)            */
  const float* norm_bias[3];
  const float* conv_weight[2];                /* sincnet.conv1d.{1,2}.weight  [60][80][5], [60][60][5]  */
  const float* conv_bias[2];
  const float* tdnn_weight[5];                /* tdnns.{0,3,6,9,12}.weight [C_out][C_in][kernel]        */
  const float* tdnn_bias[5];                  /* tdnns.{0,3,6,9,12}.bias [C_out]                        */
  const float* bn_weight[5];                  /* tdnns.{2,5,8,11,14}.weight [C_out]                     */
  const float* bn_bias[5];
  const float* bn_mean[5];                    /* tdnns.{2,5,8,11,14}.running_mean                       */
  const float* bn_var[5];                     /* tdnns.{2,5,8,11,14}.running_var                        */
  int32_t dimension;                          /* embedding size (512 for pyannote/embedding)            */
  const float* embedding_weight;              /* embedding.weight [dimension][3000]                     */
  const float* embedding_bias;                /* [dimension]                                            */
} b200_xvec_weights;
/* Loads XVectorSincNet into the ctx's own slot: a PyanNet, a WeSpeaker ResNet and an XVectorSincNet stay resident
 * side by side.  fp16 (hi, lo) splits and the BatchNorm scale / shift are made here, once. */
int b200_xvec_load(b200_ctx* ctx, const b200_xvec_weights* w);

/* XVectorMFCC (models/embedding/xvector.py:42-202): torchaudio's MFCC with its defaults at 16 kHz (n_mfcc 40, DCT-II
 * "ortho", log_mels False: centred reflect-padded STFT with n_fft 400 and hop 200, power spectrum, 128-filter mel bank,
 * AmplitudeToDB("power", top_db 80) over each whole utterance, DCT) in front of the TDNN stack, pooling and Linear of
 * XVectorSincNet (same fields and meaning as in b200_xvec_weights; tdnns.0 has 40 input channels).  The three MFCC
 * buffers are used as loaded. */
typedef struct b200_xvec_mfcc_weights {
  const float* dct_mat;                       /* mfcc.dct_mat [128][40]                                 */
  const float* window;                        /* mfcc.MelSpectrogram.spectrogram.window [400]           */
  const float* mel_fb;                        /* mfcc.MelSpectrogram.mel_scale.fb [201][128]            */
  const float* tdnn_weight[5];                /* tdnns.{0,3,6,9,12}.weight [C_out][C_in][kernel]        */
  const float* tdnn_bias[5];                  /* tdnns.{0,3,6,9,12}.bias [C_out]                        */
  const float* bn_weight[5];                  /* tdnns.{2,5,8,11,14}.weight [C_out]                     */
  const float* bn_bias[5];
  const float* bn_mean[5];                    /* tdnns.{2,5,8,11,14}.running_mean                       */
  const float* bn_var[5];                     /* tdnns.{2,5,8,11,14}.running_var                        */
  int32_t dimension;                          /* embedding size                                         */
  const float* embedding_weight;              /* embedding.weight [dimension][3000]                     */
  const float* embedding_bias;                /* [dimension]                                            */
} b200_xvec_mfcc_weights;
/* Loads XVectorMFCC into the ctx's own slot, next to the PyanNet, WeSpeaker, XVectorSincNet and SSeRiouSS slots. */
int b200_xvec_mfcc_load(b200_ctx* ctx, const b200_xvec_mfcc_weights* w);

/* SSeRiouSS (models/segmentation/SSeRiouSS.py) on the WavLM Base front end (torchaudio WAVLM_BASE / WAVLM_BASE_PLUS:
 * conv feature extractor without conv biases and GroupNorm on conv 0, 768-wide post-LN transformer of 12 layers with
 * 12 heads and gated relative position bias), then the PyanNet head: 1-4 BiLSTM layers of 128 with 768 inputs, two
 * Linear+LeakyReLU layers of 128 and the classifier (fields and layouts as in b200_seg_weights).  Keys below are those
 * of the state dict without the "wav2vec." prefix. */
#define B200_SSL_LAYERS 12
#define B200_SSL_REL_SPAN 1023
typedef struct b200_ssl_layer_weights {
  const float* in_proj_weight;                /* attention.attention.in_proj_weight [2304][768] (q, k, v)  */
  const float* in_proj_bias;                  /* [2304]                                                    */
  const float* out_proj_weight;               /* attention.attention.out_proj.weight [768][768]            */
  const float* out_proj_bias;
  const float* gru_weight;                    /* attention.gru_rel_pos_linear.weight [8][64]               */
  const float* gru_bias;                      /* [8]                                                       */
  const float* gru_const;                     /* attention.gru_rel_pos_const [12]                          */
  const float* layer_norm_weight;             /* layer_norm [768]                                          */
  const float* layer_norm_bias;
  const float* ff1_weight;                    /* feed_forward.intermediate_dense.weight [3072][768]        */
  const float* ff1_bias;
  const float* ff2_weight;                    /* feed_forward.output_dense.weight [768][3072]              */
  const float* ff2_bias;
  const float* final_layer_norm_weight;       /* final_layer_norm [768]                                    */
  const float* final_layer_norm_bias;
} b200_ssl_layer_weights;
typedef struct b200_ssl_weights {
  const float* conv0_weight;                  /* feature_extractor.conv_layers.0.conv.weight [512][1][10]  */
  const float* conv0_norm_weight;             /* feature_extractor.conv_layers.0.layer_norm (GroupNorm) [512] */
  const float* conv0_norm_bias;
  const float* conv_weight[6];                /* conv_layers.{1..6}.conv.weight [512][512][3] x4, [512][512][2] x2 */
  const float* proj_norm_weight;              /* encoder.feature_projection.layer_norm [512]               */
  const float* proj_norm_bias;
  const float* proj_weight;                   /* encoder.feature_projection.projection.weight [768][512]   */
  const float* proj_bias;
  const float* pos_conv_weight;               /* pos_conv_embed.conv weight with its weight norm folded [768][48][128] */
  const float* pos_conv_bias;                 /* [768]                                                     */
  const float* encoder_norm_weight;           /* encoder.transformer.layer_norm [768]: applied after the positional
                                                 conv's residual, before layer 0                              */
  const float* encoder_norm_bias;
  const float* rel_attn_embed;                /* layers.0.attention.rel_attn_embed.weight [320][12]        */
  const int32_t* rel_bucket;                  /* [2 * B200_SSL_REL_SPAN + 1]: bucket of the offset j - i = d at
                                                 d + 1023 (offsets beyond +-1023 take the saturated end values) */
  int32_t num_layers;                         /* transformer layers run: 12, or wav2vec_layer (1 .. 12)    */
  b200_ssl_layer_weights layer[B200_SSL_LAYERS];
  const float* layer_weights;                 /* [num_layers] softmax(wav2vec_weights); NULL: the output of layer
                                                 num_layers alone (wav2vec_layer >= 1)                      */
  int32_t lstm_layers;                        /* 1 .. 4                                                    */
  const float* lstm_w_ih[8];                  /* lstm.weight_ih_l{k}[_reverse]: [512][768] for layer 0     */
  const float* lstm_w_hh[8];
  const float* lstm_b_ih[8];
  const float* lstm_b_hh[8];
  const float* linear_weight[2];              /* linear.{0,1}.weight [128][256], [128][128]                */
  const float* linear_bias[2];
  const float* classifier_weight;             /* [num_classes][128]                                        */
  const float* classifier_bias;
} b200_ssl_weights;
/* Loads SSeRiouSS into the ctx's own slot: a PyanNet, a WeSpeaker ResNet, an XVectorSincNet and an SSeRiouSS stay
 * resident side by side.  num_classes / activation as in b200_seg_load_head. */
int b200_ssl_load(b200_ctx* ctx, const b200_ssl_weights* w, int32_t num_classes, int32_t activation);
/* SSeRiouSS.forward on windows of any length window >= 400 samples (arguments as in b200_seg_forward_window):
 * T = 1 + (window - 400) / 320 frames for window >= 400 (499 for 160000).  GroupNorm statistics are taken over the
 * whole padded window.  Windows run in sub-batches of at most ssl_max_batch x 160000 samples (option ssl_max_batch,
 * default 32: 320 s); one window longer than that returns B200_STATUS_INVALID naming the option. */
int b200_ssl_forward_window(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                            int32_t num_chunks, int32_t window, uint8_t* classes, float* logp, void* stream);
/* The same for a sigmoid head, outputs as in b200_seg_forward_scores. */
int b200_ssl_forward_scores(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                            int32_t num_chunks, int32_t window, float* scores, float* max_scores, void* stream);
/* The WavLM Base front end alone, arguments as in b200_ssl_forward_window: out[num_chunks][T][768] fp32, the LSTM
 * input of the forward (the softmax-weighted layer average, or the output of layer wav2vec_layer).  The head does not
 * run; sub-batches, ssl_max_batch and the window checks are those of the forward. */
int b200_ssl_features(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                      int32_t num_chunks, int32_t window, float* out, void* stream);

/* ---- audio ingest: Audio.__call__ / Audio.downmix_and_resample (core/io.py:223-265, 306-351) -----------------
 * pcm is a DEVICE buffer holding the raw decoded audio: B200_PCM_S16_INTERLEAVED = int16 [frame][channel] (what a
 * PCM WAV holds; half the PCIe bytes of float32) or B200_PCM_F32_PLANAR = float32 [channel][frame] (the reference's
 * in-memory {"waveform": (channel, time)} files).  channel >= 0 selects that channel (io.py:232-233), channel < 0
 * downmixes by the mean over channels (mono="downmix", io.py:241-242); when sr_in != sr_out the signal is resampled
 * with torchaudio.functional.resample's default polyphase windowed-sinc filter (io.py:246-250).  Writes
 * b200_audio_num_frames(frames_in, sr_in, sr_out) float32 samples to out (capacity checked). */
#define B200_PCM_S16_INTERLEAVED 0
#define B200_PCM_F32_PLANAR 1
int64_t b200_audio_num_frames(int64_t frames_in, int32_t sr_in, int32_t sr_out);
int b200_audio_ingest(b200_ctx* ctx, const void* pcm, int32_t format, int32_t channels, int64_t frames_in,
                      int32_t sr_in, int32_t sr_out, int32_t channel, float* out, int64_t out_capacity, void* stream);

/* ---- segmentation: Inference.infer / Inference.slide hot loop (core/inference.py:182-215, 295-313) --------
 * `wav` is a device fp32 buffer; chunk i covers wav[chunk_off[i] .. chunk_off[i]+160000), of which only the first
 * chunk_valid[i] samples are real (the rest is the zero padding of the last chunk, inference.py:270-278).
 * chunk_off / chunk_valid are HOST arrays.  Output: powerset class id per frame, classes[num_chunks][589]
 * (argmax of the LogSoftmax output, utils/powerset.py:135-140); optional log-probabilities [num_chunks][589][7]. */
int b200_seg_forward(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                     int32_t num_chunks, uint8_t* classes, float* logp, void* stream);
/* PyanNet.forward of a log-softmax head on windows of any length (models/segmentation/PyanNet.py:223-240): window i covers
 * wav[chunk_off[i] .. chunk_off[i] + window), of which the first chunk_valid[i] <= window samples are real (zero padding
 * after them, inference.py:270-278).  Every InstanceNorm normalises over the whole padded window.  F = 1 + (window - 251)
 * / 10 frames, then MaxPool 3, Conv1d 5, MaxPool 3, Conv1d 5, MaxPool 3 (589 for 160000); window >= 1261 (F >= 2).
 * Output classes[num_chunks][F] (argmax, ties to the first class), optional logp[num_chunks][F][K], K the loaded head's
 * class count.  Windows run in sub-batches of at most seg_max_batch x 160000 samples; one window longer than that
 * (5.87 h with the default) returns B200_STATUS_INVALID, and so does a loaded sigmoid head.
 * b200_seg_forward is this function with window = 160000. */
int b200_seg_forward_window(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                            int32_t num_chunks, int32_t window, uint8_t* classes, float* logp, void* stream);
/* The same for a sigmoid head (binary / multi-label problems): scores[num_chunks][F][K] fp32 in [0, 1] and / or
 * max_scores[num_chunks][F], the maximum over the K scores of each frame (VoiceActivityDetection's
 * pre_aggregation_hook, pipelines/voice_activity_detection.py:111-114, fused into the classifier); either may be NULL,
 * not both.  A loaded log-softmax head returns B200_STATUS_INVALID. */
int b200_seg_forward_scores(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                            int32_t num_chunks, int32_t window, float* scores, float* max_scores, void* stream);
/* Intermediates of the segmentation network, for testing it stage by stage (b200_seg_stages, b200_seg_head_stages).
 * Every pointer is a DEVICE buffer or NULL; after each stage the library copies that stage's result into every
 * non-NULL buffer, in the layout the next stage reads.  n windows, T frames, float2 = (scale, shift). */
typedef struct b200_seg_capture {
  void* af_wav;                 /* [n] float2: wav_norm1d as an affine of the raw samples                   */
  float* P0;                    /* [n][80][pool0] sinc conv -> |.| -> MaxPool 3                             */
  void* af0;                    /* [n][80] float2: norm1d.0 as an affine of P0                              */
  float* P1;                    /* [n][60][pool1] Conv1d 1 -> MaxPool 3 -> + bias                           */
  void* af1;                    /* [n][60] float2                                                           */
  float* P2;                    /* [n][60][pool2] Conv1d 2 -> MaxPool 3 -> + bias (pool2 = T)               */
  void* af2;                    /* [n][60] float2                                                           */
  float* x0;                    /* [n][T][64] head input: leaky_relu(P2 * scale + shift), 4 zero columns     */
  float* gx[4];                 /* per LSTM layer [n][T][1024]: input projection + b_ih + b_hh, column
                                   dir * 512 + unit * 4 + gate (i, f, g, o)                                 */
  float* y[4];                  /* per LSTM layer [n][T][256] fp32 (seg_gemm_impl 0): forward units 0..127,
                                   reverse 128..255                                                         */
  void* y_hi[4];                /* the same as fp16 (hi, lo) pairs, y = hi + lo (seg_gemm_impl 1)            */
  void* y_lo[4];
  float* z1;                    /* [n][T][128] leaky_relu(linear.0): fp32 (seg_gemm_impl 0) ...              */
  void* z1_hi;                  /* ... or fp16 (hi, lo) (seg_gemm_impl 1)                                   */
  void* z1_lo;
  float* z2;                    /* [n][T][128] leaky_relu(linear.1), fp32                                   */
  uint8_t* cls;                 /* log-softmax heads: classes [n][T] (required) and logp [n][T][K]           */
  float* logp;
  float* scores;                /* sigmoid heads: scores [n][T][K] and max_scores [n][T]                    */
  float* max_scores;
} b200_seg_capture;
/* PyanNet on n windows as b200_seg_forward_window / b200_seg_forward_scores run it (same kernels and launches, under
 * the ctx's seg_*_impl options), with its intermediates copied into cap; the classifier writes cap's outputs.  n may
 * not exceed one sub-batch (min(seg_max_batch * 160000 / window, 65535) windows), else B200_STATUS_INVALID. */
int b200_seg_stages(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                    int32_t num_chunks, int32_t window, const b200_seg_capture* cap, void* stream);
/* The segmentation head of a loaded model alone on a caller input x0[n][T][k0] (DEVICE fp32), T >= 1: the BiLSTM stack,
 * linear layers and classifier as the forward runs them, capturing gx, y, z1, z2 and the outputs into cap.  model
 * B200_SEG_HEAD_PYANNET (k0 = 64: 60 SincNet features and 4 columns the weights ignore) or B200_SEG_HEAD_SSERIOUSS
 * (k0 = 768). */
#define B200_SEG_HEAD_PYANNET 0
#define B200_SEG_HEAD_SSERIOUSS 1
int b200_seg_head_stages(b200_ctx* ctx, int32_t model, const float* x0, int32_t n, int32_t T,
                         const b200_seg_capture* cap, void* stream);
/* SincNet.forward alone (models/blocks/sincnet.py:163-184): out[num_chunks][589][60] fp32 (frame-major). */
int b200_sincnet_forward(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                         int32_t num_chunks, float* out, void* stream);
/* Powerset.to_multilabel, hard (utils/powerset.py:115-140): classes[n] -> multilabel[n][3] in {0,1} (u8). */
int b200_powerset_to_multilabel(b200_ctx* ctx, const uint8_t* classes, int64_t n, uint8_t* multilabel, void* stream);
/* The same for any powerset: num_speakers <= 32 speakers with at most max_per_frame per frame, classes in the
 * reference's order (set size 0 .. max_per_frame, itertools.combinations within each size); num_classes must be the
 * powerset's class count (at most 32), else B200_STATUS_INVALID.  multilabel[n][num_speakers]; class ids
 * >= num_classes give an all-zero row.  b200_powerset_to_multilabel is this function with (7, 3, 2). */
int b200_powerset_to_multilabel_generic(b200_ctx* ctx, const uint8_t* classes, int64_t n, int32_t num_classes,
                                        int32_t num_speakers, int32_t max_per_frame, uint8_t* multilabel,
                                        void* stream);

/* ---- embeddings: SpeakerDiarization.get_embeddings hot loop (pipelines/speaker_diarization.py:399-459) over
 * PyannoteAudioPretrainedSpeakerEmbedding.__call__ (pipelines/speaker_verification.py:704-716) and
 * WeSpeakerResNet34.forward (models/embedding/wespeaker/__init__.py:324-343), or the loaded bottleneck trunk's.  One
 * trunk pass per chunk, the three
 * local speakers share it (forward_frames + forward_embedding, :288-322); masks[num_chunks][3][589] u8 are the
 * StatsPool weights; emb[num_chunks][3][256] fp32. */
int b200_emb_forward(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                     int32_t num_chunks, const uint8_t* masks, float* emb, void* stream);
/* The same with a fused all-gather for the multi-GPU chunk pool: emb_peers[n_peers] (HOST array
 * of DEVICE pointers, n_peers <= 7) are this rank's slot inside the OTHER GPUs' gather buffers (peer memory mapped
 * over NVLink, e.g. CUDA IPC / torch symmetric memory); the epilogue of the final Linear GEMM stores every output
 * tile to `emb` and to all peers (P2P stores), so the exchange overlaps the GEMM and no collective call follows.
 * The caller synchronises the ranks afterwards (any barrier with system-scope release/acquire). */
int b200_emb_forward_push(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                          int32_t num_chunks, const uint8_t* masks, float* emb, float* const* emb_peers,
                          int32_t n_peers, void* stream);
/* P2P push of a byte range (16-byte aligned) to the same offsets of n_dsts <= 7 peer buffers: the powerset classes
 * of this rank's chunks, next to the embeddings pushed by b200_emb_forward_push. */
int b200_push(b200_ctx* ctx, const void* src, int64_t bytes, void* const* dsts, int32_t n_dsts, void* stream);
/* compute_fbank (wespeaker/__init__.py:113-139): fbank[num_chunks][998][80], global-mean centred. */
int b200_emb_fbank(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                   int32_t num_chunks, float* fbank, void* stream);
/* Host-only (no device work): the shared-frame fbank layout b200_emb_forward uses for a chunk list processed in
 * sub-batches of `sub_batch` chunks.  The reference computes 998 fbank frames per chunk (wespeaker/__init__.py:113-139)
 * although consecutive chunks of Inference.slide (core/inference.py:235-257: step = 0.1 * duration = 100 frame hops)
 * share 898 of them; overlapping, hop-aligned, full chunks are grouped into runs whose frames are computed once.
 * frame0[num_chunks]: first fbank row of each chunk inside its sub-batch; rows_per_sub_batch[ceil(n / sub_batch)]:
 * fbank rows computed per sub-batch (998 * chunks without sharing).  Returns the number of runs, < 0 on bad arguments. */
int64_t b200_emb_fbank_plan(const int64_t* chunk_off, const int32_t* chunk_valid, int32_t num_chunks, int32_t sub_batch,
                            int32_t share, int32_t* frame0, int32_t* rows_per_sub_batch);
/* ResNet.forward_frames on a given fbank (resnet.py:399-419): frames[num_chunks][C][10][125] fp32 (NCHW), C = 256 for
 * ResNet34 and 1024 for a bottleneck trunk. */
int b200_emb_trunk(b200_ctx* ctx, const float* fbank, int32_t num_chunks, float* frames, void* stream);
/* One stage of the trunk of b200_emb_trunk on B segments of width W, as the embedding paths run it (conv_impl
 * included).  Stage 0 is the stem: in = fp32 fbank[B][W][80], fmean[B][80] subtracted from it, out = NHWC fp16
 * [B][80][W][32].  Stage k >= 1 is block k - 1 (BasicBlock or Bottleneck; fmean unused): in = NHWC fp16
 * [B][H][W][C_in], H = 80, 40, 20 or 10 by the block's layer, out = NHWC fp16 [B][H'][W'][C_out].  B may not exceed
 * one embedding sub-batch, max(1, emb_max_batch * 998 / W) segments. */
int b200_emb_trunk_stage(b200_ctx* ctx, int32_t stage, const void* in, const float* fmean, int32_t B, int32_t W,
                         void* out, void* stream);
/* WeSpeakerResNet34.forward (models/embedding/wespeaker/__init__.py:324-343) on utterances of one length
 * num_samples >= 400 (a (num_utts, 1, num_samples) tensor): utterance i = wav[off[i] .. off[i] + num_samples), off a
 * HOST array.  compute_fbank (:113-139) gives T0 = 1 + (num_samples - 400) / 160 frames, the trunk
 * (resnet.py:347-368) T = T0 after layer 1 and (T + 2 - 3) / 2 + 1 after each of layers 2-4; StatsPool
 * (models/blocks/pooling.py:30-61, 76-130) weights are interpolated onto the T frames with torch's CUDA nearest index.
 * weights: NULL (mean and std(correction=1) over the T frames; T = 1 gives NaN) or fp32 DEVICE
 * [num_utts][num_speakers][num_weights], any real values.  emb: fp32 DEVICE [num_utts][max(num_speakers, 1)][256].
 * Utterances run in sub-batches of max(1, emb_max_batch * 998 / T0); one utterance longer than emb_max_batch * 998
 * fbank frames (263 472 = 43.9 min with the default) returns B200_STATUS_INVALID. */
int b200_emb_forward_utt(b200_ctx* ctx, const float* wav, const int64_t* off, int64_t num_samples, int32_t num_utts,
                         const float* weights, int32_t num_speakers, int32_t num_weights, float* emb, void* stream);
/* ResNet.forward_embedding on caller frames (resnet.py:370-397, wespeaker/__init__.py:304-322): frames fp32 DEVICE
 * NCHW [B][C][10][T] (what forward_frames returns; C = 256 for ResNet34, 1024 for a bottleneck trunk), weights and
 * emb as in b200_emb_forward_utt. */
int b200_emb_forward_embedding(b200_ctx* ctx, const float* frames, int32_t B, int32_t T, const float* weights,
                               int32_t num_speakers, int32_t num_weights, float* emb, void* stream);
/* XVectorSincNet.forward (models/embedding/xvector.py:329-349) on utterances of one length num_samples >= 4771,
 * arguments as in b200_emb_forward_utt.  SincNet gives F frames (b200_seg_forward_window's arithmetic), the TDNN
 * stack T = F - 14; StatsPool weights [num_utts][num_speakers][num_weights] (any real values, NULL = mean and
 * std(correction=1)) reach the T frames by torch's CUDA nearest index.  emb: fp32 DEVICE
 * [num_utts][max(num_speakers, 1)][dimension].  Utterances run in sub-batches of at most emb_max_batch x 160000
 * samples; one utterance longer than that (43.9 min with the default) returns B200_STATUS_INVALID. */
int b200_xvec_forward(b200_ctx* ctx, const float* wav, const int64_t* off, int64_t num_samples, int32_t num_utts,
                      const float* weights, int32_t num_speakers, int32_t num_weights, float* emb, void* stream);
/* XVectorMFCC.forward (models/embedding/xvector.py:185-202) on utterances of one length num_samples >= 2800,
 * arguments, pooling and sub-batches as in b200_xvec_forward.  MFCC gives F = 1 + num_samples / 200 frames, the TDNN
 * stack T = F - 14. */
int b200_xvec_mfcc_forward(b200_ctx* ctx, const float* wav, const int64_t* off, int64_t num_samples, int32_t num_utts,
                           const float* weights, int32_t num_speakers, int32_t num_weights, float* emb, void* stream);
/* The MFCC front end of the loaded XVectorMFCC alone: utterances as in b200_xvec_mfcc_forward (num_samples > 200) ->
 * out fp32 DEVICE [num_utts][1 + num_samples / 200][40] (frame-major, the transpose of torchaudio's layout). */
int b200_xvec_mfcc_features(b200_ctx* ctx, const float* wav, const int64_t* off, int64_t num_samples, int32_t num_utts,
                            float* out, void* stream);
/* StatsPool.forward (models/blocks/pooling.py:76-130): seq[B][F][T], weights[B][S][Tw] or NULL -> out[B][S][2F]. */
int b200_stats_pool(b200_ctx* ctx, const float* seq, const float* weights, float* out, int32_t B, int32_t F, int32_t T,
                    int32_t S, int32_t Tw, void* stream);

/* ---- overlap-add / reconstruction (core/inference.py:498-620, pipelines/utils/diarization.py:150-268,
 * pipelines/speaker_diarization.py:480-528).  seg[num_chunks][589][3] u8 in {0,1}; start_frame[num_chunks] DEVICE
 * int32 array with the global frame index of each chunk's first frame (non-decreasing; computed on the host as
 * inference.py:596 does); num_frames = size of the global grid. */
int b200_speaker_count(b200_ctx* ctx, const uint8_t* seg, const int32_t* start_frame, int32_t num_chunks,
                       int32_t num_frames, uint8_t* count, void* stream);
/* SpeakerDiarization.reconstruct + to_diarization (pipelines/speaker_diarization.py:480-528,
 * pipelines/utils/diarization.py:221-268): per frame, the `count` most active clusters (ties: lower cluster index).
 * hard_clusters[num_chunks][3] int8 DEVICE (-2 = inactive/unassigned, values >= num_clusters_out are ignored);
 * count[num_frames] u8 device (already capped); out: discrete[num_frames][num_clusters_out] u8 with
 * num_clusters_out >= max(K, max(count)), at most 127 (hard clusters are int8 like the reference's
 * constrained_argmax; up to 32 clusters the per-frame counters stay in registers). */
int b200_reconstruct(b200_ctx* ctx, const uint8_t* seg, const int8_t* hard_clusters, const int32_t* start_frame,
                     int32_t num_chunks, int32_t num_frames, const uint8_t* count, int32_t num_clusters_out,
                     uint8_t* discrete, void* stream);

/* Inference.aggregate (core/inference.py:498-620), the generic float overlap-add behind the aggregated
 * (skip_aggregation=False) Inference output and the VAD / OSD pipelines: scores[num_chunks][589][K] fp32 (NaN =
 * missing), hamming / warm_up: DEVICE fp64[589] windows or NULL (= ones) -> out[num_frames][K] fp32, bit-identical to
 * numpy's mixed float32/float64 arithmetic (see post.cu). */
int b200_aggregate(b200_ctx* ctx, const float* scores, const int32_t* start_frame, int32_t num_chunks,
                   int32_t num_frames, int32_t num_classes, const double* hamming, const double* warm_up,
                   int32_t skip_average, float missing, float epsilon, float* out, void* stream);
/* The same for chunks of any frames_per_chunk frames: scores[num_chunks][frames_per_chunk][K], hamming / warm_up
 * fp64[frames_per_chunk] or NULL.  b200_aggregate is this function with frames_per_chunk = 589. */
int b200_aggregate_window(b200_ctx* ctx, const float* scores, const int32_t* start_frame, int32_t num_chunks,
                          int32_t num_frames, int32_t frames_per_chunk, int32_t num_classes, const double* hamming,
                          const double* warm_up, int32_t skip_average, float missing, float epsilon, float* out,
                          void* stream);
/* VoiceActivityDetection's pre-aggregation step (pipelines/voice_activity_detection.py:111-114: max over the
 * speakers of the multilabel output) straight from the powerset classes: speech[n] fp32 in {0,1}. */
int b200_powerset_speech(b200_ctx* ctx, const uint8_t* classes, int64_t n, float* speech, void* stream);
/* The same for any powerset (arguments and checks as b200_powerset_to_multilabel_generic): speech[n] = 1 where the
 * class is a non-empty speaker set.  b200_powerset_speech is this function with (7, 3, 2). */
int b200_powerset_speech_generic(b200_ctx* ctx, const uint8_t* classes, int64_t n, int32_t num_classes,
                                 int32_t num_speakers, int32_t max_per_frame, float* speech, void* stream);

/* Onsets / offsets of a discrete diarization discrete[num_frames][num_clusters] u8 (to_annotation ->
 * Binarize(onset=offset=0.5), pipelines/utils/diarization.py:188-218, utils/signal.py:254-318) as unordered events
 * k * (num_frames + 1) + f.  buf (DEVICE int32[2 + 2 * cap]) = [n_on, n_off, on[cap], off[cap]]; counts may exceed
 * cap (then only cap events were stored: call again with a larger buffer). */
int b200_frame_transitions(b200_ctx* ctx, const uint8_t* discrete, int32_t num_frames, int32_t num_clusters,
                           int32_t cap, int32_t* buf, void* stream);

/* ---- clustering (pipelines/clustering.py:77-140, 572-669; utils/vbx.py; scipy linkage/fcluster) --------------- */
/* filter_embeddings: clean-frame counts per (chunk, speaker): out[num_chunks][3] int32, plus active[num_chunks][3] u8
 * = any frame active (inactive speakers, speaker_diarization.py:681). */
int b200_clean_frames(b200_ctx* ctx, const uint8_t* seg, int32_t num_chunks, int32_t* clean, uint8_t* active,
                      void* stream);
/* linkage(X, "centroid", "euclidean") (scipy, called at clustering.py:600-602 and :374-376): x[n][dim] fp64 device;
 * normalize: 0 = rows as given, 1 = L2-normalised in fp64, 2 = rows hold float32 values and are normalised exactly as
 * numpy does on float32 embeddings (x / np.linalg.norm(x, axis=1, keepdims=True): float32 pairwise sum, float32
 * sqrt and division; clustering.py:597-599) before widening; Z[n-1][4] fp64 device in scipy's format.
 * Problems of n <= 32768 observations run one CTA each over a dense n x n fp64 distance matrix in the ctx workspace
 * (8 n^2 bytes).  Larger ones (n >= option "linkage_grid_min") run one after another, each on the whole GPU (a
 * cooperative grid) over scipy's condensed distances, 4 n (n - 1) bytes allocated stream-ordered for the call and freed
 * before it returns (4.3 GB at n = 32 768, 17 GB at 65 536, 40 GB at 100 000); the limit is device memory
 * (B200_STATUS_OOM, with n and the bytes in the message, when the allocation fails).  Both paths emit the same Z bit
 * for bit.  At most 1 048 560 observations per problem. */
int b200_linkage_centroid(b200_ctx* ctx, const double* x, int32_t n, int32_t dim, int32_t normalize, double* Z,
                          void* stream);
/* the same (clustering.py:594-603) for num_problems independent problems in ONE launch (one CTA each; problems above
 * the threshold then take the whole-GPU path in turn): rows of problem f are
 * x[row_offsets[f] .. row_offsets[f+1]) (row_offsets: HOST int32[num_problems+1]); Z rows are concatenated, problem
 * f contributing max(n_f - 1, 0) rows. */
int b200_linkage_centroid_batched(b200_ctx* ctx, const double* x, const int32_t* row_offsets, int32_t num_problems,
                                  int32_t dim, int32_t normalize, double* Z, void* stream);
/* host only: device bytes a b200_linkage_centroid_batched call with these HOST row_offsets needs at the default
 * "linkage_grid_min" = the ctx workspace it grows to plus the per-call packed distances of its largest problem above
 * the threshold.  Negative status for bad arguments (num_problems < 1, dim < 1, decreasing offsets). */
int64_t b200_linkage_bytes(const int32_t* row_offsets, int32_t num_problems, int32_t dim);
/* fcluster(Z, t, criterion="distance") (clustering.py:604, 385): HOST arrays, labels[n] 1-based like scipy. */
int b200_fcluster_distance(const double* Z, int32_t n, double t, int32_t* labels);
/* PLDA.__call__ (core/plda.py:50-63; xvec_tf / plda_tf of utils/vbx.py:211-217): x[n][Din] fp64 device ->
 * fea[n][L]; mean1[Din], mean2[Dout], lda[Din][Dout], mu[Dout], trT[Dout][L] (= plda_tr^T[:, :L]) fp64 device. */
int b200_plda_transform(b200_ctx* ctx, const double* x, int32_t n, int32_t Din, int32_t Dout, int32_t L,
                        const double* mean1, const double* mean2, const double* lda, const double* mu,
                        const double* trT, double* fea, void* stream);
/* VBx centroids (clustering.py:620-621): W = q[:, kept]; centroids[K][dim] = W^T train / sum(W): q[n][S], kept[K]
 * (DEVICE int32 column indices), train[n][dim], all fp64 device. */
int b200_weighted_centroids(b200_ctx* ctx, const double* q, int32_t n, int32_t S, const int32_t* kept, int32_t K,
                            const double* train, int32_t dim, double* centroids, void* stream);
/* cdist(a, b, "cosine") (clustering.py:645-655): a[m][dim], b[k][dim] fp64 device -> d[m][k] fp64 device. */
int b200_cdist_cosine(b200_ctx* ctx, const double* a, int32_t m, const double* b, int32_t k, int32_t dim, double* d,
                      void* stream);
/* VBx iterations (utils/vbx.py:98-136 via cluster_vbx :140-155): fea[n][D], phi[D], gamma[n][S] (in: initial
 * responsibilities, out: final), pi[S] (out), all fp64 device; *iters (host) = iterations run. */
int b200_vbx(b200_ctx* ctx, const double* fea, const double* phi, int32_t n, int32_t D, int32_t S, double Fa,
             double Fb, int32_t max_iters, double epsilon, double* gamma, double* pi, int32_t* iters, void* stream);
/* batched: problem f has n[f] frames (consecutive rows of fea) and S[f] speakers; gamma / pi are the per-problem
 * arrays concatenated; n, S, iters (nullable) are HOST int32[num_problems].  One 8-CTA thread-block cluster per
 * problem runs all iterations (utils/vbx.py:98-136), convergence is tested on the device. */
int b200_vbx_batched(b200_ctx* ctx, const double* fea, const double* phi, const int32_t* n, const int32_t* S,
                     int32_t num_problems, int32_t D, double Fa, double Fb, int32_t max_iters, double epsilon,
                     double* gamma, double* pi, int32_t* iters, void* stream);
/* constrained_argmax / argmax (clustering.py:127-140, 658-665): soft[num_chunks][3][K] fp64 device ->
 * hard[num_chunks][3] int8 device (-2 = unassigned), K at most 127.  Constrained: the optimum that
 * scipy's linear_sum_assignment(maximize=True) returns, ties included (soft must be NaN-free).  Unconstrained:
 * np.argmax per speaker (first maximum; a NaN counts as the maximum). */
int b200_assign(b200_ctx* ctx, const double* soft, int32_t num_chunks, int32_t num_clusters, int32_t constrained,
                int8_t* hard, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200DIAR_H_ */
