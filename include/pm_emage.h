/* pm_emage.h - C ABI of libpm_emage.so: the H100 (sm_90a) kernels of the EMAGE audio->motion
 * inference hot path.
 *
 * The reference (PantoMatrix) has no FFI for this path: every op below is a stock torch.nn /
 * torch.nn.functional call made from Python (SURVEY.md section 8b).  Each entry point therefore
 * cites the reference *call site* it replaces; the Python modules in pantomatrix_b200/emage_audio
 * (same names and signatures as /root/reference/models/emage_audio/__init__.py:1-12) are the only
 * callers.  M.py = models/emage_audio/modeling_emage_audio.py, P.py = .../processing_emage_audio.py.
 *
 * Conventions
 *   - plain pointers + explicit sizes; all pointers are DEVICE pointers unless noted
 *   - activations are channels-last fp32: tensor (batch, rows, channels), row stride `ld*` in elements,
 *     batch stride `*_bs` in elements (lets callers pass column slices / overlapping windows)
 *   - `stream` is a cudaStream_t passed as void*; nothing allocates, nothing synchronises
 *   - return 0 = ok, <0 = PM_E* argument error, >0 = cudaError_t from the launch
 *   - optional split-bf16 output (`planes`, p_ps, p_ld, p_nsplit): the producer also (or only, when its fp32
 *     `out` is NULL) writes its result as p_nsplit bf16 planes (x ~ p0+p1+p2, plane stride p_ps, row stride
 *     p_ld elements): the A operand format of pm_tapgemm_tc, so no separate conversion pass is needed
 *   - plane element format: bit 8 (PM_FMT_F16) of any `nsplit` / `p_nsplit` / `out_nsplit` argument selects IEEE fp16
 *     planes instead of bf16 (same 2-byte storage).  Two fp16 planes carry 22 mantissa bits, so nsplit = 2
 *     (3 tensor-core products) gives the accuracy of 3 bf16 planes (6 products) - provided magnitudes stay below
 *     65504; an overflow becomes inf - inf = NaN in the consuming GEMM, which the host checks for.
 *   - the split rule, the same in every producer: fp16 activation planes hold 64 x (exact pre-scale).  Each plane is
 *     the running remainder rounded to nearest even (bf16: v = x; fp16: v = 64 x; plane p = RNE(v), v -= plane p),
 *     except two fp16 activation planes: plane 0 = the head of v rounded half away from zero to 11 significant bits on
 *     the fp32 bit pattern ((bits + 0x1000) & 0xFFFFE000), plane 1 = RNE(v - head).  The head is exact in fp16 for
 *     |v| >= 2^-14; of the canonical NaN it is -0, and plane 1 carries the NaN.
 */
#ifndef PM_EMAGE_H
#define PM_EMAGE_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define PM_ABI_VERSION 6
#define PM_FMT_F16 0x100
#define PM_H264_I4X4 0x100   /* pm_h264_encode / _gop / _me: bit 8 of `qp` adds Intra 4x4 (I_NxN) macroblocks */
#define PM_TC_TILE_SHIFT 16   /* pm_tapgemm_tc: N tile override in bits 16-23 of `nsplit` */
#define PM_TC_STORE_LOOP (1 << 24)   /* pm_tapgemm_tc: bit 24 of `nsplit` forces the per-element store loop */
int pm_abi_version(void);
/* cudaMemsetAsync on `stream` (a memset node under graph capture, not a kernel): zeroed slack rows, flags */
int pm_memset_async(void* ptr, int value, long long bytes, void* stream);
/* compute capability major*10+minor of the current device, or <0 */
int pm_device_cc(void);

/* ---- tap-GEMM: Conv1d (any kernel size/stride/zero padding) and Linear as one op ------------------
 * out[b,l,n] = act( bias[n] + sum_{t<taps} sum_{c<cin} A[b, l*stride + t - pad, c] * W[t,n,c]
 *                   + residual[b,l,n] ),  rows of A outside [0,rows_in) read as zero.
 * W is (taps, cout, cin) fp32 (BatchNorm already folded in by the host packer).
 * Replaces: nn.Conv1d+BatchNorm1d+LeakyReLU(+shortcut add) in BasicBlock P.py:283-294, the k=3 convs of
 * ResBlock/VQEncoderV6/VQDecoderV5 P.py:178-261, nn.Linear everywhere (MLP P.py:322-326, projections
 * M.py:288,293,297,304,323-325, MultiheadAttention in/out projections and FFN linear1/linear2 inside
 * nn.Transformer{En,De}coderLayer M.py:238-250).  fp32 SIMT reference engine (exact-order fp32 FMA). */
int pm_tapgemm_f32(const float* A, long long a_bs, int lda, int batch, int rows_in, int cin,
                   const float* W, const float* bias, int taps, int stride, int pad,
                   int rows_out, int cout,
                   const float* residual, long long r_bs, int ldr,
                   int act, float slope,
                   float* out, long long o_bs, int ldo, void* stream);

/* ---- tap-GEMM on the wgmma tensor cores (split-bf16 operands, fp32 register accumulate) ----------
 * Same contract as pm_tapgemm_f32 with stride == 1 (strided convs are passed as stride-1 problems over the
 * (rows/s, s*cin) view of the input with zero-padded taps).  A and W are `nsplit` bf16 planes (x = p0+p1+p2),
 * plane strides a_ps / w_ps elements: nsplit 1 = plain bf16, 2 = bf16x3 (p0*p0 + p0*p1 + p1*p0), 3 = bf16x6
 * (all products down to 2^-24).  W planes are (taps, w_rows, ldw) with w_rows >= cout a multiple of 64, zero
 * rows beyond cout; 128-column N tiles are used only when w_rows is a multiple of 128.  The N tile is chosen from
 * the shape and the SM count unless (nsplit >> PM_TC_TILE_SHIFT) & 0xff forces it: 1 = 64, 2 = 128 columns (tests,
 * A/B runs).  Both tiles give bit-identical results.  lda, ldw, a_bs, a_ps, w_ps must be multiples
 * of 8 elements (TMA 16-byte rule).  The activation is applied to columns < act_cols only (<=0: all).
 * The epilogue writes the fp32 result and/or its bf16 split planes (out_f32 / out_bf16 nullable): by TMA stores
 * where every output view has a 16-byte aligned base and strides (and a residual, if any, too), otherwise per
 * element; nsplit | PM_TC_STORE_LOOP forces the per-element loop (tests, A/B runs).  Both give the same bits.
 * Operands are staged by TMA (cp.async.bulk.tensor, zero fill for padding rows, tap shift folded into the
 * row coordinate); descriptors are built on the host inside this call from the raw pointers.
 * `prefetch` (nullable, 16-byte aligned): prefetch_bytes of global memory - the NEXT GEMM's packed weights - are
 * pulled into L2 by this launch (cp.async.bulk.prefetch.L2), so weight streaming overlaps the previous GEMM.
 * fp16 operands (nsplit | PM_FMT_F16): the host packs W scaled by a power of two into the top of the fp16 range;
 * `acc_scale` (its reciprocal, exact) multiplies the accumulator before bias.  Must be 1 for bf16 operands. */
int pm_tapgemm_tc(const uint16_t* A, long long a_ps, long long a_bs, int lda, int batch, int rows_in, int cin,
                  const uint16_t* W, long long w_ps, int w_rows, int ldw, int taps, int pad, int nsplit,
                  const float* bias, int rows_out, int cout,
                  const float* residual, long long r_bs, int ldr,
                  int act, int act_cols, float slope, float acc_scale,
                  float* out_f32, long long o_bs, int ldo,
                  uint16_t* out_bf16, long long ob_ps, long long ob_bs, int ldob, int out_nsplit,
                  const void* prefetch, long long prefetch_bytes, void* stream);

/* fp32 (batch, rows, ch) -> nsplit bf16 or fp16 planes by the split rule above: each plane the running remainder
 * rounded to nearest even; two fp16 planes take the half-away head of 64 x, then RNE(64 x - head). */
int pm_split_bf16(const float* x, long long x_bs, int ldx, int batch, int rows, int ch,
                  uint16_t* out, long long o_ps, long long o_bs, int ldo, int nsplit, void* stream);

/* ---- WavEncoder stem: first BasicBlock's conv1 and downsample conv on the raw waveform (Cin = 1) --
 * sequence (b, w) starts at audio + b*a_bs + w*a_ws and is n_samples long; k=15, stride 5, pad 1600.
 * Outputs are window-major: row block (w*batch + b) of (windows*batch, rows_out, cout).
 * y1 = LeakyReLU_0.01(conv1*bn1), sc = downsample conv*bn (both BN-folded): P.py:285-291,301.
 * y1 goes out as fp32 (`y1`, nullable) and / or as the next GEMM's operand planes (`planes`, nullable; dense rows of
 * p_ld elements, plane stride p_ps, p_nsplit | PM_FMT_F16 as for pm_add_layernorm_f32); at least one of the two.
 * cout 32 or 64, ksize 15; anything else returns PM_EUNSUPPORTED. */
int pm_wav_stem_f32(const float* audio, long long a_bs, long long a_ws, int batch, int windows, int n_samples,
                    const float* w1, const float* b1, const float* wd, const float* bd, int cout,
                    int ksize, int stride, int pad, int rows_out, float slope,
                    float* y1, float* sc,
                    uint16_t* planes, long long p_ps, int p_ld, int p_nsplit, void* stream);

/* ---- LayerNorm(x + r) * gamma + beta over the last dim (r nullable): post-norm residual of
 * nn.TransformerEncoderLayer / DecoderLayer (M.py:238-250), eps 1e-5.  ch must be a multiple of 128 <= 1024 */
int pm_add_layernorm_f32(const float* x, const float* r, const float* gamma, const float* beta,
                         float* out, long long rows, int ch, float eps,
                         uint16_t* planes, long long p_ps, int p_ld, int p_nsplit, void* stream);

/* ---- multi-head attention core, no masks: softmax(Q K^T / sqrt(hd)) V for Tq,Tk <= 64, hd = 192 ----
 * Q/K/V rows are (b*T + t) with row strides ldq/ldk/ldv; head h occupies columns [h*hd,(h+1)*hd).
 * Replaces scaled_dot_product_attention inside nn.MultiheadAttention (M.py:238-250 layers). */
int pm_attention_f32(const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv,
                     float* O, int ldo, int batch, int heads, int tq, int tk, int head_dim,
                     uint16_t* planes, long long p_ps, int p_ld, int p_nsplit, void* stream);

/* Same op on the wgmma tensor cores for the fp16x3 engine: Q, K, V are two-plane fp16 activations (x = (p0+p1)/64,
 * plane stride *_ps, clip stride *_bs, row stride ld* elements, *_cols valid columns; head h of Q starts at column
 * q_col0 + h*hd, likewise K and V - so the packed q|k|v projection output is consumed in place through TMA).
 * S = Q K^T and O = P V run as 3-product fp16 wgmma (M=64) with S and O in registers, softmax in fp32 registers.
 * Output: fp32 O (nullable) and / or two fp16 planes (p_nsplit = 2 | PM_FMT_F16). */
int pm_attention_tc(const uint16_t* Q, long long q_ps, long long q_bs, int ldq, int q_cols, int q_col0,
                    const uint16_t* K, long long k_ps, long long k_bs, int ldk, int k_cols, int k_col0,
                    const uint16_t* V, long long v_ps, long long v_bs, int ldv, int v_cols, int v_col0,
                    float* O, int ldo, int batch, int heads, int tq, int tk, int head_dim,
                    uint16_t* planes, long long p_ps, int p_ld, int p_nsplit, void* stream);

/* ---- broadcast adds: out[b,t,:] = ((x[b,t,:] + first) + second), each of first/second chosen by code:
 * 0 = nothing, 1 = pe[t,:] (PeriodicPositionalEncoding P.py:341-343), 2 = spk[b,:] (speaker embedding
 * row repeated over t, M.py:285-286).  x nullable (treated as 0).  Preserves the reference's add order
 * (M.py:291,298-299,307-308,320-322). */
int pm_add_rows_f32(const float* x, const float* pe, const float* spk, int first, int second,
                    float* out, int batch, int rows, int ch,
                    uint16_t* planes, long long p_ps, int p_ld, int p_nsplit, void* stream);
/* out[r,:] = a[r,:] + b[r,:] for `rows` rows of `ch` columns with row strides lda / ldb / ldo (M.py:312,320-325; column
 * ranges of wider tensors are read and written in place, e.g. the forward and backward halves of a BiLSTM output,
 * camn:265).  A dense tensor of n elements is one row of n, or n / ch rows of ch with planes (ch % 4 == 0). */
int pm_add2_f32(const float* a, long long lda, const float* b, long long ldb, float* out, long long ldo,
                long long rows, long long ch,
                uint16_t* planes, long long p_ps, int p_ld, int p_nsplit, void* stream);

/* ---- window assembly (M.py:384-391 and 267-268 fused): builds one window's motion-encoder input.
 * motion/mask: (batch, total_len, ch) full-sequence tensors, either may be NULL = inference()'s defaults (identity
 * rot6d + zero trans/contact; all masked, M.py:369-377); seed: (batch, pre, ch) decoded last frames, clip stride seed_bs.
 * For frame f<pre: v = mask==0 ? motion : seed (seed NULL = the first window, whose seed is motion[:, :pre] itself,
 * M.py:379), window mask forced 0; else v = motion, m = mask.
 * out = (m == 1) ? mask_embedding[c] : v. */
int pm_window_input_f32(const float* motion, const float* mask, const float* seed, const float* mask_embedding,
                        float* out, int batch, int total_len, int start, int win_len, int pre, int ch, long long seed_bs,
                        uint16_t* planes, long long p_ps, int p_ld, int p_nsplit, void* stream);

/* ---- VQ ------------------------------------------------------------------------------------------ */
/* index = argmin_k ( |z|^2 + |e_k|^2 - 2 z.e_k ) evaluated in fp32, first minimum wins (a row of NaNs yields 0, like
 * torch.argmin): EmageVQVAEConv.decode_from_latent M.py:60-65, Quantizer.map2index P.py:158-164.
 * e2 = precomputed |e_k|^2 (n_codes).  Writes int64 indices.  e_dim must be 256.
 *   pm_l2_argmin_tc      n_codes == 256: persistent wgmma kernel - fp16 tensor-core screen of all 256 scores per row with a
 *                        rigorous error bound, exact fp32 re-scoring of every row whose best two screened distances
 *                        are within that bound; each z row is read from HBM once (1 KB + 8 B written per row).
 *                        max_ctas > 0 caps the persistent grid (<= 0: one CTA per SM).
 *   pm_l2_argmin_simt_f32  n_codes a multiple of 64: register-tiled fp32 SIMT kernel (sequential-k fp32 FMA).
 *   pm_l2_argmin_f32     dispatcher the product calls: tc for 256-code codebooks, simt otherwise. */
int pm_l2_argmin_f32(const float* z, long long rows, int rows_per_batch, long long z_bs,
                     const float* codebook, const float* e2, int n_codes, int e_dim, long long* index, void* stream);
int pm_l2_argmin_tc(const float* z, long long rows, int rows_per_batch, long long z_bs,
                    const float* codebook, const float* e2, int n_codes, int e_dim, long long* index, int max_ctas,
                    void* stream);
int pm_l2_argmin_simt_f32(const float* z, long long rows, int rows_per_batch, long long z_bs,
                          const float* codebook, const float* e2, int n_codes, int e_dim, long long* index, void* stream);
/* index = first argmax over the last dim: torch.max(F.log_softmax(x,2),2)[1], M.py:398-401 (monotone).
 * Row r of the (batch, rows_per_batch, ch) view lives at x + (r / rows_per_batch)*x_bs + (r % rows_per_batch)*ldx
 * (rows_per_batch <= 0: one dense matrix; the same convention addresses z in pm_l2_argmin_* with ld = 256), so the
 * tail frames of a window are read in place.  nonfinite (nullable): set to 1 when any element read is NaN / inf. */
int pm_row_argmax_f32(const float* x, long long rows, int ch, int ldx, int rows_per_batch, long long x_bs,
                      long long* index, int* nonfinite, void* stream);
/* out[r,:] = codebook[index[r],:]: Quantizer.get_codebook_entry P.py:166-170, nn.Embedding M.py:285-286.
 * n_table = rows of `codebook`; indices outside [0, n_table) are clamped (never an out-of-bounds read). */
int pm_gather_rows_f32(const float* codebook, long long n_table, const long long* index, long long rows, int ch,
                       float* out, uint16_t* planes, long long p_ps, int p_ld, int p_nsplit, void* stream);
/* |e_k|^2 per codebook row (done once at pack time) */
int pm_row_sqnorm_f32(const float* x, int rows, int ch, float* out, void* stream);

/* ---- pose composition: EmageVQModel.decode M.py:135-188 + rotation conversions P.py:6-104 ---------
 * face (bt,106) | upper (bt,78) | hands (bt,180) | lower (bt,61) decoder outputs (any may be NULL = the
 * reference's zero branch) -> expression (bt,100), axis_angle (bt,165), motion4inf (bt,337). */
int pm_pose_compose_f32(const float* face, const float* upper, const float* hands, const float* lower,
                        float* expression, float* axis_angle, float* motion4inf, long long bt, void* stream);

/* ---- global translation: velocity2position P.py:107-115 as used by get_global_motion M.py:195-205 --
 * rec (batch, t, ld) global-AE output; vel = rec[..., 54:57]; x/z integrated sequentially with dt,
 * y copied; ref_trans (batch,3) start position. */
int pm_global_trans_f32(const float* rec, int ld, int vel_off, const float* ref_trans, int ref_bs, float dt,
                        float* trans, int batch, int t, void* stream);

/* ---- audio front-end: decode output -> 16 kHz mono fp32, the resampling inside librosa.load(path, sr=16000) at
 * test_emage_audio.py:17 (T.py:17), train_emage_audio.py:48 (TR.py:48) and test_camn_audio.py:15.
 * pcm: interleaved (batch, n_in, channels) samples, int16 (is_int16 = 1, converted as v / 32768) or fp32 (is_int16 = 0);
 * clip stride in_bs elements.  Channels are summed in fp32 (x.mean(axis=1) order of the host reader) and divided by
 * `channels` (1..8, else PM_EUNSUPPORTED).  out (batch, n_out) fp32, clip stride out_bs, n_out = ceil(n_in*up/down):
 *   out[m] = sum_k h[k] * u[(m + n_pre_remove)*down - k],  u = mono signal upsampled by zero insertion, zero outside
 *   [0, n_in) - scipy.signal.resample_poly(padtype='constant') with h its front-padded filter.
 * bank: (up, taps) fp32, phase-major: bank[p*taps + j] = h[p + up*j] (zero past the end); up == down == 1 with
 * bank = {1} is the pure convert-and-mix.  fp32 FMA accumulation, each output in a fixed order (deterministic,
 * independent of batch position).  n_in == 0 writes nothing. */
int pm_resample_poly_f32(const void* pcm, int is_int16, long long in_bs, int batch, long long n_in, int channels,
                         const float* bank, int up, int down, int taps, long long n_pre_remove,
                         float* out, long long out_bs, void* stream);

/* ---- CaMN / DisCo (BASELINE configs[2],[3]) ------------------------------------------------------- */
/* One bidirectional nn.LSTM layer, zero initial state (camn:205-217,264-271; disco:212-216,255).  xproj (batch, t,
 * ldx >= 8*hidden) holds W_ih x + b_ih + b_hh for both directions (column dir*4H + gate*H + unit, gates i,f,g,o);
 * whh (2, 4H, H) fp32; y (batch, t, ldy >= 2H) receives [forward h | backward h].  `barrier` = 4 uint32 of scratch.
 * hidden must be 512.  Persistent cooperative kernel, W_hh resident in shared memory. */
int pm_lstm_bidir_f32(const float* xproj, long long x_bs, int ldx, const float* whh,
                      float* y, long long y_bs, int ldy, unsigned int* barrier,
                      int batch, int t, int hidden, void* stream);
/* Conditioning columns of the layer-0 LSTM input (camn:238-263, disco:229-253): for clip b < batch, row r < t, writes
 * out + b*o_bs + r*ldo + [0, spk_dim + pose_dims + 1) = [spk[speaker_id[b]] | seed pose | seed flag].
 * speaker_id: int64[batch], clamped to [0, n_spk) like pm_gather_rows_f32 (range checks belong to the caller).
 * seed: (batch, >= min(seed_frames, seed_len), pose_dims) rows with clip stride seed_bs and row stride seed_ld, nullable
 * (= zeros); seed_len is the length of the caller's seed sequence.  Row r shows seed row j = r when r < seed_len, else
 * j = r - (t - seed_len) (a shorter seed is extended by its own last t - seed_len rows; t <= 2*seed_len).  Seed row j is
 * (seed[j], 1) when j < min(seed_frames, seed_len), else zeros.  A pure copy: no arithmetic. */
int pm_lstm_cond_f32(const float* spk, long long n_spk, int spk_dim, const long long* speaker_id,
                     const float* seed, long long seed_bs, int seed_ld, int seed_len, int seed_frames, int pose_dims,
                     float* out, long long o_bs, int ldo, int batch, int t, void* stream);
/* rot6d (rows, n_sel*6) of the selected joints -> axis-angle (rows, 165), zeros at unselected joints: camn:274-277.
 * slot: device int32[55], position of joint j among the selected ones or -1. */
int pm_rot6d_to_aa_f32(const float* rot6d, long long rows, int n_sel, const int* slot, float* out, void* stream);
/* DisCo content mix disco:250-251: out[r,:] = softmax(sel[r,0:2])[0]*c1[r,:] + [1]*c2[r,:] (out row stride ldo) */
int pm_softmax2_mix_f32(const float* sel, const float* c1, const float* c2, float* out, long long rows, int ch, int ldo,
                        void* stream);

/* ---- SMPL-X body model (pantomatrix_b200/body_model.py): the smplx forward pass that every consumer of generated poses
 * runs next (emage_utils/motion_rep_transfer.py:38-50, emage_utils/motion_io.py:117-140, datasets/foot_contact.py:46-58).
 * Frames are rows r = b*t + i of `batch` clips of `t` frames; every per-frame input has a clip stride *_bs and a frame
 * stride *_ts in elements and a dense last dimension (views are read in place).
 *
 * pm_smplx_fk_f32: rest joints, Rodrigues and forward kinematics of every frame in one launch.
 *   poses (batch, t, 165) axis-angle, joint-major; joint j is used when bit j of joint_mask is set, else it reads as zero;
 *   pose_mean[165] (the hand means) is added afterwards.  betas (batch, 300) per clip and expr (batch, t, 100) per frame,
 *   both nullable (= zeros); transl (batch, t, 3) nullable.
 *   J = j_template (55*3) + j_dirs^T [betas | expr] with j_dirs (400, 55*3) = J_regressor . shapedirs.
 *   R_j = I + sin K + (1 - cos) K K, angle = |r + 1e-8| (smplx batch_rodrigues).  G_j = G_parent [R_j | J_j - J_parent],
 *   evaluated one tree level at a time: level_order[55] lists the joints by depth, level l is
 *   level_order[level_start[l] .. level_start[l+1]), n_levels <= 55; parents[55] with -1 at the root.
 *   Writes joints (rows, 55, 3) dense = G_j[:, 3] + transl, and (each nullable):
 *     rel_transforms (rows, 55, 12): A_j = G_j - [0 | G_j (J_j, 0)], the 3x4 rows of smplx's relative transforms;
 *     the vertex GEMM's A operand row [betas | expr | (R_1 - I) .. (R_54 - I)] (886 values, R row-major) as fp32 `feat`
 *     (row stride ld_feat >= 886) and / or as operand planes (p_nsplit | PM_FMT_F16 as for pm_add_layernorm_f32). */
int pm_smplx_fk_f32(const float* poses, long long pose_bs, long long pose_ts,
                    const float* betas, long long b_bs,
                    const float* expr, long long e_bs, long long e_ts,
                    const float* transl, long long t_bs, long long t_ts,
                    long long joint_mask, int batch, int t,
                    const float* j_template, const float* j_dirs, const float* pose_mean,
                    const int* parents, const int* level_order, const int* level_start, int n_levels,
                    float* joints, float* rel_transforms, float* feat, int ld_feat,
                    uint16_t* planes, long long p_ps, int p_ld, int p_nsplit, void* stream);
/* pm_smplx_skin_f32: linear blend skinning in place.  verts (rows, ld >= 3*n_verts) holds v_posed (the vertex GEMM's
 * output, vertex-major xyz) and receives (sum_j w_vj A_j) (v_posed, 1) + transl.  Weights in CSR form: row_ptr
 * (n_verts + 1), col / val (row_ptr[n_verts]).  rel_transforms (rows, 55, 12) from pm_smplx_fk_f32; transl as there
 * (nullable; t = frames per clip). */
int pm_smplx_skin_f32(float* verts, long long ld, long long rows, int n_verts,
                      const int* row_ptr, const int* col, const float* val, const float* rel_transforms,
                      const float* transl, long long t_bs, long long t_ts, int t, void* stream);
/* pm_motion_rep_f32: get_motion_rep_tensor (emage_utils/motion_rep_transfer.py:31-72).  poses (batch, t, 165) as above,
 * joints (batch, t, 55, 3) dense -> rep15d (batch, t, 55*15) dense, per joint [position | velocity | rot6d (quaternion
 * route, P.py:63-104) | angular velocity].  Velocities: (x[i+1] - x[i-1]) / two_dt inside a clip, one-sided over dt at
 * both ends (t >= 2). */
int pm_motion_rep_f32(const float* poses, long long pose_bs, long long pose_ts, const float* joints,
                      int batch, int t, float dt, float two_dt, float* rep15d, void* stream);

/* ---- SMPL-X mesh render (pantomatrix_b200/render.py): emage_utils/fast_render.py's frames of `views` (1 or 2)
 * 480 x 720 image views side by side, views * 480 x 720 RGB uint8, row 0 at the top, black background; view k is the
 * frame's k-th 480-column block.  Two views: render_one_sequence_with_face (fast_render.py:286-321; 56-68
 * do_render_one_frame, 80-92 np.hstack) and render_one_sequence (323-361); one: render_one_sequence_no_gt (363-391).
 * Fixed scene (fast_render.py:30-57): OrthographicCamera(xmag=1, ymag=1, znear 0.05, zfar 100) at create_pose_camera(-2), so pixel x =
 * (x_view / xmag + 1) * 240 and y = (1 - y_view / ymag) * 360 (the aspect ratio is ignored: a 1.5x vertical stretch);
 * DirectionalLight at create_pose_light(-30), direction toward the light l = (0, 0.5, 0.866); colour 220.
 * A chunk holds `frames` frames of `views` views.  With one view, verts1 / v1_fs and the second transform are not read
 * (verts1 may be NULL).  Three launches per chunk:
 *
 * pm_mesh_vertex_f32: one thread per (frame, view, vertex).  View k reads verts_k + frame * vk_fs (V rows of xyz, the
 *   body model's vertex buffer in place), applies p * scale_k + offset_k in fp32 (multiply, then add), then the view
 *   transform and the projection in fp32, each operation rounded on its own.  Writes xy (frames, views, V, 2) int32 =
 *   the pixel coordinates * 256 rounded to nearest even (8 sub-pixel bits), or INT_MIN where a coordinate is not finite
 *   or beyond the +-2^20-pixel guard band; depth (frames, views, V) = -z_view fp32; normal (frames, views, V, 3) fp32 =
 *   the normalised sum (0 when it is 0) of cross(b - a, c - a) of the transformed corners over the incident faces, in
 *   ascending face index: vf_ptr (V + 1) / vf_face, a CSR of the faces of each vertex.  faces (F, 3) int32.
 * pm_mesh_raster: one thread per (frame, view, triangle).  A triangle with an INT_MIN corner or zero area is skipped;
 *   one with negative area has corners 1 and 2 swapped (both sides are drawn).  Corner k's weight is the int64 edge
 *   function of the edge from corner k+1 to k+2, w_k = dx (cy - y) - dy (cx - x), at pixel centres (p * 256 + 128);
 *   a centre is covered when every w_k > 0, or w_k = 0 on a top-left edge (dy < 0, or dy = 0 and dx > 0).  The
 *   bounding box is clamped to the viewport.  Depth = fp32(((w0 d0 + w1 d1) + w2 d2) / area2), fp64 and each operation
 *   rounded; pixels outside [znear, zfar] are clipped.  atomicMin of (depth bits << 32 | triangle id) into vis
 *   (frames, views, 720, 480) uint64, which the caller clears to all ones (pm_memset_async 0xff): the nearest triangle
 *   wins, ties to the lower id, whatever the execution order.
 * pm_mesh_shade_u8: one thread per pixel of vis.  Background (all ones) is 0; otherwise the triangle's weights at the
 *   pixel centre over area2 interpolate its corner normals, and value = rint(220 max(0, n.l / |n|)) is written to R, G
 *   and B of out + frame * out_fs + (y * views * 480 + view * 480 + x) * 3 (out_fs >= 720 * views * 480 * 3 bytes). */
int pm_mesh_vertex_f32(const float* verts0, long long v0_fs, const float* verts1, long long v1_fs,
                       int n_verts, int frames, float scale0, float ox0, float oy0, float oz0,
                       float scale1, float ox1, float oy1, float oz1, const int* faces,
                       const int* vf_ptr, const int* vf_face, int* xy, float* depth, float* normal,
                       int views, void* stream);
int pm_mesh_raster(const int* xy, const float* depth, int n_verts, const int* faces, int n_faces,
                   int frames, unsigned long long* vis, int views, void* stream);
int pm_mesh_shade_u8(const unsigned long long* vis, const int* xy, const float* normal, int n_verts,
                     const int* faces, int frames, unsigned char* out, long long out_fs, int views, void* stream);
/* pm_time_upsample_f32: motion_io.time_upsample_numpy (the npz writer's upsample=30 // pose_fps) as the renderer reads
 * its output back, float32.  x (batch, t, channels) with clip / frame strides x_bs / x_ts and a dense last dimension ->
 * out (batch, k t, channels) dense.  k = 1 copies.  Otherwise, with n = k t, output frame j sits at
 * pos = j * step, step = (t-1) / (n-1) in fp64 (numpy's linspace; pos = t-1 exactly for j = n-1, 0 for every j when
 * t = 1), lo = clamp(floor(pos), 0, max(t-2, 0)), frac = pos - lo, a = x[lo], b = x[min(lo+1, t-1)], d = fp32(b - a)
 * and out = fp32(double(a) + double(d) * frac), each operation rounded on its own. */
int pm_time_upsample_f32(const float* x, long long x_bs, long long x_ts, int batch, int t, int channels, int k,
                         float* out, void* stream);

/* ---- PNG encoding of RGB8 frames (pantomatrix_b200/png.py, DESIGN.md section 11) --------------------------------
 * n_frames frames of h rows x w pixels of RGB8, each dense (row stride 3 w bytes), frame f at frames + f * f_fs.  Frame
 * f becomes one PNG file in data + f * cap, by one rule:
 *   scanlines: filter type 1 (Sub) on every row; S = h rows of s = 3 w + 1 bytes, byte 0 of a row 1, byte 1 + i
 *     raw[i] - raw[i - 3] mod 256 (raw[i] for i < 3);
 *   parse, per row, from its first byte: at frame position p the candidate distances, in the order
 *     (1, 2, 3, 4, 5, 6, 7, 8, 9, 12, s, s - 3, s + 3, s - 6, s + 6), are valid when 1 <= d <= min(p, 32768); L_d is the
 *     longest run <= min(258, row end - p) with S[p + j] == S[p + j - d] (overlap allowed, the source may lie in earlier
 *     rows).  If max L_d >= 3 a match of that length at the first d reaching it, else the literal S[p];
 *   deflate: one block, BFINAL = 1, BTYPE = 01 (fixed Huffman codes, RFC 1951 3.2.6), every row's tokens in row order,
 *     end-of-block; codes bit-reversed into the LSB-first stream, extra bits not;
 *   zlib: 0x78 0x01, the deflate data, Adler-32 of S big-endian;
 *   PNG: signature, IHDR (w, h, depth 8, colour type 2, 0, 0, 0), one IDAT with the zlib stream, IEND; each chunk's
 *     CRC-32 over its type and data.
 * Bound: every token costs at most 9 bits per byte of S it covers, so a file has at most
 *   ceil((3 + 9 h s + 7) / 8) + 63 bytes; every entry point requires that bound <= 2^31, cap >= it, cap a multiple of 4,
 *   data 4-byte aligned.  Workspace: row_bits and row_adler, n_frames * h entries each.  Launch order on one stream:
 *   pm_memset_async(data, 0, n_frames * cap), pm_png_count, pm_png_scan, pm_png_emit, pm_png_crc.
 * pm_png_count: one thread per (frame, row): filters on the fly, parses, writes the row's bit count to row_bits and
 *   its Adler-32 partials (sum of its bytes, sum of (s - i) x byte i, both mod 65521; wsum in the high word).
 * pm_png_scan: one CTA per frame: row_bits becomes each row's bit offset in its slot, nbytes[f] the file's size; writes
 *   everything but the block's data and IDAT's CRC, which it seeds with the part that does not depend on the data.
 * pm_png_emit: one thread per (frame, row): the parse again, ORing the row's bits into the slot at its offset.
 * pm_png_crc: one thread per 1 KiB block of IDAT's type and data: the block's CRC register moved to the chunk's end,
 *   XORed into the CRC bytes (the CRC is linear, so the result does not depend on the order). */
int pm_png_count(const unsigned char* frames, long long f_fs, int n_frames, int h, int w, long long* row_bits,
                 unsigned long long* row_adler, void* stream);
int pm_png_scan(int n_frames, int h, int w, long long* row_bits, const unsigned long long* row_adler,
                unsigned char* data, long long cap, long long* nbytes, void* stream);
int pm_png_emit(const unsigned char* frames, long long f_fs, int n_frames, int h, int w, const long long* row_off,
                unsigned char* data, long long cap, void* stream);
int pm_png_crc(int n_frames, int h, int w, unsigned char* data, long long cap, const long long* nbytes, void* stream);

/* ---- H.264 encoding of RGB8 frames (pantomatrix_b200/video.py, DESIGN.md section 12) ----------------------------
 * n_frames frames of h rows x w pixels of RGB8 (h, w multiples of 16; at most 36864 macroblocks and 543 per side,
 * level 5.1), each dense, frame f at frames + f * f_fs and at index f mod clip_len of its clip.  Frame f becomes one
 * sample in data + f * cap, by one rule:
 *   colour: Y = ((66 R + 129 G + 25 B + 128) >> 8) + 16 per pixel; with Rs, Gs, Bs the sums over each 2x2 block,
 *     Cb = ((-38 Rs - 74 Gs + 112 Bs + 512) >> 10) + 128, Cr = ((112 Rs - 94 Gs - 18 Bs + 512) >> 10) + 128 (>> floors);
 *   stream: Constrained Baseline (profile 66, constraint_set0/1), level 5.1, CAVLC, 4:2:0; SPS and PPS are built on
 *     the host (video.sps / video.pps);
 *   picture: IDR, nal_ref_idc 3, idr_pic_id = (f mod clip_len) mod 2; one I slice (slice_type 7) per macroblock row:
 *     first_mb_in_slice = row w / 16, frame_num 0, slice_qp_delta = qp - 26, disable_deblocking_filter_idc 1;
 *   macroblock: Intra16x16 with mb_qp_delta 0, chroma DC; luma DC (left column mean, 128 in column 0) or, when the left
 *     macroblock exists and its SAD against the source Y is strictly lower, Horizontal.  qbits = 15 + qp / 6,
 *     f = 2^qbits / 3, MF the standard table by position class; AC level = sgn(W) ((|W| MF + f) >> qbits); luma DC
 *     D = H4 WD H4, level = sgn(D) (((|D| >> 1) MF0 + 2 f) >> (qbits + 1)); chroma DC D = H2 WD H2, level =
 *     sgn(D) ((|D| MF0 + 2 f) >> (qbits + 1)) at QPc (table 8-15, offset 0).  cbpLuma 15 if any AC level, else 0;
 *     cbpChroma 2 if any chroma AC level, else 1 if any chroma DC level, else 0.  Reconstruction per 8.5 bit for bit;
 *   I_PCM (mb_type 25, source samples) instead, when the Intra16x16 macroblock_layer() would pass 3200 bits or a level
 *     would need level_prefix > 15;
 *   framing: each slice one NAL unit with emulation prevention, prefixed by its length (4 bytes, big-endian).
 * Bound: a slice has at most P = ceil((62 + 3200 w / 16 + 8) / 8) RBSP bytes and P / 2 emulation prevention bytes, so
 *   slice_cap >= slice_bound = 4 + P + P / 2 and cap >= (h / 16) slice_bound.  Launch order on one stream:
 *   pm_memset_async(data, 0, n_frames * cap), pm_h264_encode, pm_h264_gather.
 * pm_h264_encode: one warp per (frame, row): the slice into scratch + (f h / 16 + row) slice_cap, its length prefix
 *   included, and its byte count into slice_bytes.
 * pm_h264_gather: one CTA per (frame, row): the slice copied to its offset in the frame's slot; nbytes[f] the sum.
 *
 * pm_h264_encode_gop: the same with keyframe interval 1 <= gop <= clip_len; gop 1 is pm_h264_encode (recon unused).
 * n_frames is a multiple of clip_len.  Any gop >= clip_len gives the bytes of gop = clip_len, so a caller with a
 * larger gop passes clip_len.  Frame t of a clip is an IDR frame when t mod gop == 0, coded as above with idr_pic_id =
 * (t div gop) mod 2, else a P frame against the reconstruction of frame t - 1:
 *   SPS (video.sps(h, w, gop)): max_num_ref_frames 1 when gop > 1; the PPS is unchanged;
 *   P picture: one P slice per row, nal_ref_idc 2, nal_unit_type 1: first_mb_in_slice, slice_type 5, pps id 0,
 *     frame_num = (t mod gop) mod 16 (4 bits, wraps), num_ref_idx_active_override_flag 0,
 *     ref_pic_list_modification_flag_l0 0, adaptive_ref_pic_marking_mode_flag 0, slice_qp_delta, and
 *     disable_deblocking_filter_idc 1;
 *   motion: always (0, 0).  The macroblock above lies in another slice, so the P_Skip vector and every predictor are
 *     (0, 0); the prediction is the co-located 16x16 luma and 8x8 chroma of the reference, and a row reads only the
 *     same row of the reference;
 *   macroblock: the inter candidate is source - reference with the 4x4 transform of all 16 luma coefficients (no luma
 *     DC Hadamard), the chroma DC / AC split as intra, and f = 2^qbits / 6 for every level.  P_Skip when every inter
 *     level is 0 (the reconstruction is the reference).  Else P_L0_16x16 (mb_type 0, mvd (0, 0), coded_block_pattern
 *     by Table 9-4's Inter column: luma bit b8 when a 4x4 block of 8x8 block b8 has a level, chroma 0 / 1 / 2 as intra;
 *     mb_qp_delta 0 only when cbp > 0; luma residual_block(16) per 4x4 block of each set 8x8 bit) when the luma SAD
 *     against the reference is <= the Intra16x16 candidate's SAD, else Intra16x16 as above with mb_type + 5.  I_PCM
 *     (mb_type 30) in the same cases as above.  nC: a P_Skip neighbour counts 0, I_PCM 16.  mb_skip_run ue(v) before
 *     every coded macroblock, and after the last one when the slice ends in skips;
 *   bound: a slice has at most P = ceil((70 + 3201 w / 16 + 8) / 8) RBSP bytes (the longest slice header; at most 3201
 *     bits per macroblock with its share of the skip runs), so slice_cap >= 4 + P + P / 2, and data's slots hold
 *     (h / 16) times that (video.slot_bytes(h, w, gop)).
 * One warp per (chain, row), a chain being one GOP of one clip: the warp codes the chain's frames in order and keeps
 * the row's reconstruction (luma 16 x w, then Cb and Cr 8 x w / 2) in recon + (chain h / 16 + row) recon_stride,
 * recon_stride >= 24 w, (n_frames / clip_len) ceil(clip_len / gop) (h / 16) rows of workspace.  Each GOP's IDR frame
 * writes it before the P frames read it, so it needs no clearing.  Launch order: as pm_h264_encode.
 * pm_h264_gather checks cap and slice_cap against the gop = 1 bound only; with gop > 1 the caller sizes both by the
 * gop > 1 bound above (video.slice_bytes(w, gop), video.slot_bytes(h, w, gop)). */
int pm_h264_encode(const unsigned char* frames, long long f_fs, int n_frames, int clip_len, int h, int w, int qp,
                   unsigned char* scratch, long long slice_cap, int* slice_bytes, void* stream);
int pm_h264_encode_gop(const unsigned char* frames, long long f_fs, int n_frames, int clip_len, int h, int w, int qp,
                       unsigned char* scratch, long long slice_cap, int* slice_bytes, int gop, unsigned char* recon,
                       long long recon_stride, void* stream);
/* pm_h264_encode_me: pm_h264_encode_gop (gop 2 .. clip_len) with motion search range 1 <= search <= 32 whole pixels.
 * Everything but the inter macroblocks' vectors is the rule above (GOP structure, headers, SPS, PPS, intra, I_PCM,
 * nC, skip runs, cbp mapping):
 *   reference: the whole reconstruction of frame t - 1 (luma h x w, chroma h / 2 x w / 2), read at clipped
 *     coordinates outside it (8.4.2.2);
 *   integer search: every (dx, dy), |dx|, |dy| <= search, whose 16x16 luma block lies inside the frame; vectors in
 *     quarter-pel units; J(mv) = SAD_Y(mv) + LAMBDA[qp] (b(mvx) + b(mvy)), b(v) the bits of se(v), SAD_Y against the
 *     motion-compensated luma, measured against a zero predictor (every macroblock's search is independent); lowest
 *     J, ties to the smaller |mvx| + |mvy|, then smaller mvy, then smaller mvx;
 *   sub-pel: the 8 neighbours at +-2 of the integer winner, then the 8 at +-1 of the half-pel winner, in raster order,
 *     each replacing the centre only when its J is strictly lower.  Luma by 8.4.2.2.1 (6-tap, j from unrounded
 *     intermediates, quarter positions rounded averages), chroma by 8.4.2.2.2 (the luma vector in eighth chroma
 *     samples, bilinear);
 *   LAMBDA[qp] = floor(sqrt(0.85 2^((qp - 12) / 3)) + 0.5) in float64: 0 0 0 0 0 0 0 1 1 1 1 1 1 1 1 1 1 2 2 2 2 3 3 3
 *     4 4 5 5 6 7 7 8 9 10 12 13 15 17 19 21 23 26 30 33 37 42 47 53 59 66 74 83;
 *   macroblock: P_Skip when every level of the zero-motion inter candidate is 0 (vector (0, 0), 8.4.1.1), else the
 *     inter candidate at the searched vector (source - MC prediction, transform and quantisation as above) is
 *     P_L0_16x16 when its luma SAD <= the Intra16x16 candidate's, else Intra16x16; a non-zero vector with no level is
 *     P_L0_16x16 with cbp 0; I_PCM as above;
 *   mvd = mv - mvp, se(v) x then y; mvp (8.4.1.3, B and C never available) is the left macroblock's vector when it is
 *     P_L0_16x16, else (0, 0);
 *   bound: as gop > 1 above (the mvd counts toward the 3200 bits).
 * Workspaces: recon, two whole-frame reconstructions (Y, Cb, Cr planes, 3 h w / 2 bytes each) per chain,
 * recon_stride >= 3 h w apart; mv, mv_len >= chains (h / 16) (w / 16) int16 (x, y) pairs, 4-byte aligned; chains =
 * (n_frames / clip_len) ceil(clip_len / gop).  Neither needs clearing.  Launches, on one stream with no host
 * synchronisation: the code kernel for frame 0 of every chain (IDR, into buffer 0), then for k = 1 .. gop - 1 the
 * search kernel (one CTA per macroblock of every chain's frame k, the vectors into mv) and the code kernel (one warp
 * per (chain, row), frame k against buffer (k - 1) mod 2, into buffer k mod 2).  Launch order around it and slot
 * sizes: as pm_h264_encode_gop. */
int pm_h264_encode_me(const unsigned char* frames, long long f_fs, int n_frames, int clip_len, int h, int w, int qp,
                      unsigned char* scratch, long long slice_cap, int* slice_bytes, int gop, unsigned char* recon,
                      long long recon_stride, int search, short* mv, long long mv_len, void* stream);
/* Intra 4x4: qp | PM_H264_I4X4 (bit 8) in pm_h264_encode, pm_h264_encode_gop (forwarded at gop 1) and
 * pm_h264_encode_me; every other bit above the quantiser is refused.  Without the bit every byte is the rule above.
 * With it, in I and P slices, every coded macroblock also has an I_NxN candidate:
 *   availability (6.4.11.4): the macroblock above is another slice and the one to the right is not coded, so blocks of
 *     the top block row have no above samples, above-right samples come only from blocks of the same macroblock
 *     coded before (luma4x4BlkIdx order; missing ones are p[3, -1] when the above samples exist, 8.3.1.2), and the
 *     left (and, in block rows 1..3, above-left) samples of block column 0 come from the left macroblock's
 *     reconstruction, whatever its type (constrained_intra_pred_flag stays 0);
 *   mode per 4x4 block, in luma4x4BlkIdx order: the candidates are the modes 8.3.1.2 defines from the available
 *     samples; J = SAD(source, prediction) + LAMBDA[qp] b, b = 1 when the mode equals predIntra4x4PredMode, else 4;
 *     lowest J, ties to the lower mode.  predIntra4x4PredMode (8.3.1.1) is 2 for every top-row block and every block
 *     of the frame's column 0, and a left neighbour outside an I_NxN macroblock counts as mode 2;
 *   residual: the 4x4 transform of all 16 coefficients, quantised with f = 2^qbits / 3, reconstructed by 8.5.12 with
 *     the DC scaled like every other position; each block is reconstructed before the next is predicted;
 *   choice: J4 = the sum of the 16 blocks' J, J16 = the Intra16x16 candidate's SAD (DC or Horizontal as above); the
 *     macroblock is I_NxN when J4 + 6 LAMBDA[qp] < J16.  In P slices the intra cost is min(J16, J4 + 6 LAMBDA[qp]),
 *     and the inter candidate (zero-motion or searched) wins when its luma SAD is <= that cost; the P_Skip test and
 *     the vectors do not change;
 *   syntax: mb_type I_NxN (ue(0) in I slices, ue(5) in P slices), 16 x (prev_intra4x4_pred_mode_flag, or 0 and
 *     rem_intra4x4_pred_mode), intra_chroma_pred_mode 0 (chroma DC, coded as for Intra16x16), coded_block_pattern by
 *     Table 9-4's Intra column (luma bit b8 when a 4x4 block of 8x8 block b8 has a level), mb_qp_delta 0 only when
 *     cbp > 0, residual_block(16) per 4x4 block of each set 8x8 bit; nC by 9.2.1 (P_Skip 0, a clear cbp bit 0,
 *     I_PCM 16, an Intra16x16 AC block its TotalCoeff);
 *   I_PCM replaces an I_NxN macroblock in the same cases as above (over 3200 bits, a level_prefix above 15), so the
 *     slice bounds, slot sizes, SPS, PPS and MP4 boxes are unchanged.
 * The launches are as without the bit (other kernel instances, the same workspaces). */
int pm_h264_gather(int n_frames, int h, int w, const unsigned char* scratch, long long slice_cap,
                   const int* slice_bytes, unsigned char* data, long long cap, long long* nbytes, void* stream);

/* ---- FLAC encoding of recorded samples (pantomatrix_b200/flac.py, DESIGN.md section 13) ----------------------------
 * batch clips of n >= 1 samples x channels (1..8), clip b at pcm + b * clip_stride samples, each dense (n, channels):
 * int16 at bps 16, or int32 holding -2^23 .. 2^23 - 1 at bps 24.  Frame k of clip b (samples 4096 k onward, the last
 * frame may be shorter; F = ceil(n / 4096) per clip) becomes one FLAC frame in data + (b F + k) * cap, by one rule:
 *   header: sync 0xFFF8; block-size code 1100 (4096) or 0111 with bs - 1 in 16 bits; rate code 0100..1010 for 8, 16,
 *     22.05, 24, 32, 44.1 and 48 kHz, else 1100 (8-bit kHz) for a whole number of kHz below 256, else 1101 (16-bit
 *     Hz); channel assignment; sample size 100 (16) or 110 (24); frame number k UTF-8 coded; CRC-8 (poly 0x07).  At
 *     most 13 bytes (k < 2^21);
 *   subframes, per channel (no wasted bits, no LPC): the fewest bits of CONSTANT (all samples equal), FIXED order
 *     0..4 (order <= bs) and VERBATIM, ties to that order, then the lower order, partition order and parameter.
 *     FIXED residuals e are coded as u = 2e (e >= 0) or -2e - 1 by partitioned Rice: partition order p in 0..8 with
 *     2^p dividing bs and bs >> p >= order (partition 0 holds bs >> p minus order residuals); each partition's k is
 *     the one with the fewest count (k + 1) + sum(u >> k) bits; method 00 (4-bit k <= 14) unless 01 (5-bit k <= 30)
 *     is strictly smaller; no escape codes;
 *   stereo: the best subframes of L, R, S = L - R (at bps + 1) and M = (L + R) >> 1 (arithmetic, at bps); the pair
 *     with the fewest bits of independent (L R), left/side (L S), side/right (S R) and mid/side (M S), ties in that
 *     order.  Other channel counts are independent;
 *   end: zero bits to a byte boundary, CRC-16 (poly 0x8005) of the whole frame, big-endian.
 * Bound: the minimum never passes independent VERBATIM, so a frame of bs samples has at most
 *   18 + ceil(channels (8 + bps bs) / 8) bytes; cap >= that bound for bs = min(n, 4096), cap a multiple of 4, data
 *   4-byte aligned.  An int32 frame holding a sample outside -2^23 .. 2^23 - 1 is not coded: nbytes = -1, slot zero.
 * Workspace: rec, 66 int32 per (clip, frame, candidate), candidates = 4 (L, R, S, M) for stereo, else channels.
 * Launch order on one stream: pm_memset_async(data, 0, batch F cap), pm_flac_analyse, pm_flac_emit.
 * pm_flac_analyse: one CTA per (clip, frame, candidate): the candidate's best subframe (bits, type, order, p, method
 *   and the partitions' k) into its record.
 * pm_flac_emit: one CTA per (clip, frame): the assignment, the header, each subframe ORed into the slot at its bit
 *   offset (a block scan of the code lengths), the CRC-16, and nbytes. */
int pm_flac_analyse(const void* pcm, long long clip_stride, int batch, int n, int channels, int bps, int* rec,
                    void* stream);
int pm_flac_emit(const void* pcm, long long clip_stride, int batch, int n, int channels, int bps, int rate,
                 const int* rec, unsigned char* data, long long cap, long long* nbytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif
