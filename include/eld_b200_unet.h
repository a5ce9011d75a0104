/* eld_b200_unet.h - U-Net part of the C ABI (included by eld_b200.h).
 *
 * Replaces what PyTorch-eager dispatches to cuDNN/ATen for UNetSeeInDark (reference
 * models/arch/Unet.py:6-91) and ELDModel.optimize_parameters (models/ELD_model.py:469-475).
 * Activations are NHWC bf16 with an explicit channel pitch (so a concat buffer is just a wider
 * pitch: torch.cat at Unet.py:69,74,79,84 disappears); weights are bf16 K-major GEMM operands
 * packed from the fp32 PyTorch-layout master copy by eld_pack_weights.
 */
#ifndef ELD_B200_UNET_H
#define ELD_B200_UNET_H

/* kinds for eld_pack_weights: source layout is PyTorch's (Conv2d OIHW, ConvTranspose2d IOHW).  The packed
 * operand is OPAQUE: the logical K-major matrix listed below, stored as the shared-memory image the tiles
 * consume (blocks [n_tile][tap][64-channel chunk], 64B/128B swizzle applied) so that a block is one linear
 * bulk copy.  Same element count as the source.  The K side of the operand (cin for the fprop kinds, cout for the
 * dgrad kinds) and its row count must be multiples of 32, and a row count above 256 a multiple of 256 (a block holds
 * up to 256 rows; a partial last block would span the addresses of a whole one, past the operand's end): conv fprop
 * cout, conv / deconv dgrad cin in {32, 64, ..., 256, 512, 768, ...}; deconv fprop 4*cout likewise.  Other shapes:
 * ELD_E_ARG, nothing written. */
#define ELD_PACK_CONV_FPROP    0  /* [cout][ (kh*3+kw)*cin + ci ]            <- W[co][ci][kh][kw]      */
#define ELD_PACK_CONV_DGRAD    1  /* [cin ][ (kh*3+kw)*cout + co ]           <- W[co][ci][2-kh][2-kw]  */
#define ELD_PACK_DECONV_FPROP  2  /* [(kh*2+kw)*cout + co][ci]               <- Wt[ci][co][kh][kw]     */
#define ELD_PACK_DECONV_DGRAD  3  /* [ci][(kh*2+kw)*cout + co]               <- Wt[ci][co][kh][kw]     */
int eld_pack_weights(eld_ctx* ctx, const float* w, void* packed_bf16, int cout, int cin, int kind, void* stream);

#define ELD_ACT_NONE  0
#define ELD_ACT_LRELU 1  /* max(0.2x, x)  (Unet.py:102-104), fused into the producing tile           */
#define ELD_ACT_MASK  2  /* multiply by d lrelu/dx of `aux`, autograd of max(0.2x, x): 1 if aux > 0, 0.2 if aux < 0,
                          * 0.6 at +-0 and +-Inf (the arguments tie), 1.2 at NaN: backward of lrelu */

/* y[n,h,w,y_c0:y_c0+cout] = act( conv3x3_pad1(x[n,h,w,x_c0:x_c0+cin]) + bias )   nn.Conv2d(k=3,p=1), Unet.py:11-44.
 * With ELD_PACK_CONV_DGRAD weights (cin/cout swapped) the same tile is the data gradient.
 * cin % 32 == 0, cout % 32 == 0 (above 256 a multiple of 256, as the packed operand); any h, w >= 1 (partial tiles are
 * masked).  bias may be NULL, at most 1024 entries.  y (and aux): 32-byte aligned, pitch and first channel multiples
 * of 16 (the epilogue uses 256-bit accesses).  Every channel range [c0, c0 + c) lies inside its tensor's pitch.
 * A call that breaks one of these rules returns ELD_E_ARG and writes nothing; the same holds for the calls below. */
int eld_conv3x3_bf16(eld_ctx* ctx, const void* x, int x_pitch, int x_c0, int cin, const void* w_packed,
                     const float* bias, void* y, int y_pitch, int y_c0, int cout, int n, int h, int w,
                     int act, const void* aux, int aux_pitch, int aux_c0, void* stream);

/* nn.ConvTranspose2d(cin, cout, 2, stride=2) (Unet.py:30,34,38,42) as GEMM + pixel-shuffle epilogue:
 * y[n, 2h+kh, 2w+kw, y_c0+co] = sum_ci x[n,h,w,ci] Wt[ci][co][kh][kw] + bias[co].  (h, w) = INPUT grid.
 * cin % 32 == 0; cout a power of two >= 32 (the epilogue stores 32 channels of one output sub-pixel at a time) and at
 * most 1024; any h, w >= 1.  bias may be NULL.  y: as for eld_conv3x3_bf16. */
int eld_deconv2x2_bf16(eld_ctx* ctx, const void* x, int x_pitch, int x_c0, int cin, const void* w_packed,
                       const float* bias, void* y, int y_pitch, int y_c0, int cout, int n, int h, int w,
                       void* stream);

/* data gradient of the above: dx[n,h,w,ci] = sum_{kh,kw,co} dy[n,2h+kh,2w+kw,co] Wt[ci][co][kh][kw],
 * optionally times the LeakyReLU derivative of aux (the deconv input activation; act = ELD_ACT_NONE or ELD_ACT_MASK).
 * cin % 32 == 0 (above 256 a multiple of 256), cout % 32 == 0; h % 8 == 0 and w % 16 == 0 (the gather loads whole
 * 8 x 16 tiles of the input grid).  dx and aux: as y and aux of eld_conv3x3_bf16. */
int eld_deconv2x2_dgrad_bf16(eld_ctx* ctx, const void* dy, int dy_pitch, int dy_c0, int cout,
                             const void* w_packed, void* dx, int dx_pitch, int dx_c0, int cin,
                             int n, int h, int w, int act, const void* aux, int aux_pitch, int aux_c0,
                             void* stream);

/* Weight gradients, accumulated (+=) in f32 into the PyTorch-layout gradient `dw` (zero it once per
 * step): conv dW[co][ci][kh][kw] += sum_pixels dz[.,co] * x[. + (kh-1,kw-1), ci]   (autograd of Unet.py:11-44);
 * deconv dWt[ci][co][kh][kw] += sum_pixels x[n,h,w,ci] * dy[n,2h+kh,2w+kw,co].  (h, w) = x's grid.
 * cin % 32 == 0, cout % 32 == 0, h % 4 == 0, w % 16 == 0 (whole 4 x 16 reduction chunks). */
int eld_conv3x3_wgrad_bf16(eld_ctx* ctx, const void* x, int x_pitch, int x_c0, int cin,
                           const void* dz, int dz_pitch, int dz_c0, int cout,
                           float* dw, int n, int h, int w, void* stream);
int eld_deconv2x2_wgrad_bf16(eld_ctx* ctx, const void* x, int x_pitch, int x_c0, int cin,
                             const void* dy, int dy_pitch, int dy_c0, int cout,
                             float* dw, int n, int h, int w, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Whole-network step.  Parameters / gradients / Adam moments are FLAT fp32 device buffers in the
 * reference's state_dict order (conv1_1.weight, conv1_1.bias, ... conv10_1.bias; Unet.py:11-46), conv
 * weights OIHW, deconv weights IOHW - so released checkpoints copy in 1:1 and DDP all-reduces one buffer.
 */
typedef struct eld_unet eld_unet;
size_t eld_unet_param_count(void);                                   /* 7,760,484 for UNetSeeInDark(4,4) */
int    eld_unet_param_offset(const char* layer, int is_bias, size_t* offset, size_t* count);
size_t eld_unet_workspace_bytes(int n, int h, int w, int train);     /* activations (+gradients) + packed weights; train = 1 also
                                                                      * holds what the forward tiles leave for the backward: slope
                                                                      * words (2 bits per masked activation element) and pool codes
                                                                      * (1.5 bytes per pooled element: maxima + slope bits) */
/* Inference (train = 0): h % 16 == 0 and w % 16 == 0, as for the reference network.  Training (train = 1):
 * h % 128 == 0, w % 256 == 0.  Both: n * h * w < 2^26 pixels (the head's 32-bit index), or ELD_E_ARG before the
 * workspace is looked at - e.g. at most 255 frames of 512 x 512.  The caller owns `workspace` (device memory) for the
 * lifetime of the object.
 * Creation synchronises (a cudaMemset of the workspace, the kernels' shared-memory opt-in): create the object outside any
 * CUDA graph capture.  eld_unet_train_step (per-launch profiling off, eld_unet_profile) neither synchronises nor
 * allocates - memsets on `stream`, kernels with
 * programmatic stream serialization - so it captures into a graph (programmatic edges) and replays; the graph keeps
 * addressing this object's workspace, which must outlive it. */
int    eld_unet_create(eld_ctx* ctx, int n, int h, int w, int train, void* workspace, size_t bytes, eld_unet** out);
void   eld_unet_destroy(eld_unet* u);
/* The same network with 3-channel frames on either side (ELDModel.initialize, ELD_model.py:377-389: in_channels = 3 for
 * --stage_in srgb, out_channels = 3 for --stage_out srgb): conv1_1 becomes [32][cin][3][3], conv10_1 [cout][32][1][1];
 * everything else, and the meaning of every other entry point, is unchanged (x is [n][cin][h][w], out / target / dout
 * [n][cout][h][w]).  cin, cout in {3, 4}. */
size_t eld_unet_param_count_io(int cin, int cout);
int    eld_unet_param_offset_io(const char* layer, int is_bias, int cin, int cout, size_t* offset, size_t* count);
int    eld_unet_create_io(eld_ctx* ctx, int n, int h, int w, int train, void* workspace, size_t bytes,
                          int cin, int cout, eld_unet** out);
int    eld_unet_grad_buckets_io(int cin, int cout, size_t* offsets, int max_offsets);
/* ELDModel.forward (ELD_model.py:422-432): x f32 NCHW [n][4][h][w] -> out f32 NCHW [n][4][h][w] */
int    eld_unet_forward(eld_unet* u, const float* params, const float* x, float* out, void* stream);
/* forward + pixel loss (L1: mean |out-target|, losses.py:32; or MSE, see eld_unet_set_loss) + backward (ELD_model.py:411-420): grads is zeroed
 * and filled - or, after eld_unet_set_accumulate(u, 1), this call's gradients are added to what grads holds; *loss (device
 * float) receives this call's mean absolute error either way.  No optimizer step, no host sync. */
int    eld_unet_train_step(eld_unet* u, const float* params, const float* x, const float* target,
                           float* out, float* grads, float* loss, void* stream);
/* The autograd seam (ELDModel.backward_G, ELD_model.py:411-420: `loss.backward()` through netG): after an
 * eld_unet_forward on a train = 1 object (activations stay in the workspace), back-propagate the caller's
 * dout = d(loss)/d(out) (f32 NCHW) into `grads` (zeroed and filled, like eld_unet_train_step).  Any loss the caller likes.
 * The gradient of the input frame is not computed here; eld_unet_input_grad gives it on request. */
int    eld_unet_backward(eld_unet* u, const float* params, const float* x, const float* dout, float* grads, void* stream);
/* d(loss)/d(x) of the last eld_unet_backward / eld_unet_train_step on this object, stream-ordered after it:
 * dx f32 NCHW [n][cin][h][w], overwritten.  bf16 conv1_1 gradient and weights, fp32 accumulation.  Fails on an object
 * created with train = 0 and when no backward or train step has run since the last forward. */
int    eld_unet_input_grad(eld_unet* u, const float* params, float* dx, void* stream);
/* Several forwards before their backwards (a loss that calls the network twice, torch.utils.checkpoint, a retained
 * graph): what a forward leaves for its backward - activations, pool codes, slope words, packed weights - is its FORWARD
 * STATE.  A train = 1 object holds one in its workspace (the built-in state, which eld_unet_forward / eld_unet_backward /
 * eld_unet_train_step use); a caller may give a forward a state of its own and later back-propagate from that state,
 * whatever ran on the object in between.  state == NULL means the built-in state, so eld_unet_forward(u, ...) is
 * eld_unet_forward_state(u, NULL, ...) and eld_unet_backward likewise.  A caller state is device memory of
 * eld_unet_state_bytes(n, h, w, cin, cout) bytes at any address (laid out from its first 1 KB boundary); a non-NULL state
 * needs an object created with train = 1.  The backward writes only its own scratch and `grads`, so a state stays valid
 * after a backward that read it and may be back-propagated again.  Launches, grids and tiles are those of
 * eld_unet_forward / eld_unet_backward; eld_unet_input_grad follows either backward as before. */
size_t eld_unet_state_bytes(int n, int h, int w, int cin, int cout);   /* 0 for bad arguments */
int    eld_unet_forward_state(eld_unet* u, void* state, const float* params, const float* x, float* out, void* stream);
int    eld_unet_backward_state(eld_unet* u, void* state, const float* params, const float* x, const float* dout,
                               float* grads, void* stream);
/* Frozen parameters (p.requires_grad_(False) in the reference, ELD_model.py:473-475): which gradients the following
 * eld_unet_train_step / eld_unet_backward compute.  flags: one byte per parameter tensor in state_dict order (46: weight
 * and bias of every layer), nonzero = trainable; input_grad != 0 keeps the data-gradient chain running down to conv1_1
 * so that eld_unet_input_grad stays valid.  A layer's weight-gradient launch runs when its weight or its bias trains;
 * the data-gradient chain runs from the head down to the deepest tensor something still needs (a trainable layer below
 * it, or the frame), and a concat's skip half only when the encoder side needs it.  The `grads` range of a frozen tensor
 * reads zero; every bucket event is still recorded.  Default (and after all ones, input_grad = 1): everything, as
 * before.  Host-side only: no launch, no synchronisation. */
int    eld_unet_set_trainable(eld_unet* u, const uint8_t* flags, int n_flags, int input_grad);
/* Pixel loss of eld_unet_train_step (models/losses.py:29-36, --loss): 0 = nn.L1Loss (default), 1 = nn.MSELoss. */
#define ELD_LOSS_L1 0
#define ELD_LOSS_L2 1
int    eld_unet_set_loss(eld_unet* u, int kind);
/* Gradient accumulation over micro-batches (loss.backward() adding into .grad, DistributedDataParallel.no_sync()): with
 * on != 0, every following eld_unet_train_step adds its gradients to `grads` instead of zeroing it first, so k steps on k
 * micro-batches leave the sum of their gradients (scale it in the optimizer step: each step's loss is its own batch's
 * mean).  The step launches the kernels of a plain step in the same order, without the memset of `grads`; bucket events
 * mark the accumulated sum final.  A frozen tensor's range of `grads` is never written, so it keeps what it held: keep
 * one eld_unet_set_trainable mask over a window.  Governs eld_unet_train_step only (eld_unet_backward still zeroes and
 * fills).  Default off.  Host-side only: no launch, no synchronisation.  ELD_E_ARG for NULL or an object created with
 * train = 0. */
int    eld_unet_set_accumulate(eld_unet* u, int on);
/* Data-parallel overlap (SURVEY 8e; the reference is single-GPU, ELD_model.py:187-190): the flat gradient is final in
 * eld_unet_grad_buckets() = 4 contiguous ranges in backward-completion order (decoder upv6..conv10_1, bottleneck
 * conv5_*, encoder conv2_1..conv4_2, first layer conv1_1..conv1_2); offsets[2k], offsets[2k+1] = first element, element
 * count of bucket k.
 * After eld_unet_bucket_events(u, 1) every eld_unet_train_step records an event on its stream when bucket k of `grads`
 * is final; eld_unet_wait_bucket makes `stream` (the caller's communication stream) wait for it - the caller then
 * all-reduces grads[offset, offset+count) there while the rest of backward runs, and runs Adam on a bucket once its
 * all-reduce has joined the compute stream. */
int    eld_unet_grad_buckets(size_t* offsets, int max_offsets);      /* returns the bucket count (4) */
int    eld_unet_bucket_events(eld_unet* u, int enable);
int    eld_unet_wait_bucket(eld_unet* u, int bucket, void* stream);
/* Per-launch timing (CUDA events on the launch stream) of the steps issued after eld_unet_profile(u, 1);
 * eld_unet_profile_read synchronises, returns name[32] / ms / algorithmic FLOPs / algorithmic bytes per
 * launch and clears the log.  Used by bench.py for the live roofline numbers. */
int    eld_unet_profile(eld_unet* u, int enable);
/* Measurement aid (no reference counterpart): a one-thread kernel on `stream` that compares %clock64 with %globaltimer
 * for ~20 us and writes the SM clock in MHz that the preceding kernels were running at to *out_mhz_device. */
int    eld_clock_probe(eld_ctx* ctx, float* out_mhz_device, void* stream);
int    eld_unet_profile_read(eld_unet* u, int max, char* names32, float* ms, double* flops, double* bytes, int* count);
/* Where intermediate tensor `name` of the last step lives in the caller's workspace (for tests and debugging; no launch,
 * no synchronisation).  dims = {n, h, w, units per pixel}, *elem_bytes = 2 (bf16) / 4 (f32, uint32) / 1 (bytes).
 * Names: activations a1_1, cat9, p1, ... a9_2; gradients dz9_2 ... dz1_1, dcat9 ... dcat6 (the whole planar buffer: up
 * plane [n][h][w][units/2], then the skip plane), dp1 ... dp4; pool codes pc1 ... pc4 (one byte per pooled element:
 * maxima and neg bits) and pt1 ... pt4 (half a byte: tie bits); slope words sign:<activation> (neg bits) and
 * tie:<activation> (uint32, one per pixel and 32 channels each); packed operands wf:<layer>, wd:<layer> (dims
 * {1, 1, 1, element count}); the [tap][ci][co] staging of the conv weight gradients gtmp (f32, parameter offsets).
 * ELD_E_ARG for an unknown name and, on an object created with train = 0, for a training-only one. */
int    eld_unet_buffer(const eld_unet* u, const char* name, void** ptr, int dims[4], int* elem_bytes);
/* torch.optim.Adam step (ELD_model.py:400-401,475) on the flat buffers; grads are multiplied by
 * grad_scale first (1/world_size after a SUM all-reduce), then weight_decay * params is added.  step counts from 1.
 * ELD_E_ARG, nothing written: a NULL argument, step < 1. */
int    eld_adam_step(eld_ctx* ctx, float* params, const float* grads, float* m, float* v, size_t n,
                     float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                     float grad_scale, void* stream);
/* The same update on n_segs ranges of the flat buffers in ONE launch: segs (host) = (offset, count) pairs, steps (host) =
 * each range's own step count (torch.optim.Adam's per-parameter state['step']: a tensor that was frozen for a while has
 * taken fewer steps).  Elements outside the ranges are not touched.  n_segs <= 64.  ELD_E_ARG, nothing written: a NULL
 * argument, a step count < 1, more than 64 ranges, two ranges that share an element (empty ranges share none). */
int    eld_adam_step_segments(eld_ctx* ctx, float* params, const float* grads, float* m, float* v, const size_t* segs,
                              const int* steps, int n_segs, float lr, float beta1, float beta2, float eps,
                              float weight_decay, float grad_scale, void* stream);
/* Capturable Adam (torch.optim.Adam(capturable=True)): the same update, with the learning rate and the step counters in
 * DEVICE memory, read when the kernels run, so that a CUDA graph that captured the call is right on every replay.
 * *lr (device float) is the learning rate; a step counter (device int) holds the steps its elements have taken so far
 * (>= 0), and this call updates them with the bias corrections of step counter + 1 (1 - beta^t by device powf, which may
 * differ from the host powf of eld_adam_step by an ulp) and leaves counter + 1 behind.
 * Mechanism: two launches on `stream`.  The update kernel reads lr and the counters (thread s of each block derives range
 * s's bias corrections into shared memory) and never writes a counter; a one-block kernel issued after it increments
 * each counter once.  No thread reads a counter after it has been incremented.
 * eld_adam_step_capturable: elements [0, n), one counter `step`.
 * eld_adam_step_segments_capturable: n_segs ranges as for eld_adam_step_segments (segs, host), steps (host) = one device
 * counter per range; a counter named by several ranges takes one step.  Ranges holding no element still step their
 * counters; n_segs == 0 launches nothing.
 * ELD_E_ARG, nothing written and nothing launched: a NULL argument (a NULL counter among steps included), more than 64
 * ranges, two ranges that share an element. */
int    eld_adam_step_capturable(eld_ctx* ctx, float* params, const float* grads, float* m, float* v, size_t n,
                                const float* lr, int* step, float beta1, float beta2, float eps, float weight_decay,
                                float grad_scale, void* stream);
int    eld_adam_step_segments_capturable(eld_ctx* ctx, float* params, const float* grads, float* m, float* v,
                                         const size_t* segs, int* const* steps, int n_segs, const float* lr,
                                         float beta1, float beta2, float eps, float weight_decay, float grad_scale,
                                         void* stream);
/* torch.optim.Adam's parameter groups: the update of eld_adam_step_segments with each range's own hyperparameters, in
 * ONE launch.  ranges (host): n_ranges entries, each the elements [offset, offset + count) of the flat buffers, their
 * step count (>= 1) and their group's lr, betas, eps and weight decay; grad_scale applies to every range.  The same
 * hyperparameters in every range give eld_adam_step_segments' result bit for bit.  Elements outside the ranges are not
 * touched.  n_ranges <= 64.
 * ELD_E_ARG, nothing written and nothing launched: a NULL argument, a step count < 1, more than 64 ranges, two ranges that
 * share an element (empty ranges share none), an lr, eps or weight_decay that is negative or not finite, a beta outside
 * [0, 1). */
typedef struct {
    size_t offset, count;
    int    step;
    float  lr, beta1, beta2, eps, weight_decay;
} eld_adam_range;
int    eld_adam_step_ranges(eld_ctx* ctx, float* params, const float* grads, float* m, float* v,
                            const eld_adam_range* ranges, int n_ranges, float grad_scale, void* stream);
/* The capturable form (as eld_adam_step_segments_capturable): each range names its own device step counter and its own
 * device learning rate, read when the kernels run; ranges of one parameter group share one lr pointer, so a replay reads
 * each group's current rate.  A range's bias corrections use its own betas.  Two launches on `stream` (the update, then
 * the counters' increment); a counter named by several ranges takes one step; n_ranges == 0 launches nothing.
 * ELD_E_ARG, nothing written and nothing launched: a NULL argument (a NULL counter or lr among the ranges included),
 * more than 64 ranges, two ranges that share an element, an eps or weight_decay that is negative or not finite, a beta
 * outside [0, 1).  The device lr is not read on the host: the caller keeps it a finite number >= 0. */
typedef struct {
    size_t       offset, count;
    int*         step;          /* device */
    const float* lr;            /* device */
    float        beta1, beta2, eps, weight_decay;
} eld_adam_range_dev;
int    eld_adam_step_ranges_capturable(eld_ctx* ctx, float* params, const float* grads, float* m, float* v,
                                       const eld_adam_range_dev* ranges, int n_ranges, float grad_scale, void* stream);
/* torch.optim.Adam's other update rules, per range: eld_adam_step_ranges(_capturable) with `flags` in every record, a
 * set of
 *   ELD_ADAM_AMSGRAD     (amsgrad=True)   vmax <- max(vmax, v), NaN if either is (torch.maximum); the denominator is
 *                                         sqrt(vmax) / sqrt(1 - beta2^t) + eps.  vmax is laid out like m and v.
 *   ELD_ADAM_MAXIMIZE    (maximize=True)  the scaled gradient's sign flipped before the weight decay.
 *   ELD_ADAM_DECOUPLED   (decoupled_weight_decay=True, torch.optim.AdamW) a non-zero weight decay multiplies the
 *                                         parameters by 1 - lr * weight_decay (fp32, rounded once; the device lr in the
 *                                         capturable form) instead of adding weight_decay * params to the gradient.
 * Flags 0 in every range give eld_adam_step_ranges(_capturable)'s result bit for bit, and a range's flags 0 give that
 * range the plain update's bits in any call.  vmax is read and written only on AMSGRAD ranges and may be NULL when no
 * range has that flag.  One update launch (plus the counters' increment in the capturable form), as the plain calls.
 * ELD_E_ARG, nothing written and nothing launched: every refusal of the plain call, flag bits other than these three,
 * a NULL vmax while some range has ELD_ADAM_AMSGRAD. */
#define ELD_ADAM_AMSGRAD   1u
#define ELD_ADAM_MAXIMIZE  2u
#define ELD_ADAM_DECOUPLED 4u
typedef struct {
    size_t   offset, count;
    int      step;
    float    lr, beta1, beta2, eps, weight_decay;
    unsigned flags;
} eld_adam_range_ex;
typedef struct {
    size_t       offset, count;
    int*         step;          /* device */
    const float* lr;            /* device */
    float        beta1, beta2, eps, weight_decay;
    unsigned     flags;
} eld_adam_range_dev_ex;
int    eld_adam_step_ranges_ex(eld_ctx* ctx, float* params, const float* grads, float* m, float* v, float* vmax,
                               const eld_adam_range_ex* ranges, int n_ranges, float grad_scale, void* stream);
int    eld_adam_step_ranges_ex_capturable(eld_ctx* ctx, float* params, const float* grads, float* m, float* v,
                                          float* vmax, const eld_adam_range_dev_ex* ranges, int n_ranges,
                                          float grad_scale, void* stream);

#endif
