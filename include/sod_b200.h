/* sod_b200.h — C ABI of libsod_b200.so: the H100 (sm_90a) data-parallel hot path of
 * lartpang/Distributed-SOD-Project.
 *
 * The reference is pure Python and has NO FFI layer of its own (SURVEY §8b): its hot path is reached
 * through five Python call sites.  Each entry point below replaces the arithmetic behind one of them;
 * the citation on each says which (paths relative to the reference repository).  A maintainer of the
 * reference binds these with `ctypes` exactly as INTEGRATION.md shows.
 *
 * Conventions
 *  - plain C: raw device pointers, element counts as int64_t, dtype enums, `void* stream` = cudaStream_t.
 *  - the caller owns every buffer; the library allocates nothing and never synchronises the stream.
 *  - return value: 0 ok; <0 contract error (sod_strerror); >0 a cudaError_t from the launch.
 *  - re-entrant; callable from any host thread (PyTorch's autograd thread calls the *_bwd entries).
 *  - collective entries (anything taking a sod_comm) must be called in the same order on every rank.
 */
#ifndef SOD_B200_H
#define SOD_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SOD_ABI_VERSION 7
#define SOD_MAX_WORLD 8
#define SOD_MAX_SEGMENTS 16
#define SOD_COMM_MAX_BLOCKS 1024   /* flag rows per channel */
#define SOD_COMM_CHANNELS 4        /* barrier channels: 0 gradient reduce+SGD or +Adam, 3 plain all-reduce (1,2 reserved; the
                                      SyncBN exchange uses tagged packets, not flags) */

typedef enum { SOD_F32 = 0, SOD_BF16 = 1, SOD_F16 = 2 } sod_dtype;

enum {
    SOD_OK = 0,
    SOD_EINVAL = -1,       /* null pointer / negative size / bad enum */
    SOD_EALIGN = -2,       /* pointer or offset not 16-byte aligned */
    SOD_EWORKSPACE = -3,   /* workspace too small */
    SOD_EUNSUPPORTED = -4, /* shape outside what the kernels cover (e.g. C % 8 != 0) */
    SOD_ECOMM = -5         /* bad communicator (world > SOD_MAX_WORLD, missing peer pointer …) */
};

int sod_version(void);
const char* sod_strerror(int code);
/* sm count / compute capability of the current device; the hot path refuses anything but sm_90 */
int sod_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ------------------------------------------------------------------------------------------------
 * (3) BCE-with-logits + CEL, forward AND backward in one kernel.
 * Replaces: torch.nn.BCEWithLogitsLoss (train.py:203) + CEL.forward (loss/CEL.py:15-20) as summed by
 *           get_total_loss (utils/pipeline_ops.py:37-42), and their autograd backward (train.py:302).
 *   total = w_bce*BCE(reduction) + w_cel*CEL;  grad = grad_scale * d total / d logits
 * scalars_out[8] (device, fp32): bce, cel, total, sum_p, sum_t, sum_pt, bce_sum(unreduced), n
 * mode: 0 auto (resident when the tensor fits the grid's shared memory, ≈5.4 M elements, else ring-streamed), 1 force the
 *       shared-memory-resident single-read kernel, 2 force the ring-streamed kernel (producer warp + shared-memory ring;
 *       phase 2 re-streams what did not stay resident, newest first, with L2 eviction hints)
 * workspace: sod_loss_workspace_bytes() bytes, 16-byte aligned; contents need not be initialised.
 * ------------------------------------------------------------------------------------------------ */
size_t sod_loss_workspace_bytes(void);
int sod_loss_bce_cel_fwd_bwd(const void* logits, int logits_dtype, const void* mask, int mask_dtype,
                             void* grad_logits, int grad_dtype, float* scalars_out, int64_t n,
                             int reduction_sum, float w_bce, float w_cel, float grad_scale, float eps,
                             int mode, void* workspace, size_t workspace_bytes, void* stream);
/* the same with grad = (*grad_scale_dev) * grad_scale * d total / d logits, rounded once to the logits dtype: the amp loss
 * scale is applied before the rounding (fp16 logits at a mean over millions of pixels would otherwise round the unscaled
 * gradient, ≈1/n, into fp16's subnormal range).  grad_scale_dev: device fp32 scalar, read at execution time. */
int sod_loss_bce_cel_fwd_bwd_scaled(const void* logits, int logits_dtype, const void* mask, int mask_dtype,
                                    void* grad_logits, int grad_dtype, float* scalars_out, int64_t n,
                                    int reduction_sum, float w_bce, float w_cel, float grad_scale, const float* grad_scale_dev,
                                    float eps, int mode, void* workspace, size_t workspace_bytes, void* stream);
/* grad *= *scale_dev (device scalar): only for the case where the loss is not the root of backward */
int sod_scale_by_device_scalar(void* grad, int dtype, int64_t n, const float* scale_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Symmetric-memory communicator (one process per GPU; all ranks on one NVSwitch domain).
 * Built by the host from torch.distributed._symmetric_memory (buffer_ptrs / multicast_ptr): `peer[r]`
 * is rank r's arena as mapped into THIS process, `mc` the multicast (NVLS) mapping of the same arena
 * or 0.  Replaces the NCCL communicator of dist.init_process_group (train.py:73-77) for the hot path.
 * The first sod_comm_flag_bytes() bytes of every arena are the signal area and must be zeroed once
 * (before the first collective, followed by a process-group barrier).
 * ------------------------------------------------------------------------------------------------ */
typedef struct {
    int32_t rank;
    int32_t world;
    uint64_t peer[SOD_MAX_WORLD];
    uint64_t mc;
    uint64_t arena_bytes;
    uint32_t* error_flag;   /* device word in local memory; set non-zero on a barrier timeout */
    uint64_t timeout_cycles;/* bounded spin in SM clock cycles; 0 = default (~20 s for barriers, ~2 s for packets) */
    uint32_t* block_seq;    /* device array [SOD_COMM_CHANNELS*SOD_COMM_MAX_BLOCKS] in LOCAL memory, zeroed once:
                               per-block barrier sequence numbers, advanced by the kernels themselves, so the
                               collectives carry no host-side sequence number and replay inside CUDA graphs */
} sod_comm;
size_t sod_comm_flag_bytes(void);

/* ------------------------------------------------------------------------------------------------
 * (1) gradient all-reduce ⊕ unscale ⊕ SGD-momentum.
 * Replaces: apex DDP(delay_allreduce=True) flat all-reduce + ×1/W (train.py:185), amp unscale
 *           (train.py:299), torch.optim.SGD.step as configured by make_optimizer
 *           (utils/pipeline_ops.py:295-313; train.py:303), and optimizer.zero_grad (train.py:297).
 * Flat fp32 buffers of n elements (n % 4 == 0), laid out group-major; `segs` (host array) gives each
 * contiguous range its lr / weight_decay / momentum; SOD_SEG_FROZEN ranges receive the averaged
 * gradient but p and v are left alone (the reference leaves `div_2.*` out of every param group).
 *   g = (Σ_ranks grad) * inv_scale / world + wd*p ;  v = mu*v + g ;  p -= lr*v
 * world==1 (comm NULL): purely local.  world>1: grad and param live in the arena at grad_off/param_off;
 * rank r reduces shard r (NVLS multimem.ld_reduce when comm->mc != 0 and algo allows, else peer loads
 * in rank order), updates its shard of p and v, and writes the new p to every rank (multimem.st / peer
 * stores).  `mom` is the local momentum buffer, full length n (only shard r is used when world>1).
 * found_inf (device, may be NULL): when non-NULL and *found_inf != 0 the whole step is skipped.
 * flags: SOD_SGD_ZERO_GRAD zeroes the local gradient buffer(s) on the way out.
 * Mixed precision ("fp32 master" of apex amp, train.py:183): `grad16` (bf16, same flat layout, may be NULL) holds
 * the gradients autograd produced in bf16 — the kernel adds them to `grad` in registers, so no bf16→fp32 cast
 * kernel and no fp32 accumulation kernel run per tensor; `shadow16` (bf16, may be NULL) receives the rounded copy
 * of every updated parameter, which the next forward's convolutions consume directly (no per-iteration weight
 * cast).  Ranges flagged SOD_SEG_GRAD16 take their gradient from `grad16` alone.  With world>1 `grad16` lives in the
 * arena too (grad16_off) and those ranges are reduced from the bf16 values themselves; sod_grad_merge_bf16 is only needed
 * when fp32 gradients were ALSO written for such a range (a forward outside autocast).  `shadow16` is the LOCAL bf16
 * buffer every rank refreshes from the all-gathered parameters.
 * ------------------------------------------------------------------------------------------------ */
enum { SOD_SEG_FROZEN = 1,
       SOD_SEG_GRAD16 = 2 /* the gradient of this range exists ONLY in the bf16 buffer (`grad16`): the fp32 buffer is neither read
                             nor cleared there, and with world>1 the bf16 values themselves cross NVLink (summed in fp32) */,
       SOD_SEG_NESTEROV = 4 /* SGD only: Nesterov momentum, v = mu*v + g ; p -= lr*(g + mu*v) (torch.optim.SGD nesterov=True,
                               the reference's `nesterov` key for sgd_trick / f3_trick, utils/pipeline_ops.py:258,312) */ };
typedef struct {
    int64_t begin, end;        /* element range, multiples of 4 */
    float lr, weight_decay, momentum;
    int32_t flags;
} sod_sgd_segment;
enum { SOD_SGD_ZERO_GRAD = 1, SOD_ALGO_NO_MULTIMEM = 2,
       SOD_DEBUG_TIMING = 4 /* syncbn: per-CTA globaltimer stamps behind the workspace (tools/bn_phases.py) */,
       SOD_BN_ACCUMULATE_PARAM_GRADS = 8 /* syncbn_bwd: dgamma/dbeta += (write straight into the bound .grad) */,
       SOD_ALGO_FORCE_MULTIMEM = 16 /* use NVLS even at world 2, where the default is peer loads */,
       SOD_BN_BWD_MASK_FROM_X = 32 /* syncbn_bwd: re-derive the ReLU mask from x with the forward's arithmetic instead
                                      of reading y (one input stream less); needs relu, beta and dres == NULL */,
       SOD_BN_L2_HINTS = 64 /* syncbn_bwd: L2 eviction-priority hints on the bulk copies — evict-last for chunks that
                               are fetched twice, evict-first for last uses */,
       SOD_BN_LAUNCH_COOP = 128 /* syncbn_fwd/bwd: cooperative launch (driver-guaranteed co-residency of the grid) */,
       SOD_BN_LAUNCH_PDL = 256 /* syncbn_fwd/bwd: programmatic dependent launch (prologue overlaps the producer's tail) */,
       SOD_GRAD16_F16 = 512 /* step kernels, sod_grad_merge_bf16, sod_grad_check_ranges: `grad16` and `shadow16` hold fp16
                               (amp with dtype fp16) instead of bf16; the shadow is rounded to nearest, = param.half() */ };

/* lr_dev (device, fp32[nseg], may be NULL): when given, the learning rate of segment i is read from lr_dev[i] at
 * execution time instead of segs[i].lr — a captured CUDA graph then follows CustomScheduler
 * (utils/pipeline_ops.py:225-229, stepped per epoch train.py:240-241 or per iteration train.py:288-289) with one
 * small H2D copy per change and no re-capture. */
int sod_sgd_momentum(float* param, float* mom, float* grad, void* grad16, void* shadow16, int64_t n,
                     const sod_sgd_segment* segs, int nseg, const float* lr_dev, float inv_scale,
                     const uint32_t* found_inf, int flags, void* stream);
/* grad16_off (world>1): arena offset of the symmetric bf16 gradient buffer, or 0.  Ranges flagged SOD_SEG_GRAD16 are reduced
 * from it (peer loads of the bf16 values, fp32 sum in rank order — half the reduce-scatter bytes and no merge pre-pass);
 * all other ranges from the fp32 buffer at grad_off as before. */
int sod_allreduce_sgd(const sod_comm* comm, uint64_t grad_off, uint64_t grad16_off, uint64_t param_off, float* mom,
                      void* shadow16, int64_t n, const sod_sgd_segment* segs, int nseg, const float* lr_dev,
                      float inv_scale, const uint32_t* found_inf, int flags, void* stream);

/* ------------------------------------------------------------------------------------------------
 * (1b) gradient all-reduce ⊕ unscale ⊕ Adam — the same two kernels as above with the update rule of
 *      torch.optim.Adam (amsgrad=False, maximize=False, L2 weight decay folded into g), which the reference builds
 *      for optim "adam" (utils/pipeline_ops.py:287-294).  Per element, with t = step_dev[segment] + 1:
 *   g = (Σ_ranks grad) * inv_scale / world + wd*p ;  m += (1-β1)*(g-m) ;  v = β2*v + (1-β2)*g*g
 *   p -= fp32(lr / (1-β1^t)) * m / (sqrt(v) / fp32(sqrt(1-β2^t)) + eps)      (bias corrections in fp64)
 * exp_avg (m) and exp_avg_sq (v) are local fp32 buffers of n elements, laid out like `param`; with world>1 rank r
 * only reads and writes its shard of them.  Everything else — segments, SOD_SEG_FROZEN / SOD_SEG_GRAD16, grad16,
 * shadow16, lr_dev, found_inf, flags, the arena offsets — means what it means for the SGD entry points above.
 * step_dev (device, int32[SOD_ADAM_STEP_WORDS], zeroed once by the caller): step_dev[i] is the number of steps segment i
 * has taken; the last CTA of the launch advances every non-frozen segment's count, so a captured CUDA graph replays
 * with the right bias correction.  When *found_inf != 0 nothing but the gradients changes (the counts included).
 * step_dev[SOD_MAX_SEGMENTS] is a ticket word the kernel uses and leaves at 0.  One step_dev per stream at a time.
 * SOD_SEG_NESTEROV is refused here (SOD_EINVAL), as are β outside [0, 1) and eps < 0.  β1 and β2 enter the
 * arithmetic as the shortest decimal that rounds to the given fp32 value (0.999f → 0.999), as torch's Python floats do.
 * ------------------------------------------------------------------------------------------------ */
#define SOD_ADAM_STEP_WORDS (SOD_MAX_SEGMENTS + 1)
typedef struct {
    int64_t begin, end;        /* element range, multiples of 4 */
    float lr, weight_decay, beta1, beta2, eps;
    int32_t flags;
} sod_adam_segment;
int sod_adam(float* param, float* exp_avg, float* exp_avg_sq, float* grad, void* grad16, void* shadow16, int64_t n,
             const sod_adam_segment* segs, int nseg, const float* lr_dev, int32_t* step_dev,
             float inv_scale, const uint32_t* found_inf, int flags, void* stream);
int sod_allreduce_adam(const sod_comm* comm, uint64_t grad_off, uint64_t grad16_off, uint64_t param_off,
                       float* exp_avg, float* exp_avg_sq, void* shadow16, int64_t n, const sod_adam_segment* segs,
                       int nseg, const float* lr_dev, int32_t* step_dev, float inv_scale,
                       const uint32_t* found_inf, int flags, void* stream);

/* ------------------------------------------------------------------------------------------------
 * (1c) device-resident dynamic loss scale — apex amp O1 with fp16 (train.py:183,299): initial scale 2^16; a step whose
 *      gradients hold an inf or NaN is skipped and halves the scale (never below 1); `growth_interval` clean steps in a row
 *      double it.  The step entry points below are the four above with `sod_loss_scaler* scaler` in place of
 *      (inv_scale, found_inf): they read found_inf and 1/scale at execution time, and the last CTA applies the rules
 *      (ticket, like step_dev of sod_adam):
 *        overflow: scale = max(scale/2, 1), unskipped = 0      clean: unskipped += 1, scale = min(2*scale, 2^24) when
 *        unskipped % growth_interval == 0 (apex's max_loss_scale; a larger scale set by the caller only halves on overflow)
 *      found_inf is left set to the step's verdict; the caller clears it before the next step's first check (with
 *      world > 1: after the previous step, which stream order gives).  A captured CUDA graph replays the whole protocol with
 *      no host round trip.  One scaler per stream at a time; `ticket` starts at 0 and is left at 0.
 * world > 1: `scaler` lives in the arena (the same offset on every rank); after its start barrier the kernel ORs the
 * found_inf words of all ranks, so every rank skips or steps on the same verdict and the scalers stay bit-identical.
 * ------------------------------------------------------------------------------------------------ */
typedef struct {
    uint32_t found_inf;        /* non-zero: a gradient of this step is inf/NaN (OR-ed in by the checks below) */
    float scale;
    int32_t unskipped;         /* clean steps since the last overflow (apex's `unskipped`) */
    int32_t growth_interval;
    uint32_t ticket;
    uint32_t reserved[3];
} sod_loss_scaler;
int sod_sgd_momentum_scaler(float* param, float* mom, float* grad, void* grad16, void* shadow16, int64_t n,
                            const sod_sgd_segment* segs, int nseg, const float* lr_dev, sod_loss_scaler* scaler, int flags,
                            void* stream);
int sod_allreduce_sgd_scaler(const sod_comm* comm, uint64_t grad_off, uint64_t grad16_off, uint64_t param_off, float* mom,
                             void* shadow16, int64_t n, const sod_sgd_segment* segs, int nseg, const float* lr_dev,
                             sod_loss_scaler* scaler, int flags, void* stream);
int sod_adam_scaler(float* param, float* exp_avg, float* exp_avg_sq, float* grad, void* grad16, void* shadow16, int64_t n,
                    const sod_adam_segment* segs, int nseg, const float* lr_dev, int32_t* step_dev, sod_loss_scaler* scaler,
                    int flags, void* stream);
int sod_allreduce_adam_scaler(const sod_comm* comm, uint64_t grad_off, uint64_t grad16_off, uint64_t param_off,
                              float* exp_avg, float* exp_avg_sq, void* shadow16, int64_t n, const sod_adam_segment* segs,
                              int nseg, const float* lr_dev, int32_t* step_dev, sod_loss_scaler* scaler, int flags,
                              void* stream);

/* Multi-tensor gather of bf16 gradients into the flat bf16 gradient buffer (`grad16` above): item i copies
 * numel elements from the dense tensor `src` to dst16[dst_offset ...] (dst_offset % 8 == 0).  Replaces the
 * per-parameter accumulate kernels autograd launches at the end of backward (train.py:302): the weight gradients are
 * left where cuDNN wrote them and collected by ONE launch (per SOD_GATHER_MAX_ITEMS tensors). */
#define SOD_GATHER_MAX_ITEMS 160
typedef struct {
    const void* src;
    int64_t dst_offset, numel;
} sod_gather_item;
int sod_grad_gather16(const sod_gather_item* items, int nitems, void* dst16, int64_t dst_elems, void* stream);
/* the same gather for dtype SOD_BF16 or SOD_F16, which also does *found_inf |= any(!isfinite(what it copied)): the amp
 * overflow check of the stolen weight gradients costs no pass of its own */
int sod_grad_gather16_checked(const sod_gather_item* items, int nitems, void* dst16, int64_t dst_elems, int dtype,
                              uint32_t* found_inf, void* stream);
/* grad[i] += float(grad16[i]); grad16[i] = 0   (world>1 pre-pass, one launch over the flat buffers); sod_grad_merge16 is the
 * same with `flags` (SOD_GRAD16_F16: grad16 is fp16) */
int sod_grad_merge_bf16(float* grad, void* grad16, int64_t n, void* stream);
int sod_grad_merge16(float* grad, void* grad16, int64_t n, int flags, void* stream);
/* *found_inf |= any(!isfinite(grad)) — the amp overflow check (train.py:299), one read of grad */
int sod_grad_nonfinite(const float* grad, int64_t n, uint32_t* found_inf, void* stream);
/* the amp overflow check of the gradients the checked gather does not see: range i is grad16[begin, end) when its flags
 * carry SOD_SEG_GRAD16 (fp16 with SOD_GRAD16_F16 in `flags`, else bf16), grad[begin, end) otherwise.  Ranges need no
 * alignment; any number of them (one launch per SOD_CHECK_MAX_RANGES). */
#define SOD_CHECK_MAX_RANGES 128
typedef struct {
    int64_t begin, end;
    int32_t flags;
} sod_check_range;
int sod_grad_check_ranges(const float* grad, const void* grad16, int64_t n, const sod_check_range* ranges, int nranges,
                          int flags, uint32_t* found_inf, void* stream);

/* plain in-place SUM all-reduce of fp32 data at arena offset `off` (BASELINE config 5 sweep; also the
 * scalar loss mean of utils/tensor_ops.py:60-64 with scale = 1/W).  algo: 0 auto, 1 one-shot, 2 two-shot */
int sod_allreduce_f32(const sod_comm* comm, uint64_t off, int64_t n, float scale, int algo, int flags,
                      void* stream);

/* ------------------------------------------------------------------------------------------------
 * (2) SyncBatchNorm, statistics exchange fused with normalize/affine (+ optional pre-add, residual, ReLU).
 * Replaces: apex convert_syncbn_model/SyncBatchNorm forward+backward (train.py:180) — local Welford +
 *           2 all_gathers + elementwise forward; reduce + 2 all_reduces + elementwise backward.
 * Data layout: channels-last matrices [M = N*H*W rows, C channels] (dtype ∈ bf16/f16/f32; C a power-of-two
 * multiple of 8, C ≤ 2048), fp32 gamma/beta/running stats/saved stats.
 *   z = x (+ pre_add);  mean/var over M*world rows;  y = relu?((z-mean)*invstd*gamma + beta (+ residual))
 * conv_bias1/2 (per-channel, dtype conv_bias_dtype, may be NULL): biases of the convolution(s) producing x / pre_add,
 *   folded in here — z = x (+ pre_add) + b1 + b2 — so that the bias-less convolution output needs no separate
 *   bias-add pass; the backward adds Σ_rows dz (the bias gradient, LOCAL like dgamma/dbeta) into dconv_bias1/2.
 * training=0: uses running stats, no exchange.  comm may be NULL (world 1).
 * stats_off: arena offset of the exchange slot for this call (sod_syncbn_exchange_bytes(C) bytes; the host
 * rotates ≥2 slots); seq/epoch: the packet tag — it must be unique among all syncbn calls (forward AND
 * backward) that share a workspace / slot and identical on all ranks for the same call.  epoch == NULL: tag =
 * seq (31 bits; one global host call counter does it).  epoch != NULL (CUDA-graph replay): tag =
 * 2^31 | (*epoch << 10) | (seq & 1023), with seq the call index inside the captured iteration and *epoch a
 * device counter the captured iteration increments once.
 * workspace: sod_syncbn_workspace_bytes(rows, C) bytes, zero-filled once, then owned by the library.
 * ------------------------------------------------------------------------------------------------ */
size_t sod_syncbn_workspace_bytes(int64_t rows, int channels);
size_t sod_syncbn_exchange_bytes(int channels);
int sod_syncbn_fwd(const void* x, const void* pre_add, const void* residual, void* y, int dtype,
                   const float* gamma, const float* beta, float* running_mean, float* running_var,
                   float* save_mean, float* save_invstd, int64_t rows, int channels, float momentum,
                   float eps, int relu, int training, const sod_comm* comm, uint64_t stats_off, uint32_t seq,
                   const uint32_t* epoch, int64_t* num_batches_tracked /* += 1 when training; may be NULL */,
                   const void* conv_bias1, const void* conv_bias2, int conv_bias_dtype, void* workspace,
                   size_t workspace_bytes, int flags, void* stream);
/* dz = d/d(x) = d/d(pre_add); dres = relu-masked dy (written only if non-NULL; may alias nothing);
 * dgamma/dbeta: LOCAL sums (the gradient all-reduce averages them with every other parameter).
 * y: the forward's output, read for the ReLU mask (may be NULL when relu == 0 or with SOD_BN_BWD_MASK_FROM_X);
 * beta: read only with SOD_BN_BWD_MASK_FROM_X (may be NULL otherwise). */
int sod_syncbn_bwd(const void* dy, const void* x, const void* pre_add, const void* y, void* dz, void* dres,
                   int dtype, const float* gamma, const float* beta, const float* save_mean,
                   const float* save_invstd, float* dgamma, float* dbeta, int64_t rows, int channels, int relu,
                   const sod_comm* comm, uint64_t stats_off, uint32_t seq, const uint32_t* epoch, const void* conv_bias1,
                   const void* conv_bias2, void* dconv_bias1, void* dconv_bias2, int conv_bias_dtype, void* workspace,
                   size_t workspace_bytes, int flags, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Resampling ops on either side of the SyncBN kernels (SURVEY §8f.1), channels-last [N,H,W,C], C % 8 == 0.
 * sod_upsample2x_bilinear_*: bilinear ×2, align_corners=False — `cus_sample` / `upsample_add`
 *   (utils/tensor_ops.py:12-25; call sites network/TestModel.py:100-126, module/MyLightModule.py:42-52);
 *   `add` (may be NULL) is the tensor `upsample_add` sums with, already at the output size.  (h, w) = INPUT size.
 *   The backward is a gather (no atomics): deterministic.
 * sod_avgpool2x2_*: AvgPool2d((2,2), stride=2) — `h2l_pool` (module/MyLightModule.py:14); (h_out, w_out) = OUTPUT size.
 * ------------------------------------------------------------------------------------------------ */
int sod_upsample2x_bilinear_fwd(const void* x, const void* add, void* y, int n, int h, int w, int c, int dtype, void* stream);
int sod_upsample2x_bilinear_bwd(const void* dy, void* dx, int n, int h, int w, int c, int dtype, void* stream);
int sod_avgpool2x2_fwd(const void* x, void* y, int n, int h_out, int w_out, int c, int dtype, void* stream);
int sod_avgpool2x2_bwd(const void* dy, void* dx, int n, int h_out, int w_out, int c, int dtype, void* stream);

/* Column sum of a channels-last matrix [rows, c] (c a power-of-two multiple of 8, ≤ 2048) into out[c] (same dtype, fp32
 * accumulation, deterministic): the bias gradient Σ_rows dy of a convolution that does not feed a BatchNorm — the five
 * `trans*` 1x1 convolutions of network/TestModel.py:32-36 — which autograd otherwise computes with a generic reduction.
 * workspace: sod_colsum_workspace_bytes() bytes, zero-filled once, then owned by the library (one stream at a time). */
size_t sod_colsum_workspace_bytes(void);
int sod_colsum(const void* x, void* out, int64_t rows, int c, int dtype, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Weight-standardised GroupNorm ResNet-50 backbone (reference backbone/wsgn/customized_func.py:12-29, resnet.py).
 *
 * sod_groupnorm_fwd / _bwd — y = act(GroupNorm(x) [+ residual]) on a channels-last [n·hw, c] matrix, groups ==
 * SOD_GN_GROUPS, biased variance, fp32 accumulation.  c must be a multiple of groups (else SOD_EINVAL) and a
 * power-of-two multiple of 8, ≤ 2048 (else SOD_EUNSUPPORTED); x, y, dy, dx, dres, residual and the workspace 16-byte
 * aligned, save_stats 8-byte aligned (SOD_EALIGN).  save_stats: [n·groups] (mean, rstd) pairs written by the forward
 * and read by the backward.  The backward reads y for the ReLU mask (relu != 0) and writes dx, dres = masked dy (may be
 * NULL) and dγ, dβ over the whole batch — added into dgamma / dbeta with SOD_BN_ACCUMULATE_PARAM_GRADS, stored
 * otherwise.  Deterministic: per-CTA partials merged in fixed order by the last CTA to arrive (integer tickets).
 * workspace: at least sod_groupnorm_workspace_bytes(n, hw, c, groups) bytes (0 for a shape the kernels refuse),
 * zero-filled once, then owned by the library (one stream at a time).  sod_groupnorm_splits: the CTAs per sample the
 * launch uses on the current device (the geometry of oracle/wsgn_geometry.py).
 *
 * sod_ws_fwd / _bwd — weight standardisation of `filters` filters of k = C·R·S fp32 weights each (dense per filter,
 * any memory order): w_hat = (w − μ) / (σ + eps) with the unbiased σ, written once rounded in `dtype`; the backward
 * takes dw_hat in `dtype` and writes the fp32 dw of that expression (added into dw with
 * SOD_BN_ACCUMULATE_PARAM_GRADS).  One CTA per filter, deterministic.  k must be > 1.
 * ------------------------------------------------------------------------------------------------ */
#define SOD_GN_GROUPS 32
size_t sod_groupnorm_workspace_bytes(int n, int64_t hw, int c, int groups);
int sod_groupnorm_splits(int n, int64_t hw, int c, int groups);
int sod_groupnorm_fwd(const void* x, const void* residual, void* y, int dtype, const float* gamma, const float* beta,
                      float* save_stats, int n, int64_t hw, int c, int groups, float eps, int relu, void* workspace,
                      size_t workspace_bytes, void* stream);
int sod_groupnorm_bwd(const void* dy, const void* x, const void* y, void* dx, void* dres, int dtype, const float* gamma,
                      const float* save_stats, float* dgamma, float* dbeta, int n, int64_t hw, int c, int groups,
                      int relu, void* workspace, size_t workspace_bytes, int flags, void* stream);
int sod_ws_fwd(const float* w, void* w_hat, int dtype, int filters, int k, float eps, void* stream);
int sod_ws_bwd(const float* w, const void* dw_hat, int dtype, float* dw, int filters, int k, float eps, int flags,
               void* stream);

/* ------------------------------------------------------------------------------------------------
 * 32-group 3×3 convolutions of the weight-standardised GroupNorm ResNeXt-50 32×4d backbone (reference
 * backbone/wsgn/resnext.py `conv2`): padding 1, dilation 1, no bias, C_in = C_out = c, groups == SOD_GCONV_GROUPS,
 * c / groups ∈ {4, 8, 16, 32}, stride 1 or 2, any h, w ≥ 1 (else SOD_EUNSUPPORTED; c not a multiple of groups, a bad
 * dtype or a non-positive size is SOD_EINVAL).  Activations channels-last [n, h, w, c] / [n, ho, wo, c] with
 * ho = (h − 1) / stride + 1 (likewise wo) in `dtype`; (h, w) is the size of x in every entry.  w_hat is
 * [c][3][3][c / groups] in `dtype` (a channels-last weight's memory order); the weight gradient dw_hat is fp32 in the
 * same order (what sod_ws_bwd reads with dtype SOD_F32).  fp32 accumulation; fp32 activations are computed in fp32
 * (no TF32), 16-bit ones on tensor cores.  Every pointer 16-byte aligned (SOD_EALIGN).
 *
 * sod_gconv3x3_fwd: y from x.  sod_gconv3x3_dgrad: dx from dy (the transposed convolution).
 * sod_gconv3x3_wgrad: dw_hat from x and dy, stored (not accumulated).  The pixels are split into
 * sod_gconv3x3_wgrad_splits(...) fixed chunks (oracle/gconv_geometry.py; a function of the shape only), whose fp32
 * partials go to the workspace — at least sod_gconv3x3_wgrad_workspace_bytes(...) bytes, 0 for a refused shape — and
 * are added in chunk order by a second launch.  Deterministic; no refusal launches anything.
 * ------------------------------------------------------------------------------------------------ */
#define SOD_GCONV_GROUPS 32
int sod_gconv3x3_fwd(const void* x, const void* w_hat, void* y, int dtype, int n, int h, int w, int c, int groups,
                     int stride, void* stream);
int sod_gconv3x3_dgrad(const void* dy, const void* w_hat, void* dx, int dtype, int n, int h, int w, int c, int groups,
                       int stride, void* stream);
int sod_gconv3x3_wgrad_splits(int n, int h, int w, int c, int groups, int stride);
size_t sod_gconv3x3_wgrad_workspace_bytes(int n, int h, int w, int c, int groups, int stride);
int sod_gconv3x3_wgrad(const void* x, const void* dy, float* dw_hat, int dtype, int n, int h, int w, int c, int groups,
                       int stride, void* workspace, size_t workspace_bytes, void* stream);

/* MaxPool2d(kernel 3, stride 2, padding 1) of the ResNet stem (backbone/origin/resnet.py `maxpool`; `div_4` in
 * backbone/origin/from_origin.py:7-15), channels-last [N,H,W,C], C % 8 == 0; (h, w) = INPUT size, output
 * ((h-1)/2+1, (w-1)/2+1).  argmax: one byte per OUTPUT element (window position kh*3+kw), written by the forward and
 * read by the backward, which is a deterministic gather with fp32 accumulation.  Ties / NaN as torch: first maximum
 * in (kh, kw) scan order, NaN propagates.  (Checked against torch by the GPU tests and enabled by default.) */
int sod_maxpool3x3s2_fwd(const void* x, void* y, void* argmax, int n, int h, int w, int c, int dtype, void* stream);
int sod_maxpool3x3s2_bwd(const void* dy, const void* argmax, void* dx, int n, int h, int w, int c, int dtype, void* stream);

/* MaxPool2d(kernel 2, stride 2) of VGG16-BN (backbone/origin/vgg.py `make_layers` "M"; the first op of `div_4` … `div_32`
 * in backbone/origin/from_origin.py:18-25), channels-last [N,H,W,C], fp32 / bf16 / fp16; (h, w) = INPUT size, output
 * (h/2, w/2) (floor mode).  argmax: one byte per OUTPUT element (window position kh*2+kw, or 4 for a window with
 * nothing above -inf other than the first, where torch's index points outside the window).  Ties / NaN as torch: first
 * maximum in (kh, kw) scan order, NaN propagates.  The backward writes every dx element: dy at the window position the
 * byte names, 0 elsewhere and on the row / column floor mode drops (bit-identical to torch's).  h < 2, w < 2 or
 * C % 8 != 0 → SOD_EUNSUPPORTED, a pointer not 16-byte aligned → SOD_EALIGN; a refused call writes nothing. */
int sod_maxpool2x2s2_fwd(const void* x, void* y, void* argmax, int n, int h, int w, int c, int dtype, void* stream);
int sod_maxpool2x2s2_bwd(const void* dy, const void* argmax, void* dx, int n, int h, int w, int c, int dtype, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Data-side neighbours of the iteration (SURVEY §8f.2, §8f.4).
 *
 * sod_preprocess_batch — the per-sample tensor transforms and the multi-scale collate of the reference's loader as one
 * kernel over a uint8 batch: ToTensor + Normalize (utils/dataset.py:86-96), mask ToTensor (:110-116), optional
 * left-right flip (utils/joint_transforms.py:19-23; flip_u8[i] != 0 mirrors sample i), and the collate's
 * F.interpolate(img, bilinear, align_corners=False) / F.interpolate(mask, nearest) to (ho, wo)
 * (utils/dataset.py:125-132).  img_u8 [n,hs,ws,3] HWC, mask_u8 [n,hs,ws] (may be NULL together with out_mask),
 * out_img: storage [n,ho,wo,3] = a channels-last [n,3,ho,wo] tensor of out_dtype, out_mask fp32 [n,1,ho,wo].
 *
 * sod_saliency_* — sufficient statistics of the reference's evaluation metrics (utils/saliency_metric.py:8-239 as
 * driven by train.py:383-412): quantize = ToPILImage's mul(255).byte() (optionally after a sigmoid); head = per image
 * {min_u, max_u, max_gt, 0, n_fg, Σy, Σx, 0} (int64[8]); hist = per image uint32[4 quadrants][2 gt][256 k] joint
 * histogram of k = u - min_u, quadrants split at split_yx[2i], split_yx[2i+1] (rows < y / cols < x first), counters
 * ADDED to (zero them first).  Integer arithmetic only: results are exact and order independent.
 * ------------------------------------------------------------------------------------------------ */
int sod_preprocess_batch(const void* img_u8, const void* mask_u8, const void* flip_u8, void* out_img, int out_dtype,
                         float* out_mask, int n, int hs, int ws, int ho, int wo, const float* mean3,
                         const float* std3, void* stream);
int sod_saliency_quantize(const void* pred, int dtype, void* out_u8, int64_t n, int apply_sigmoid, void* stream);
int sod_saliency_head(const void* pred_u8, const void* gt_u8, int n, int h, int w, int64_t* head, void* stream);
int sod_saliency_hist(const void* pred_u8, const void* gt_u8, int n, int h, int w, const int64_t* head,
                      const int32_t* split_yx, uint32_t* hist, void* stream);

/* The same two metric kernels over a ragged batch: image i of pred_u8 and gt_u8 starts at byte offsets[i] and is
 * hw[2i] × hw[2i+1] (device arrays; every h·w < 2^31).  sod_saliency_head / sod_saliency_hist are the special case of
 * equal sizes. */
int sod_saliency_head_ragged(const void* pred_u8, const void* gt_u8, int n, const int64_t* offsets, const int32_t* hw,
                             int64_t* head, void* stream);
int sod_saliency_hist_ragged(const void* pred_u8, const void* gt_u8, int n, const int64_t* offsets, const int32_t* hw,
                             const int64_t* head, const int32_t* split_yx, uint32_t* hist, void* stream);

/* sod_saliency_wfm — the weighted F-measure's per-image sums (utils/saliency_metric.py:232-303) on the nearest
 * foreground pixels scipy's `distance_transform_edt(gt == 0, return_indices=True)` picks, ties included.  Three
 * launches; `head` is sod_saliency_head's output for the same images (it gives the binarisation and the prediction's
 * min / max).  sums[i] = {ΣEw over the foreground, ΣEw over the background, n_fg, 0} in float64, all 0 for an image
 * without foreground; the host forms Q from them.  The sums are reduced in a fixed order: bit-identical from run to
 * run and whatever else is in the batch.  coef_host: 50 HOST doubles, the reference's 7×7 Gaussian (σ = 5) row-major,
 * then log(0.5)/5.  nearest_yx (may be NULL): int32 [Σ h·w][2], images back to back in batch order, (y, x) of each
 * pixel's nearest foreground pixel, (−1, −1) in an image without foreground.  The ragged form also takes the sizes as a
 * HOST array hw_host (the same values as hw).  workspace: sod_saliency_wfm_workspace_bytes(n, sizes) bytes, 16-byte
 * aligned (for the fixed form, n copies of (h, w)); it returns 0 for invalid or unsupported sizes.  SOD_EWORKSPACE and
 * every other refusal launch nothing; images of 2^31 pixels or more, or wider than 2^21, are SOD_EUNSUPPORTED. */
size_t sod_saliency_wfm_workspace_bytes(int n, const int32_t* hw_host);
int sod_saliency_wfm(const void* pred_u8, const void* gt_u8, int n, int h, int w, const int64_t* head,
                     const double* coef_host, void* workspace, size_t workspace_bytes, double* sums, int32_t* nearest_yx,
                     void* stream);
int sod_saliency_wfm_ragged(const void* pred_u8, const void* gt_u8, int n, const int64_t* offsets, const int32_t* hw,
                            const int32_t* hw_host, const int64_t* head, const double* coef_host, void* workspace,
                            size_t workspace_bytes, double* sums, int32_t* nearest_yx, void* stream);

/* ------------------------------------------------------------------------------------------------
 * sod_resize_u8 — Pillow's `Image.resize((w, h), filter)` for 8-bit images, box = the whole image, reducing_gap=None,
 * bit for bit: the reference's `ToPILImage()(out).resize(gt.size)` (BICUBIC, train.py:392-395) and torchvision
 * `Resize((S, S))` on a PIL image (BILINEAR, utils/dataset.py:97-104).  channels 1 ("L") or 3 ("RGB", HWC).
 * Ragged batch: image i of src starts at byte src_off[i] and is src_hw[2i] × src_hw[2i+1]; it is written at dst_off[i]
 * as dst_hw[2i] × dst_hw[2i+1] (all four arrays on the device).  The workspace holds the per-image coefficient tables
 * and intermediate rows; sod_resize_u8_workspace_bytes takes the same sizes as HOST arrays and returns 0 for invalid
 * arguments.  An image whose part of the workspace does not fit in workspace_bytes is left unwritten.
 * ------------------------------------------------------------------------------------------------ */
#define SOD_RESIZE_BILINEAR 2     /* PIL.Image.Resampling.BILINEAR */
#define SOD_RESIZE_BICUBIC 3      /* PIL.Image.Resampling.BICUBIC */
size_t sod_resize_u8_workspace_bytes(int n, const int32_t* src_hw, const int32_t* dst_hw, int channels, int filter);
int sod_resize_u8(const void* src, const int64_t* src_off, const int32_t* src_hw, void* dst, const int64_t* dst_off,
                  const int32_t* dst_hw, int n, int channels, int filter, void* workspace, size_t workspace_bytes,
                  void* stream);

/* ------------------------------------------------------------------------------------------------
 * sod_augment_u8 — the reference's random training augmentation after JointResize (utils/joint_transforms.py:20-48,
 * utils/dataset.py:86-95), bit for bit, for given per-sample parameters, over n images "RGB" S×S×3 (HWC) and masks
 * "L" S×S, each packed back to back:
 *   RandomHorizontallyFlip → RandomRotate: img.rotate(deg, BILINEAR), mask.rotate(deg, NEAREST), fill 0 →
 *   ColorJitter(0.1, 0.1, 0.1) on the image: brightness / contrast / saturation in ops[] order, each
 *   Image.blend(degenerate, img, factor).
 * `params` is a HOST array of n entries; it is validated and copied into the workspace (no host pointer is kept).
 * rot[] is Pillow's output → input matrix of `Image.rotate(deg)` as its Python code computes it; identity = 1 when
 * deg % 360 == 0 (Pillow copies).  ops[] is a permutation of {0: brightness, 1: contrast, 2: saturation}.
 * Two launches over images × row tiles.  Returns SOD_EINVAL on null pointers, n <= 0, S <= 0, a workspace smaller than
 * sod_augment_u8_workspace_bytes(n), or ops[] that is not a permutation.  src and dst must not overlap.
 * ------------------------------------------------------------------------------------------------ */
typedef struct sod_augment_param {
    double rot[6];
    int32_t flip;        /* mirror left-right before the rotation */
    int32_t identity;
    int32_t ops[3];
    float factor[3];     /* brightness, contrast, saturation (indexed by op id) */
} sod_augment_param;
size_t sod_augment_u8_workspace_bytes(int n);
int sod_augment_u8(const void* img, const void* mask, void* img_out, void* mask_out, int n, int size,
                   const sod_augment_param* params, void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SOD_B200_H */
