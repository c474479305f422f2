/*
 * shifu_b200.h - C ABI of the H100-native tabular-DNN train/score hot path.
 *
 * This is the drop-in boundary (SURVEY.md section 8b, seam B3).  The reference has no
 * native boundary of its own for this path: its arithmetic is reached through
 *   - Python  tf.Session.run          shifu-tensorflow-on-yarn/src/main/resources/ssgd_monitor.py:276,281
 *   - Java    TF-Java JNI (libtensorflow_jni 1.4.0)
 *                                     shifu-tensorflow-eval/src/main/java/ml/shifu/shifu/tensorflow/TensorflowModel.java:63-88,169
 * Every entry point below names the reference call it stands in for.  A JNI shim
 * (java/, csrc/jni_shim.c) and a ctypes binding (shifu-tensorflow_b200/_capi.py) sit on top of
 * exactly these symbols; see INTEGRATION.md.
 *
 * Conventions
 *   - every function returns 0 on success, a negative sb_status on failure;
 *     sb_last_error() returns a thread-local message for the last failure on this thread.
 *   - the caller owns all host buffers; the library owns all device memory.
 *   - one handle = one CUDA device.  Handles are not thread-safe except sb_model_score*,
 *     which is re-entrant (the reference scorer is called from many threads,
 *     TensorflowModel.java:53 has no lock).
 *   - flat parameter order is layer-major [W_0 (in x out, row-major), b_0, W_1, b_1, ..., W_out, b_out],
 *     i.e. the variables weight_hidden_layer{l}, biases_hidden_layer{l}, weight_shifu_output_0,
 *     biases_shifu_output_0 of ssgd_monitor.py:59,64,99-104,121.
 *   - there is NO CPU fallback: every compute entry point fails with SB_ERR_CUDA when no
 *     sm_90 device is present.
 */
#ifndef SHIFU_B200_H
#define SHIFU_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SB_MAX_HIDDEN 32

typedef enum {
  SB_OK = 0,
  SB_ERR_INVALID = -1,   /* bad argument                                   */
  SB_ERR_CUDA = -2,      /* CUDA / driver / no device                      */
  SB_ERR_NCCL = -3,
  SB_ERR_IO = -4,        /* SavedModel / checkpoint read or write          */
  SB_ERR_STATE = -5,     /* e.g. scoring before load (IllegalStateException in TensorflowModel.java:55-57) */
  SB_ERR_FORMAT = -6     /* unsupported graph / corrupt file               */
} sb_status;

/* get_activation_fun, ssgd_monitor.py:74-88 */
typedef enum { SB_ACT_SIGMOID = 0, SB_ACT_TANH = 1, SB_ACT_RELU = 2, SB_ACT_LEAKYRELU = 3, SB_ACT_NONE = -1 } sb_act;
/* SB_LOSS_MSE = tf.losses.mean_squared_error on the sigmoid output, SUM_BY_NONZERO_WEIGHTS
 * (ssgd_monitor.py:129) - the reference's loss.  SB_LOSS_SIGMOID_CE = BASELINE.json's wording. */
typedef enum { SB_LOSS_MSE = 0, SB_LOSS_SIGMOID_CE = 1 } sb_loss;
/* ADADELTA: ssgd_monitor.py:138; ADAM: ssgd.py:57; SGD: ssgd_monitor_bk.py:81; MOMENTUM: north star.
 * ADAGRAD, RMSPROP, FTRL: the other TF 1.x optimizers in their training_ops.cc kernel forms (ApplyAdagrad; ApplyRMSProp,
 * not centered; ApplyFtrl with lr_power = -0.5 and no l2 shrinkage).  Every update is element-wise in fp32 with correctly
 * rounded square roots and divisions.  Optimizer state (s1 / s2) per parameter and its start value, written when the
 * trainer is created (sb_trainer_set_params and sb_trainer_init_xavier leave the state as it is, for every optimizer):
 *   ADADELTA  accum = 0, accum_update = 0     ADAM     m = 0, v = 0         SGD   -
 *   MOMENTUM  accum = 0                       ADAGRAD  accum = initial_accumulator
 *   RMSPROP   ms = 1 (TF's ones initializer), mom = 0                     FTRL  accum = initial_accumulator, linear = 0
 *   RPROP     prev = 0, step = learning_rate
 * FTRL sets a parameter to exactly 0 while |linear| <= l1 (also with l1 = 0 and linear = 0, e.g. a zero gradient from
 * the start), as TF does.
 * RPROP: resilient propagation in its iRPROP- form (Igel and Huesken), for full-batch gradients such as the
 * sync_replicas schedule's one update per epoch.  It uses only the sign of each gradient and computes exactly what
 * torch.optim.Rprop(lr, etas=(0.5, 1.2), step_sizes=(1e-6, 50)) computes, in fp32:
 *   p = g prev;  step = min(max(step * (p > 0 ? 1.2 : p < 0 ? 0.5 : 1), 1e-6), 50)
 *   g = p < 0 ? 0 : g;  theta -= sign(g) step  (g = +-0: theta keeps its bits);  prev = g
 * learning_rate is only the start value of step; the value 7 is not an optimizer. */
typedef enum { SB_OPT_ADADELTA = 0, SB_OPT_ADAM = 1, SB_OPT_SGD = 2, SB_OPT_MOMENTUM = 3, SB_OPT_ADAGRAD = 4,
               SB_OPT_RMSPROP = 5, SB_OPT_FTRL = 6, SB_OPT_RPROP = 8 } sb_optimizer;
/* SB_PREC_FP32: fp32 operands and fp32 accumulation end to end (what TF-CPU computes) - parity mode (CUDA cores).
 * SB_PREC_BF16: bf16 operands on the tensor cores (wgmma), fp32 accumulation, fp32 master
 *               weights and optimizer state - performance mode.
 * SB_PREC_FP32_TC: fp32-class accuracy ON the tensor cores: every fp32 operand value is split into three bf16 parts
 *               (v = p0 + p1 + p2, exact to ~2^-24), the six part products with i + j < 3 accumulate in fp32.  Same
 *               kernels as SB_PREC_BF16 over a six times longer K axis; meets the fp32 tolerances (loss / gradients
 *               1e-4, scores 1e-5).  Parity mode that is not a CUDA-core program.
 * SB_PREC_BF16X2: two parts, three products (~2^-17 relative per product): half the cost of FP32_TC. */
typedef enum { SB_PREC_FP32 = 0, SB_PREC_BF16 = 1, SB_PREC_FP32_TC = 2, SB_PREC_BF16X2 = 3 } sb_precision;

typedef struct {
  int32_t n_features;              /* FEATURE_COUNT = len(SELECTED_COLUMN_NUMS), ssgd_monitor.py:43-44 */
  int32_t n_hidden;                /* train.params.NumHiddenLayers, ssgd_monitor.py:93                 */
  int32_t hidden[SB_MAX_HIDDEN];   /* train.params.NumHiddenNodes,  ssgd_monitor.py:94                 */
  int32_t acts[SB_MAX_HIDDEN];     /* train.params.ActivationFunc,  ssgd_monitor.py:95 (sb_act)        */
  int32_t loss;                    /* sb_loss                                                          */
  int32_t optimizer;               /* sb_optimizer                                                     */
  float learning_rate;             /* train.params.LearningRate, ssgd_monitor.py:133                   */
  float rho;                       /* Adadelta rho (TF default 0.95); RMSProp decay (TF default 0.9)   */
  float epsilon;                   /* Adadelta / Adam epsilon (TF default 1e-8); RMSProp (1e-10)       */
  float beta1, beta2;              /* Adam (TF defaults 0.9 / 0.999)                                   */
  float momentum;                  /* Momentum; RMSProp momentum (TF default 0.0)                      */
  int32_t max_batch;               /* largest mini-batch (rows) a step will be given                   */
  int32_t precision;               /* sb_precision                                                     */
} sb_net_desc;
/* Optimizer fields each optimizer reads (the others are ignored, whatever they hold):
 *   ADADELTA rho, epsilon    ADAM beta1, beta2, epsilon    SGD -    MOMENTUM momentum    RPROP -
 *   RMSPROP  rho (decay, in [0, 1]), momentum (>= 0), epsilon (>= 0); a value out of range is SB_ERR_INVALID, found
 *            before any device work
 *   ADAGRAD  initial_accumulator, FTRL initial_accumulator, l1, l2: sb_trainer_set_optimizer_params (TF's defaults
 *            0.1, 0, 0 until it is called).  The descriptor's layout is unchanged, so callers built against it keep working. */

typedef struct sb_trainer sb_trainer_t;
typedef struct sb_model sb_model_t;

/* ---- library ---- */
const char* sb_version(void);
const char* sb_last_error(void);
/* number of visible CUDA devices with compute capability 10.x; <0 on error */
int sb_device_count(void);
/* free and total device memory of `device` (cudaMemGetInfo), e.g. to tell beforehand whether a set will fit in HBM */
int sb_device_mem_info(int device, uint64_t* free_bytes, uint64_t* total_bytes);
/* pinned host memory for callers that want true async H2D (JNI direct buffers) */
int sb_host_alloc(void** ptr, uint64_t bytes);
int sb_host_free(void* ptr);

/* ---- data-parallel rendezvous: replaces tf.train.Server/ClusterSpec (ssgd_monitor.py:152-166).
 * Rank 0 calls sb_nccl_unique_id and ships the 128 bytes to the other ranks by any means. ---- */
#define SB_NCCL_ID_BYTES 128
int sb_nccl_unique_id(void* out128);

/* ---- trainer: replaces model()+MonitoredTrainingSession of the worker branch
 * (ssgd_monitor.py:110-144, 251-257).  nccl_id may be NULL when world == 1. ---- */
int sb_trainer_create(const sb_net_desc* desc, int device, const void* nccl_id, int rank, int world,
                      sb_trainer_t** out);
/* (world > 1 with nccl_id == NULL: replicas driven by ONE process; they must be connected with
 * sb_trainer_set_peer_pointers before the first step, there is no NCCL fallback then.) */
int sb_trainer_destroy(sb_trainer_t* t);
/* Optional faster gradient exchange for ranks on one NVLink/NVSwitch node: a two-shot all-reduce kernel over CUDA-IPC
 * peer memory instead of NCCL.  Every rank exports its exchange buffer (64-byte cudaIpcMemHandle_t), the host
 * all-gathers the handles in rank order and hands the table to every rank.  Must be called on all ranks before the
 * next step; without it the exchange is ncclAllReduce. */
#define SB_IPC_HANDLE_BYTES 64
int sb_trainer_ipc_handle(sb_trainer_t* t, void* out64);
int sb_trainer_set_peer_handles(sb_trainer_t* t, const void* handles /* world x 64 bytes */, int32_t n_handles);
/* back to NCCL: unmap the peers (call on every rank when any rank failed to map, so that no rank runs the peer kernels) */
int sb_trainer_clear_peer_handles(sb_trainer_t* t);
/* The same peer table for trainers that live in ONE process (one host thread driving several GPUs, or several replicas
 * on one GPU in the tests): instead of IPC handles, pass every rank's exchange allocation (sb_trainer_exchange_base) as a
 * plain device pointer, in rank order; peer access between the devices is enabled here.  bases[own rank] is ignored. */
void* sb_trainer_exchange_base(sb_trainer_t* t);
int sb_trainer_set_peer_pointers(sb_trainer_t* t, void* const* bases, int32_t n);
int64_t sb_trainer_param_count(const sb_trainer_t* t);
/* variable init / restore (tf.initialize_all_variables + Saver.restore, ssgd_monitor.py:238,327) */
int sb_trainer_set_params(sb_trainer_t* t, const float* flat, int64_t n);
int sb_trainer_get_params(sb_trainer_t* t, float* flat, int64_t n);
/* xavier-uniform init on weights and biases (ssgd_monitor.py:59-68), seeded */
int sb_trainer_init_xavier(sb_trainer_t* t, uint64_t seed);
/* parity hook: the (all-reduced, mean over ranks) gradient the last step applied */
int sb_trainer_get_grads(sb_trainer_t* t, float* flat, int64_t n);
/* Deterministic training (on = 1; default 0): every reduction over CTAs of a training step is added in a fixed order,
 * so two runs with the same build, GPU model and SM count, descriptor, inputs, seed, world size and sequence of calls
 * give bit-identical parameters, optimizer state, gradients, losses and checkpoint / SavedModel files.  Call it right
 * after sb_trainer_create: SB_ERR_STATE after the first step or graph capture, after the peer exchange was set up, on a
 * wide+deep trainer (sb_trainer_set_sparse is refused on a deterministic one).  All four precisions.  A
 * deterministic trainer with world > 1 needs a peer table (sb_trainer_set_peer_handles / _pointers): without one its
 * first step returns SB_ERR_STATE (NCCL's all-reduce fixes no summation order). */
int sb_trainer_set_deterministic(sb_trainer_t* t, int32_t on);
/* Adagrad / FTRL hyperparameters the descriptor has no field for: accum's start value initial_accumulator (> 0; TF default
 * 0.1) and FTRL's l1 / l2 regularization strengths (>= 0; TF defaults 0).  Writes initial_accumulator into the state at
 * once (a device fill).  Call it right after sb_trainer_create: SB_ERR_STATE after the first step or graph capture,
 * SB_ERR_INVALID for an optimizer that reads none of them or a value out of range (both before any device work). */
int sb_trainer_set_optimizer_params(sb_trainer_t* t, float initial_accumulator, float l1, float l2);
/* Fine-tuning with frozen layers (ModelConfig train.params FixedLayers / FixedBias).  Layers are numbered from 1: hidden
 * layers 1..n_hidden, the output layer n_hidden + 1.  The weights of every listed layer, and its bias when fix_bias != 0,
 * are fixed: a step never changes their values, their optimizer state or their bf16 shadows (bit for bit, whatever the
 * optimizer - Adam, Momentum, RMSProp and FTRL would move a parameter with a zero gradient), sb_trainer_get_grads reports
 * 0 for them, and the peer exchange neither moves nor updates them.  A step skips the dW GEMM of every frozen weight
 * matrix and the dA GEMMs that nothing at or below them needs; every parameter that trains gets the gradient it gets
 * without frozen layers.  layers == NULL with n == 0 freezes nothing (the default).  SB_ERR_INVALID, before any device
 * work: a layer outside [1, n_hidden + 1], a layer listed twice, or every parameter fixed.  SB_ERR_STATE after the first
 * step or graph capture, or after the peer exchange was set up.  Every rank must fix the same parameters:
 * sb_trainer_set_peer_handles / _pointers refuse a peer that does not (SB_ERR_INVALID), so call this on every rank
 * before the exchange handles are shared. */
int sb_trainer_set_fixed_layers(sb_trainer_t* t, const int32_t* layers, int32_t n, int32_t fix_bias);

/* one sess.run([train_step, loss, global_step], feed_dict) (ssgd_monitor.py:272-276) in the
 * "clean" schedule: forward, loss, backward, gradient mean over ranks, one optimizer update.
 * X [rows, n_features] fp32 row-major, y [rows] (labels 0/1 as float), w [rows] sample weights
 * (NULL = all 1.0), all HOST memory.  loss_out (nullable) receives this rank's mini-batch loss. */
int sb_trainer_step(sb_trainer_t* t, const float* X, const float* y, const float* w, int32_t rows,
                    float* loss_out);

/* Wide+deep (BASELINE.json configs[3]; the reference only plumbs the numeric / categorical column lists,
 * TensorflowTaskExecutor.java:213-223, and has no sparse model - spec in oracle/wide_deep.py): the first hidden layer's
 * n_features = n_dense + n_onehot inputs are n_dense numeric columns followed by the one-hot expansion of n_cat categorical
 * columns.  A sparse step feeds the dense block Xd [rows, n_dense] and idx [rows, n_cat] (global one-hot column of each
 * categorical value, -1 = missing) and evaluates the one-hot block as an embedding gather (forward) / scatter-add
 * (gradient) - the SAME parameters, loss and update as sb_trainer_step on the materialised one-hot matrix. */
int sb_trainer_set_sparse(sb_trainer_t* t, int32_t n_dense, int32_t n_onehot, int32_t n_cat);
int sb_trainer_step_sparse(sb_trainer_t* t, const float* Xd, const int32_t* idx, const float* y, const float* w,
                           int32_t rows, float* loss_out);
int sb_trainer_predict_sparse(sb_trainer_t* t, const float* Xd, const int32_t* idx, int64_t rows, float* out);
int sb_trainer_eval_loss_sparse(sb_trainer_t* t, const float* Xd, const int32_t* idx, const float* y, const float* w,
                                int64_t rows, float* loss_out);

/* Same step, pipelined: returns as soon as the work is queued.  The H2D copy of this batch goes through a second
 * staging slot on a copy stream and overlaps the previous step's compute; the loss of the most recent step is read
 * with sb_trainer_last_loss (which waits).  X / y / w must be pinned (sb_host_alloc or equivalent) for the copy to be
 * truly asynchronous and must stay untouched until two further steps have been queued or sb_trainer_sync returned. */
int sb_trainer_step_async(sb_trainer_t* t, const float* X, const float* y, const float* w, int32_t rows);

/* Reference epoch-sync schedule (SyncReplicasOptimizer, ssgd_monitor.py:136-141): accumulate the
 * gradient of one mini-batch without updating; then apply the MEAN of the n accumulated
 * mini-batch gradients (averaged over ranks as well) as ONE optimizer update. */
int sb_trainer_accumulate(sb_trainer_t* t, const float* X, const float* y, const float* w, int32_t rows,
                          float* loss_out);
int sb_trainer_apply_accumulated(sb_trainer_t* t);     /* queued on the trainer's stream; sb_trainer_sync / get_params wait */
/* Same, with the divisor given explicitly: the update uses (sum over ranks of the locally accumulated gradients) /
 * total_pushes.  This is ConditionalAccumulator.take_grad(R) when ranks accepted different numbers of pushes (stale pushes
 * are dropped per worker, ssgd_monitor.py:136-141; the host-side token bookkeeping lives in trainer.py). */
int sb_trainer_apply_accumulated_mean(sb_trainer_t* t, int64_t total_pushes);

/* HBM-resident training set: load_data + np.array_split (ssgd_monitor.py:186-192) keep the whole
 * set in RAM and slice mini-batches from it; here the set lives in HBM and each step reads its
 * rows [row_offset, row_offset+rows) from there.  Calling load again replaces the set.
 * Placement: X goes to HBM when it fits in the free device memory beside a reserve (16 bytes per row for y, w, the n_nz
 * prefix counts and a row order, the conversion windows, and as much again as the trainer's step buffers).  A set that
 * does not fit is kept in mapped pinned host memory in the same layout (tensor-core modes: the bf16 parts, bit for bit
 * what HBM would hold; fp32 mode: the fp32 rows); y, w and the prefix counts stay in HBM.  Steps over a host set read
 * their batch's rows over PCIe first (tensor-core modes: gather_batch_kernel into the step's batch buffer; fp32 mode:
 * the host-batch load kernel), and compute exactly what they compute over the same set in HBM.  If the pinned
 * allocation fails the call returns SB_ERR_CUDA with the byte count it asked for, and no set is loaded. */
int sb_trainer_load_dataset(sb_trainer_t* t, const float* X, const float* y, const float* w, int64_t n_rows);
/* 1 when the loaded set's X lives in pinned host memory, 0 when it is in HBM or no set is loaded */
int sb_trainer_dataset_on_host(const sb_trainer_t* t);
/* (X / y / w of sb_trainer_load_dataset, sb_trainer_eval_loss and sb_trainer_predict may be HOST or DEVICE pointers on the
 * trainer's device: sb_text_parse_device hands the parsed set over without a host round trip.) */
int sb_trainer_step_resident(sb_trainer_t* t, int64_t row_offset, int32_t rows, float* loss_out);
/* same, but does not wait for the GPU: the loss of step i is readable after sb_trainer_sync */
int sb_trainer_step_resident_async(sb_trainer_t* t, int64_t row_offset, int32_t rows);
/* The inner loop of an epoch in one call (`for i in range(total_batch): sess.run(train_step)`, ssgd_monitor.py:268-276):
 * n_steps consecutive update steps over rows [row_offsets[i], row_offsets[i]+rows) of the resident set, identical to
 * n_steps calls of sb_trainer_step_resident_async.  Does not wait for the GPU; steps are replayed four per captured
 * graph, so the turn-around between two graphs is paid once per four steps. */
int sb_trainer_run_resident(sb_trainer_t* t, const int64_t* row_offsets, int32_t n_steps, int32_t rows);
int sb_trainer_accumulate_resident(sb_trainer_t* t, int64_t row_offset, int32_t rows, float* loss_out);
/* forward + loss only over resident rows, no gradient, no update: what a sess.run whose push the accumulator drops as stale
 * still reports (its loss), ssgd_monitor.py:276 */
int sb_trainer_loss_resident(sb_trainer_t* t, int64_t row_offset, int32_t rows, float* loss_out);
/* Read the resident set through a row order: after this call, the resident entry points (step_resident[_async],
 * run_resident, accumulate_resident, loss_resident) address logical row r as row rows[r] of the set loaded by
 * sb_trainer_load_dataset, and check their offsets against n instead of the set's length.  Any list of in-range rows
 * (1 <= n < 2^31; repeats allowed), HOST memory; it is copied (4 bytes per row on the device), and checked on the host
 * before any device work (SB_ERR_INVALID).  rows == NULL with n == 0 goes back to the physical order.  SB_ERR_STATE
 * without a resident set.  Loading a new set drops the order.  Waits for the queued steps; captured step graphs are
 * reused.  eval_loss, predict, host-batch and sparse steps are unaffected.  An ordered step gathers its batch into the
 * step's batch buffer first (gather_batch_kernel) - every epoch can draw new mini-batches without a second copy of the
 * set. */
int sb_trainer_set_row_order(sb_trainer_t* t, const int64_t* rows, int64_t n);
int sb_trainer_last_loss(sb_trainer_t* t, float* loss_out);
/* the loss curve: mini-batch loss of update steps first_step .. first_step + n - 1 (1-based global_step values; the last
 * 8192 steps are kept).  Every step's tail kernel posts its (loss sum, n_nz) into pinned host memory, so asynchronous
 * calls (sb_trainer_run_resident / _step_async) lose no per-step loss (`loss` fetched by every sess.run, ssgd_monitor.py:276).
 * Waits for the queued work. */
int sb_trainer_loss_history(sb_trainer_t* t, int64_t first_step, int32_t n, float* out);
int sb_trainer_sync(sb_trainer_t* t);
/* Make every replica identical to rank `root`: parameters, optimizer state and the step counter (ncclBroadcast on the
 * trainer's communicator).  The reference keeps ONE copy of the variables on the parameter servers, initialised or restored
 * by the chief only (ssgd_monitor.py:203-206, 251-257); replicas get the same effect by calling this on all ranks after
 * init / restore on the root.  No-op when world == 1. */
int sb_trainer_broadcast_state(sb_trainer_t* t, int32_t root);
/* cudaStream_t the trainer launches on (for CUDA-event timing by the caller) */
void* sb_trainer_stream(sb_trainer_t* t);
/* number of this library's kernels launched by one step at this batch size (bench.py's gpu_launches) */
int sb_trainer_kernels_per_step(sb_trainer_t* t, int32_t rows);

/* validation pass: sess.run([loss, global_step]) on the valid set (ssgd_monitor.py:281-284);
 * forward + loss only, any number of rows (processed in max_batch chunks with the reduction of
 * ONE big batch: sum w*(..)^2 over all rows / count of non-zero weights over all rows). */
int sb_trainer_eval_loss(sb_trainer_t* t, const float* X, const float* y, const float* w, int64_t rows,
                         float* loss_out);
/* forward only: sigmoid outputs for rows (host) */
int sb_trainer_predict(sb_trainer_t* t, const float* X, int64_t rows, float* out);

/* checkpoint / resume (MonitoredTrainingSession(checkpoint_dir=...), ssgd_monitor.py:251-257):
 * params + optimizer state + step counter as one flat blob. */
int sb_trainer_save_checkpoint(sb_trainer_t* t, const char* path);
int sb_trainer_load_checkpoint(sb_trainer_t* t, const char* path);
int64_t sb_trainer_global_step(const sb_trainer_t* t);

/* simple_save + export_generic_config (ssgd_monitor.py:457-490): SavedModel dir (saved_model.pb with
 * tag "serve", signature "serving_default" shifu_input_0 -> shifu_output_0, variables/ tensor bundle)
 * plus GenericModelConfig.json. */
int sb_trainer_export_savedmodel(sb_trainer_t* t, const char* export_dir);

/* ---- scorer: replaces TensorflowModel.init / compute (TensorflowModel.java:112-172, 53-94) ---- */
/* SavedModelBundle.load(modelPath, tags) + feed/fetch by op name */
int sb_model_load(const char* saved_model_dir, const char* input_name, const char* output_name,
                  const char* tag, int device, int precision, sb_model_t** out);
/* build directly from a topology + flat parameters (no file) */
int sb_model_create(const sb_net_desc* desc, const float* flat_params, int64_t n, int device, sb_model_t** out);
int sb_model_destroy(sb_model_t* m);
int32_t sb_model_n_features(const sb_model_t* m);
int32_t sb_model_n_layers(const sb_model_t* m);
/* batched compute(): X [rows, n_features] fp32 host -> out [rows] fp32 host */
int sb_model_score(sb_model_t* m, const float* X, int64_t rows, float* out);
/* compute(MLData): one row of doubles -> double (double->float cast at TensorflowModel.java:64-68).
 * Concurrent calls on one handle share device batches of up to 128 rows; a lone call is scored at once.  A row's
 * score is the same whichever rows share its batch. */
int sb_model_score_row_f64(sb_model_t* m, const double* row, int32_t n, double* out);
/* device-resident scoring (X, out are DEVICE pointers on the model's device), asynchronous on the
 * model's stream; sb_model_sync waits. */
int sb_model_score_device(sb_model_t* m, const float* dX, int64_t rows, float* dOut);
/* Column sensitivity (varsel filterBy SE / ST, per-row reason codes).  With s(x) the score sb_model_score computes in
 * the model's precision mode, for row r and list position k:
 *   d[r,k] = s(x_r) - s(x_r with column cols[k] set to values[k])
 *   sum_sq[k] = sum_r w_r d^2,  sum[k] = sum_r w_r d,  *w_sum = sum_r w_r.
 * cols == NULL && n_cols == 0: every column in order; otherwise n_cols >= 1 columns in [0, n_features), in any order,
 * repeats allowed; outputs follow list positions.  values: NULL (every value 0, the mean of a ZSCALE-normalised column)
 * or one finite value per list position.  w: NULL weighs every row 1.  deltas: nullable, row-major [rows, n_cols].
 * X, w and deltas may be host or device pointers on the model's device; sum_sq, sum (n_cols each) and w_sum are host
 * memory.  Synchronous; takes the model's device lock, so it is safe beside compute() callers on the same handle.
 * Guarantees:
 *   - same bits on repeat: every output is bit-identical across calls with the same inputs, and the sums do not depend
 *     on whether deltas was requested or on whether X / w are host or device pointers;
 *   - zero when nothing changes: d is exactly +0 wherever x[r, cols[k]] == values[k] (the base score each delta is
 *     taken against comes out of the same launches as the perturbed scores);
 *   - fixed-order sums: accumulated in fp64, over rows in a fixed tree per row chunk and over row chunks in order.
 * Layer 0's pre-activation z0 is computed once per row; each (row, column) pair is the rank-1 update
 * z0 + (v - x_c) W0[c, :] followed by layers 1..L.  The scores are s within the model's precision (not bit-identical to
 * sb_model_score's: z0 is kept in fp32 and updated before the activation).  Rows go in chunks of
 * R = clamp(max_batch / (n_cols + 1), 64, max_batch / 2) rows; a chunk's list positions in pieces of up to
 * max_batch / R - 1 columns, each one forward of R (columns + 1) pair rows.
 * Errors, all reported before any device work: a null model SB_ERR_STATE; null X / sum_sq / sum / w_sum, rows < 0, a bad
 * cols / n_cols pair, a column out of range or a non-finite value SB_ERR_INVALID.  rows = 0 returns zeros. */
int sb_model_sensitivity(sb_model_t* m, const float* X, const float* w, int64_t rows, const int32_t* cols, int32_t n_cols,
                         const float* values, double* sum_sq, double* sum, double* w_sum, float* deltas);
/* Per-row reason codes: for each row, the k list positions whose deltas rank first, computed on the GPU without
 * materialising the [rows, n_cols] deltas.  d[r,j] is sb_model_sensitivity's delta, with the same cols / n_cols / values
 * rules.  Ranking order (total, so the result is unique): the key is d for SB_REASON_RAISE (the values that push the
 * score up the most), -d for SB_REASON_LOWER and |d| for SB_REASON_MAGNITUDE; a larger key ranks first; keys compare as
 * floats (-0 == +0); a NaN key ranks after every other key; equal keys rank by the smaller list position.
 * Outputs, row-major: pos [rows, k] int32, the list positions best first; d [rows, k] their deltas; scores (nullable)
 * [rows] the base score s(x_r) the deltas are taken against.  That score is computed as this call computes it (z0 kept
 * in fp32), so it is not bit-identical to sb_model_score's.
 * Every returned d[r,i] is bit-identical to deltas[r, pos[r,i]] of sb_model_sensitivity on the same model and inputs:
 * the call runs the same row chunks, pieces and launches up to the pair scores, and merges each piece's deltas into a
 * running top k per row on the device.
 * X, pos, d and scores may be host or device pointers on the model's device.  Synchronous; takes the model's device
 * lock, so it is safe beside compute() callers on the same handle.  rows = 0 returns SB_OK and writes nothing.
 * Errors, all reported before any device work: a null model SB_ERR_STATE; null X / pos / d, rows < 0, a bad cols / n_cols
 * pair, a column out of range, a non-finite value, k < 1, k > min(n_cols, 32) or an unknown order SB_ERR_INVALID. */
enum { SB_REASON_RAISE = 0, SB_REASON_LOWER = 1, SB_REASON_MAGNITUDE = 2 };
int sb_model_reason_codes(sb_model_t* m, const float* X, int64_t rows, const int32_t* cols, int32_t n_cols, const float* values,
                          int32_t k, int32_t order, int32_t* pos, float* d, float* scores);
int sb_model_sync(sb_model_t* m);
void* sb_model_stream(sb_model_t* m);
/* Test hooks of the scorer.  stats[SB_DEBUG_MSTAT_WORDS] since creation = {compute() batches run, rows they scored,
 * the largest batch, batches run by the one-launch fp32 kernel, batches run by the captured tensor-core graph,
 * one-launch fp32 forwards of any entry point}. */
#define SB_DEBUG_MSTAT_WORDS 6
enum { SB_DEBUG_MSTAT_BATCHES = 0, SB_DEBUG_MSTAT_ROWS = 1, SB_DEBUG_MSTAT_MAX_FILL = 2, SB_DEBUG_MSTAT_SMALL = 3,
       SB_DEBUG_MSTAT_GRAPH = 4, SB_DEBUG_MSTAT_SMALL_LAUNCHES = 5 };
int sb_debug_model_batch_stats(sb_model_t* m, int64_t* stats, int32_t n_stats);
/* The next compute() batch waits until k rows are queued or timeout_ms have passed (k = 0: no wait). */
int sb_debug_model_hold(sb_model_t* m, int32_t k, int32_t timeout_ms);
/* The kernels the model's last forward launched, "+"-joined into out (cap bytes, truncated to fit): "score_rows" for
 * an fp32 batch of up to 128 rows, otherwise the batch load, one GEMM per hidden layer and the output layer, e.g.
 * "load_batch<bf16>+gemm_wide+gemm_wide+gemm_pp<FWD>+out_layer_rows<1>"; "none" before the first forward.  Every
 * scoring entry point runs its rows in forwards of at most max_batch rows (16384 in fp32, 65536 in bf16, 32768 in the
 * split modes), so after a call this names the launches of its last piece.  After sb_model_sensitivity: the launches
 * of its last row chunk's z0 and last piece, e.g.
 * "load_batch<bf16>+gemm_tc<128,F32>+sens_perturb<bf16>+gemm_pp<FWD>+gemm_pp<FWD>+out_layer_rows<1>+sens_reduce".
 * After sb_model_reason_codes: the same, ending in "sens_topk" instead of "sens_reduce". */
int sb_debug_model_routes(sb_model_t* m, char* out, int32_t cap);
/* the device bytes the model allocated for its network, workspace and staging (a test hook) */
int sb_debug_model_bytes(sb_model_t* m, int64_t* out);

/* ---- bagged models: Shifu trains train.baggingNum models per run (models/model0 .. model{K-1}) and `shifu eval` scores
 * every one of them per row and reports their mean, max, min and median beside the members' scores.  An ensemble is K
 * member models on one device and one stream that share one staged copy of the rows: each chunk of rows is copied in and
 * converted to the GEMM operand (load_batch_kernel) once, and every member's forward reads it.
 * Members must share n_features and precision; their hidden widths, depths and activations may differ.  Each member
 * scores each chunk with its own launches at its own max_batch, the one sb_model_score uses at that precision, and the
 * ensemble chunks rows at that size, so member g's scores are bit-identical to what an sb_model_t of the same member
 * computes from the same rows through sb_model_score / sb_model_score_device.
 * The statistics, per row, over the K member scores s_0 .. s_{K-1}:
 *   mean    ((s_0 + s_1) + ...) + s_{K-1} summed in fp32 in member order, then divided by (float)K
 *   max     the largest value (of equal values, the first in member order); min likewise
 *   median  with the values sorted (equal values in member order): K odd the middle value; K even (a + b) / 2 in fp32 of
 *           the two middle values a <= b.  The reference scorer's sources are not part of this project, so this even-K
 *           convention is defined here, not taken from Shifu.
 *   If any member's score is NaN, all four statistics are the quiet NaN 0x7fc00000.
 * Errors, all found before any device work: k < 1 or k > SB_ENSEMBLE_MAX, a null argument, members whose n_features
 * differ, descriptors whose precision differs, a parameter count that does not fit its descriptor, both outputs null,
 * rows < 0, or a row length != n_features in sb_ensemble_score_row_f64 are SB_ERR_INVALID; a null handle SB_ERR_STATE;
 * sb_ensemble_load reports a member's load errors exactly as sb_model_load does.  rows = 0 returns SB_OK and writes
 * nothing. ---- */
#define SB_ENSEMBLE_MAX 32
typedef struct sb_ensemble sb_ensemble_t;
/* K SavedModel directories, each loaded as sb_model_load loads one (SavedModelBundle.load per models/model<g>), every
 * member at `precision` */
int sb_ensemble_load(const char* const* dirs, int32_t k, const char* input_name, const char* output_name, const char* tag,
                     int device, int precision, sb_ensemble_t** out);
/* K topologies + flat parameter vectors, each as sb_model_create takes one */
int sb_ensemble_create(const sb_net_desc* descs, const float* const* flats, const int64_t* n_params, int32_t k, int device,
                       sb_ensemble_t** out);
int sb_ensemble_destroy(sb_ensemble_t* e);
int32_t sb_ensemble_size(const sb_ensemble_t* e);
/* K compute() calls per row plus the statistics: X [rows, n_features] fp32, host or device; scores [rows, k] (member
 * order) and stats [rows, 4] = {mean, max, min, median}, host or device; either output may be NULL, not both.
 * Synchronous, like sb_model_score. */
int sb_ensemble_score(sb_ensemble_t* e, const float* X, int64_t rows, float* scores, float* stats);
/* the same with DEVICE pointers, asynchronous on the ensemble's stream, like sb_model_score_device; sb_ensemble_sync waits */
int sb_ensemble_score_device(sb_ensemble_t* e, const float* dX, int64_t rows, float* dScores, float* dStats);
/* compute(MLData) of every member: one row of doubles -> out[k + 4] doubles (the k member scores, then mean, max, min,
 * median).  Concurrent calls on one handle share device batches of up to 128 rows, as sb_model_score_row_f64's do; a
 * lone call is scored at once. */
int sb_ensemble_score_row_f64(sb_ensemble_t* e, const double* row, int32_t n, double* out);
int sb_ensemble_sync(sb_ensemble_t* e);
void* sb_ensemble_stream(sb_ensemble_t* e);
/* Test hooks.  routes: the launches of the ensemble's last chunk, "+"-joined, e.g. for two bf16 members
 * "load_batch<bf16>+gemm_wide+gemm_pp<FWD>+out_layer_rows<1>+gemm_pp<FWD>+out_layer_rows<1>+ensemble_stats", for an
 * fp32 chunk of up to 128 rows "score_rows+score_rows+ensemble_stats"; "none" before the first.  bytes: the device bytes
 * the ensemble allocated (every member's network and workspace, the one input staging, the member score slots). */
int sb_debug_ensemble_routes(sb_ensemble_t* e, char* out, int32_t cap);
int sb_debug_ensemble_bytes(sb_ensemble_t* e, int64_t* out);
/* Explaining the ensemble's score (DESIGN §6j): column sensitivity and per-row reason codes of one statistic of the
 * members' scores.  With s_g(x) member g's score as sb_model_sensitivity computes it for that member alone (z0 in fp32,
 * the rank-1 update, layers 1..L) and S(x) the statistic `stat` of s_0 .. s_{K-1} under exactly the rules above (fp32
 * mean in member order, first-wins max / min, the even-K median (a + b) * 0.5f, a NaN giving the quiet NaN):
 *   d[r,k] = S(x_r) - S(x_r with column cols[k] set to values[k]).
 * Every other rule is sb_model_sensitivity's / sb_model_reason_codes': cols / n_cols / values, w, the sums, deltas, k,
 * order, the outputs and where they may live, and their guarantees (the same bits on repeat; sums that do not depend on
 * deltas or on the pointer kinds; d exactly +0 wherever x[r, cols[k]] == values[k]; fp64 sums added in a fixed order;
 * every reason-code d bit-identical to sb_ensemble_sensitivity's delta at its position; scores = S(x_r) as the call
 * computes it).  Rows go in the chunks and pieces sb_model_sensitivity uses at the members' shared max_batch: each row
 * chunk is loaded once and each member computes its own z0; per piece every member runs its perturbation and forward
 * into its score slot, so member g's pair scores are bit-identical to those of an sb_model_t of member g, and one launch
 * forms S of every pair.  A one-member ensemble gives sb_model_sensitivity's bits for every stat.
 * Synchronous; takes the ensemble's device lock, so it is safe beside sb_ensemble_score_row_f64 callers.
 * Errors, all found before any device work: a null handle SB_ERR_STATE; a stat outside 0..3 SB_ERR_INVALID; otherwise
 * as the model functions report them.  The routes after a call: the last row chunk's load and every member's z0 GEMM,
 * then per member in member order its sens_perturb, its layers and its output unit, then "ensemble_stat", then
 * "sens_reduce" or "sens_topk". */
enum { SB_STAT_MEAN = 0, SB_STAT_MAX = 1, SB_STAT_MIN = 2, SB_STAT_MEDIAN = 3 };
int sb_ensemble_sensitivity(sb_ensemble_t* e, int32_t stat, const float* X, const float* w, int64_t rows,
                            const int32_t* cols, int32_t n_cols, const float* values,
                            double* sum_sq, double* sum, double* w_sum, float* deltas);
int sb_ensemble_reason_codes(sb_ensemble_t* e, int32_t stat, const float* X, int64_t rows, const int32_t* cols,
                             int32_t n_cols, const float* values, int32_t k, int32_t order,
                             int32_t* pos, float* d, float* scores);

/* ---- model performance: what `shifu eval` reports about a scored set (ROC AUC, PR AUC, KS, and the gains / ROC / PR /
 * score-bucket lists), computed on the GPU from one radix sort of the scores.  Shifu's evaluator is not part of this
 * project, so the quantities are defined here.
 * Rows.  Each added row has a score s (fp32), a target y and a weight w.  y must be exactly 0 or 1 (-0 counts as 0); w must
 * be finite and >= 0, and is 1 for every row when the caller passes no weights.  A row whose s is NaN, whose y is any other
 * value, or whose w is negative, NaN or +-inf is invalid.  +-inf scores are valid; -0 and +0 are the same score.
 * Thresholds.  t_1 > t_2 > ... > t_m are the distinct scores; run j is the set of rows with s = t_j.  p_j, n_j count its
 * positives and negatives, wp_j, wn_j are their weight sums in fp64.  TP_j = sum_{i<=j} p_i, and likewise FP_j, WTP_j and
 * WFP_j: the rows flagged at threshold t_j (s >= t_j).  P, N, Wp and Wn are the totals.  Every row counts once in the
 * unweighted metrics, rows with w = 0 included.
 * Metrics (sb_perf_summary):
 *   auc    A2 / (2 P N), A2 = sum_j n_j (2 TP_{j-1} + p_j): the Mann-Whitney statistic with ties counted half.  A2 and
 *          2 P N are exact int64 values and the result is one fp64 division of their fp64 values; up to 1.34e8 rows both
 *          are below 2^53, so auc is the correctly rounded value of the exact fraction.
 *   w_auc  sum_j wn_j (WTP_{j-1} + wp_j / 2) / (Wp Wn) in fp64.
 *   ap     average precision (area under the PR curve): sum_j (p_j / P) TP_j / (TP_j + FP_j); w_ap the same with the
 *          weighted values (a run with wp_j = 0 adds 0).
 *   ks     max_j |TP_j N - FP_j P| / (P N): the numerator is exact in int64 (so is the argmax), and the value is one fp64
 *          division of the two int64 values; ks_score is t_j of the first j (the highest threshold) that attains it.
 *          w_ks / w_ks_score: the same in fp64 with the weighted values and the same tie-break.
 *   A metric whose denominator is 0 is the quiet NaN (a single-class set; a zero weight total for the weighted ones), and
 *   so is its ks_score.  An empty handle's summary has zero counts and NaN metrics.
 * Guarantees: every result depends only on the rows and their arrival order, not on how they were split into adds, on
 * whether the pointers were host or device, or on timing.  The sort is stable and every fp64 sum runs in a fixed order, so
 * results are bit-identical on repeat.  WTP_j and WFP_j never decrease along the table.  At most 2^31 - 1 rows per handle.
 * Memory: the handle holds each row's 32-bit key and payload, their sort double buffer and the run table: at most 53 device
 * bytes per row of capacity (every score distinct), plus 13 MB (12 MB of it the host-row staging, allocated at the first add
 * that reads host memory, and 48 bytes per level of the largest sb_perf_points call).  The capacity is allocated at the first add (or by reserve_rows), grows to
 * max(rows held, 1.5 x capacity) rounded up to 4096 rows, and is freed by sb_perf_destroy.
 * Errors: a null handle is SB_ERR_STATE.  Null scores or y, rows < 0, score_stride < 1, a row total over 2^31 - 1, an unknown
 * axis, a level out of range, a NaN level or n < 0 are SB_ERR_INVALID, reported before any device work.  Invalid rows are
 * counted on the device; while the handle holds any, sb_perf_summary_get, sb_perf_points and sb_debug_perf_runs return
 * SB_ERR_INVALID with the three counts in the message, until sb_perf_reset. ---- */
typedef struct sb_perf sb_perf_t;
/* no device: SB_ERR_CUDA.  reserve_rows (0 .. 2^31 - 1) pre-sizes the row capacity. */
int sb_perf_create(int device, int64_t reserve_rows, sb_perf_t** out);
int sb_perf_destroy(sb_perf_t* p);
/* forget every row (and every invalid-row count), keep the allocations */
int sb_perf_reset(sb_perf_t* p);
/* Append rows: scores[r * score_stride], y[r], w[r] (w NULL: 1).  With score_stride = 4 a caller can pass the mean column
 * of sb_ensemble_score_device's stats; with stride K, member g's scores.  Host or device pointers on p's device.  When all
 * of them are device pointers the call is queued on p's stream, after the work that was queued on after_stream (nullable,
 * e.g. sb_model_stream(m)) at the time of the call, with no host synchronise.  Otherwise it returns once the rows have been
 * read.  rows = 0 adds nothing.  The sort runs when a result is asked for after new rows arrived. */
int sb_perf_add(sb_perf_t* p, const float* scores, int32_t score_stride, const float* y, const float* w, int64_t rows,
                void* after_stream);
typedef struct {
  int64_t rows, pos, neg, n_distinct;   /* rows held, P, N, m */
  double w_pos, w_neg;                  /* Wp, Wn */
  double auc, w_auc, ap, w_ap, ks, w_ks;
  float ks_score, w_ks_score;
} sb_perf_summary;
/* synchronous */
int sb_perf_summary_get(sb_perf_t* p, sb_perf_summary* out);
/* Operating points, one per level (synchronous).  For SB_PERF_ACTION_RATE, SB_PERF_RECALL and SB_PERF_FPR a level l lies in
 * [0, 1]: the point is the first run j (the highest threshold) whose axis value reaches l, the axis values being
 * (TP_j + FP_j) / (P + N), TP_j / P and FP_j / N as fp64 divisions (weighted != 0: (WTP_j + WFP_j) / (Wp + Wn), WTP_j / Wp,
 * WFP_j / Wn); an axis whose denominator is 0 is SB_ERR_INVALID.  These give Shifu's gains, ROC and PR lists.  For
 * SB_PERF_SCORE, l is any non-NaN value: the point is the last run with t_j >= l (the score-bucket list), or, when there is
 * none, the empty point {threshold +inf, all counts 0}.  Each point is {t_j, TP_j, FP_j, WTP_j, WFP_j}. */
enum { SB_PERF_ACTION_RATE = 0, SB_PERF_RECALL = 1, SB_PERF_FPR = 2, SB_PERF_SCORE = 3 };
typedef struct { float threshold; int64_t tp, fp; double w_tp, w_fp; } sb_perf_point;
int sb_perf_points(sb_perf_t* p, int32_t axis, int32_t weighted, const double* levels, int32_t n, sb_perf_point* out);
int sb_perf_sync(sb_perf_t* p);
void* sb_perf_stream(sb_perf_t* p);
/* Test hooks: the first min(cap, m) rows of the run table (t_j and the cumulative TP / FP / WTP / WFP; any output may be
 * NULL) with *n_runs = m, and the device bytes the handle holds. */
int sb_debug_perf_runs(sb_perf_t* p, float* t, int64_t* tp, int64_t* fp, double* wtp, double* wfp, int64_t cap, int64_t* n_runs);
int sb_debug_perf_bytes(sb_perf_t* p, int64_t* out);

/* ---- text ingest: the per-cell float() loop of load_data (ssgd_monitor.py:387-419) on the GPU ----
 * text: the gunzipped, delim-separated lines (must end with '\n'), HOST memory.  col_map[c] gives the role of text
 * column c: >= 0 feature index (into X [rows, n_feat] row-major), SB_COL_TARGET, SB_COL_WEIGHT, SB_COL_SKIP; columns
 * >= n_map are skipped.  y <- float(target cell); w <- weight cell with "negative -> 1.0", 1.0 when the line has no
 * weight column.  Every value is float32(float64(text)) exactly as numpy feeds the reference's fp32 placeholders.
 * Cells the exact fast path declines (> 15-19 significant digits, |exp| > 22, nan/inf, malformed) are NOT written:
 * they are listed in flags[0..min(n_flags, flag_cap)) for the caller to resolve with its own float(); slot -100 marks
 * a line whose number of feature cells / target cell is wrong.  col_map must name every feature index 0 .. n_feat - 1
 * exactly once, the target exactly once and the weight at most once, with no entry outside [SB_COL_WEIGHT, n_feat);
 * any other map is SB_ERR_INVALID before any device work (shared by sb_text_parse_device and the host hook). */
#define SB_COL_SKIP (-1)
#define SB_COL_TARGET (-2)
#define SB_COL_WEIGHT (-3)
typedef struct { int64_t row; int32_t slot; int32_t len; int64_t offset; } sb_cell_flag;
int sb_text_parse(const char* text, int64_t n_bytes, char delim, const int32_t* col_map, int32_t n_map, int32_t n_feat,
                  float* X, float* y, float* w, int64_t max_rows, int64_t* n_rows_out, sb_cell_flag* flags,
                  int64_t flag_cap, int64_t* n_flags_out, int device);
/* The same parse with the result left ON THE DEVICE: *dX [rows, n_feat], *dy, *dw are cudaMalloc'ed by the library (release
 * with sb_device_free) and go straight into sb_trainer_load_dataset / sb_trainer_eval_loss; only the flag list (cells for
 * the caller's float(), patched in with sb_device_patch_f32) and 4 bytes per row (weights, for the n_nz prefix counts) ever
 * reach the host.  kernel_ms_out (nullable): device time of the three parsing kernels (HBM-bound: text read twice for the
 * line index, once for the cells; X written once) - bench.py's `ingest` roofline. */
int sb_text_parse_device(const char* text, int64_t n_bytes, char delim, const int32_t* col_map, int32_t n_map, int32_t n_feat,
                         float** dX, float** dy, float** dw, int64_t* n_rows_out, sb_cell_flag* flags, int64_t flag_cap,
                         int64_t* n_flags_out, int device, float* kernel_ms_out);
int sb_device_alloc_f32(float** out, int64_t n, int device);
int sb_device_free(void* p);
int sb_device_patch_f32(float* d_base, int64_t index, float value);
int sb_device_read_f32(const float* d_src, int64_t n, float* host_out);
/* d_dst[i, :] = d_src[rows_host[i], :] - the train / valid split of the parsed set (the Bernoulli coins of
 * ssgd_monitor.py:396 are drawn on the host from the caller's RNG; only the row indices travel) */
int sb_device_gather_rows(const float* d_src, int32_t n_cols, const int64_t* rows_host, int64_t n, float* d_dst, int device);

/* test hook: the same parsing state machine run on the host (CPU unit tests of the number parser; not a product path) */
int sb_debug_text_parse_host(const char* text, int64_t n_bytes, char delim, const int32_t* col_map, int32_t n_map,
                             int32_t n_feat, float* X, float* y, float* w, int64_t max_rows, int64_t* n_rows_out,
                             sb_cell_flag* flags, int64_t flag_cap, int64_t* n_flags_out);

/* ---- file-format helpers used by the host mirrors and tests ---- */
/* write a SavedModel for an arbitrary MLP (host only, no GPU needed) */
int sb_savedmodel_write(const char* export_dir, const sb_net_desc* desc, const float* flat_params, int64_t n);
/* parse a SavedModel into topology + flat parameters (host only).  flat may be NULL to query n_params. */
int sb_savedmodel_read(const char* saved_model_dir, const char* input_name, const char* output_name,
                       const char* tag, sb_net_desc* desc_out, int32_t* out_act, float* flat, int64_t flat_cap,
                       int64_t* n_params);

/* ---- kernel-level test hooks (parity tests of single kernels through the C ABI) ---- */
/* D[M,N] = A * B^T on the wgmma path: A, B are fp32 host arrays that are rounded to bf16 on the device; D fp32 host.
 * split_k >= 1.  Operand layouts: a_mn = 0: A is [M,K] (K-major), 1: A is [K,M] (MN-major); b_mn likewise for
 * B ([N,K] or [K,N]).  Instantiated combinations: (0,0) dA GEMM, (0,1) forward GEMM, (1,1) dW GEMM.
 * cfg_cg = 1 forces a 128 x cfg_bn tile (cfg_bn 64|128, or 256 for (1,1)); cfg_cg = 0 lets the planner choose.  Any
 * other cfg_cg is SB_ERR_INVALID. */
int sb_debug_gemm_bf16_cfg(const float* A, const float* B, float* D, int32_t M, int32_t N, int32_t K,
                           int32_t split_k, int32_t a_mn, int32_t b_mn, int32_t cfg_cg, int32_t cfg_bn, int device);

/* One forward (kind 0), dA (kind 1) or dW (kind 2) GEMM of a training step at `precision` (sb_precision), launched by the
 * step's own per-layer launch code on a network built so that the GEMM is one of its layers: the step's planning, tensor
 * maps, part pairs and kernel instantiations.  All matrices are fp32 row-major on the host; the tensor-core modes store
 * them as np bf16 parts (np = 1 BF16, 2 BF16X2, 3 FP32_TC) split as the step splits them.  out receives [np, M, N]: each
 * part's bf16 widened to fp32 (FP32: the fp32 values, one part).
 *   kind 0: out = the parts of act(A[row0 .. row0 + M - 1] W + addend + bias).  A [a_rows, K], W [K, N], bias [N].
 *           a_rows > M or row0 > 0: the batch is read at a row offset, as a step on the HBM-resident set reads it (tensor-
 *           core modes).  addend [M, N] (nullable): a wide+deep step, whose layer 0 adds the embedding sums.
 *           clear_n4 > 0 (tensor-core modes): the GEMM's idle producer warps clear a buffer of clear_n4 float4, as on a
 *           resident step.
 *   kind 1: out = the parts of (A W^T) * act'(aux), colsum[N] += its column sums.  A = dZ_l [M, K], W = W_l [N, K],
 *           aux = A_{l-1} [M, N] (stored as np parts).
 *   kind 2: grad[M, N] += A^T dZ over the K batch rows, rows r0 .. r1 - 1 only (an exchange chunk; r0 a multiple of 8,
 *           FP32: the whole matrix).  A [a_rows, M] with the batch at row0 (resident as for kind 0), dZ passed in W [K, N].
 * sms: the grid cap (the SMs a dW GEMM may take, or the Net's SM count for the forward and dA plans; a small value puts
 * several tiles on each CTA); 0 = every SM.  route (nullable, route_cap bytes) receives the kernel and tile launched, e.g.
 * "gemm_tc<128,DW>", "gemm_dw", "gemm_tc<64,FWD,GENERIC>", "gemm_pp<DA>", "gemm_wide", "gemm_f32<DA>".
 * Before the launch the 64 rows past M of every output part and its pad columns N .. round_up(N, 8) - 1, the gradient
 * outside its in/out region (kind 1: the column sums; kind 2: rows r0 .. r1 - 1) and 256 floats behind it, and the cleared
 * buffer with 256 floats behind it are filled with a sentinel.  *guard returns how many of these changed, and how many
 * floats of the cleared range are not +0, except that a pad column of a batch row may hold what the kernels store beyond N:
 * kind 0 the parts of act(0) (the tile is 0 there), kind 1 +-0.  Every argument is checked before any device work; a bad
 * one is SB_ERR_INVALID. */
int sb_debug_gemm_layer(int32_t kind, int32_t precision, const float* A, const float* W, const float* bias, const float* aux,
                        const float* addend, float* out, float* colsum, float* grad, int32_t* guard, char* route,
                        int32_t route_cap, int32_t M, int32_t N, int32_t K, int32_t a_rows, int32_t row0, int32_t act,
                        int32_t r0, int32_t r1, int32_t sms, int64_t clear_n4, int device);

/* Timeline of the last step (trainer created with SB_STEP_TRACE=1 in the environment): for each GEMM launch of the
 * step, 16 %globaltimer stamps (ns) of its CTA 0: [0] entry, [1] setup done, [2] dependencies resolved, [3] first TMA
 * issued, [4] first stage landed, [5] MMAs of the first tile issued, [6] first accumulator complete, [7] first
 * epilogue done, [8] exit.  names = comma-separated kernel roles.  Measurement aid; no reference counterpart. */
int sb_debug_step_trace(sb_trainer_t* t, uint64_t* stamps, int32_t cap_kernels, char* names, int32_t names_cap, int32_t* n_kernels);
/* micro-benchmark of one tile configuration: average device milliseconds per launch over `iters` back-to-back launches
 * (CUDA events on the launching stream, operands L2-warm) */
int sb_debug_gemm_bench(const float* A, const float* B, float* D, int32_t M, int32_t N, int32_t K, int32_t split_k,
                        int32_t a_mn, int32_t b_mn, int32_t cfg_cg, int32_t cfg_bn, int device, int32_t iters,
                        float* ms_out);

/* One plain-bf16 forward (da = 0) or dA (da = 1) GEMM of a training step through the kernel the step plans for it, with
 * its fused epilogue.  Operands are fp32 on the host, rounded to bf16 on the device:
 *   forward: out = bf16(act(A W + bias))               A [M,K], W [K,N], bias [N]
 *   dA     : out = bf16((A W^T) * act'(aux)),          A [M,K], W [N,K], aux [M,N] (an activation output);
 *            colsum[N] = column sums of the fp32 product before rounding (nullable)
 * out [M,N] receives the bf16 results widened to fp32.  bm_wg = 0 lets the planner choose the tile, 64 or 128 forces
 * the rows of a ping-pong warpgroup tile, 256 the forward GEMM's 128 x 256 tile (invalid for dA).  iters > 0: afterwards, average device milliseconds per launch over `iters` back-to-back
 * launches into *ms_out. */
int sb_debug_gemm_epilogue(const float* A, const float* W, const float* bias, const float* aux, float* out, float* colsum,
                           int32_t M, int32_t N, int32_t K, int32_t da, int32_t act, int32_t bm_wg, int device,
                           int32_t iters, float* ms_out);

/* The last hidden layer of a training step with the output layer fused into its GEMM (gemm_fwd_out_kernel, N <= 256),
 * launched the way the step launches it:
 *   a = act(A W + bias) (fp32),  z = a . wo + bo,  y_hat = sigmoid(z),  loss term and dz (SUM_BY_NONZERO_WEIGHTS),
 *   dZ = dz * wo * act'(a) as np bf16 parts,  db_L += sum_r dZ,  dw_o += sum_r dz a,  db_o += sum_r dz,
 *   loss_sum += sum_r loss term.
 * A [a_rows, K] fp32; the batch is rows row0 .. row0 + M - 1, read at a row offset as a step reads the HBM-resident set.
 * W [K, N], bias [N], wo [N] fp32.  A and W are split into np bf16 parts on the device (np = 1: plain bf16).
 * y, w [M]; n_nz is the count of non-zero w.  g_bL [N], g_wo [N], g_bo [1] and loss_sum [1] are in/out: the kernel
 * adds into the values passed in.  dZ [np, M, N] receives each part's bf16 widened to fp32.  Before the launch every
 * part's pad columns N .. round_up(N, 8) - 1 and 64 rows past M are filled with a sentinel; *guard returns how many of
 * them changed, except that a pad column of a batch row may hold +-0 (the tile is 0 beyond N and the bulk tensor store
 * writes a row's last 16-byte piece whole).  grid = 0: the step's grid (one CTA per 64-row tile, at most one per SM);
 * 1 .. SMs: that many CTAs, each running several tiles.  No PDL, no trace. */
int sb_debug_gemm_fwd_out(const float* A, const float* W, const float* bias, const float* wo, float bo, const float* y,
                          const float* w, float* dZ, float* g_bL, float* g_wo, float* g_bo, float* loss_sum, int32_t* guard,
                          int32_t M, int32_t N, int32_t K, int32_t a_rows, int32_t row0, int32_t act, int32_t loss,
                          int32_t np, int32_t grid, int device);

/* The output layer of a step at `precision` (sb_precision) on its own (out_layer_rows_kernel / out_layer_kernel), launched
 * by the step's own launch code on a network whose last hidden layer (width H, activation act) holds A_L:
 *   z = A_L . wo + bo,  y_hat = sigmoid(z),  loss term and dz (SUM_BY_NONZERO_WEIGHTS, n_nz = the count of non-zero w),
 *   dZ = dz * wo * act'(A_L),  db_L += sum_r dZ,  dw_o += sum_r dz A_L,  db_o += sum_r dz,  loss_sum += sum_r loss term.
 * A [M, H] fp32 host, stored as the step stores A_L: np bf16 parts split as the step splits them (np = 1 BF16, 2 BF16X2,
 * 3 FP32_TC) or fp32.  wo [H]; y, w [M] (do_loss = 1).  (do_loss, do_bwd) = (1, 1): a training step; (1, 0): an
 * evaluation (y_hat and the loss); (0, 0): a score (y_hat only; y and w may be null).  yhat [M] (nullable unless
 * do_loss = 0) receives y_hat; dZ [np, M, H] each part's bf16 widened to fp32 (FP32: one part); g_bL [H], g_wo [H], g_bo
 * and loss_sum are in/out: the kernel adds into the values passed in.  det = 1: the deterministic instantiation,
 * launched twice on the same network from the same initial values; the results are the second launch's and
 * *repeat_same (nullable) is 1 if every output bit, guards included, equals the first launch's (-1 for det = 0).
 * sms: the SM count the launch code plans for (0 = every SM).  route (nullable, route_cap bytes) receives the kernel
 * instantiation launched, e.g. "out_layer_rows<2,DET>", "out_layer<bf16>", "out_layer<float>".
 * Before the launch, A_L's pad columns and the 64 rows past M of every part hold NaN, and so do y and w past M (all of
 * them for a score) and n_nz for a score.  The 64 rows past M of dZ and y_hat, dZ's pad columns, the flat gradient
 * outside the g_bL / g_wo / g_bo slots (all of it unless do_bwd) and 256 floats behind it, and the step-scalar words
 * other than the loss sum (and that one too unless do_loss) are filled with a sentinel or the input value; *guard returns
 * how many of them changed, except that a pad column of a batch row may hold +-0 on a backward (the 16-byte pieces of
 * dZ reach into it).  On a score or an evaluation dZ must stay the sentinel too.  Every argument is checked before any
 * device work (do_bwd needs do_loss; M, H >= 1; sms up to the device's SM count); a bad one is SB_ERR_INVALID. */
int sb_debug_out_layer(int32_t precision, int32_t det, int32_t do_loss, int32_t do_bwd, const float* A, const float* wo, float bo,
                       const float* y, const float* w, float* yhat, float* dZ, float* g_bL, float* g_wo, float* g_bo,
                       float* loss_sum, int32_t* guard, int32_t* repeat_same, char* route, int32_t route_cap, int32_t M, int32_t H,
                       int32_t act, int32_t loss, int32_t sms, int device);

/* The wide+deep first layer's embedding kernels (embed_gather_kernel, embed_scatter_kernel), launched by the step's own
 * launch code on a network with 3 dense columns and n_onehot one-hot columns of n_cat categorical columns, hidden [H].
 * W_e [n_onehot, H] fp32 is put into the parameters and stored as the step stores it (np bf16 shadow parts, or fp32);
 * idx [rows, n_cat] holds one-hot columns in [0, n_onehot) or -1 (missing), checked as the sparse entry points check it.
 *   scatter = 0: out [rows, H] = E, E[r] = sum over c with idx[r, c] >= 0 of W_e[idx[r, c]] (every part).
 *   scatter = 1: out [n_onehot, H] is in/out, W_e's rows of the flat gradient: row j gains the sum over every (r, c) with
 *                idx[r, c] = j of dZ_0[r], where dZ [rows, H] fp32 is stored as the step stores dZ_0 (np parts or fp32).
 *                We may be null.
 * W_e's dense neighbours, b_0 and the output layer hold NaN, and so do dZ_0's pad columns and 64 rows past the batch.
 * Before the launch E's pad columns and its 64 rows past the batch (gather), or the flat gradient outside W_e's rows and
 * 256 floats behind it (scatter-add), are filled with a sentinel; *guard returns how many of them changed.  Every argument
 * is checked before any device work; a bad one is SB_ERR_INVALID. */
int sb_debug_embed(int32_t precision, int32_t scatter, const float* We, const int32_t* idx, const float* dZ, float* out,
                   int32_t* guard, int32_t rows, int32_t H, int32_t n_onehot, int32_t n_cat, int device);

/* ---- test hooks of the peer-memory gradient exchange (csrc/xchg_p2p.cuh), on a trainer with a peer table ---- */
/* Read (write = 0) or write (1) one raw buffer of this rank's parameter arena, after waiting for the trainer's stream:
 * which = SB_DEBUG_BUF_THETA / _S1 / _S2 / _GRAD: float[n_params] (no gather from the run owners: a non-owner's stale
 * master and state stay visible); SB_DEBUG_BUF_SHADOW + l: the bf16 shadow of hidden layer l as uint16 bits
 * [np, in, ld_out], pad columns out .. ld_out - 1 included (tensor-core modes only, else SB_ERR_STATE).  Writing theta
 * leaves the shadows alone; write = 2 (theta only) also refreshes them.  A wrong length is SB_ERR_INVALID.
 * The step's input stage (sb_debug_first_kernel), on any trainer:
 *   SB_DEBUG_BUF_BATCH_X: layer 0's batch operand.  Tensor-core modes: Xb as uint16 bits [np, max_batch, ldx] with
 *     ldx = round_up(F, 8), or round_up(n_dense, 8) once sb_trainer_set_sparse was called; fp32 mode: Xf [max_batch, F].
 *   SB_DEBUG_BUF_BATCH_Y / _W: float[max_batch], the labels / weights a step's descriptor points at: ordY / ordW of
 *     ordered steps while a row order is set or the bf16 set is in host memory, else the host staging buffers (a host step without w reads ones instead).
 *   SB_DEBUG_BUF_SCAL: float[4], the step scalars of descriptor slot (0, 0) (loss sum, n_nz, 2 unused).
 *   SB_DEBUG_BUF_DS_X: the resident set: uint16 bits [np, ds_rows, round_up(F, 8)] (tensor-core modes) or float
 *     [ds_rows, F] (fp32 mode); _DS_Y / _DS_W: float[ds_rows]; _DS_P: int32[ds_rows + 1], the prefix counts of the
 *     non-zero weights (tensor-core modes only, else SB_ERR_STATE).  Read-only; without a loaded set SB_ERR_STATE.
 * A bad id, a write to a read-only id and a bad write mode are SB_ERR_INVALID before the trainer is looked at. */
#define SB_DEBUG_BUF_THETA 0
#define SB_DEBUG_BUF_S1 1
#define SB_DEBUG_BUF_S2 2
#define SB_DEBUG_BUF_GRAD 3
#define SB_DEBUG_BUF_SHADOW 4
#define SB_DEBUG_BUF_BATCH_X (SB_DEBUG_BUF_SHADOW + SB_MAX_HIDDEN)
#define SB_DEBUG_BUF_BATCH_Y (SB_DEBUG_BUF_BATCH_X + 1)
#define SB_DEBUG_BUF_BATCH_W (SB_DEBUG_BUF_BATCH_X + 2)
#define SB_DEBUG_BUF_SCAL (SB_DEBUG_BUF_BATCH_X + 3)
#define SB_DEBUG_BUF_DS_X (SB_DEBUG_BUF_BATCH_X + 4)
#define SB_DEBUG_BUF_DS_Y (SB_DEBUG_BUF_BATCH_X + 5)
#define SB_DEBUG_BUF_DS_W (SB_DEBUG_BUF_BATCH_X + 6)
#define SB_DEBUG_BUF_DS_P (SB_DEBUG_BUF_BATCH_X + 7)
int sb_debug_trainer_buffer(sb_trainer_t* t, int32_t which, void* host, int64_t n, int32_t write);
/* Queue what a step queues before layer 0, and wait for it: the batch's descriptor into slot (0, 0), then the step's first
 * kernel (enqueue_first), which clears the gradient buffer [0, n_params) when clear = 1.
 *   X != NULL: host rows, staged as sb_trainer_step stages them (X [rows, F], y, w nullable), or on a sparse trainer as
 *              sb_trainer_step_sparse does (X = the dense block [rows, n_dense], idx [rows, n_cat]);
 *   X == NULL: rows [row_offset, row_offset + rows) of the resident set, as a resident step reads them (through the row
 *              order if one is set); y, w and idx must be NULL.
 * route (route_cap bytes) receives the kernels launched, "+"-joined: "load_batch<bf16>", "load_batch<fp32>",
 * "gather_batch<bf16>", "gather_batch<fp32>" (a sparse step's load is followed by "+embed_gather"), or "none" for a
 * bf16-resident batch, whose descriptor write publishes n_nz and layer 0 reads the set in place.  Changes neither the step count nor any captured step.  Read the results with sb_debug_trainer_buffer. */
int sb_debug_first_kernel(sb_trainer_t* t, const float* X, const float* y, const float* w, const int32_t* idx, int64_t row_offset,
                          int32_t rows, int32_t clear, char* route, int32_t route_cap);
/* on = 1: the next sb_trainer_load_dataset places the set in pinned host memory whatever its size (0: by size, the
 * default), so that the host-memory path can be compared with the same set in HBM.  A test hook, not an option. */
int sb_debug_force_host_set(sb_trainer_t* t, int32_t on);
/* Queue one exchange of the slots in slot_mask exactly as a step does, and return without waiting: the descriptor of
 * the next update (global step + 1 and its lr_t, gradient scale `gscale` (0: 1 / world), epoch + 1), then the step's
 * exchange launch on the trainer's stream - its slot and work tables, grid rule (alone: as the last launch of a step)
 * and kernel choice.  grid > 0 replaces the grid rule.  Every rank of the peer table must queue the same exchange before
 * any of them is waited for (sb_trainer_sync, which also reports a peer that never arrived).  *lr_t_out, *grid_out
 * (nullable) receive the lr_t and grid used, route (route_cap bytes) the kernel launched, e.g. "xchg_ll<4>",
 * "xchg_update<16>".  A mask outside the trainer's slots is SB_ERR_INVALID, no peer table SB_ERR_STATE; both are found
 * before any device work. */
int sb_debug_exchange(sb_trainer_t* t, int32_t slot_mask, float gscale, int32_t grid, int32_t alone, float* lr_t_out,
                      int32_t* grid_out, char* route, int32_t route_cap);
/* The exchange's ownership tables.  info[SB_DEBUG_XINFO_WORDS] = {slots, SMs, LL protocol, replicas share the device,
 * rank, world, np, 0, slot_begin[8], slot_end[8]}.  work (nullable: query *n_work) receives SB_DEBUG_XWORK_WORDS int64
 * per run of the optimizer's work table: {off, count, out_dim, mat_off, ld_out, np, hidden layer whose shadow the run
 * refreshes or -1, part_stride}.  The runs of slot s are [slot_begin[s], slot_end[s]). */
#define SB_DEBUG_XINFO_WORDS 24
#define SB_DEBUG_XWORK_WORDS 8
int sb_debug_exchange_layout(sb_trainer_t* t, int32_t* info, int32_t info_cap, int64_t* work, int64_t work_cap, int32_t* n_work);
/* Test hook of the single-GPU optimizer (csrc/kernels.cuh optimizer_kernel), on a world-1 trainer.  Queue one update
 * without waiting: the descriptor of the next update (global step + 1 and its lr_t, gradient scale `gscale` (0: 1 / world),
 * epoch + 1), then the optimizer over the raw gradient buffer - tail = 0: one launch over the whole work table, as
 * sb_trainer_apply_accumulated and a step without the split tail queue it; tail = 1: the step's split tail (layer 0's
 * runs on the main stream, the others on the side stream, then the join).  *lr_t_out (nullable) receives lr_t, route
 * (route_cap bytes) the launches, "+"-joined, each as "optimizer<base|ext|rprop>@<main|side>[first run,end run)".  A bad
 * gscale or tail, or tail = 1 with one hidden layer, is SB_ERR_INVALID; world > 1 is SB_ERR_STATE; both are found before
 * any device work. */
int sb_debug_optimizer(sb_trainer_t* t, float gscale, int32_t tail, float* lr_t_out, char* route, int32_t route_cap);

#ifdef __cplusplus
}
#endif
#endif /* SHIFU_B200_H */
