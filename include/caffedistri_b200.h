/*
 * caffedistri_b200.h -- C ABI of libcaffedistri_b200.so
 *
 * H100-native replacement for the inter-executor gradient-sync hot path of
 * yahoo/CaffeOnSpark's libcaffedistri.so (CaffeNet<float> behind the
 * com.yahoo.ml.jcaffe.CaffeNet JNI class).  Plain pointers and sizes only; no
 * C++/torch types.  Every entry point names the reference interface it
 * replaces (paths relative to the reference repo root):
 *   J  = caffe-distri/src/main/java/com/yahoo/ml/jcaffe/CaffeNet.java
 *   JN = caffe-distri/src/main/cpp/jni/JniCaffeNet.cpp
 *   CN = caffe-distri/src/main/cpp/CaffeNet.cpp
 *   CH = caffe-distri/include/CaffeNet.hpp
 *
 * Conventions (mirroring JN): functions that return `int` status return 1 for
 * true/success and 0 for false/failure unless stated otherwise; integer
 * getters return -1 on failure (JN:235-249,479-580); the message behind a
 * failure is available from cos_last_error() (thread-local), which is what the
 * JNI shim turns into a java.lang.Exception (src/main/cpp/common.cpp:111-116).
 * The handle is the value the reference stores in BaseObject.address (a long).
 *
 * There is NO CPU fallback: every compute entry point fails (0 / -1 with an
 * error string) when no CUDA device is usable.
 */
#ifndef CAFFEDISTRI_B200_H_
#define CAFFEDISTRI_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define COS_API __attribute__((visibility("default")))

/* J:21-23 connection types.  RDMA and SOCKET both select the NVLink peer-memory
 * transport here (there is no socket or verbs data path in this library). */
#define COS_CONNECTION_NONE 0
#define COS_CONNECTION_RDMA 1
#define COS_CONNECTION_SOCKET 2

/* gradient wire precision of the reduce-scatter (weights/history stay fp32) */
#define COS_GRAD_FP32 0
#define COS_GRAD_BF16 1

/* solver type (SolverParameter.type); history layout per type, see cos_net_history */
#define COS_SOLVER_SGD 0  /* "SGD": momentum SGD, history = P floats */
#define COS_SOLVER_ADAM 1 /* "Adam": history = 2P floats, m of every blob then v of every blob */

/* all-reduce algorithm selection (cos_net_set_option "algo") */
#define COS_ALGO_AUTO 0
#define COS_ALGO_TWO_SHOT 1 /* reduce-scatter -> fused SGD -> weight push (sharded PS, reference structure) */
#define COS_ALGO_ONE_SHOT 2 /* every rank reduces + updates everything, no weight push (small P) */

typedef struct cos_net cos_net; /* opaque; == CaffeNet<float>* of the reference (JN:96-99) */

/* One input blob of train()/predict(): what a com.yahoo.ml.jcaffe.FloatBlob
 * hands over (JN:383-413, common.cpp GetFloatBlobVector): host fp32 data in
 * NCHW order owned by the caller for the duration of the call. */
typedef struct cos_blob {
  const float* data;
  int num, channels, height, width;
} cos_blob;

/* Solver + learnable-parameter layout, the information the reference reads
 * from the solver/net prototxt (caffe.proto SolverParameter :102-, ParamSpec
 * :283-304) and from Net::learnable_params() (parallel.cpp:27-57). */
typedef struct cos_solver_desc {
  int nblobs;               /* learnable blobs, learnable_params() order */
  const int64_t* counts;    /* elements per blob */
  const float* lr_mult;     /* ParamSpec.lr_mult   (NULL = all 1.0) */
  const float* decay_mult;  /* ParamSpec.decay_mult (NULL = all 1.0) */
  const char* lr_policy;    /* fixed|step|exp|inv|multistep|poly|sigmoid */
  float base_lr, gamma, power;
  int stepsize;
  const int* stepvalues;
  int nstepvalues;
  int max_iter;
  float momentum, weight_decay;
  int test_iter, test_interval;
  const char* snapshot_prefix; /* may be NULL */
  int grad_dtype;              /* COS_GRAD_FP32 | COS_GRAD_BF16 */
  int init_iter;               /* iteration to resume from (0) */
  int regularization_l1;       /* SolverParameter.regularization_type: 0 = "L2" (default), 1 = "L1" */
  int solver_type;             /* COS_SOLVER_SGD (0, default) | COS_SOLVER_ADAM; momentum is Adam's beta1 */
  float momentum2;             /* Adam's beta2 (SolverParameter.momentum2, 0.999 in a prototxt) */
  float delta;                 /* Adam's epsilon (SolverParameter.delta, 1e-8 in a prototxt) */
  int iter_size;               /* SolverParameter.iter_size: forward/backward passes per step (0 is read as 1);
                                  the step scales the accumulated gradient by 1/iter_size (SGDSolver::Normalize) */
} cos_solver_desc;

/* Gradient producer = Net::ForwardBackward of the reference (solver.cpp:221-223),
 * out of scope for this library and supplied by the embedding runtime.  Called
 * from cos_net_train on the calling thread after the input blobs were staged
 * to the device: `inputs[i]` are DEVICE pointers (same shapes as the host
 * blobs), it must enqueue on `cuda_stream` work that ACCUMULATES the local
 * gradient into cos_net_diff() using the weights in cos_net_data(), and write
 * the scalar loss to the DEVICE float `loss_dev`.  Return 0 on success.
 * With iter_size k > 1 it is called k times per step, each time with its own
 * `loss_dev`; cos_net_last_loss() then reports the float mean of the k losses. */
typedef int (*cos_forward_backward_fn)(void* user, int solver_index, const cos_blob* inputs, int ninputs,
                                       float* loss_dev, void* cuda_stream);

/* ---------------------------------------------------------------- errors */
COS_API const char* cos_last_error(void);
COS_API const char* cos_version(void);

/* ------------------------------------------ the 18 JNI natives (J:60-230) */

/* J:60-69 allocate / JN:14-89.  cluster_size==1 -> local net (CH LocalCaffeNet),
 * else connection_type RDMA|SOCKET -> NVLink peer net (CH Socket/RDMACaffeNet),
 * anything else fails like the reference's missing switch case (JN:41-64).
 * Parses the solver prototxt and the net it names to derive the layout. */
COS_API int cos_net_allocate(const char* solver_conf_file, const char* model_file, const char* state_file,
                             int num_local_devices, int cluster_size, int node_rank, int is_training,
                             int connection_type, int start_device_id, int validation_net_id, cos_net** out);

/* Same, with the layout given directly instead of parsed from prototxt. */
COS_API int cos_net_allocate_desc(const cos_solver_desc* desc, int num_local_devices, int cluster_size,
                                  int node_rank, int is_training, int connection_type, int start_device_id,
                                  cos_net** out);

/* J:72 deallocate / JN:96-99 */
COS_API void cos_net_deallocate(cos_net* net);

/* J:125 localAddresses / JN:106-159, CN:394-404.  Returns the number of
 * addresses (0 for a local net, cluster_size otherwise; "" at the own rank)
 * or -1.  *addresses points to an array owned by the net, valid until the
 * next call or deallocate. */
COS_API int cos_net_local_addresses(cos_net* net, const char* const** addresses);

/* J:80 connect / JN:184-228, CN:456-480.  `addresses` is indexed by rank; NULL
 * array or NULL entries are allowed (common.cpp:57-77).  A malformed or
 * unreachable address returns 0 (CaffeNetTest.connectbogus). */
COS_API int cos_net_connect(cos_net* net, const char* const* addresses, int naddresses);

/* J:86 sync / JN:166-177, CN:497-504: zero-payload control barrier over all
 * executors (no-op returning 1 on a local net, CH:91). */
COS_API int cos_net_sync(cos_net* net);

/* J:99 init / JN:256-270, CN:585-654: bind the calling thread to the solver's
 * device; solver_index < 0 -> 0. */
COS_API int cos_net_init(cos_net* net, int solver_index, int enable_nn);

/* J:120 train / JN:383-413, CN:707-729: ONE Solver::Step (solver.cpp:194-273):
 * stage the input blobs host->device, run the gradient producer iter_size
 * times on that one batch (the reference's data layer is Reset to the fed
 * batch, so every pass of a Step reads it), then the fused scale +
 * reduce-scatter + Normalize + SGD/momentum update + weight all-gather kernel,
 * ++iter.  data==NULL -> 0 with error "data is NULL" (JN:391-395). */
COS_API int cos_net_train(cos_net* net, int solver_index, const cos_blob* data, int ndata);

/* One Solver::Step over `passes` distinct micro-batches: `data` holds passes
 * groups of ndata blobs, group i is what pass i's producer call sees.  passes
 * must equal the solver's iter_size; the effective batch is passes x the
 * micro-batch.  Same staging, pipelining, loss and sync as cos_net_train.
 * 1/0 with the reason in cos_last_error(). */
COS_API int cos_net_train_accumulate(cos_net* net, int solver_index, const cos_blob* data, int ndata, int passes);

/* Untransformed input formats of cos_net_train_raw / cos_data_transform: what the JVM hands Caffe's
 * DataTransformer.  F32_NCHW is a FloatBlob (Transform(Blob*, Blob*): one mirror / crop draw per batch);
 * U8_NHWC is a vector of 8-bit images, each height x width x channels interleaved (Transform(cv::Mat):
 * one draw per image). */
#define COS_RAW_F32_NCHW 0
#define COS_RAW_U8_NHWC 1
typedef struct cos_raw_blob {
  const void* data; /* host memory, owned by the caller for the duration of the call */
  int format;       /* COS_RAW_* */
  int num, channels, height, width;
} cos_raw_blob;
/* train() on untransformed host blobs, one per staged input (data-layer top) in order: stage them, apply each input's
 * transform_param on the device, then run the registered producer and the fused sync exactly as train() does.  An
 * input without a transform_param (the label) must be F32_NCHW with its top's element count; it is copied.  The net
 * must have been allocated from a prototxt; mean files are read by the first call.  With iter_size k every pass
 * transforms again with its own draws.  Returns when the caller's memory has been read.  1/0 + cos_last_error(). */
COS_API int cos_net_train_raw(cos_net* net, int solver_index, const cos_raw_blob* data, int ndata);
/* The transform kernel alone, only enqueued on cuda_stream: in, out and mean are device pointers, mean_values a host
 * array of nmean floats (1 or channels; at most 64).  mean (channels x height x width of the input) and mean_values
 * exclusive; neither: x * scale.  out is num x channels x crop x crop fp32 (x height x width when crop_size is 0).
 * key seeds the draws (DESIGN.md, "Input transform on the device").  1/0 + cos_last_error(). */
COS_API int cos_data_transform(const void* in, int format, int num, int channels, int height, int width, float* out,
                               int crop_size, int mirror, const float* mean, const float* mean_values, int nmean,
                               float scale, uint64_t key, void* cuda_stream);
/* Decoded 8-bit images of any size, one cv::Mat each (format COS_RAW_U8_IMAGES of cos_net_train_raw).  For this
 * format the cos_raw_blob fields mean: data points to num cos_raw_image, each with its own size; channels is shared by
 * all images; height and width are the resize target (OpenCV's 8-bit INTER_LINEAR, as the reference's -resize), or
 * 0, 0 for no resize.  Each image is then transformed as a U8_NHWC image is, with its draws taken on its post-resize
 * size; Caffe's per-image checks (crop, top size, mean size) apply to that size.  Every call must repeat the first
 * call's num, channels and target; the images' own sizes may change from call to call. */
#define COS_RAW_U8_IMAGES 2
typedef struct cos_raw_image {
  const void* data; /* host, height x width x channels uint8, interleaved (a decoded cv::Mat) */
  int height, width;
} cos_raw_image;
/* One image of a ragged batch on the device: byte offset into the arena, its height and width. */
typedef struct cos_image_geometry {
  int64_t offset;
  int height, width;
} cos_image_geometry;
/* The COS_RAW_U8_IMAGES kernel alone, only enqueued on cuda_stream.  in (the images, each at its geometry's offset),
 * geometry (num entries), out and mean are device pointers; mean_values is a host array as for cos_data_transform.
 * resize_height x resize_width is the target, or 0 x 0.  out is num x channels x out_height x out_width fp32: crop x crop
 * with a crop, else every image's post-resize size.  mean is channels x mean_height x mean_width, every image's
 * post-resize size.  Geometry the host cannot see is checked by the kernel: an image it cannot take (a side below 1,
 * below the crop, or off the output or mean size) comes out as NaN.  1/0 + cos_last_error(). */
COS_API int cos_image_transform(const void* in, const cos_image_geometry* geometry, int num, int channels,
                                int resize_height, int resize_width, float* out, int out_height, int out_width,
                                int crop_size, int mirror, const float* mean, int mean_height, int mean_width,
                                const float* mean_values, int nmean, float scale, uint64_t key, void* cuda_stream);
/* Host only: one line per staged input of a solver or net prototxt, with its name, shape, scale, mirror, crop and
 * mean source (mean files are read and checked).  Returns the text length and copies it with its NUL when cap exceeds
 * it (buf may be NULL), or -1 + error naming the layer. */
COS_API int cos_input_transform_plan(const char* prototxt, char* buf, int cap);

/* J:110 predict / JN:277-376: forward-only; not on the sync path -> always
 * fails with "predict: not supported" (returns -1).  Kept for symbol parity. */
COS_API int cos_net_predict(cos_net* net, int solver_index, const cos_blob* data, int ndata,
                            const char* const* output_blob_names, int nnames, cos_blob* outputs);

/* J:220,227 validation / aggregateValidationOutputs (JN:420-470): not on the
 * sync path; return 0 with an error string. */
COS_API int cos_net_validation(cos_net* net, const cos_blob* data, int ndata);
COS_API int cos_net_aggregate_validation_outputs(cos_net* net);

/* J:133-165 integer getters / JN:235-249,479-580; -1 on invalid index. */
COS_API int cos_net_device_id(cos_net* net, int solver_index);
COS_API int cos_net_get_init_iter(cos_net* net, int solver_index);
COS_API int cos_net_get_max_iter(cos_net* net, int solver_index);
COS_API int cos_net_get_test_iter(cos_net* net, int solver_index);
COS_API int cos_net_get_test_interval(cos_net* net);

/* J:171 snapshot / JN:537-548, CN:735-738 -> Solver::Snapshot (solver.cpp:400-425):
 * writes stock-Caffe binaryproto files <prefix>_iter_<n>.caffemodel (NetParameter)
 * and .solverstate (SolverState) and returns the iteration, -1 on failure.  With
 * snapshot_format: HDF5 (sgd_solver.cpp:279-323, net.cpp:867-917) the files are
 * <prefix>_iter_<n>.caffemodel.h5 / .solverstate.h5 in HDF5's original file layout,
 * written without libhdf5 (csrc/hdf5_io.cpp): /data/<layer>/<j>, /iter, /learned_net,
 * /current_step, /history/<i>.  Called on rank 0 only, like
 * the reference (CaffeProcessor.scala:454-465); NOT collective: the history
 * shards of the other ranks are read through their mapped arenas. */
COS_API int cos_net_snapshot(cos_net* net);
/* The path snapshot() writes for `iter` (== CaffeNet.java:192-207 snapshotFilename). 1/0. */
COS_API int cos_net_snapshot_filename(cos_net* net, int iter, int is_state, char* buf, int cap);

/* J:177,185 getValidationOutputBlobNames / getValidationOutputBlobs
 * (JN:587-673): no validation net here; return -1 with an error string. */
COS_API int cos_net_get_validation_output_blob_names(cos_net* net, const char* const** names);
COS_API int cos_net_get_validation_output_blobs(cos_net* net, int length, cos_blob* outputs);

/* ------------------- hot-path surface for a native gradient producer ------ */

/* Register Net::ForwardBackward (see cos_forward_backward_fn). */
COS_API int cos_net_set_forward_backward(cos_net* net, cos_forward_backward_fn fn, void* user);

/* The built-in gradient producer (DESIGN.md section 14): a forward/backward engine built from the TRAIN phase of a
 * Caffe net prototxt, on this library's own sm_90a kernels.  It runs MemoryData / CoSData / Input, Convolution (group
 * 1, dilation 1), Pooling (MAX, AVE), InnerProduct (any axis), ReLU, Sigmoid, BatchNorm, LRN (WITHIN_CHANNEL), Slice,
 * Embed over fp32 token ids (a CoSData INT_ARRAY top), Reshape, RNN (without expose_hidden; its hidden state is kept
 * per engine from call to call, zero at first, and not snapshotted) over time-major CoSData tops (transpose: true),
 * MVN (its top the bottom's legacy 4-D shape; in place it computes the out-of-place result), Crop (its reference
 * bottom only gives a shape, so a per-pixel CoSData label can be cropped to a score map), SPP (MAX or AVE), Tile (not
 * in place), the other layers DESIGN.md section 14 lists, and one loss layer, SoftmaxWithLoss or ContrastiveLoss among
 * them (default normalisation); Accuracy and Silence are skipped.
 * Named params are shared as in Caffe.  Every other layer, and loss_param or an unknown filler type, is refused with an
 * error naming the layer.  Every use of a learnable blob adds its gradient into diff_ once per call; results are
 * bitwise reproducible.
 * A label outside [0, classes), or an Embed id that is not an integer in [0, input_dim), sets the net's device status
 * word: the next synchronising call fails with a message. */
/* Attach the built-in engine to every local solver of `net` and register it as the producer.
 * net_prototxt NULL = the net the solver file named at allocate; otherwise a solver or net prototxt whose layout must
 * equal the net's.  fill_weights 1 = initialise data_ from the prototxt fillers (only when no model_file was
 * restored), drawn from the cos_net_fill generator keyed by (the solver's random_seed, blob index); random_seed absent
 * or negative = seed 0, so every rank fills identically.  1/0. */
COS_API int cos_net_use_native_producer(cos_net* net, const char* net_prototxt, int fill_weights);
/* One Net::ForwardBackward with the registered producer on DEVICE inputs, no sync: accumulates into diff_, writes the
 * loss to the device float loss_dev.  cuda_stream NULL = the net's stream.  1/0. */
COS_API int cos_net_forward_backward(cos_net* net, int solver_index, const cos_blob* inputs, int ninputs,
                                     float* loss_dev, void* cuda_stream);
/* Host only, no device: the engine's plan for a solver or net prototxt as text (one op per line).  Returns the text
 * length and copies it with its NUL when cap exceeds it (buf may be NULL to ask for the length), or -1 + error. */
COS_API int cos_native_producer_plan(const char* prototxt, char* buf, int cap);

/* Flat device buffers of Params<Dtype> (parallel.hpp:22-45): data_ and diff_,
 * each cos_net_param_count() = P fp32 elements, blobs laid out back to back in
 * learnable_params() order, and the start of the solver's history_: P floats for
 * SGD; 2P for Adam, the m of every blob followed by the v of every blob
 * (AdamPreSolve order, adam_solver.cpp:8-17). */
COS_API float* cos_net_data(cos_net* net, int solver_index);
COS_API float* cos_net_diff(cos_net* net, int solver_index);
COS_API float* cos_net_history(cos_net* net, int solver_index);
COS_API int64_t cos_net_param_count(cos_net* net);

/* SocketSync::chunk (socket_sync_cpu.cpp:46-54): shard of `rank`. 1/0. */
COS_API int cos_net_shard(cos_net* net, int rank, uint64_t* offs, uint64_t* size);

/* Current iteration (Solver::iter()) and the rate GetLearningRate()
 * (sgd_solver.cpp:27-63) yields for it. */
COS_API int cos_net_iter(cos_net* net);
COS_API float cos_net_learning_rate(cos_net* net);
COS_API float cos_net_last_loss(cos_net* net);

/* THE HOT PATH.  Everything of Solver::Step after ForwardBackward plus the
 * next step's on_start, as one kernel launch on `cuda_stream` (NULL = the
 * net's own stream): diff *= 1/N, reduce-scatter over NVLink peer memory in
 * the reference's summation order, L2 decay, momentum SGD, w -= h, push of the
 * new weights to every peer, optional diff := 0 (ClearParamDiffs of the next
 * Step), ++iter.  Asynchronous: returns after the launch.  Collective: every
 * rank must call it once per iteration. */
COS_API int cos_net_sync_step(cos_net* net, int solver_index, void* cuda_stream);

/* on_start() alone (socket_sync_cpu.cpp:102-105): all-gather of the owned
 * weight shards.  connect() runs it once; exposed for tests. Collective. */
COS_API int cos_net_all_gather_weights(cos_net* net, int solver_index, void* cuda_stream);

/* Wait for the net's outstanding device work and surface device-side errors
 * (barrier time-outs).  1 = ok. */
COS_API int cos_net_synchronize(cos_net* net);

/* Options: "algo" (COS_ALGO_*), "zero_diff" (0/1, default 1),
 * "grid" (CTAs, 0 = auto), "block" (threads, 0 = auto), "kernel" (-1 = auto,
 * 0 = LDG/STG pull kernel, 1 = TMA bulk-copy pull pipeline, 2 = push kernel
 * (stores only, bf16 cast in registers), 3 = NVLS multimem kernel, 4 = LL kernel
 * (flag-in-data words, no barrier / fence; small nets, cluster_size <= 8)),
 * "barrier_timeout_ms", "one_shot_max_bytes", "ll_max_bytes" / "push_max_bytes" /
 * "nvls_min_bytes" (AUTO thresholds on the message size 4P), "push_vecs" (push / LL
 * kernel grid sizing; an Adam net refuses 1 and 3: cos_net_sync_step then returns 0 without launching),
 * "timing" (CUDA events around each launch, default 0), "initial_gather" (0 =
 * connect() skips the first on_start(); the caller then runs
 * cos_net_all_gather_weights itself), "nvls" (-1 = auto: join an NVSwitch
 * multicast team at connect() when cluster_size >= 6, the wire is fp32 and
 * 4P >= nvls_min_bytes (32 MiB); 0 = never; 1 = always try.  The in-switch sum matches the
 * reference to 1e-5, not bitwise: set 0 for bit-exact runs), "nvls_unroll",
 * "nvls_p2p" (share of plain-P2P vectors in the NVLS kernel), "train_pipeline"
 * (1 = cos_net_train returns once its batch has left host memory; 0 = after the
 * whole step), "trace" (record %globaltimer at the kernel's phase boundaries and inside
 * the two barriers), "iter" / "current_step" (the solver's iteration counter and
 * multistep position, e.g. to restart a benchmark from the same state).
 * Read-only via get_option: "resolved_algo", "resolved_kernel", "nvls_active",
 * "transport", "default_grid", "trace_0".."trace_12".  1/0. */
COS_API int cos_net_set_option(cos_net* net, const char* name, int64_t value);
COS_API int64_t cos_net_get_option(cos_net* net, const char* name);

/* Device time in ms of the last completed cos_net_sync_step / all_gather
 * launch (CUDA events on the launching stream), -1 if none. */
COS_API float cos_net_last_kernel_ms(cos_net* net);
/* Kernels launched by this net so far (bench.py gpu_launches). */
COS_API int64_t cos_net_launch_count(cos_net* net);
/* Seeded synthetic fill of one flat buffer ON THE DEVICE (which: 0 = data_, 1 = diff_,
 * 2 = the whole history, 2P floats for Adam): out[i] = amp * u_i, u_i uniform in [-1, 1) from a counter-based
 * generator keyed by (seed, stream) -- the generator the oracle's driver uses
 * (oracle/ref_driver.cpp), so benchmarks and parity runs need no host copy of the
 * 4P-byte tensors.  Asynchronous on the net's stream; 1/0. */
COS_API int cos_net_fill(cos_net* net, int solver_index, int which, uint64_t seed, uint64_t stream, float amp);

/* ------------ native layers for the gradient producer (DESIGN.md section 10) ------ */
/* Memory-bound layers of CaffeNet / CIFAR-10-quick as single passes.  Every tensor is a
 * contiguous NCHW fp32 DEVICE buffer of the given sizes.  The calls only enqueue kernels on
 * `cuda_stream` (NULL = the legacy default stream): they never allocate, synchronise or query
 * the device, so they may be captured into a CUDA graph.  1 = launched; 0 = bad arguments or a
 * failed launch (no GPU: there is no CPU path), with the reason in cos_last_error(). */

/* Cross-channel LRN (Caffe's ACROSS_CHANNELS, zero padding at the channel ends), local_size
 * odd and <= 15:  s_c = k + alpha/local_size * sum_{|c'-c| <= local_size/2} x_c'^2,
 * y_c = x_c * s_c^-beta.  The backward recomputes s from x (nothing else is stored). */
COS_API int cos_lrn_forward(const float* x, float* y, int num, int channels, int height, int width, int local_size,
                            float alpha, float beta, float k, void* cuda_stream);
COS_API int cos_lrn_backward(const float* x, const float* dy, float* dx, int num, int channels, int height, int width,
                             int local_size, float alpha, float beta, float k, void* cuda_stream);

/* LRN within the channel (Caffe's WITHIN_CHANNEL: split, square, AVE pool local_size x local_size with pad
 * local_size/2 and stride 1, power with shift 1, scale alpha and power -beta, product), local_size odd and <= 15:
 * s = 1 + alpha/local_size^2 * sum of x^2 over the window centred on (h, w), clipped to the plane;  y = x * s^-beta.
 * Caffe does not use k for this region, so there is none.  The backward recomputes s from x.  Not in place: y, and
 * dx, must not overlap an input. */
COS_API int cos_lrn_within_forward(const float* x, float* y, int num, int channels, int height, int width,
                                   int local_size, float alpha, float beta, void* cuda_stream);
COS_API int cos_lrn_within_backward(const float* x, const float* dy, float* dx, int num, int channels, int height,
                                    int width, int local_size, float alpha, float beta, void* cuda_stream);

/* conv bias + ReLU + MAX pooling (ceil mode, pad 0; either order of ReLU and pooling gives the same
 * result).  x is the conv output WITHOUT bias, bias has `channels` elements, y and index are
 * num x channels x pooled_height x pooled_width with pooled_* the ceil-mode sizes (checked).
 * index holds the position of the window's first maximum of x + bias (0 .. kernel^2-1), or 255
 * when that maximum is <= 0 (no gradient flows).  kernel <= 15. */
COS_API int cos_bias_relu_maxpool_forward(const float* x, const float* bias, float* y, uint8_t* index, int num,
                                          int channels, int height, int width, int kernel, int stride,
                                          int pooled_height, int pooled_width, void* cuda_stream);
/* dx (num x channels x height x width, written densely) and dbias (channels, overwritten) from dy and
 * the forward's index.  bias_partials is num * channels floats of scratch.  Deterministic. */
COS_API int cos_bias_relu_maxpool_backward(const float* dy, const uint8_t* index, float* dx, float* bias_partials,
                                           float* dbias, int num, int channels, int height, int width, int kernel,
                                           int stride, int pooled_height, int pooled_width, void* cuda_stream);

/* The same four layers with bf16 activations (x, y, dy, dx: uint16_t bit patterns of bfloat16, for the
 * mixed-precision producer).  Arguments, checks and launch rules are those of the fp32 calls above; bias,
 * bias_partials and dbias stay fp32.  Arithmetic is fp32 as in the fp32 calls: every y and dx element is the
 * fp32 call's result on the upcast inputs rounded once to bf16 (round to nearest even), index is the fp32 call's
 * index, and dbias equals the fp32 call's dbias on the upcast dy bit for bit. */
COS_API int cos_lrn_forward_bf16(const uint16_t* x, uint16_t* y, int num, int channels, int height, int width,
                                 int local_size, float alpha, float beta, float k, void* cuda_stream);
COS_API int cos_lrn_backward_bf16(const uint16_t* x, const uint16_t* dy, uint16_t* dx, int num, int channels,
                                  int height, int width, int local_size, float alpha, float beta, float k,
                                  void* cuda_stream);
COS_API int cos_lrn_within_forward_bf16(const uint16_t* x, uint16_t* y, int num, int channels, int height, int width,
                                        int local_size, float alpha, float beta, void* cuda_stream);
COS_API int cos_lrn_within_backward_bf16(const uint16_t* x, const uint16_t* dy, uint16_t* dx, int num, int channels,
                                         int height, int width, int local_size, float alpha, float beta,
                                         void* cuda_stream);
COS_API int cos_bias_relu_maxpool_forward_bf16(const uint16_t* x, const float* bias, uint16_t* y, uint8_t* index,
                                               int num, int channels, int height, int width, int kernel, int stride,
                                               int pooled_height, int pooled_width, void* cuda_stream);
COS_API int cos_bias_relu_maxpool_backward_bf16(const uint16_t* dy, const uint8_t* index, uint16_t* dx,
                                                float* bias_partials, float* dbias, int num, int channels, int height,
                                                int width, int kernel, int stride, int pooled_height,
                                                int pooled_width, void* cuda_stream);

/* The bias+ReLU+max-pool calls run shared-memory staged kernels where cos_pool_fast_path() returns 1 and
 * per-element kernels (the reference path) elsewhere; both write the same bits.  For tests and benchmarks only:
 * cos_layers_set_reference_kernels(1) makes every later launch in the process take the reference path, 0 (the
 * default) restores the choice by geometry.  The initial value is COS_LAYERS_REFERENCE_KERNELS from the environment
 * (set and not "0": on), read once when the library loads.  cos_layers_reference_kernels() returns the setting.
 * cos_pool_fast_path() is a pure host function of the shape: 1 = staged kernels, 0 = reference path (whatever the
 * switch says). */
COS_API void cos_layers_set_reference_kernels(int on);
COS_API int cos_layers_reference_kernels(void);
COS_API int cos_pool_fast_path(int num, int channels, int height, int width, int kernel, int stride);

/* Caffe's BatchNorm layer (batch_norm_layer.cpp; DESIGN.md section 13), x contiguous NCHW (a 2-axis
 * num x channels bottom passes height = width = 1).  mean_blob and var_blob have `channels` floats and
 * scale_blob one: the layer's three learnable blobs, usually pointers into data_.  save holds 2 * channels
 * floats: the mean, then the variance, the forward normalised with (the backward reads them).  workspace is
 * 2 * (num + 1) * channels floats of scratch.  Same launch rules as the calls above; deterministic.
 * Not in place: y must not alias x, and dx must not alias x or dy (the backward reads both twice); such
 * calls are rejected.  A Caffe net with top == bottom passes a separate output buffer.
 * use_global_stats 0: y = (x - mean) / powf(var + eps, 0.5) with the biased batch variance E((x - mean)^2),
 *   and the blobs are updated in place: s = s * f + 1, mean_blob = mean + f * mean_blob,
 *   var_blob = M / (M - 1) * var + f * var_blob (M = num * height * width, factor 1 when M <= 1),
 *   f = moving_average_fraction, one fp32 rounding per operation.
 * use_global_stats 1: mean = mean_blob / s and var = var_blob / s (0 when s == 0); the blobs are only read.
 * The backward writes dx only: (dy - sum(dy) / M - x^ * sum(dy * x^) / M) / std in training mode and dy / std
 * with global statistics; the blobs get no gradient. */
COS_API int cos_batch_norm_forward(const float* x, float* y, float* mean_blob, float* var_blob, float* scale_blob,
                                   float* save, float* workspace, int num, int channels, int height, int width,
                                   int use_global_stats, float moving_average_fraction, float eps, void* cuda_stream);
COS_API int cos_batch_norm_backward(const float* x, const float* dy, float* dx, const float* save, float* workspace,
                                    int num, int channels, int height, int width, int use_global_stats, float eps,
                                    void* cuda_stream);
/* bf16 activations (x, y, dy, dx); statistics, save and workspace stay fp32.  Every y and dx element is the fp32
 * call's result on the upcast inputs rounded once to bf16, and save and the blobs equal the fp32 call's bit for bit. */
COS_API int cos_batch_norm_forward_bf16(const uint16_t* x, uint16_t* y, float* mean_blob, float* var_blob,
                                        float* scale_blob, float* save, float* workspace, int num, int channels,
                                        int height, int width, int use_global_stats, float moving_average_fraction,
                                        float eps, void* cuda_stream);
COS_API int cos_batch_norm_backward_bf16(const uint16_t* x, const uint16_t* dy, uint16_t* dx, const float* save,
                                         float* workspace, int num, int channels, int height, int width,
                                         int use_global_stats, float eps, void* cuda_stream);

/* Caffe's MVN layer (mvn_layer.cu; DESIGN.md section 14): `rows` contiguous rows of `dim` fp32 elements, each
 * normalised on its own (a Caffe bottom has num * channels rows, or num with across_channels).  With
 * alpha = (float)(1.0 / dim) and one fp32 rounding per operation:
 *   forward   y = x - mu, mu = sum(x) * alpha; with normalize_variance y = (x - mu) / s, s = powf(var, 0.5) + eps
 *             (glibc's powf), var = sum((x - mu)^2) * alpha
 *   backward  with normalize_variance dx = (dy + c * (y * A + B)) / s, c = (float)(-1.0 / dim), A = sum(y * dy),
 *             B = sum(dy) (Caffe's formula, the exact derivative only where s >> eps); mean-only dx = dy - B * alpha
 * stats holds 5 * rows floats, row vectors in this order: sum(x), sum((x - mu)^2) and s (written by the forward;
 * 0 and 1 mean-only), then A and B (written by the backward, which reads s).  workspace is
 * cos_mvn_workspace_floats(rows, dim) floats (NULL when that is 0).  The row sums' order is fixed by (rows, dim):
 * results are bitwise identical from run to run.  y may be x, and dx may be y or dy.  Same launch rules as the
 * calls above; rows * dim must be below 2^31 (else "bad shape"). */
COS_API long long cos_mvn_workspace_floats(long long rows, long long dim);
COS_API int cos_mvn_forward(const float* x, float* y, float* stats, float* workspace, long long rows, long long dim,
                            int normalize_variance, float eps, void* cuda_stream);
COS_API int cos_mvn_backward(const float* y, const float* dy, float* dx, float* stats, float* workspace,
                             long long rows, long long dim, int normalize_variance, void* cuda_stream);

/* Caffe's Crop layer (crop_layer.cpp; DESIGN.md section 14) over contiguous fp32 blobs of `naxes` axes (1 to 32):
 *   forward   y[i_0, .., i_{n-1}] = x[i_0 + offsets[0], .., i_{n-1} + offsets[n-1]] over top_shape
 *   backward  dx over bottom_shape: dy at the mapped index inside the window, +0 outside it; every element written
 * Both are bit-exact copies (NaN payloads, infinities, subnormals and -0 arrive as they are), one launch each.  The
 * window must lie inside the bottom (else "the window leaves the bottom").  Same launch rules as the calls above. */
COS_API int cos_crop_forward(const float* x, float* y, int naxes, const long long* bottom_shape,
                             const long long* top_shape, const long long* offsets, void* cuda_stream);
COS_API int cos_crop_backward(const float* dy, float* dx, int naxes, const long long* bottom_shape,
                              const long long* top_shape, const long long* offsets, void* cuda_stream);

/* Convolution on TF32 tensor cores (DESIGN.md section 10.2): x [n, c, h, w], w [k, c / groups, r, s] and
 * y [n, k, p, q] contiguous fp32 NCHW, p = (h + 2 pad_h - r) / stride_h + 1, q likewise; any geometry whose tensors
 * have fewer than 2^31 elements.  Every operand is rounded to TF32 (cvt.rna) and the products are summed in fp32, in
 * an order fixed by the shape: repeated calls give the same bits.
 *   forward          y = conv(x, w) (+ bias[k] when bias is not NULL)
 *   backward_data    dx from dy and w (any stride)
 *   backward_filter  dw from x and dy; workspace is cos_conv_workspace_floats(...) floats (NULL when that is 0)
 * Same launch rules as the calls above. */
COS_API long long cos_conv_workspace_floats(int n, int c, int h, int w, int k, int r, int s, int stride_h,
                                            int stride_w, int pad_h, int pad_w, int groups);
COS_API int cos_conv_forward(const float* x, const float* weight, const float* bias, float* y, int n, int c, int h,
                             int w, int k, int r, int s, int stride_h, int stride_w, int pad_h, int pad_w, int groups,
                             void* cuda_stream);
COS_API int cos_conv_backward_data(const float* dy, const float* weight, float* dx, int n, int c, int h, int w, int k,
                                   int r, int s, int stride_h, int stride_w, int pad_h, int pad_w, int groups,
                                   void* cuda_stream);
COS_API int cos_conv_backward_filter(const float* x, const float* dy, float* dweight, float* workspace, int n, int c,
                                     int h, int w, int k, int r, int s, int stride_h, int stride_w, int pad_h,
                                     int pad_w, int groups, void* cuda_stream);

/* Caffe's SPP layer (spp_layer.cpp; DESIGN.md section 14) over a contiguous fp32 [num, channels, height, width] bottom
 * with pyramid_height levels (1 to 16), MAX (max_pool != 0) or AVE.  Level l pools 2^l x 2^l windows of kernel
 * ceil(H / 2^l), stride the kernel and pad (kernel * 2^l - H + 1) / 2 (likewise for the width), as
 * SPPLayer::GetPoolingParam sets them.
 *   forward   y [num, channels * (4^pyramid_height - 1) / 3]: each sample's level l from channels * (4^l - 1) / 3 on,
 *             ordered (channel, row, column), bit for bit Caffe's Split + Pooling + Flatten + Concat; with MAX,
 *             argmax (int32, y's size) gets each window's first maximum (-1 when no value is > -FLT_MAX)
 *   backward  dx (the bottom's size, every element written) = the levels' Pooling gradients added in level order, as
 *             Caffe's Split adds them; argmax is the forward's (unused for AVE, may be NULL)
 * A geometry with a level whose pad is not below its kernel is refused.  One launch each; same launch rules as the
 * calls above. */
COS_API int cos_spp_forward(const float* x, float* y, int* argmax, int num, int channels, int height, int width,
                            int pyramid_height, int max_pool, void* cuda_stream);
COS_API int cos_spp_backward(const float* dy, const int* argmax, float* dx, int num, int channels, int height,
                             int width, int pyramid_height, int max_pool, void* cuda_stream);

/* Caffe's Tile layer (tile_layer.cpp; DESIGN.md section 14) over a contiguous fp32 bottom of `naxes` axes
 * (bottom_shape) repeated `tiles` times along `axis` (canonical, 0 .. naxes - 1): with outer = count(0, axis) and
 * inner = count(axis), the top is [outer, tiles, inner] in memory, at most 2^31 - 1 elements.
 *   forward   y[o, t, d] = x[o, d], every bit copied
 *   backward  dx[o, d] = dy[o, 0, d], then dy[o, t, d] added for t = 1 .. tiles - 1 in order, each add rounded once
 *             in fp32: Backward_cpu's copy and axpys bit for bit (a column of -0 stays -0); every element written
 * One launch each; same launch rules as the calls above. */
COS_API int cos_tile_forward(const float* x, float* y, int naxes, const long long* bottom_shape, int axis, int tiles,
                             void* cuda_stream);
COS_API int cos_tile_backward(const float* dy, float* dx, int naxes, const long long* bottom_shape, int axis,
                              int tiles, void* cuda_stream);

/* --------------------- transport object (reference: util/socket.hpp) ------ */
/* PeerAdapter = SocketAdapter + SocketChannel of the reference
 * (socket.hpp:22-89): a listener thread on a per-process endpoint whose
 * address string travels through Spark; channels carry only control messages
 * and memory handles (file descriptors), never tensor payload. */
typedef struct cos_adapter cos_adapter;
COS_API cos_adapter* cos_adapter_create(int cluster_size, int rank);
COS_API void cos_adapter_destroy(cos_adapter* a);
COS_API const char* cos_adapter_address(cos_adapter* a);
COS_API int cos_adapter_connect(cos_adapter* a, const char* const* addresses, int naddresses);
/* CTRL barrier (socket_sync_cpu.cpp:135-163 with data=false). 1/0. */
COS_API int cos_adapter_barrier(cos_adapter* a, int timeout_ms);
/* Offer a file descriptor under `key` / fetch the one `peer` offered. */
COS_API int cos_adapter_offer_fd(cos_adapter* a, const char* key, int fd, const void* meta, int meta_len);
COS_API int cos_adapter_fetch_fd(cos_adapter* a, int peer, const char* key, void* meta, int meta_cap,
                                 int timeout_ms);

/* ---------------- snapshot file utilities (host only, Caffe binaryproto) ------ */
/* Write / read the subset of caffe.proto the snapshots use (NetParameter.layer[].blobs[],
 * SolverState) without libprotobuf.  Blob k has shape_ndims[k] dims taken in order from
 * dims_flat; consecutive blobs with the same layer name form one layer.  Readers return
 * the element count of the requested blob (copied into `out` when cap allows) or -1. */
COS_API int cos_caffemodel_write(const char* path, const char* net_name, int nblobs, const char* const* layer_names,
                                 const char* const* layer_types, const int* shape_ndims, const int64_t* dims_flat,
                                 const float* const* data);
COS_API int64_t cos_caffemodel_read(const char* path, const char* layer_name, int blob_index, float* out,
                                    int64_t cap);
COS_API int cos_solverstate_write(const char* path, int iter, int current_step, const char* learned_net, int nblobs,
                                  const int* shape_ndims, const int64_t* dims_flat, const float* const* data);
/* blob_index < 0: returns the number of history blobs. */
COS_API int64_t cos_solverstate_read(const char* path, int* iter, int* current_step, char* learned_net,
                                     int learned_cap, int blob_index, float* out, int64_t cap);

/* -------------------------- host helpers (pure functions, no device) ------ */
/* HDF5 twins of the two writers above (snapshot_format: HDF5).  cos_caffemodel_read / cos_solverstate_read
 * recognise HDF5 files by their signature, so they read either format. */
COS_API int cos_caffemodel_write_h5(const char* path, int nblobs, const char* const* layer_names, const int* shape_ndims,
                                    const int64_t* dims_flat, const float* const* data);
COS_API int cos_solverstate_write_h5(const char* path, int iter, int current_step, const char* learned_net, int nblobs,
                                     const int* shape_ndims, const int64_t* dims_flat, const float* const* data);
/* One dataset of ANY old-style HDF5 file by absolute path ("/data", "/history/3"): returns the element count
 * (float32 copied, int32 converted to float), fills up to max_dims dims and *ndims; -1 on failure.  Used to pin the
 * reader on libhdf5-written files. */
COS_API int64_t cos_hdf5_read_dataset(const char* path, const char* dataset, int64_t* dims, int max_dims, int* ndims,
                                      float* out, int64_t cap);

COS_API void cos_chunk(uint64_t param_count, int cluster_size, int peer, uint64_t* offs, uint64_t* size);
COS_API float cos_learning_rate(const char* lr_policy, float base_lr, float gamma, float power, int stepsize,
                                const int* stepvalues, int nstepvalues, int max_iter, int iter,
                                int* current_step);
/* Parse solver prototxt (+ the net prototxt it names) into a layout; arrays
 * are written up to `cap` blobs.  Returns nblobs or -1. */
COS_API int cos_parse_solver(const char* solver_conf_file, cos_solver_desc* desc, int64_t* counts,
                             float* lr_mult, float* decay_mult, int cap, char* lr_policy_buf,
                             char* snapshot_prefix_buf, int strcap, int* stepvalues, int stepcap,
                             int* batch_size);

#ifdef __cplusplus
}
#endif
#endif /* CAFFEDISTRI_B200_H_ */
