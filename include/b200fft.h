/* b200fft -- C ABI of the H100-native batched complex FFT backend.
 *
 * This is the drop-in boundary for RustFFT's FftPlanner / Fft::process hot path: the entry points
 * a `src/cuda/` backend of the reference (next to src/avx, src/sse) would bind over FFI.  Plain
 * pointers and sizes only.  Citations are relative to the reference tree (RustFFT 6.4.1).
 *
 *   reference interface                                     replaced by
 *   ------------------------------------------------------  ---------------------------------------
 *   FftPlannerAvx::new() -> Result<Self,()>                  b200fft_device_count()
 *     (src/avx/avx_planner.rs:121-164, probed in             (0 devices => the Rust shim's new() returns
 *      FftPlanner::new, src/plan.rs:72-94)                    Err(()) and the next backend is tried)
 *   FftPlanner::plan_fft(len, direction) -> Arc<dyn Fft<T>>  b200fft_plan_create() / b200fft_plan_destroy()
 *   FftPlannerScalar::design_fft_for_len -> Recipe           b200fft_plan_create_from_recipe()  (the host keeps
 *     (src/plan.rs:134-226,412-425) + build_fft (:315-410)     planning; the library builds what the recipe says)
 *     (src/plan.rs:101-126; instances cached per             (the shim keeps RustFFT's FftCache,
 *      (len, direction), src/fft_cache.rs:5-38)               src/fft_cache.rs, above this call)
 *   Length::len / Direction::fft_direction                   b200fft_plan_len() / b200fft_plan_direction()
 *     (src/lib.rs:140-181)
 *   Fft::get_{inplace,outofplace,immutable}_scratch_len      b200fft_plan_scratch_len()   (always 0: a backend
 *     (src/lib.rs:262-277)                                    may report 0, src/lib.rs:259-261)
 *   Fft::process / process_with_scratch (in place)           b200fft_exec_host_inplace()
 *     (src/lib.rs:195-211)
 *   Fft::process_outofplace_with_scratch /                   b200fft_exec_host_outofplace()
 *   Fft::process_immutable_with_scratch (src/lib.rs:231-255)
 *   -- (no reference equivalent: device-resident batch)      b200fft_exec_device() / b200fft_exec_device_ws()
 *
 * Semantics kept from the reference:
 *   - unnormalised, natural order, forward sign exp(-2*pi*i*k*n/N)   (src/lib.rs:81-89, src/twiddles.rs:11)
 *   - Complex<T> is repr(C) {re, im}: a buffer is float2[] / double2[], interleaved       (CHANGELOG.md:139)
 *   - a buffer of n_complex = batch*len elements is `batch` independent contiguous transforms
 *                                                                     (src/array_utils.rs:151-177)
 *   - len == 0 is a silent no-op (src/fft_helper.rs:16-18); len 0 and 1 plan fine (src/plan.rs:873-882)
 *   - the reference PANICS on bad arguments (src/common.rs:13-104); here every call returns a status and
 *     b200fft_last_error() returns the same message text; the Rust shim turns non-zero into panic!().
 *   - plan handles are immutable and may be used concurrently from many threads, like Arc<dyn Fft<T>>
 *     (src/lib.rs:184 `Sync + Send`, examples/concurrency.rs:17-29).
 *
 * There is NO CPU fallback: without a CUDA device every plan/exec call fails with B200FFT_ERR_NO_DEVICE.
 */
#ifndef B200FFT_H
#define B200FFT_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200fft_plan b200fft_plan;

enum {
    B200FFT_OK = 0,
    B200FFT_ERR_INVALID_ARG = -1,   /* null pointer, unknown enum value */
    B200FFT_ERR_NO_DEVICE = -2,     /* no CUDA device / not an sm_90 part */
    B200FFT_ERR_CUDA = -3,          /* a CUDA runtime call failed; see b200fft_last_error() */
    B200FFT_ERR_BUFFER_TOO_SMALL = -4, /* "Provided FFT buffer was too small" (src/common.rs:19-24) */
    B200FFT_ERR_NOT_MULTIPLE = -5,  /* "Input FFT buffer must be a multiple of FFT length" (src/common.rs:25-31) */
    B200FFT_ERR_LEN_MISMATCH = -6,  /* "input buffer and output buffer must have the same length" (src/common.rs:50) */
    B200FFT_ERR_UNSUPPORTED = -7,   /* length outside what this build can plan */
    B200FFT_ERR_WORKSPACE = -8      /* caller-provided workspace too small */
};

enum { B200FFT_FORWARD = 0, B200FFT_INVERSE = 1 };  /* FftDirection, src/lib.rs:147-171 */
enum { B200FFT_F32 = 0, B200FFT_F64 = 1 };          /* Complex<f32> / Complex<f64> */

/* Number of usable (compute capability 10.x) devices.  Returns status; *n = 0 when there is none. */
int b200fft_device_count(int* n);

/* Build a plan: picks the kernel sequence for `len`, builds twiddle / chirp / index tables on the host
 * (angles evaluated in extended precision, rounded once -- src/twiddles.rs:6-23 contract) and uploads them. */
int b200fft_plan_create(b200fft_plan** out, uint64_t len, int direction, int precision, int device);
int b200fft_plan_destroy(b200fft_plan* plan);

/* Planning owned by the caller (the Rust host code of a `src/cuda/` backend keeps src/plan.rs's design_fft_* and hands the
 * decomposition over as data): a flattened recipe tree, node 0 = the root, in the vocabulary of the reference's Recipe enum
 * (src/plan.rs:134-226).  The library maps each node onto its kernels or returns B200FFT_ERR_UNSUPPORTED; tables are always
 * recomputed here in extended precision (src/twiddles.rs:6-23 contract), so no host twiddles cross the boundary.
 *   kind          reference Recipe                      a, b, child
 *   AUTO          --                                    this library's own choice for `len`
 *   POW2          Radix4 / Butterfly2..32               --  (len = 2^k: one CTA pass up to 2^14, two passes up to 2^24)
 *   SMOOTH        RadixN / Butterfly3..31               --  (prime factors <= 31, one CTA pass)
 *   MIXED_RADIX   MixedRadix / MixedRadixSmall          len = a * b, two passes (a x b)
 *   GOOD_THOMAS   GoodThomasAlgorithm(+Small)           len = a * b, gcd(a, b) = 1, two passes without twiddles
 *   RADER         RadersAlgorithm                       len = a * p (a = 0 or 1: len = p prime; a in 2..8: MixedRadix{a x Rader(p)}
 *                                                       fused); child = node of the inner FFT of length p - 1 (0 = AUTO)
 *   BLUESTEIN     BluesteinsAlgorithm                   child = node of the inner FFT, length M >= 2 len - 1 (0 = AUTO)
 *   CLUSTER       MixedRadix, on chip                   len = 2^14 .. 2^17 (f32): both passes inside one thread-block cluster, the
 *                                                       transpose through distributed shared memory (one pass over HBM);
 *                                                       a = 1: half tiles (4096 points per CTA, 2^14 .. 2^16) */
enum {
    B200FFT_RECIPE_AUTO = 0,
    B200FFT_RECIPE_POW2 = 1,
    B200FFT_RECIPE_SMOOTH = 2,
    B200FFT_RECIPE_MIXED_RADIX = 3,
    B200FFT_RECIPE_GOOD_THOMAS = 4,
    B200FFT_RECIPE_RADER = 5,
    B200FFT_RECIPE_BLUESTEIN = 6,
    B200FFT_RECIPE_CLUSTER = 7,
    B200FFT_RECIPE_COLUMNS = 8 /* internal to the 2-D plans: len = a * b, a-point FFTs down the columns of [a][b] images */
};
typedef struct b200fft_recipe_node {
    uint32_t kind;  /* B200FFT_RECIPE_* */
    uint32_t child; /* index of the inner-FFT node (RADER / BLUESTEIN); 0 = let the library choose */
    uint64_t len;   /* length of this node's transform */
    uint64_t a, b;  /* MIXED_RADIX / GOOD_THOMAS: the split; RADER: a = outer radix */
} b200fft_recipe_node;
int b200fft_plan_create_from_recipe(b200fft_plan** out, const b200fft_recipe_node* nodes, uint32_t n_nodes, int direction,
                                    int precision, int device);

/* The decomposition a plan was built as, in the same node vocabulary (node 0 = root): a plan can be stored as data and rebuilt
 * bit-identically with b200fft_plan_create_from_recipe -- plan serialisation for callers that cache plans across processes
 * (the reference keeps its Recipe in memory only, src/plan.rs:134-226).  Returns the number of nodes (at most 2 today); writes
 * min(cap, n) of them when `nodes` is not NULL. */
int b200fft_plan_recipe(const b200fft_plan* plan, b200fft_recipe_node* nodes, uint32_t cap);

uint64_t b200fft_plan_len(const b200fft_plan* plan);
int b200fft_plan_direction(const b200fft_plan* plan);
int b200fft_plan_precision(const b200fft_plan* plan);
/* which: 0 = in place, 1 = out of place, 2 = immutable.  Host-visible scratch the caller must supply: 0. */
uint64_t b200fft_plan_scratch_len(const b200fft_plan* plan, int which);
/* Human-readable description of the chosen algorithm tree, e.g. "FourStep{256x256}".  Returns length or <0. */
int b200fft_plan_describe(const b200fft_plan* plan, char* buf, uint64_t cap);
/* Kernel launches one exec of `batch` transforms issues (bench.py reports it as gpu_launches). */
uint64_t b200fft_plan_launches(const b200fft_plan* plan, uint64_t batch);

/* Trait-conformant host paths: host memory owned by the caller (pageable or pinned), n_complex = batch*len elements;
 * synchronous.  The batch flows in 64 MiB slices through a three-stage pipeline (copy in | kernels | copy out, one stream each)
 * over a ring of four device buffers owned by the plan (created on the first call, reused afterwards).  Pinned / registered
 * memory is copied from and to directly; pageable memory is staged through a pinned ring by a small pool of copy threads. */
int b200fft_exec_host_inplace(const b200fft_plan* plan, void* buffer, uint64_t n_complex);
int b200fft_exec_host_outofplace(const b200fft_plan* plan, const void* input, void* output, uint64_t n_complex);

/* Device-resident path (the measured one): d_in / d_out hold batch*len elements on the plan's device,
 * d_in == d_out allowed; asynchronous on `cuda_stream` (a cudaStream_t, NULL = default stream).
 * Plans that need an intermediate buffer take it from the stream-ordered allocator. */
int b200fft_exec_device(const b200fft_plan* plan, const void* d_in, void* d_out, uint64_t batch, void* cuda_stream);
/* Same, with a caller-provided device workspace of at least b200fft_workspace_bytes(plan, batch) bytes, 128-byte aligned
 * (the passes address it through TMA and drop consumed lines with discard.global.L2; B200FFT_ERR_INVALID_ARG otherwise). */
uint64_t b200fft_workspace_bytes(const b200fft_plan* plan, uint64_t batch);
int b200fft_exec_device_ws(const b200fft_plan* plan, const void* d_in, void* d_out, uint64_t batch,
                           void* cuda_stream, void* d_workspace, uint64_t workspace_bytes);

/* Real-input / real-output transforms of even length on top of the complex plans (SURVEY 8(f).4: what the `realfft` crate adds above
 * RustFFT's Fft trait; RustFFT itself has none).  forward: batch * len reals -> batch * (len/2 + 1) complex (the non-redundant half of the
 * spectrum); inverse: the reverse, unnormalised (inverse(forward(x)) = len * x), equal to len * numpy.fft.irfft(X, len) for any X: the
 * imaginary parts of X[0] and X[len/2] are ignored, as numpy ignores them.  Device-resident entry points (asynchronous on the stream)
 * and synchronous host ones (plain copies in and out, not pipelined). */
typedef struct b200fft_real_plan b200fft_real_plan;
int b200fft_real_plan_create(b200fft_real_plan** out, uint64_t len, int precision, int device);
int b200fft_real_plan_destroy(b200fft_real_plan* plan);
uint64_t b200fft_real_workspace_bytes(const b200fft_real_plan* plan, uint64_t batch);
int b200fft_real_forward_device(const b200fft_real_plan* plan, const void* d_real_in, void* d_complex_out, uint64_t batch, void* cuda_stream);
int b200fft_real_inverse_device(const b200fft_real_plan* plan, const void* d_complex_in, void* d_real_out, uint64_t batch, void* cuda_stream);
int b200fft_real_forward_host(const b200fft_real_plan* plan, const void* real_in, void* complex_out, uint64_t batch);
int b200fft_real_inverse_host(const b200fft_real_plan* plan, const void* complex_in, void* real_out, uint64_t batch);

/* 2-D complex transforms of row-major [height][width] images (batch of them, contiguous): the width-point plan over all rows, then one
 * strided pass of height-point FFTs down the columns (SURVEY 8(f).4; the same two steps a caller of RustFFT writes with two plans and two
 * transposes).  height: prime factors <= 31 and at most 4096 (f64: 2048); width: any length b200fft_plan_create accepts. */
typedef struct b200fft_plan2d b200fft_plan2d;
int b200fft_plan2d_create(b200fft_plan2d** out, uint64_t height, uint64_t width, int direction, int precision, int device);
int b200fft_plan2d_destroy(b200fft_plan2d* plan);
int b200fft_exec2d_device(const b200fft_plan2d* plan, const void* d_in, void* d_out, uint64_t batch, void* cuda_stream);
int b200fft_exec2d_host(const b200fft_plan2d* plan, const void* in, void* out, uint64_t batch);

/* 2-D real-input / real-output transforms of row-major [height][width] real images (a batch of them, contiguous; what
 * numpy.fft.rfft2 / irfft2 compute over the last two axes).  forward: batch * H * W reals -> batch * H * (W/2 + 1) complex, equal
 * to numpy.fft.rfft2(x), unnormalised, forward sign as everywhere here.  inverse: the reverse, unnormalised, so
 * inverse(forward(x)) = H * W * x.  For any half spectrum X it equals H * W * numpy.fft.irfft2(X, s=(H, W)): the inverse column
 * transforms, then numpy's irfft of every row, which keeps only the real parts of the DC and Nyquist entries.  So of columns 0 and
 * W/2 only the Hermitian parts (X[k1][k] + conj X[-k1][k]) / 2 count; the rest cannot be represented by a real image.
 * width: even, >= 2, with W/2 any length b200fft_plan_create accepts; height: >= 1, prime factors <= 31 and at most 4096
 * (f64: 2048); B200FFT_ERR_UNSUPPORTED otherwise.  Two passes over half-size complex data: the W/2-point complex plan over the
 * rows, then one column pass that applies the real unpack (forward) or pack (inverse) on its load; height 1 is the 1-D real
 * transform of length W.  Out of place only: overlapping input and output ranges are B200FFT_ERR_INVALID_ARG.  batch == 0 is a
 * silent no-op.  Plans are immutable and thread safe; the device entry points are asynchronous on the stream and take their
 * workspace from the stream-ordered allocator (CUDA-graph capturable). */
typedef struct b200fft_real_plan2d b200fft_real_plan2d;
int b200fft_real_plan2d_create(b200fft_real_plan2d** out, uint64_t height, uint64_t width, int precision, int device);
int b200fft_real_plan2d_destroy(b200fft_real_plan2d* plan);
/* e.g. "Real2d{62x256,rows=Direct{128}}" (rows: the W/2-point row plan's description).  Returns length or <0. */
int b200fft_real_plan2d_describe(const b200fft_real_plan2d* plan, char* buf, uint64_t cap);
int b200fft_real2d_forward_device(const b200fft_real_plan2d* plan, const void* d_real_in, void* d_complex_out, uint64_t batch, void* cuda_stream);
int b200fft_real2d_inverse_device(const b200fft_real_plan2d* plan, const void* d_complex_in, void* d_real_out, uint64_t batch, void* cuda_stream);
/* Same on host memory, synchronous (plain copies in and out, not pipelined). */
int b200fft_real2d_forward_host(const b200fft_real_plan2d* plan, const void* real_in, void* complex_out, uint64_t batch);
int b200fft_real2d_inverse_host(const b200fft_real_plan2d* plan, const void* complex_in, void* real_out, uint64_t batch);

/* 3-D complex transforms of row-major [depth][height][width] volumes (a batch of them, contiguous; numpy.fft.fftn over the last three
 * axes, unnormalised, forward sign as everywhere here).  Replaces the caller's composition of b200fft_exec2d_* over the batch * D
 * slices, a transpose that makes D the last axis, the D-point 1-D plan and a transpose back.  The width-point plan runs over every
 * row (d_in -> d_out), then the H axis and the D axis each run in place on d_out, one pass per axis; an axis of length 1 is
 * skipped.  An axis of length 2^k <= 4096 (f64: 2048) runs a compiled pass down the strided axis (one read and one write, no
 * workspace); any other length <= 4096 (f64: 2048) with prime factors <= 31 runs the 2-D plans' column pass, which needs its
 * columns fewer than 2^31 elements apart (H * W for the D axis); anything else is B200FFT_ERR_UNSUPPORTED, naming the axis.
 * width: any length b200fft_plan_create accepts.  d_in == d_out (in place) is allowed, and out of place leaves the input intact;
 * any other overlap is B200FFT_ERR_INVALID_ARG.  batch == 0 is a silent no-op.  Plans are immutable and thread safe; the device
 * entry point is asynchronous on the stream (CUDA-graph capturable). */
typedef struct b200fft_plan3d b200fft_plan3d;
int b200fft_plan3d_create(b200fft_plan3d** out, uint64_t depth, uint64_t height, uint64_t width, int direction, int precision, int device);
int b200fft_plan3d_destroy(b200fft_plan3d* plan);
/* e.g. "Fft3d{256x256x256,rows=Direct{256},cols=Axis{256,F=16},depth=Axis{256,F=16}}", "...,cols=Columns{100 down [100x100]}"
 * (rows: the width-point plan; cols: the H axis; depth: the D axis; absent when the axis has length 1).  Returns length or <0. */
int b200fft_plan3d_describe(const b200fft_plan3d* plan, char* buf, uint64_t cap);
/* d_in, d_out: batch * D * H * W complex values on the plan's device; asynchronous on `cuda_stream`. */
int b200fft_exec3d_device(const b200fft_plan3d* plan, const void* d_in, void* d_out, uint64_t batch, void* cuda_stream);
/* Same on host memory, synchronous (plain copies in and out, not pipelined). */
int b200fft_exec3d_host(const b200fft_plan3d* plan, const void* in, void* out, uint64_t batch);

/* 3-D real-input / real-output transforms of row-major [depth][height][width] real volumes (numpy.fft.rfftn / irfftn over the last
 * three axes).  Replaces the caller's composition of b200fft_real2d_* over the batch * D slices with a transpose, the D-point
 * complex plan and a transpose back.  forward: batch * D * H * W reals -> batch * D * H * (W/2 + 1) complex, unnormalised: the 2-D
 * real transform of every [H][W] slice, then the D axis in place on the output.  inverse: the reverse, unnormalised, so
 * inverse(forward(x)) = D * H * W * x; numpy's order (inverse complex transforms over D and H, then irfft over W), so for ANY half
 * spectrum X it equals D * H * W * numpy.fft.irfftn(X, s=(D, H, W)).  The inverse runs the D axis out of place into a workspace of
 * one spectrum's size from the stream-ordered allocator, then the 2-D real inverse from there: the input is never written.  depth 1
 * is exactly b200fft_real_plan2d.  width and height follow b200fft_real_plan2d_create; depth follows the axis routes of
 * b200fft_plan3d_create.  Out of place only: overlapping input and output ranges are B200FFT_ERR_INVALID_ARG.  batch == 0 is a
 * silent no-op.  Plans are immutable and thread safe; the device entry points are asynchronous on the stream (CUDA-graph capturable). */
typedef struct b200fft_real_plan3d b200fft_real_plan3d;
int b200fft_real_plan3d_create(b200fft_real_plan3d** out, uint64_t depth, uint64_t height, uint64_t width, int precision, int device);
int b200fft_real_plan3d_destroy(b200fft_real_plan3d* plan);
/* e.g. "Real3d{64x64x64,plane=Real2d{64x64,rows=Direct{32}},depth=Axis{64,F=32}}".  Returns length or <0. */
int b200fft_real_plan3d_describe(const b200fft_real_plan3d* plan, char* buf, uint64_t cap);
int b200fft_real3d_forward_device(const b200fft_real_plan3d* plan, const void* d_real_in, void* d_complex_out, uint64_t batch, void* cuda_stream);
int b200fft_real3d_inverse_device(const b200fft_real_plan3d* plan, const void* d_complex_in, void* d_real_out, uint64_t batch, void* cuda_stream);
/* Same on host memory, synchronous (plain copies in and out, not pipelined). */
int b200fft_real3d_forward_host(const b200fft_real_plan3d* plan, const void* real_in, void* complex_out, uint64_t batch);
int b200fft_real3d_inverse_host(const b200fft_real_plan3d* plan, const void* complex_in, void* real_out, uint64_t batch);

/* Batched FFT convolution (SURVEY 8(f).4; what scipy.signal.fftconvolve / oaconvolve do): every row of a batch of rows of
 * signal_len samples, contiguous, is convolved with ONE filter of filter_len taps fixed at plan time.  Plain sums, no scaling;
 * the result equals scipy.signal.fftconvolve(row, filter, mode):
 *   FULL   signal_len + filter_len - 1 outputs, output t = full-convolution index t
 *   SAME   signal_len outputs starting at full index (filter_len - 1) / 2 (scipy's centring)
 *   VALID  signal_len - filter_len + 1 outputs starting at full index filter_len - 1; needs signal_len >= filter_len
 * Domains: COMPLEX rows and filter of float2 / double2; REAL rows and filter of float / double, real output (two rows share one
 * complex transform).  Cross-correlation of x with h is the convolution of x with conj(h[::-1]) (the reversed, conjugated filter).
 * filter: host memory, filter_len elements, 1 <= filter_len <= 2048 (B200FFT_ERR_UNSUPPORTED otherwise).  One launch and one pass
 * over device memory per call, any signal length (overlap-save: blocks of M = 256..4096 points, M - filter_len + 1 outputs each,
 * FFT -> * FFT(filter) -> inverse FFT inside one CTA).  No workspace.  Out of place only: overlapping input and output ranges are
 * B200FFT_ERR_INVALID_ARG.  signal_len == 0 or batch == 0 is a silent no-op.  Plans are immutable and thread safe. */
typedef struct b200fft_conv_plan b200fft_conv_plan;
enum { B200FFT_CONV_FULL = 0, B200FFT_CONV_SAME = 1, B200FFT_CONV_VALID = 2 };
enum { B200FFT_CONV_COMPLEX = 0, B200FFT_CONV_REAL = 1 };
int b200fft_conv_plan_create(b200fft_conv_plan** out, uint64_t signal_len, const void* filter, uint64_t filter_len, int mode,
                             int domain, int precision, int device);
int b200fft_conv_plan_destroy(b200fft_conv_plan* plan);
/* Samples per output row (0 for a NULL plan). */
uint64_t b200fft_conv_output_len(const b200fft_conv_plan* plan);
/* e.g. "OverlapSave{n=100000,m=255,M=2048,L=1794,full,real}".  Returns length or <0. */
int b200fft_conv_describe(const b200fft_conv_plan* plan, char* buf, uint64_t cap);
/* d_in: batch * signal_len samples, d_out: batch * output_len samples on the plan's device; asynchronous on `cuda_stream`. */
int b200fft_conv_device(const b200fft_conv_plan* plan, const void* d_in, void* d_out, uint64_t batch, void* cuda_stream);
/* Same on host memory, synchronous (plain copies in and out, not pipelined). */
int b200fft_conv_host(const b200fft_conv_plan* plan, const void* in, void* out, uint64_t batch);

/* Batched multi-channel FFT convolution: C filters of filter_len taps each (host memory, row-major [C][filter_len], fixed at plan
 * time), every output row convolved with its own filter.  Modes, domains, output lengths and filter limits as for b200fft_conv_*;
 * plain sums, no scaling.  The output is batch * C rows of output_len samples, row (b, c) at (b C + c) output_len.  Layouts:
 *   PER_CHANNEL  input batch * C rows of signal_len samples, row (b, c) at (b C + c) signal_len:  y[b][c] = x[b][c] (*) h[c]
 *                = scipy.signal.fftconvolve(x, h[None], mode, axes=-1) for x of shape [batch][C][signal_len]
 *   SHARED       input batch rows, a filter bank over each:  y[b][c] = x[b] (*) h[c]
 *                = scipy.signal.fftconvolve(x[:, None, :], h[None], mode, axes=-1) for "full" and "valid" (for "same", scipy crops
 *                the channel axis to x's: broadcast x to [batch][C][signal_len] first)
 * One launch and one pass over device memory per call, like the single-filter plans; the C spectra stay on the device with the
 * plan.  C = 1 is exactly the b200fft_conv plan.  channels == 0 is B200FFT_ERR_INVALID_ARG; spectrum tables above 2^31 bytes are
 * B200FFT_ERR_UNSUPPORTED.  Out of place only.  signal_len == 0 or batch == 0 is a silent no-op.  Immutable and thread safe. */
typedef struct b200fft_chconv_plan b200fft_chconv_plan;
enum { B200FFT_CHCONV_PER_CHANNEL = 0, B200FFT_CHCONV_SHARED = 1 };
int b200fft_chconv_plan_create(b200fft_chconv_plan** out, uint64_t signal_len, uint64_t channels, const void* filters, uint64_t filter_len,
                               int mode, int domain, int layout, int precision, int device);
int b200fft_chconv_plan_destroy(b200fft_chconv_plan* plan);
/* Samples per output row (0 for a NULL plan). */
uint64_t b200fft_chconv_output_len(const b200fft_chconv_plan* plan);
/* e.g. "ChannelOverlapSave{n=65536,m=255,C=64,M=2048,L=1794,full,real,per_channel}".  Returns length or <0. */
int b200fft_chconv_describe(const b200fft_chconv_plan* plan, char* buf, uint64_t cap);
/* d_in: batch * C * signal_len samples (SHARED: batch * signal_len), d_out: batch * C * output_len samples, on the plan's device;
 * asynchronous on `cuda_stream`. */
int b200fft_chconv_device(const b200fft_chconv_plan* plan, const void* d_in, void* d_out, uint64_t batch, void* cuda_stream);
/* Same on host memory, synchronous (plain copies in and out, not pipelined). */
int b200fft_chconv_host(const b200fft_chconv_plan* plan, const void* in, void* out, uint64_t batch);

/* Batched 2-D FFT convolution of real images: every [height][width] image of a batch of real images (row-major, contiguous) is
 * convolved with ONE real filter of [filter_height][filter_width] taps (row-major, host memory) fixed at plan time.  Plain sums,
 * no scaling; the result equals scipy.signal.fftconvolve(image, filter, mode) in 2-D, with the B200FFT_CONV_* modes per axis:
 *   FULL   (H + kh - 1) x (W + kw - 1) outputs
 *   SAME   H x W outputs starting at full index ((kh - 1) / 2, (kw - 1) / 2) (scipy's centring, also for a filter larger than the image)
 *   VALID  (H - kh + 1) x (W - kw + 1) outputs starting at full index (kh - 1, kw - 1); needs H >= kh and W >= kw (the inputs are
 *          not swapped as scipy does)
 * Cross-correlation of an image with h is the convolution with h[::-1, ::-1] (the filter reversed along both axes).
 * Any H, W, kh, kw >= 1, odd widths included.  The plan runs a circular convolution of P x Q, Q = 2 M, with P >= H + kh - 1 - r0
 * and Q >= W + kw - 1 - c0 ((r0, c0) = the first output's full index), which leaves every output alias-free; P and M are the
 * smallest 7-smooth numbers >= those bounds (and >= 2) and must be at most 4096 (f64: 2048), B200FFT_ERR_UNSUPPORTED otherwise.
 * Three passes over half-size complex data: M-point row FFTs of the images, one column pass (real unpack, P-point FFT, product
 * with the filter's spectrum, inverse P-point FFT, only the output rows stored), inverse M-point row FFTs with the real pack that
 * store only the output columns.  Out of place only: overlapping input and output ranges are B200FFT_ERR_INVALID_ARG.
 * batch == 0 is a silent no-op.  Plans are immutable and thread safe; the device entry point is asynchronous on the stream and
 * takes its two workspaces from the stream-ordered allocator (CUDA-graph capturable). */
typedef struct b200fft_conv2d_plan b200fft_conv2d_plan;
int b200fft_conv2d_plan_create(b200fft_conv2d_plan** out, uint64_t height, uint64_t width, const void* filter, uint64_t filter_height,
                               uint64_t filter_width, int mode, int precision, int device);
int b200fft_conv2d_plan_destroy(b200fft_conv2d_plan* plan);
/* Output image shape: *out_height x *out_width per input image.  Returns status. */
int b200fft_conv2d_output_shape(const b200fft_conv2d_plan* plan, uint64_t* out_height, uint64_t* out_width);
/* e.g. "Conv2d{1080x1920,k=31x31,full,pad=1120x1960}" (pad = P x Q).  Returns length or <0. */
int b200fft_conv2d_describe(const b200fft_conv2d_plan* plan, char* buf, uint64_t cap);
/* d_in: batch * H * W reals, d_out: batch * Ho * Wo reals on the plan's device; asynchronous on `cuda_stream`. */
int b200fft_conv2d_device(const b200fft_conv2d_plan* plan, const void* d_in, void* d_out, uint64_t batch, void* cuda_stream);
/* Same on host memory, synchronous (plain copies in and out, not pipelined). */
int b200fft_conv2d_host(const b200fft_conv2d_plan* plan, const void* in, void* out, uint64_t batch);

/* Batched real-to-real transforms: DCTs and DSTs of types II, III and IV (what the `rustdct` crate's Dct2 / Dct3 / Dct4 / Dst2 / Dst3
 * / Dst4 traits add above RustFFT's Fft).  A buffer holds batch * len reals (float / double), contiguous rows; d_in == d_out (in
 * place) is allowed, any other overlap of the input and output ranges is B200FFT_ERR_INVALID_ARG.  Unnormalised; for a row x and
 * n, k in 0 .. len - 1 (N = len):
 *   DCT2  X[k] = sum x[n] cos(pi (2n+1) k / 2N)                              = scipy.fft.dct(x, 2) / 2
 *   DCT3  X[k] = x[0] / 2 + sum_{n>=1} x[n] cos(pi n (2k+1) / 2N)            = scipy.fft.dct(x, 3) / 2
 *   DCT4  X[k] = sum x[n] cos(pi (2n+1)(2k+1) / 4N)                          = scipy.fft.dct(x, 4) / 2
 *   DST2  X[k] = sum x[n] sin(pi (2n+1)(k+1) / 2N)                           = scipy.fft.dst(x, 2) / 2
 *   DST3  X[k] = (-1)^k x[N-1] / 2 + sum_{n<=N-2} x[n] sin(pi (n+1)(2k+1) / 2N) = scipy.fft.dst(x, 3) / 2
 *   DST4  X[k] = sum x[n] sin(pi (2n+1)(2k+1) / 4N)                          = scipy.fft.dst(x, 4) / 2
 * so DCT3(DCT2(x)) = DST3(DST2(x)) = DCT4(DCT4(x)) = DST4(DST4(x)) = (N/2) x.  len == 0 plans and is a silent no-op.
 * len = 2^k with 4 <= len <= 32768 (f64: 16384) runs in one pass (one read and one write, no workspace; buffers aligned to two
 * elements, B200FFT_ERR_INVALID_ARG otherwise).  Every other length runs a pre kernel, a complex plan and a post kernel over a
 * workspace from the stream-ordered allocator: the len/2-point plan for even len, the len-point plan for odd len (DCT4 / DST4:
 * 2 len points); a length whose complex plan cannot be built is B200FFT_ERR_UNSUPPORTED.  Any batch runs, in chunks where a launch would exceed its index range.  batch == 0 is a silent no-op.
 * Plans are immutable and thread safe; the device entry point is asynchronous on the stream (CUDA-graph capturable). */
typedef struct b200fft_dct_plan b200fft_dct_plan;
enum { B200FFT_DCT2 = 0, B200FFT_DCT3 = 1, B200FFT_DCT4 = 2, B200FFT_DST2 = 3, B200FFT_DST3 = 4, B200FFT_DST4 = 5 };
int b200fft_dct_plan_create(b200fft_dct_plan** out, uint64_t len, int kind, int precision, int device);
int b200fft_dct_plan_destroy(b200fft_dct_plan* plan);
/* e.g. "Dct2{n=4096,fused,M=2048}", "Dst4{n=1001,inner=Bluestein{...}}" (inner: the complex plan's description).  Returns length or <0. */
int b200fft_dct_describe(const b200fft_dct_plan* plan, char* buf, uint64_t cap);
/* d_in, d_out: batch * len reals on the plan's device; asynchronous on `cuda_stream`. */
int b200fft_dct_device(const b200fft_dct_plan* plan, const void* d_in, void* d_out, uint64_t batch, void* cuda_stream);
/* Same on host memory, synchronous (plain copies in and out, not pipelined). */
int b200fft_dct_host(const b200fft_dct_plan* plan, const void* in, void* out, uint64_t batch);

/* Batched 2-D and 3-D DCTs / DSTs: the same kind (B200FFT_DCT2 .. B200FFT_DST4) along each of the last `rank` (2 or 3) axes of
 * contiguous row-major arrays of shape[0] x .. x shape[rank-1] reals; a buffer holds `batch` such arrays.  Unnormalised: the result
 * is scipy.fft.dctn / dstn(x, type, axes = the last rank axes) / 2^rank, so DCT3n(DCT2n(x)) = DST3n(DST2n(x)) = DCT4n(DCT4n(x)) =
 * DST4n(DST4n(x)) = prod(shape[i] / 2) x.  Every axis length the 1-D plan of that kind accepts is supported; an axis whose 1-D plan
 * cannot be built is that plan's error, prefixed with the axis.  Arrays of zero elements and batch == 0 are silent no-ops.
 * The last axis runs the 1-D plan over every row (in -> out); every other axis then runs in place on out, one pass per axis: a
 * fused column pass for power-of-two lengths 4 .. 4096 (f64: 2048), one read and one write with no workspace; any other length
 * transposes slabs into a workspace from the stream-ordered allocator, runs the 1-D plan there and transposes back.
 * d_in == d_out (in place) is allowed; any other overlap is B200FFT_ERR_INVALID_ARG.  When the last axis runs a fused 1-D plan the
 * buffers must be aligned to two elements (B200FFT_ERR_INVALID_ARG otherwise).  Plans are immutable and thread safe; the device
 * entry point is asynchronous on the stream (CUDA-graph capturable). */
typedef struct b200fft_dctn_plan b200fft_dctn_plan;
int b200fft_dctn_plan_create(b200fft_dctn_plan** out, const uint64_t* shape, int rank, int kind, int precision, int device);
int b200fft_dctn_plan_destroy(b200fft_dctn_plan* plan);
/* e.g. "Dct2{512x512,rows=Dct2{n=512,fused,M=256},cols=fused{M=256,F=16}}",
 * "Dst3{1080x1920,rows=Dst3{n=1920,inner=...},cols=transposed{Dst3{n=1080,inner=...}}}": the last axis first (3-D: rows, cols,
 * then depth).  Returns length or <0. */
int b200fft_dctn_describe(const b200fft_dctn_plan* plan, char* buf, uint64_t cap);
/* d_in, d_out: batch * prod(shape) reals on the plan's device; asynchronous on `cuda_stream`. */
int b200fft_dctn_device(const b200fft_dctn_plan* plan, const void* d_in, void* d_out, uint64_t batch, void* cuda_stream);
/* Same on host memory, synchronous (plain copies in and out, not pipelined). */
int b200fft_dctn_host(const b200fft_dctn_plan* plan, const void* in, void* out, uint64_t batch);

/* Batched short-time Fourier transforms of real rows.  A plan fixes a real `window` of n_fft taps (host memory, in the plan's
 * precision; n_fft even and >= 2), the hop (1 <= hop <= n_fft), signal_len and `center`.  A signal buffer holds batch contiguous
 * rows of signal_len reals; a spectrum buffer holds batch * frames * (n_fft/2 + 1) complex values, frame-major: row r, frame f,
 * bin k at (r frames + f) (n_fft/2 + 1) + k (torch.stft's [bins][frames] layout is the transpose of the last two axes).
 *   forward  S[f][k] = sum_u w[u] xp[f hop + u] exp(-2 pi i k u / n_fft),  u < n_fft, k <= n_fft/2   (unnormalised)
 *            xp = x reflect-padded by n_fft/2 on each side when center (torch's pad_mode "reflect"; needs signal_len > n_fft/2),
 *            else xp = x (needs signal_len >= n_fft);  frames = 1 + (signal_len + (center ? n_fft : 0) - n_fft) / hop
 *   inverse  the least-squares inverse, torch.istft(..., center, length = signal_len): every frame's irfft (normalised by 1/n_fft)
 *            times the window, overlap-added, divided by the window envelope env[p] = sum_f w[p - f hop]^2, with the first
 *            n_fft/2 samples dropped when center, and zeros past the last frame.  So inverse(forward(x)) = x.  This is the one
 *            transform here that is normalised: the division by the envelope is part of what an inverse STFT is, and the 1/n_fft
 *            folds into the same multiply (one table entry per sample, evaluated in long double and rounded once).  The
 *            imaginary parts of bins 0 and n_fft/2 are ignored, as numpy's irfft ignores them.
 * The inverse needs the NOLA condition, env > 1e-11 at every returned sample; it is checked at plan time in long double, and a plan
 * that fails it (e.g. a periodic Hann window without center) runs its forward but returns B200FFT_ERR_UNSUPPORTED from the inverse.
 * n_fft = 2^k with 4 <= n_fft <= 32768 (f64: 16384) runs the forward in one pass: one read of the signal and one write of the
 * spectrum, no workspace.  Every other n_fft frames and windows into a workspace and runs the real plan of n_fft points from it
 * (an n_fft whose real plan cannot be built is that plan's error); the inverse always runs the real plan's inverse into a workspace
 * of whole rows of frames, then one overlap-add pass.  Workspaces come from the stream-ordered allocator (CUDA-graph capturable)
 * in chunks of at most 2^27 reals (the inverse: at least one row).  signal_len and frames * n_fft must stay below 2^31
 * (B200FFT_ERR_UNSUPPORTED).  Bad parameters and null pointers are B200FFT_ERR_INVALID_ARG.  Out of place only: overlapping input
 * and output ranges are B200FFT_ERR_INVALID_ARG.  batch == 0 is a silent no-op.  Plans are immutable and thread safe; the device
 * entry points are asynchronous on the stream. */
typedef struct b200fft_stft_plan b200fft_stft_plan;
int b200fft_stft_plan_create(b200fft_stft_plan** out, uint64_t signal_len, const void* window, uint64_t n_fft, uint64_t hop, int center,
                             int precision, int device);
int b200fft_stft_plan_destroy(b200fft_stft_plan* plan);
/* e.g. "Stft{n=16000,n_fft=512,hop=128,center,frames=126,fused,M=256}",
 * "Stft{n=16000,n_fft=400,hop=160,center,frames=101,rows=Real{Smooth{...}}}" (rows: the real plan's complex plan).  Returns length or <0. */
int b200fft_stft_describe(const b200fft_stft_plan* plan, char* buf, uint64_t cap);
/* Frames per row (0 for a NULL plan). */
uint64_t b200fft_stft_frames(const b200fft_stft_plan* plan);
/* d_signal: batch * signal_len reals, d_spectrum: batch * frames * (n_fft/2 + 1) complex values on the plan's device; asynchronous
 * on `cuda_stream`. */
int b200fft_stft_forward_device(const b200fft_stft_plan* plan, const void* d_signal, void* d_spectrum, uint64_t batch, void* cuda_stream);
int b200fft_stft_inverse_device(const b200fft_stft_plan* plan, const void* d_spectrum, void* d_signal, uint64_t batch, void* cuda_stream);
/* Same on host memory, synchronous (plain copies in and out, not pipelined). */
int b200fft_stft_forward_host(const b200fft_stft_plan* plan, const void* signal, void* spectrum, uint64_t batch);
int b200fft_stft_inverse_host(const b200fft_stft_plan* plan, const void* spectrum, void* signal, uint64_t batch);

/* Batched chirp-z transforms on the unit circle (scipy.signal.czt / zoom_fft).  For each contiguous row x of n samples and
 * k = 0 .. m - 1:
 *   y[k] = sum_{t<n} x[t] exp(-2 pi i (start + k step) t)     (unnormalised, like every transform here)
 * with start and step in turns (cycles per sample): scipy.signal.czt(x, m, w = exp(-2 pi i step), a = exp(2 pi i start)), and
 * zoom_fft(x, [f1, f2], m, fs, endpoint) is start = f1 / fs, step = (f2 - f1) / (fs m) (endpoint: / (fs (m - 1))).  start = 0,
 * step = 1/n, m = n is the DFT; a negative step walks the circle backwards.  Only arcs of the unit circle: spirals (|a| != 1 or
 * |w| != 1) are not supported.  The tables use the exact phase of the given doubles: start t + step t^2 / 2 is reduced mod 1 in
 * 128-bit integers (to 2^-124 turns), evaluated in long double and rounded once, so that the error stays at FFT level up to
 * n + m - 1 = 2^24 (forming w^(k^2/2) in double, as scipy does, loses accuracy as k^2 grows).
 * domain B200FFT_CONV_COMPLEX: rows of complex samples; B200FFT_CONV_REAL: rows of reals (half the bytes read); the output is
 * complex either way, batch * m values.  L = max(8, next_pow2(n + m - 1)) <= 4096 runs in one pass (Bluestein's fused kernel
 * with the CZT's tables): one read of x and one write of y, no workspace.  8192 <= L <= 2^24 runs a pre-chirp pass, the L-point
 * forward plan, a multiply pass, the L-point inverse plan and a post-chirp pass on a workspace from the stream-ordered allocator
 * (CUDA-graph capturable), in chunks of whole rows of at most 2^27 complex values (one row at least).  n + m - 1 > 2^24 is
 * B200FFT_ERR_UNSUPPORTED.  n = 0, m = 0, a start or step that is not finite, an unknown domain or precision, null pointers
 * and overlapping input and output ranges are B200FFT_ERR_INVALID_ARG.  batch == 0 is a silent no-op.  Plans are immutable and
 * thread safe; the device entry point is asynchronous on the stream. */
typedef struct b200fft_czt_plan b200fft_czt_plan;
int b200fft_czt_plan_create(b200fft_czt_plan** out, uint64_t n, uint64_t m, double start, double step, int domain, int precision,
                            int device);
int b200fft_czt_plan_destroy(b200fft_czt_plan* plan);
/* e.g. "Czt{n=2000,m=1000,L=4096,real,fused}", "Czt{n=1000000,m=4096,L=1048576,complex,inner=FourStep{1024x1024}}" (inner: the
 * L-point forward plan).  Returns length or <0. */
int b200fft_czt_describe(const b200fft_czt_plan* plan, char* buf, uint64_t cap);
/* d_in: batch * n samples (complex, or real for B200FFT_CONV_REAL), d_out: batch * m complex values, on the plan's device;
 * asynchronous on `cuda_stream`. */
int b200fft_czt_device(const b200fft_czt_plan* plan, const void* d_in, void* d_out, uint64_t batch, void* cuda_stream);
/* Same on host memory, synchronous (plain copies in and out, not pipelined). */
int b200fft_czt_host(const b200fft_czt_plan* plan, const void* in, void* out, uint64_t batch);

/* Batched analytic signals of real rows (scipy.signal.hilbert(x, axis=-1)).  For each contiguous row x of N reals the output row
 * is N complex values z = x + i y:
 *   y[n] = sum_m x[m] (2/N) sum_{0<k<N/2} sin(2 pi k (n - m) / N)
 * that is ifft(fft(x) h) with h = 1, 2, ..., 2, (1 at N/2 for even N), 0, ...  The analytic signal is normalised by definition:
 * unlike the library's FFTs, the real part is x, copied bit for bit on every path.  N = 1 gives z = x; N = 0 plans and every
 * call is a silent no-op.  Power-of-two N from 4 to 32768 (f64: 16384) run in one pass: one read of x, one write of z, no
 * workspace.  Other even N run the N/2-point forward plan on x read as complex pairs, a pass on the spectrum and the N/2-point
 * inverse plan on a workspace from the stream-ordered allocator (CUDA-graph capturable), in chunks of whole rows of at most 2^27
 * complex values (one row at least), then a pass that writes z.  Odd N run in the output buffer itself (x promoted to complex, the
 * N-point forward plan, a sign multiply, the N-point inverse plan, x written into the real parts).  A length whose complex plan
 * (N/2 points for even N, N for odd N) this build cannot make is B200FFT_ERR_UNSUPPORTED.  Even N read x as pairs: a device
 * input that does not start at an even element is B200FFT_ERR_INVALID_ARG, as are an unknown precision, null pointers and
 * overlapping input and output ranges (out of place only).  batch == 0 is a silent no-op.  Plans are immutable and thread safe;
 * the device entry point is asynchronous on the stream. */
typedef struct b200fft_hilbert_plan b200fft_hilbert_plan;
int b200fft_hilbert_plan_create(b200fft_hilbert_plan** out, uint64_t len, int precision, int device);
int b200fft_hilbert_plan_destroy(b200fft_hilbert_plan* plan);
/* e.g. "Hilbert{n=4096,fused,M=2048}", "Hilbert{n=48000,inner=SmoothFourStep{64x375,compiled}}" (inner: the forward complex plan), "Hilbert{n=1,identity}",
 * "Hilbert{n=0,empty}".  Returns length or <0. */
int b200fft_hilbert_describe(const b200fft_hilbert_plan* plan, char* buf, uint64_t cap);
/* d_in: batch * len reals, d_out: batch * len complex values, on the plan's device; asynchronous on `cuda_stream`. */
int b200fft_hilbert_device(const b200fft_hilbert_plan* plan, const void* d_in, void* d_out, uint64_t batch, void* cuda_stream);
/* Same on host memory, synchronous (plain copies in and out, not pipelined). */
int b200fft_hilbert_host(const b200fft_hilbert_plan* plan, const void* in, void* out, uint64_t batch);

/* Batched modified DCTs of real rows (rustdct's Mdct).  A plan fixes N = len (even, >= 2), a real `window` of 2N taps (host memory,
 * in the plan's precision; any values) and signal_len L >= 1.  A row x is padded as xp = N zeros, x, zeros up to (frames + 1) N
 * samples, frames = ceil(L / N) + 1, and frame f covers xp[f N, f N + 2N).  A signal buffer holds batch contiguous rows of L reals; a
 * coefficient buffer holds batch * frames * N reals, frame-major: row r, frame f, coefficient k at (r frames + f) N + k.
 *   forward  C[f][k] = sum_{n<2N} w[n] xp[f N + n] cos(pi/N (n + 1/2 + N/2)(k + 1/2)),  k < N   (unnormalised, as rustdct defines
 *            it: row f is rustdct's process_mdct(xp[fN .. fN+N], xp[fN+N .. fN+2N]))
 *   inverse  y = (2/N) sum_f w[n] sum_k C[f][k] cos(pi/N (n + 1/2 + N/2)(k + 1/2)) placed at f N + n and overlap-added, cropped to
 *            [N, N + L): the sum of rustdct's process_imdct outputs times 2/N.  If w[n]^2 + w[n+N]^2 = 1 and w[2N-1-n] = w[n]
 *            (sine, Vorbis, KBD windows) then inverse(forward(x)) = x, the first and last N samples included.  Any other window
 *            computes the same formula (no envelope division).  The 2/N folds into one window table entry per tap, evaluated in long
 *            double and rounded once.
 * N = 2^k with 64 <= N <= 512 (f64: 64 <= N <= 16384) runs the forward in one pass: the quarter fold of the windowed frames, then the
 * N-point DCT-IV, one read of the signal and one write of the coefficients, no workspace (the lengths where that pass beat the
 * general route on an H100; README).  Every other even N folds into the coefficient
 * buffer and runs the N-point Dct4 plan on it in place (the environment variable B200FFT_MDCT_ROUTE=general, read once per process,
 * sends power-of-two N down this route too).  The inverse runs the Dct4 plan from the coefficients into a workspace of whole rows
 * of frames (stream-ordered allocator, CUDA-graph capturable; chunks of at most 2^27 reals, one row at least), then one overlap-add
 * pass.  Odd N is B200FFT_ERR_UNSUPPORTED (the fold needs N/2); so are L >= 2^31 and frames * N >= 2^31.  An N whose Dct4 plan
 * cannot be built is that plan's error.  len = 0, L = 0, an unknown precision, null pointers and overlapping input and output ranges
 * (out of place only) are B200FFT_ERR_INVALID_ARG, and so is a coefficient buffer that does not start at an even element when the
 * N-point Dct4 is a one-pass plan (the power-of-two N above: the fused passes move coefficient pairs).  The signal buffer takes any
 * offset.  batch == 0 is a silent no-op.  Plans are immutable and thread safe; the device entry points are asynchronous on the
 * stream. */
typedef struct b200fft_mdct_plan b200fft_mdct_plan;
int b200fft_mdct_plan_create(b200fft_mdct_plan** out, uint64_t len, const void* window, uint64_t signal_len, int precision, int device);
int b200fft_mdct_plan_destroy(b200fft_mdct_plan* plan);
/* e.g. "Mdct{n=512,L=48000,frames=95,fused,M=256}", "Mdct{n=960,L=48000,frames=51,dct=Dct4{n=960,inner=...}}" (dct: the N-point
 * Dct4 plan of the general forward).  Returns length or <0. */
int b200fft_mdct_describe(const b200fft_mdct_plan* plan, char* buf, uint64_t cap);
/* Frames per row (0 for a NULL plan). */
uint64_t b200fft_mdct_frames(const b200fft_mdct_plan* plan);
/* d_signal: batch * signal_len reals, d_coefs: batch * frames * len reals on the plan's device; asynchronous on `cuda_stream`. */
int b200fft_mdct_forward_device(const b200fft_mdct_plan* plan, const void* d_signal, void* d_coefs, uint64_t batch, void* cuda_stream);
int b200fft_mdct_inverse_device(const b200fft_mdct_plan* plan, const void* d_coefs, void* d_signal, uint64_t batch, void* cuda_stream);
/* Same on host memory, synchronous (plain copies in and out, not pipelined). */
int b200fft_mdct_forward_host(const b200fft_mdct_plan* plan, const void* signal, void* coefs, uint64_t batch);
int b200fft_mdct_inverse_host(const b200fft_mdct_plan* plan, const void* coefs, void* signal, uint64_t batch);

/* Message of the last failing call on this thread ("" if none). */
const char* b200fft_last_error(void);
/* Library build string: "b200fft <version> sm_90a" */
const char* b200fft_version(void);

#ifdef __cplusplus
}
#endif
#endif /* B200FFT_H */
