/*
 * pvraft_b200 -- C ABI of the H100-native (sm_90a) PV-RAFT hot path.
 *
 * The reference (weiyithu/PV-RAFT) has no FFI layer: its boundary is the Python nn.Module API
 * (SURVEY.md section 8b).  This header is the drop-in boundary underneath that API: every entry
 * point below replaces the ATen / torch-scatter op sequence of one reference function, cited as
 * `file:line` relative to the reference tree.  The Python mirror of the reference modules
 * (pvraft_b200/*.py, model/*.py) binds these symbols with ctypes -- see INTEGRATION.md.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no C++/torch types.  `stream` is a cudaStream_t
 *     passed as void*.  All pointers are DEVICE pointers on the current device.
 *   - Every call is asynchronous on `stream`, allocates nothing, never synchronises, keeps no
 *     state between calls (re-entrant); the caller owns every buffer.
 *   - Return value: 0 = ok; < 0 = pvraft_status (argument / capability error, nothing launched);
 *     > 0 = cudaError_t of the failed launch.  pvraft_last_error_string() describes the last
 *     non-zero return on the calling thread.
 *   - Tensors are contiguous fp32 unless stated.  Point-major layout [B,N,C] is used for every
 *     per-point feature array (one point's channels are contiguous), coordinates are [B,N,3].
 *   - GroupNorm statistics travel as raw double-precision sums ("stats": [B,8,2] = per sample,
 *     per group (sum, sum of squares)); producers ACCUMULATE with atomics, so the caller zeroes
 *     them (cudaMemsetAsync) before the producing call (in a fixed order with a det_workspace, see "Deterministic mode").
 *     Every producer keeps the sums accurate enough for var = sum x^2 / n - mean^2 to hold the variance to about 1e-7
 *     relative even when a group's mean is thousands of times its spread (fp32 partials are formed about a pivot value).
 *   - Weights are passed in the reference's own state_dict layouts ([Cout,Cin(,1(,1))] row-major).
 *   - Deterministic mode (what pvraft_b200 runs while torch.are_deterministic_algorithms_enabled() is true).  Every entry
 *     point that reduces floating-point values takes `void* det_workspace` as its last argument before `stream`.  NULL runs
 *     the default kernels, which accumulate with atomics in an order that varies from run to run.  Otherwise det_workspace
 *     is pvraft_*_det_workspace_bytes(...) bytes (the size query declared beside the entry point) of caller-provided,
 *     8-byte aligned scratch that the caller ZERO-FILLS before every call.  The kernels then add exact fixed-point values
 *     (Q64.64 in 128 bits) into the workspace, and one launch adds the workspace, rounded, into the destination the default
 *     kernels accumulate into.  Integer additions are exact, and every value added is a floating-point sum whose order is
 *     a function of the shapes (a point, a 128-point tile, a warp's rows of a grid sized from the shapes), so the results
 *     are bitwise identical from run to run, under graph replay, and for any SM count.  Each value added is truncated
 *     toward zero to a multiple of 2^-64, so the exact sum of n values is known to within an ABSOLUTE n * 2^-64 (terms
 *     below 2^-64 vanish); it is rounded once to double and then added to the destination.  A non-finite value, or one of
 *     magnitude >= 2^62, makes its destination entry NaN.  Same results as the default kernels up to summation order.
 *     Forward statistics are per (sample, tile / point), so with N % 128 == 0 a sample's statistics do not depend on the
 *     batch.
 */
#ifndef PVRAFT_B200_H
#define PVRAFT_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PVRAFT_VERSION 200 /* 0.2.0 */

#if defined(__GNUC__)
#define PVRAFT_API __attribute__((visibility("default")))
#else
#define PVRAFT_API
#endif

typedef enum pvraft_status {
    PVRAFT_OK = 0,
    PVRAFT_ERR_BAD_ARG = -1,     /* null pointer, non-positive size ... */
    PVRAFT_ERR_UNSUPPORTED = -2, /* shape outside what the kernels are built for */
    PVRAFT_ERR_SMEM = -3         /* working set does not fit the 227 KB shared memory of an SM */
} pvraft_status;

#define PVRAFT_KNN 32        /* model/corr.py:9, model/extractor.py:9 -- hard-coded in the reference */
#define PVRAFT_GN_GROUPS 8   /* model/corr.py:17,25 ; model/flot/gconv.py:27,30,33 */
#define PVRAFT_MOMENTS 16    /* doubles per sample for the kNN-branch moment accumulator */

PVRAFT_API int pvraft_version(void);
PVRAFT_API const char* pvraft_last_error_string(void);
/* number of SMs / max opt-in dynamic shared memory of the current device (plumbing for the host) */
PVRAFT_API int pvraft_device_info(int* sm_count, int* smem_optin_bytes);

/* ------------------------------------------------------------------------------------------------
 * All-pairs feature correlation on the Hopper tensor cores (wgmma) with an fp32-accurate 3xTF32 split.
 * Replaces CorrBlock.calculate_corr, model/corr.py:95-100: corr[b,i,j] = <fmap1[b,i,:], fmap2[b,j,:]> / sqrt(C).
 *   fmap1 [B,N,C], fmap2 [B,M,C] POINT-major f32 -> corr [B,N,M] f32.   N % 128 == 0, M % 128 == 0, C % 32 == 0.
 *   workspace: pvraft_corr_matmul_workspace_bytes(B,N,M,C) bytes (16-byte aligned) for the hi/lo operand splits.
 * --------------------------------------------------------------------------------------------- */
PVRAFT_API int64_t pvraft_corr_matmul_workspace_bytes(int B, int N, int M, int C);
PVRAFT_API int pvraft_corr_matmul_fwd(const float* fmap1, const float* fmap2, int B, int N, int M, int C, float* corr, void* workspace,
                                      void* stream);

/* ------------------------------------------------------------------------------------------------
 * The same GEMM over one window of the correlation matrix, for clouds whose N x M matrix is not built whole.
 *   pvraft_tf32_split_fwd: x [n] f32 -> hi = tf32(x), lo = tf32(x - hi) (the operand split of pvraft_corr_matmul_fwd),
 *     n % 4 == 0, 16-byte aligned buffers.  Run once per feature map and build, not once per window.
 *   pvraft_corr_matmul_window_fwd: split operands a_hi/a_lo (fmap1) [B,N,C] and b_hi/b_lo (fmap2) [B,M,C], point-major
 *     with N % 128 == 0, M % 128 == 0 (each sample's operand rows padded separately), C % 32 == 0
 *     -> corr [B, R, ldc] with R = rows rounded up to 128: corr[b,i,j] = <fmap1[b,r0+i,:], fmap2[b,c0+j,:]> / sqrt(C) for
 *     i < R, j < cols rounded up to 128.  Whole 128 x 128 tiles are written: an operand row past the caller's points (a
 *     padding row, of any content) only reaches the slab rows / columns past `rows` / `cols`, which the caller ignores.
 *     r0, c0 multiples of 128; ldc % 4 == 0; the window's whole row tiles lie inside [0, N) and its column tiles inside
 *     [0, M).  Every value is bit-identical to the same entry of pvraft_corr_matmul_fwd on the same operands.
 * --------------------------------------------------------------------------------------------- */
PVRAFT_API int pvraft_tf32_split_fwd(const float* x, int64_t n, float* hi, float* lo, void* stream);
PVRAFT_API int pvraft_corr_matmul_window_fwd(const float* a_hi, const float* a_lo, const float* b_hi, const float* b_lo, int B, int N,
                                             int M, int C, int r0, int rows, int c0, int cols, float* corr, int64_t ldc, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Correlation truncation: the K largest entries of every row of a dense correlation matrix.
 * Replaces torch.topk(corr, k, dim=2, sorted=True) in CorrBlock.init_module, model/corr.py:37-40.
 *   corr [B,N,M] -> val [B,N,K] f32, idx [B,N,K] int32 column ids, written in ASCENDING COLUMN order
 *   (value ties at the K-th place: lowest columns win).  The reference's descending-value order carries
 *   no meaning downstream; pvraft_corr_reorder rearranges every row for the lookup kernel anyway.
 * Requires 1 <= K <= min(M, 1024) and M <= 49152 (the row is staged in shared memory).
 * --------------------------------------------------------------------------------------------- */
PVRAFT_API int pvraft_corr_topk_fwd(const float* corr, int B, int N, int M, int K, float* val, int32_t* idx, void* stream);

/* ------------------------------------------------------------------------------------------------
 * The same selection over a strided window, with an optional id map: the two steps of the windowed build.
 *   corr [rows, ld] (cols <= ld valid columns per row) -> val / idx [rows, ld_out] (the first K entries of each row),
 *   the K largest of each row in ascending column order, value ties at the K-th place: lowest columns win.
 *   idx = cand_ids ? cand_ids[row * ld + j] : col_base + j for the kept column j (cand_ids [rows, ld] int32 or NULL).
 *   Per column window: col_base = first column, ld_out = W*K, val/idx offset by w*K -> the concatenated candidate lists.
 *   Merge: corr = the [rows, W*K] candidate values, cand_ids = their ids -> the row's exact top-K, because each list is in
 *   ascending column order.
 * Requires 1 <= K <= min(cols, 1024), cols <= 49152.
 * --------------------------------------------------------------------------------------------- */
PVRAFT_API int pvraft_corr_topk_window_fwd(const float* corr, int rows, int cols, int64_t ld, int K, int col_base, const int32_t* cand_ids,
                                           float* val, int32_t* idx, int64_t ld_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Bank-aware arrangement of the truncated state, once per forward (no reference counterpart: the order of
 * the K candidates inside a row carries no meaning in model/corr.py beyond fp summation order).
 * Every row of (val, idx) [rows, K] is permuted so that the 32 candidates the lookup kernel gathers with
 * one instruction fall into (nearly) distinct shared-memory banks.  Out of place; deterministic.
 * --------------------------------------------------------------------------------------------- */
PVRAFT_API int pvraft_corr_reorder(const float* val_in, const int32_t* idx_in, int64_t rows, int K, float* val_out,
                                   int32_t* idx_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Point-voxel correlation lookup (index + reduce part), one fused pass over the K candidates of
 * every point.  Replaces CorrBlock.get_voxel_feature up to (not incl.) out_conv, model/corr.py:47-71,
 * and CorrBlock.get_knn_feature up to (not incl.) knn_conv, model/corr.py:75-91.
 *   corr_val [B,N,K] f32, corr_idx [B,N,K] int32 (rows of xyz2, < M), xyz2_pad [B,M,4] = (x,y,z,0) rows of the second cloud
 *   (pvraft_xyz_pad_fwd, once per forward; 16-byte aligned, as corr_idx), coords [B,N,3]
 *   -> vox      [B,N,vox_ld]     (vox_ld >= levels*27, 0 = dense; pad columns are written as zeros so that the
 *                                consumer can read rows with 128-bit loads)  channel = level*27 + cell; mean corr of the candidates whose
 *                                round((xyz-coords)/r_level) lies in {-1,0,1}^3  (round-half-even,
 *                                true fp32 division; r_level = base_scale * 2^level)
 *   -> knn_sel  [B,N,32,4]       (corr, dx, dy, dz) of the 32 candidates nearest to coords
 *                                (distance = (dx*dx+dy*dy)+dz*dz, no FMA); order within a point is
 *                                unspecified; exact-distance ties at the 32nd place are broken deterministically
 *   -> knn_slot [B,N,32] int32   candidate slot (0..K-1) of each selected neighbour; may be NULL
 *   -> moments  [B,16] double    first/second moments of the 4-vector over the sample's N*32 edges, accumulated with
 *                                atomics into a buffer the caller has ZEROED: [0..3]=sum f_i, [4..13]=sum f_i f_j (i<=j,
 *                                row-major upper triangle), [14]=edge count, [15]=scratch (the kernel's work counter);
 *                                may be NULL (then the points are split statically)
 *   -> dbg_cube [B,N,K,levels] int8  cell id or -1 of every candidate AS DERIVED BY THE FUSED KERNEL ITSELF (the coarsest-cube
 *                                pre-test, the compaction and the per-level cell codes); test hook, NULL in production
 * K in {32,64,128,256,512,1024}; 1 <= levels <= 4; knn fixed at 32.
 * N query points (corr_val, corr_idx, coords and every output have N rows per sample), M points in the second cloud.  A cell
 * mean divides by clamp(count, 1, N) (model/corr.py:65), which differs from the count only when N < K.  The gather table is
 * staged in shared memory while M*16 bytes fit next to the warps' stages, and read from global memory (through L1/L2) otherwise.
 * det_workspace: pvraft_corr_lookup_det_workspace_bytes(B) bytes or NULL ("Deterministic mode"; it orders the moments).
 * --------------------------------------------------------------------------------------------- */
/* xyz [rows,3] -> out [rows,4] = (x,y,z,0): the gather table of the lookup kernel (one 128-bit load per candidate). */
PVRAFT_API int pvraft_xyz_pad_fwd(const float* xyz, int64_t rows, float* out, void* stream);
PVRAFT_API int pvraft_corr_lookup_fwd(const float* corr_val, const int32_t* corr_idx, const float* xyz2_pad, const float* coords,
                                      int B, int N, int M, int K, int levels, float base_scale, float* vox, int vox_ld, float* knn_sel,
                                      int32_t* knn_slot, double* moments, int8_t* dbg_cube, void* det_workspace, void* stream);
PVRAFT_API int64_t pvraft_corr_lookup_det_workspace_bytes(int B);
/* 1 when the lookup stages the gather table of a second cloud of M points in shared memory at truncate_k = K, 0 when it
 * gathers from global memory (a query for tools and tests). */
PVRAFT_API int pvraft_corr_lookup_table_in_smem(int M, int K);
/* The same lookup on the reduced-precision state of BASELINE.json configs[2] ("bf16 mode", SURVEY.md H7): correlation values as
 * bf16 bit patterns and candidate ids as uint16 (M <= 65536) -- 4 B instead of 8 B per candidate and iteration.  Index math
 * (coordinates, cells, kNN distances) stays fp32 and bit-exact; values are widened to fp32 exactly and accumulated in fp32, so
 * the outputs equal pvraft_corr_lookup_fwd on the bf16-rounded correlations.  K in {128,256,512,1024}; det_workspace as there.
 * pvraft_corr_state_pack_bf16 converts a reordered fp32/int32 state (round to nearest even). */
PVRAFT_API int pvraft_corr_lookup_bf16_fwd(const uint16_t* corr_val_bf16, const uint16_t* corr_idx_u16, const float* xyz2_pad,
                                           const float* coords, int B, int N, int M, int K, int levels, float base_scale, float* vox,
                                           int vox_ld, float* knn_sel, int32_t* knn_slot, double* moments, int8_t* dbg_cube,
                                           void* det_workspace, void* stream);
PVRAFT_API int pvraft_corr_state_pack_bf16(const float* val, const int32_t* idx, int64_t n, uint16_t* val_out, uint16_t* idx_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Generic fused (GroupNorm -> activation -> 1x1 conv [-> bias] [-> ReLU]) layer over points with
 * GroupNorm statistics of the OUTPUT accumulated on the fly.  It is the dense building block of
 * CorrBlock.out_conv[0] (model/corr.py:16), SetConv.fc2/fc3 and the fc1 pre-transform
 * (model/flot/gconv.py:26-33,58-85), FlotRefine.fc (model/refine.py:14,21).
 * --------------------------------------------------------------------------------------------- */
typedef enum pvraft_in_mode {
    PVRAFT_IN_PLAIN = 0,  /* x = in                                                     */
    PVRAFT_IN_GN = 1,     /* x = act(GN(in))            using in_stats/in_gamma/in_beta  */
    PVRAFT_IN_GN_MINMAX = 2 /* x = act(GN(in_max or in_min)): per channel picks max when the GN scale is >= 0,
                               min otherwise (max-pool over neighbours commuted with the monotone GN+LeakyReLU) */
} pvraft_in_mode;

typedef enum pvraft_act {
    PVRAFT_ACT_NONE = 0,
    PVRAFT_ACT_RELU = 1,
    PVRAFT_ACT_LRELU = 2 /* slope in act_slope (LeakyReLU 0.1, or PReLU with its learned slope) */
} pvraft_act;

typedef struct pvraft_linear_args {
    const float* in;        /* [B,N,cin] (PLAIN/GN) or the per-channel max array (GN_MINMAX) */
    const float* in_min;    /* [B,N,cin] per-channel min (GN_MINMAX only) */
    const double* in_stats; /* [B,8,2] sums of the un-normalised input (GN modes) */
    const float* in_gamma;  /* [cin] */
    const float* in_beta;   /* [cin] */
    double in_count;        /* number of elements per (sample, group) behind in_stats */
    int in_mode;            /* pvraft_in_mode */
    int in_act;             /* pvraft_act applied after the input GroupNorm */
    float in_slope;
    const float* weight;    /* [cout,w_cin] row-major; row stride w_ld floats (0 = w_cin): lets fc1.weight[:, :cin] be used in place */
    int w_ld;
    int w_cin;              /* weight columns used (0 = cin); input columns w_cin..cin-1 are padding and are ignored */
    const float* bias;      /* [cout] or NULL */
    const float* residual;  /* [B,N,cout] added to the output after bias/activation, or NULL (model/refine.py:22) */
    int out_act;            /* pvraft_act applied to the output (NONE or RELU) */
    float* out;             /* [B,N,cout] */
    double* out_stats;      /* [B,8,2] ACCUMULATED sums of `out`, or NULL (cout % 8 == 0 required) */
    int B, N, cin, cout;
} pvraft_linear_args;

/* det_workspace: pvraft_linear_det_workspace_bytes(B) bytes or NULL ("Deterministic mode"; it orders out_stats). */
PVRAFT_API int pvraft_linear_fwd(const pvraft_linear_args* a, void* det_workspace, void* stream);
PVRAFT_API int64_t pvraft_linear_det_workspace_bytes(int B);

/* ------------------------------------------------------------------------------------------------
 * The same fused layer on the Hopper tensor cores (TMA + wgmma), in one of two operand formats:
 *   - 3xTF32 (w_hi, w_lo set): fp32-accurate through a hi/lo operand split;
 *   - bf16 (w_bf16 set): activations (after the prologue) and weights rounded to bf16 (nearest even), fp32 accumulation.
 *     Prologue, epilogue, GroupNorm statistics and every tensor in memory stay fp32.
 * Up to three activation sources are concatenated along K (e.g. [h | inp | motion] of the ConvGRU,
 * model/update.py:32,36); the GroupNorm(+max/min selection)+activation prologue and the bias / ReLU / residual /
 * GroupNorm-statistics epilogue match pvraft_linear_fwd; two extra epilogues implement the ConvGRU gates
 * (model/update.py:34-39).  Requirements: points per sample N % 128 == 0; every source has a multiple of 32
 * channels; weights pre-split with pvraft_tc_weight_split into hi/lo [n_pad, K] (n_pad = cout rounded up to 16, <= 128), or
 * converted with pvraft_tc_weight_bf16 into bf16 [n_pad, K].
 * --------------------------------------------------------------------------------------------- */
typedef enum pvraft_tc_epilogue {
    PVRAFT_TC_PLAIN = 0,   /* out = act(acc + bias) (+ residual), optional output statistics                  */
    PVRAFT_TC_GRU_ZR = 1,  /* acc = [z|r] pre-activations (n_pad = 128): out = sigmoid(z), out2 = sigmoid(r) * h */
    PVRAFT_TC_GRU_Q = 2,   /* acc = q pre-activation: out = (1 - z) * h + z * tanh(acc + bias)                  */
    PVRAFT_TC_FLOW = 3     /* FlowHead tail (model/update.py:72) + RAFT update (model/RAFTSceneFlow.py:45-46), cout = 64:
                              out[B,N,3] = delta = w3 . relu(acc + bias) + b3; coords2_out = coords2 + delta;
                              flow_out = coords2_out - coords1 (the last two optional)                         */
} pvraft_tc_epilogue;

typedef struct pvraft_tc_linear_args {
    const float* in[3];     /* activation sources [B,N,in_channels[i]]; unused entries NULL */
    int in_channels[3];
    const float* in_min;    /* per-channel minima paired with in[0] (GroupNorm prologue with max/min selection) or NULL */
    const double* in_stats; /* [B,8,2] -> GroupNorm prologue on source 0 (further sources are taken as they are), or NULL */
    const float* in_gamma;
    const float* in_beta;
    double in_count;
    int in_act;             /* pvraft_act */
    float in_slope;
    const float* w_hi;      /* [n_pad, K] tf32 high parts, K = sum of in_channels */
    const float* w_lo;      /* [n_pad, K] tf32 low parts */
    int n_pad, cout;
    const float* bias;      /* [cout] or NULL (GRU_ZR: bias of z; GRU_Q: bias of q) */
    const float* bias2;     /* GRU_ZR: bias of r */
    int out_act;
    const float* residual;  /* PLAIN: [B,N,cout] added to the output, or NULL.  GRU epilogues: per-point term added to the
                               pre-activations ([B,N,128] = [z|r] for GRU_ZR, [B,N,64] for GRU_Q) -- the contribution of the
                               context features, constant over the RAFT iterations -- or NULL */
    float* out;             /* [B,N,cout] */
    float* out2;            /* GRU_ZR: r*h [B,N,64] */
    const float* h;         /* GRU epilogues: previous hidden state [B,N,64] */
    const float* z;         /* GRU_Q: update gate [B,N,64] */
    double* out_stats;      /* [B,8,2] accumulated, or NULL */
    int epilogue;           /* pvraft_tc_epilogue */
    int B, N;
    const float* tail;      /* PLAIN, or NULL: [B,N,3] copied into output columns cout..cout+2 (out row stride cout+3 = n_pad):
                               the MotionEncoder's `cat([out, flow])`, model/update.py:20 */
    const float* w3;        /* FLOW: flow_head.out_conv.2.weight [3,64] */
    const float* b3;        /* FLOW: flow_head.out_conv.2.bias [3] */
    const float* coords1;   /* FLOW: [B,N,3] or NULL */
    const float* coords2;   /* FLOW: [B,N,3] or NULL */
    float* coords2_out;     /* FLOW: [B,N,3] or NULL (may alias coords2) */
    float* flow_out;        /* FLOW: [B,N,3] or NULL */
    int params_settled;     /* nonzero: w_hi, w_lo (or w_bf16), bias, bias2, w3, b3 were last written at least three launches ago
                               on this stream (or before a synchronisation).  The kernel is launched with programmatic stream
                               serialization and then fetches them while the previous kernel drains.  0 is always safe. */
    const uint16_t* w_bf16; /* [n_pad, K] bf16 weights, or NULL.  Set: bf16 operands, and w_hi, w_lo must be NULL
                               (PVRAFT_ERR_BAD_ARG otherwise) */
} pvraft_tc_linear_args;

/* det_workspace: pvraft_tc_linear_det_workspace_bytes(B) bytes or NULL ("Deterministic mode"; it orders out_stats). */
PVRAFT_API int pvraft_tc_linear_fwd(const pvraft_tc_linear_args* a, void* det_workspace, void* stream);
PVRAFT_API int64_t pvraft_tc_linear_det_workspace_bytes(int B);

/* ---------------------------------------------------------------------------------------------
 * The update chain of one RAFT iteration in one launch: the same five layers and the same bits as the five
 * pvraft_tc_linear_fwd calls they replace, with the intermediates (cc, motion, r*h) kept on chip:
 *   cc     = relu(W_cc [PReLU(GN(y1)) | kfeat] + b_cc)            (conv_corr folded into the feature head)
 *   motion = [relu(W_m [cc | cflow] + b_m) (61) | flow (3)]        (MotionEncoder.conv, model/update.py:19-20)
 *   z, r   = sigmoid(W_zr [net | inp | motion] + [b_z | b_r])     (ConvGRU, model/update.py:34-35)
 *   net_out = (1 - z) net + z tanh(W_q [r*net | inp | motion] + b_q)   (model/update.py:36-39)
 *   p_out  = W_fc1[:, :64] net_out                                 (flow-head SetConv fc1 pre-transform, no bias)
 * Weights pre-split with pvraft_tc_weight_split into hi/lo, [n_pad, K] row-major -- or, for bf16 operands, converted with
 * pvraft_tc_weight_bf16 into w_bf16 (then the same bits as the five bf16 pvraft_tc_linear_fwd calls) -- in this order:
 *   0 W_cc [64,192], 1 W_m [64,128] (61 rows + zero padding), 2 [W_z; W_r] [128,192], 3 W_q [64,192], 4 W_fc1 [64,64].
 * Requirements: N % 128 == 0, hidden = context = 64, y1_channels = 128 (PVRAFT_ERR_UNSUPPORTED otherwise); net_out != net.
 * No reductions: the results do not depend on the launch configuration.
 * --------------------------------------------------------------------------------------------- */
typedef struct pvraft_update_chain_args {
    const float* y1;         /* [B,N,y1_channels] pre-GroupNorm lookup features */
    const double* y1_stats;  /* [B,8,2] GroupNorm sums of y1 */
    const float* gn_gamma;   /* [y1_channels] */
    const float* gn_beta;
    double gn_count;         /* elements per group and sample */
    float gn_slope;          /* PReLU slope after the GroupNorm */
    const float* kfeat;      /* [B,N,64] */
    const float* cflow;      /* [B,N,64] */
    const float* flow;       /* [B,N,3] */
    const float* net;        /* [B,N,hidden] */
    const float* inp;        /* [B,N,context] */
    const float* w_hi[5];
    const float* w_lo[5];
    const float* b_cc;       /* [64] */
    const float* b_m;        /* [61] */
    const float* b_z;        /* [64] */
    const float* b_r;        /* [64] */
    const float* b_q;        /* [64] */
    float* net_out;          /* [B,N,hidden] */
    float* p_out;            /* [B,N,64] */
    int B, N, hidden, context, y1_channels;
    const uint16_t* w_bf16[5];  /* bf16 weights, or all NULL: all five set selects bf16 operands, with w_hi, w_lo all NULL */
} pvraft_update_chain_args;

PVRAFT_API int pvraft_update_chain_fwd(const pvraft_update_chain_args* a, void* stream);
/* hi = tf32(w), lo = tf32(w - hi) of the window w[0:rows, col0:col0+cols] of a row-major matrix with row stride ld,
 * written zero-padded as [rows_pad, cols_pad]. */
PVRAFT_API int pvraft_tc_weight_split(const float* w, int rows, int cols, int ld, int col0, int rows_pad, int cols_pad,
                           float* hi, float* lo, void* stream);
/* bf16(w) (round to nearest even) of the same window, written zero-padded as [rows_pad, cols_pad]: the w_bf16 operand. */
PVRAFT_API int pvraft_tc_weight_bf16(const float* w, int rows, int cols, int ld, int col0, int rows_pad, int cols_pad,
                          uint16_t* out, void* stream);

/* out[B,N,C] (or channel-major [B,C,N] when transpose_out != 0) = act(GN(in)) -- the trailing
 * GroupNorm+LeakyReLU of SetConv (model/flot/gconv.py:33,82-83) when nothing follows it. */
PVRAFT_API int pvraft_gn_act_fwd(const float* in, const double* stats, const float* gamma, const float* beta, double count,
                      int act, float slope, int B, int N, int C, int transpose_out, float* out, const float* slope_dev, void* stream);
/* slope_dev (here and in pvraft_gn_act_bwd): optional DEVICE pointer to the slope -- the one-element nn.PReLU weight -- read by the
 * kernel instead of `slope`; the training path uses it so that a parameter the optimizer changes every step needs no host read-back. */

/* ------------------------------------------------------------------------------------------------
 * Correlation feature head (+ optional MotionEncoder), one persistent kernel.
 *  feature stage (when y1 != NULL): out_conv[1:] on the voxel branch + knn_conv/max/knn_out on the
 *    kNN branch, summed.  Replaces model/corr.py:17-19 (GN, PReLU, Conv1d 128->64), :24-29,:91-93, :45.
 *      y1 [B,N,128] = out_conv[0] output (pvraft_linear_fwd) with y1_stats [B,8,2];
 *      knn_sel [B,N,32,4], moments [B,16] from pvraft_corr_lookup_fwd  -> corr_feat [B,N,64] (may be NULL)
 *  motion stage (when motion != NULL): MotionEncoder.forward, model/update.py:15-21, on the feature
 *    just computed (or on corr_in [B,N,64] when y1 == NULL) and flow [B,N,3] -> motion [B,N,64]
 *    (channels 0..60 learned, 61..63 = flow).
 * --------------------------------------------------------------------------------------------- */
typedef struct pvraft_corrfeat_args {
    const float* y1;
    const double* y1_stats;
    const float* gn1_gamma; /* corr_block.out_conv.1.weight [128] */
    const float* gn1_beta;  /* corr_block.out_conv.1.bias   [128] */
    const float* prelu1;    /* corr_block.out_conv.2.weight [1]   */
    const float* w_out;     /* corr_block.out_conv.3.weight [64,128] */
    const float* b_out;     /* corr_block.out_conv.3.bias   [64]  */
    const float* knn_sel;
    const double* moments;
    const float* w_knn;     /* corr_block.knn_conv.0.weight [64,4] */
    const float* b_knn;     /* corr_block.knn_conv.0.bias   [64]   */
    const float* gnk_gamma; /* corr_block.knn_conv.1.weight [64]   */
    const float* gnk_beta;  /* corr_block.knn_conv.1.bias   [64]   */
    const float* preluk;    /* corr_block.knn_conv.2.weight [1]    */
    const float* w_kout;    /* corr_block.knn_out.weight [64,64]   */
    const float* b_kout;    /* corr_block.knn_out.bias   [64]      */
    float* corr_feat;       /* [B,N,64] or NULL */
    const float* corr_in;   /* [B,N,64], used only when y1 == NULL */
    const float* flow;      /* [B,N,3] */
    const float* w_cc; const float* b_cc;   /* update_block.motion_encoder.conv_corr [64,64],[64] */
    const float* w_cf; const float* b_cf;   /* update_block.motion_encoder.conv_flow [64,3],[64]  */
    const float* w_cm; const float* b_cm;   /* update_block.motion_encoder.conv      [61,128],[61] */
    float* motion;          /* [B,N,64] or NULL */
    int B, N;
} pvraft_corrfeat_args;

PVRAFT_API int pvraft_corr_feature_fwd(const pvraft_corrfeat_args* a, void* stream);

/* ------------------------------------------------------------------------------------------------
 * The ALU part of the feature head, for the tensor-core path (the 1x1 convolutions around it run as pvraft_tc_linear_fwd):
 *   kfeat[b,n,c] = max over the 32 selected candidates of PReLU(GroupNorm(knn_conv.0(f)))      (model/corr.py:86-92)
 *   cflow[b,n,c] = relu(conv_flow(flow))                                                        (model/update.py:17)
 * knn_sel [B,N,32,4] and moments [B,PVRAFT_MOMENTS] come from pvraft_corr_lookup_fwd; the GroupNorm statistics follow
 * from the moments, so no pass over the [B,64,N,32] tensor of the reference is needed.  flow/cflow may be NULL.
 * --------------------------------------------------------------------------------------------- */
typedef struct pvraft_knn_branch_args {
    const float* knn_sel;
    const double* moments;
    const float* w_knn;     /* corr_block.knn_conv.0.weight [64,4] */
    const float* b_knn;     /* corr_block.knn_conv.0.bias   [64]   */
    const float* gnk_gamma; /* corr_block.knn_conv.1.weight [64]   */
    const float* gnk_beta;  /* corr_block.knn_conv.1.bias   [64]   */
    const float* preluk;    /* corr_block.knn_conv.2.weight [1]    */
    float preluk_host;      /* the same slope as known to the host (selects the convex fast path without a device read);
                               NaN = read it from `preluk` (costs one stream synchronisation) */
    float* kfeat;           /* [B,N,64] */
    const float* flow;      /* [B,N,3] or NULL */
    const float* w_cf; const float* b_cf;   /* update_block.motion_encoder.conv_flow [64,3],[64] */
    float* cflow;           /* [B,N,64] or NULL */
    int B, N;
} pvraft_knn_branch_args;

PVRAFT_API int pvraft_knn_branch_fwd(const pvraft_knn_branch_args* a, void* stream);

/* ------------------------------------------------------------------------------------------------
 * ConvGRU.  Replaces model/update.py:31-40 with x = [inp, motion] (update.py:84).
 *   net, inp, motion [B,N,64] -> net_out [B,N,64]   (net_out may alias net)
 * --------------------------------------------------------------------------------------------- */
typedef struct pvraft_gru_args {
    const float* net;
    const float* inp;
    const float* motion;
    const float* w_z; const float* b_z;     /* update_block.gru.convz [64,192],[64] */
    const float* w_r; const float* b_r;     /* update_block.gru.convr */
    const float* w_q; const float* b_q;     /* update_block.gru.convq */
    float* net_out;
    int B, N;
} pvraft_gru_args;

PVRAFT_API int pvraft_gru_fwd(const pvraft_gru_args* a, void* stream);

/* ------------------------------------------------------------------------------------------------
 * SetConv edge stage: per point, over its 32 graph neighbours j:  y_e = P_j - P_i + W_e . (x_j - x_i)
 * (x = point coordinates; x_j - x_i is the graph's edge feature), reduced to per-channel max and min over the neighbours, with the
 * GroupNorm statistics of all N*32*C pre-activation values accumulated.  Replaces the gather +
 * fc1 + (statistics of) gn1 + max-pool of SetConv.forward, model/flot/gconv.py:65-80.
 *   fc1p [B,N,C], nbr [B,N,32] int32 (LOCAL neighbour ids), edge_feats [B,N,32,3] (= graph.edge_feats),
 *   w_fc1 [C,cin+3] (columns cin..cin+2 are read)
 *   -> ymax, ymin [B,N,C]; stats [B,8,2] accumulated.   C % 8 == 0, C <= 128.
 *   order [B,N] int32 or NULL: the LOCAL point processed r-th in every sample (pvraft_point_order_fwd: a Morton rank table).
 *   It changes no result, only which points a CTA works on at the same time, so that their overlapping neighbourhoods are
 *   gathered from L1 instead of L2.
 *   plan: the gather plan of (nbr, order), pvraft_edge_plan_fwd (16-byte aligned).  The kernel copies each tile's distinct rows
 *   into shared memory from it, or gathers the tile from global memory when it has more distinct rows than the table holds at
 *   this C; either way the results are the same bits.
 *   det_workspace: pvraft_setconv_edge_det_workspace_bytes(B) bytes or NULL ("Deterministic mode").
 * --------------------------------------------------------------------------------------------- */
PVRAFT_API int pvraft_setconv_edge_fwd(const float* fc1p, const int32_t* nbr, const float* edge_feats, const float* w_fc1, int cin,
                                       int B, int N, int C, float* ymax, float* ymin, double* stats, const int32_t* order,
                                       const void* plan, void* det_workspace, void* stream);
PVRAFT_API int64_t pvraft_setconv_edge_det_workspace_bytes(int B);

/* Gather plan of a kNN graph for pvraft_setconv_edge_fwd, independent of the features and of C: per tile of 32 consecutive
 * positions of the processing order (never straddling two samples), the distinct rows its 32 x 32 neighbour references and
 * 32 centres name, in slot order, and the slot of every reference.  nbr [B,N,32] int32, order [B,N] int32 or NULL (as for
 * pvraft_setconv_edge_fwd) -> plan, pvraft_edge_plan_bytes(B, N) bytes, sample-major: the plan of the first b samples of a
 * batch is its first pvraft_edge_plan_bytes(b, N) bytes.  Record layout in csrc/edge_plan.cuh. */
PVRAFT_API int pvraft_edge_plan_fwd(const int32_t* nbr, const int32_t* order, int B, int N, void* plan, void* stream);
PVRAFT_API int64_t pvraft_edge_plan_bytes(int B, int N);

/* ------------------------------------------------------------------------------------------------
 * FlowHead output stage + RAFT coordinate update.  Replaces model/update.py:69,71-72 (conv1, cat,
 * out_conv) after the SetConv's last GroupNorm+LeakyReLU (gconv.py:82-83), and
 * model/RAFTSceneFlow.py:45-46 (coords2 += delta; flow = coords2 - coords1).
 *   z3 [B,N,64] (setconv.fc3 output) + z3_stats, net [B,N,64], coords1/coords2 [B,N,3]
 *   -> delta [B,N,3], coords2_out [B,N,3] (may alias coords2), flow_out [B,N,3] (may be NULL)
 * --------------------------------------------------------------------------------------------- */
typedef struct pvraft_flowout_args {
    const float* z3;
    const double* z3_stats;
    const float* gn3_gamma; const float* gn3_beta; /* setconv.gn3 [64] */
    const float* net;
    const float* w_c1; const float* b_c1;          /* flow_head.conv1 [64,64],[64] */
    const float* w_o0; const float* b_o0;          /* flow_head.out_conv.0 [64,128],[64] */
    const float* w_o2; const float* b_o2;          /* flow_head.out_conv.2 [3,64],[3] */
    const float* coords1;
    const float* coords2;
    float* delta;
    float* coords2_out;
    float* flow_out;
    int B, N;
} pvraft_flowout_args;

PVRAFT_API int pvraft_flow_out_fwd(const pvraft_flowout_args* a, void* stream);

/* ------------------------------------------------------------------------------------------------
 * k nearest neighbours.  Backs knn_point (model/pointconv.py:28-39) and the adjacency of
 * Graph.construct_graph (model/flot/graph.py:53-60, which argsorts a full N x N matrix).
 *   xyz [B,N,3] (candidates), query [B,S,3] -> idx [B,S,k] int32 LOCAL candidate ids, unordered;
 *   rel [B,S,k,3] = xyz[idx] - query (the graph's edge features, graph.py:69-74), or NULL.
 * mode 0: distance = (|q|^2 + |x|^2) - 2 q.x      (graph.py:53-57 op order)
 * mode 1: distance = (-2 q.x + |q|^2) + |x|^2     (pointconv.py:21-24 op order)
 * with q.x = fma(qz,xz, fma(qy,xy, qx*xx)) and |.|^2 = (x*x+y*y)+z*z.  1 <= k <= 32, N >= k.
 * Ties at the k-th place: lowest candidate id.
 * workspace: pvraft_knn_workspace_bytes(B, N) bytes of device scratch (16-byte aligned) enable the
 * uniform-grid search for N >= 64 (the index sorted in shared memory up to N = 16384, by pvraft_grid_index_fwd's
 * counting sort above); with workspace == NULL (or N < 64) the brute-force kernel runs.  Both return the same
 * neighbours in the same order.
 * --------------------------------------------------------------------------------------------- */
PVRAFT_API int64_t pvraft_knn_workspace_bytes(int B, int N);
PVRAFT_API int pvraft_knn_fwd(const float* xyz, const float* query, int B, int N, int S, int k, int mode, int32_t* idx,
                   float* rel, void* workspace, void* stream);

/* A spatially coherent order of every cloud: perm[b, r] = index of the point that comes r-th along a Morton (Z-order) curve
 * over the cells of the kNN grid.  No counterpart in the reference (point order carries no meaning in model/*.py); the
 * RAFT driver uses it to make the SetConv gathers of consecutive points overlap in L1/L2.  64 <= N <= 16384;
 * workspace: pvraft_knn_workspace_bytes(B, N) bytes. */
PVRAFT_API int pvraft_point_order_fwd(const float* xyz, int B, int N, int32_t* perm, void* workspace, void* stream);

/* Uniform-grid index of S clouds of any size (no counterpart in the reference), the search structure of the kNN graphs
 * beyond 16384 points and of the *_grid_fwd searches below.  Built on the device with no host synchronisation (capturable):
 * per sample the bounding box, cells of edge h ~ cbrt(3 * volume / N) (at most max(32768, N) cells and 1024 along an axis),
 * and the points counting-sorted by cell id.
 *   xyz [S,N,3], offset [S,N,3] or NULL: the index is of xyz + offset (one fp32 add per coordinate), e.g. W = P + flow.
 *   workspace: pvraft_grid_index_workspace_bytes(S, N) bytes, 16-byte aligned; it holds, every block 16-byte aligned:
 *   float4 pts[S*N] (x, y, z, |p|^2 in cell order) | int32 ids[S*N] (the original ids) | int32 key[S*N] | int32 rank[S*N] |
 *   int32 cell_start[S * (cells + 1)] | per-sample grid parameters | scratch.  The order of the points inside a cell varies
 *   from run to run (an atomic histogram); every search on the index ranks on (distance, id), so its results do not.
 * Null pointers, S or N < 1 return PVRAFT_ERR_BAD_ARG, S > 65535 PVRAFT_ERR_UNSUPPORTED. */
PVRAFT_API int64_t pvraft_grid_index_workspace_bytes(int S, int N);
PVRAFT_API int pvraft_grid_index_fwd(const float* xyz, const float* offset, int S, int N, void* workspace, void* stream);

/* ================================================================================================
 * Gradient contract (SURVEY.md section 8b): what tools/engine.py:131-147 differentiates through.
 * The training path runs layer by layer; each backward entry point below pairs with a forward one.
 * Parameter-gradient outputs are ACCUMULATED with atomics into buffers the caller has zeroed (in an order that varies from
 * run to run; in a fixed order with a det_workspace, see "Deterministic mode").  The det_workspace of each entry point is
 * pvraft_<name>_det_workspace_bytes(...) bytes, declared beside it.
 * ============================================================================================= */

/* 1x1 convolution (pvraft_linear_fwd without prologue / activation), weight and bias gradient:
 *   x [rows,cin], dy [rows,cout]  ->  dW[o,i] += sum_r dy[r,o] x[r,i]  (row stride dw_ld floats, 0 = cin),  db[o] += sum_r dy[r,o] (or NULL).
 * The data gradient dx = dy . W is pvraft_linear_fwd with the transposed weight.  cin <= 256, cout <= 128. */
PVRAFT_API int pvraft_linear_wgrad(const float* x, const float* dy, int64_t rows, int cin, int cout, float* dW, int dw_ld, float* db,
                                   void* det_workspace, void* stream);
PVRAFT_API int64_t pvraft_linear_wgrad_det_workspace_bytes(int cin, int cout);
/* The same gradients on the tensor cores with bf16 operands (the 'bf16-mixed' training mode): the autograd of nn.Conv1d(k=1)
 * in model/update.py and model/flot/gconv.py, for the per-point layers of the RAFT loop.
 *   x [rows,cin], dy [rows,cout]  ->  dW[o,i] += sum_r bf16(dy[r,o]) bf16(x[r,i])  (round to nearest even, fp32 accumulation;
 *   row stride dw_ld floats, 0 = cin),  db[o] += sum_r dy[r,o]  (fp32, from the unrounded dy; or NULL).
 * rows >= 1; cin in {32,64,...,192} and cout in {32,64,96,128} (PVRAFT_ERR_UNSUPPORTED otherwise). */
PVRAFT_API int pvraft_tc_wgrad_bf16(const float* x, const float* dy, int64_t rows, int cin, int cout, float* dW, int dw_ld, float* db,
                                    void* det_workspace, void* stream);
PVRAFT_API int64_t pvraft_tc_wgrad_bf16_det_workspace_bytes(int cin, int cout);

/* GroupNorm(8) + activation backward (model/corr.py:17-18,25-26; model/flot/gconv.py:27-36 via autograd in the reference):
 *   x, dy [B,rows,C]; stats [B,8,2] raw sums of x (as produced in the forward); count = rows * C/8; act/slope as pvraft_gn_act_fwd
 *   -> dx [B,rows,C]; dgamma, dbeta [C] double (accumulated); dslope [1] double (PReLU slope gradient, or NULL);
 *      gsum [B,8,2] double scratch, ZEROED by the caller. */
PVRAFT_API int pvraft_gn_act_bwd(const float* x, const float* dy, const double* stats, const float* gamma, const float* beta, double count,
                                 int act, float slope, int B, int64_t rows, int C, double* gsum, double* dgamma, double* dbeta,
                                 double* dslope, float* dx, const float* slope_dev, const uint8_t* arg, void* det_workspace, void* stream);
PVRAFT_API int64_t pvraft_gn_act_bwd_det_workspace_bytes(int B, int C);
/* Backward of a linear layer with cin <= 4 and cout in {16,32,48,64,96,128} (the SetConv edge term and the knn_conv: rows = B*N*32) in one
 * pass over dy: dW [cout,dw_ld] += dy^T x, db [cout] += column sums (or NULL), dx [rows,cin] = dy W (or NULL).  W is [cout,w_ld]. */
PVRAFT_API int pvraft_linear_bwd_small(const float* x, const float* dy, const float* W, int64_t rows, int cin, int cout, int w_ld, float* dW,
                                       int dw_ld, float* db, float* dx, void* det_workspace, void* stream);
PVRAFT_API int64_t pvraft_linear_bwd_small_det_workspace_bytes(int cin, int cout);
/* GroupNorm + activation + max over each point's 32 consecutive rows, fused (model/flot/gconv.py:76-80, model/corr.py:87-92):
 *   x [B, pts*32, C] -> y [B,pts,C], arg [B,pts,C] uint8 (first row attaining the maximum); count = pts*32 * C/8.
 * Its backward is pvraft_gn_act_bwd with `arg` set and dy = d y [B,pts,C]: the dense, 31/32-zero gradient of the max is never formed. */
PVRAFT_API int pvraft_gn_act_maxk_fwd(const float* x, const double* stats, const float* gamma, const float* beta, double count, int act,
                           float slope, int B, int64_t pts_per_sample, int C, float* y, uint8_t* arg, const float* slope_dev, void* stream);

/* SetConv edge stage, layer-wise (model/flot/gconv.py:65-73, fc1 factorised as in pvraft_setconv_edge_fwd):
 *   forward : E[b,n,j,:] <- P[b,nbr[b,n,j],:] - P[b,n,:] + E[b,n,j,:]  (in place; E = W_e . edge_feats from pvraft_linear_fwd),
 *             stats [B,8,2] accumulated sums of the result (or NULL)
 *   backward: dP[b,nbr,:] += dT[b,n,j,:]; dP[b,n,:] -= sum_j dT[b,n,j,:]   (dP zeroed by the caller; dE = dT)
 *   P [B,N,C], nbr [B,N,32] int32 local ids, E/dT [B,N,32,C]. */
PVRAFT_API int pvraft_edge_fwd(const float* P, const int32_t* nbr, float* E, int B, int N, int C, double* stats, void* det_workspace,
                               void* stream);
PVRAFT_API int64_t pvraft_edge_fwd_det_workspace_bytes(int B);
PVRAFT_API int pvraft_edge_bwd(const float* dT, const int32_t* nbr, int B, int N, int C, float* dP, void* det_workspace, void* stream);
PVRAFT_API int64_t pvraft_edge_bwd_det_workspace_bytes(int B, int N, int C);

/* max over the 32 neighbours (model/flot/gconv.py:80, model/corr.py:92): x [pts,32,C] -> y [pts,C], arg [pts,C] uint8 (first
 * maximum); backward writes dx [pts,32,C] = dy at arg, 0 elsewhere. */
PVRAFT_API int pvraft_maxk_fwd(const float* x, int64_t pts, int C, float* y, uint8_t* arg, void* stream);
PVRAFT_API int pvraft_maxk_bwd(const float* dy, const uint8_t* arg, int64_t pts, int C, float* dx, void* stream);

/* Backward of pvraft_corr_lookup_fwd w.r.t. corr_val (model/corr.py:47-66,84; indices and coordinates carry no gradient:
 * corr.py:52-62 is under no_grad and RAFTSceneFlow.py:41 detaches the coordinates; the gradient w.r.t. the gather table
 * is pvraft_corr_lookup_xyz_bwd):
 *   g_vox [B,N,vox_ld], g_sel [B,N,32,4] (channel 0 used), knn_slot [B,N,32] from the forward, xyz2_pad [B,M,4]
 *   -> d_corr [B,N,K] (overwritten).  The means' divisor is clamp(count, 1, N), as in the forward. */
PVRAFT_API int pvraft_corr_lookup_bwd(const int32_t* corr_idx, const float* xyz2_pad, const float* coords, const int32_t* knn_slot,
                                      const float* g_vox, int vox_ld, const float* g_sel, int B, int N, int M, int K, int levels,
                                      float base_scale, float* d_corr, void* stream);
/* Backward of pvraft_corr_lookup_fwd's kNN 4-vectors w.r.t. the gather table (model/corr.py:42,88-89: knn_xyz =
 * truncate_xyz2[slot] - coords; the voxel branch's index math carries no gradient):
 *   corr_idx [B,N,K] (stored order, ids < M), knn_slot [B,N,32] from the forward, g_sel [B,N,32,4] (channels 1..3 used)
 *   -> d_xyz2[b, corr_idx[b,n,knn_slot[b,n,j]], c] += g_sel[b,n,j,1+c]   (d_xyz2 [B,M,3] ACCUMULATED, zeroed by the caller).
 * 32 <= K <= M. */
PVRAFT_API int pvraft_corr_lookup_xyz_bwd(const int32_t* corr_idx, const int32_t* knn_slot, const float* g_sel, int B, int N, int M, int K,
                                          float* d_xyz2, void* det_workspace, void* stream);
PVRAFT_API int64_t pvraft_corr_lookup_xyz_bwd_det_workspace_bytes(int B, int M);

/* Backward of the truncated correlation (model/corr.py:95-100 + the top-k gather of :37-38), sparse over the K kept entries:
 *   g [B,N,K], idx [B,N,K] (same stored order, ids < M), fmap1 [B,N,C], fmap2 [B,M,C] point-major
 *   -> d_fmap1 [B,N,C] (overwritten), d_fmap2 [B,M,C] (ACCUMULATED, zeroed by the caller).  C in {32,64,128,256}. */
PVRAFT_API int pvraft_corr_init_bwd(const float* g, const int32_t* idx, const float* fmap1, const float* fmap2, int B, int N, int M, int C,
                                    int K, float* d_fmap1, float* d_fmap2, void* det_workspace, void* stream);
PVRAFT_API int64_t pvraft_corr_init_bwd_det_workspace_bytes(int B, int M, int C);

/* Training extras on the device (SURVEY.md 8f row f3).  est, gt [points,3]; mask [points] (> 0 = valid) or NULL.
 *   pvraft_flow_metrics_fwd: acc[6] double, ZEROED by the caller, accumulates over the valid points
 *       [0] sum |ex|+|ey|+|ez|  (tools/loss.py:34-38: loss = acc[0] / (3 acc[1]))      [1] number of valid points
 *       [2] sum ||e||           (tools/metric.py:24-29: EPE = acc[2] / acc[1])
 *       [3],[4],[5] points with (epe<.05 or rel<.05), (epe<.1 or rel<.1), (epe>.3 or rel>.1), rel = epe/(||gt||+1e-4)  (metric.py:66-77)
 *   pvraft_flow_l1_bwd: d_est = g[0] * weight * sign(est - gt) / (3 acc[1]) on valid points, 0 elsewhere; g is a DEVICE scalar
 *       (the upstream gradient), acc the forward's accumulator: no host synchronisation between forward and backward. */
PVRAFT_API int pvraft_flow_metrics_fwd(const float* est, const float* gt, const float* mask, int64_t points, double* acc, void* det_workspace,
                                       void* stream);
PVRAFT_API int64_t pvraft_flow_metrics_det_workspace_bytes(void);
PVRAFT_API int pvraft_flow_l1_bwd(const float* est, const float* gt, const float* mask, int64_t points, const double* acc, const float* g,
                       float weight, float* d_est, void* stream);

/* Self-supervised losses (no counterpart in the reference, which trains on ground truth only): the Chamfer distance between
 * the first cloud moved by the flow and the second cloud, and the smoothness of the flow over the first cloud's kNN graph.
 * S = n*B samples (n predictions of a batch of B, stacked); sample s pairs with batch entry s % B, so the second cloud and the
 * graph are never copied per prediction.  ||v||^2 is (vx*vx + vy*vy) + vz*vz of the fp32 difference vector, rounded to
 * nearest at every step, never contracted.  Null pointers, S < 1, B < 1, S % B != 0, N < 1, M < 1 and k outside 1..32 return
 * PVRAFT_ERR_BAD_ARG before any launch.
 *   pvraft_chamfer_fwd: a [S,N,3] (W = P1 + flow), b [B,M,3] (P2)
 *       -> nn_ab [S,N] int32: argmin_j ||a[s,i] - b[s%B,j]||^2;  nn_ba [S,M] int32: argmin_i ||a[s,i] - b[s%B,j]||^2
 *          (exact ties: the lowest index), and acc [S,2] double, ZEROED by the caller, accumulates the sums of the minima
 *          (acc[s,0] over i, acc[s,1] over j): C_s = acc[s,0] / N + acc[s,1] / M.  A brute-force search: 2 S N M pairs.
 *   pvraft_chamfer_bwd: g [S] the DEVICE upstream gradient of C_s
 *       -> d_a [S,N,3] += 2 g_s/N (a_i - b_nn(i)) and, for every j, d_a[nn_ba(j)] += 2 g_s/M (a_nn(j) - b_j);  d_b [B,M,3] the
 *          negated terms at the other end of each pair (or NULL).  Both ACCUMULATED, zeroed by the caller.
 *   pvraft_flow_smooth_fwd: f [S,N,3], nbr [B,N,k] int32 local ids (sample s uses nbr[s % B])
 *       -> acc [S] double (ZEROED by the caller) += sum_i sum_e ||f[s,nbr[i,e]] - f[s,i]||:  S_s = acc[s] / (N k).
 *   pvraft_flow_smooth_bwd: g [S] DEVICE -> d_f [S,N,3] (ACCUMULATED, zeroed by the caller): for every edge (i, j = nbr[i,e]),
 *       u = g_s/(N k) (f_j - f_i)/||f_j - f_i|| (0 where f_j = f_i), d_f[j] += u, d_f[i] -= u. */
PVRAFT_API int pvraft_chamfer_fwd(const float* a, const float* b, int S, int B, int N, int M, int32_t* nn_ab, int32_t* nn_ba, double* acc,
                                  void* det_workspace, void* stream);
PVRAFT_API int64_t pvraft_chamfer_fwd_det_workspace_bytes(int S);
PVRAFT_API int pvraft_chamfer_bwd(const float* a, const float* b, const int32_t* nn_ab, const int32_t* nn_ba, const float* g, int S, int B,
                                  int N, int M, float* d_a, float* d_b, void* det_workspace, void* stream);
/* The same pvraft_chamfer_fwd results (nn_ab, nn_ba bitwise; acc up to summation order) from a search on uniform-grid
 * indices of b and of a instead of 2 S N M pairs.  workspace: pvraft_chamfer_grid_workspace_bytes(S, B, N, M) bytes,
 * 16-byte aligned (the indices: pvraft_grid_index_workspace_bytes(B, M) + pvraft_grid_index_workspace_bytes(S, N));
 * det_workspace: pvraft_chamfer_fwd_det_workspace_bytes(S) bytes or NULL. */
PVRAFT_API int64_t pvraft_chamfer_grid_workspace_bytes(int S, int B, int N, int M);
PVRAFT_API int pvraft_chamfer_grid_fwd(const float* a, const float* b, int S, int B, int N, int M, int32_t* nn_ab, int32_t* nn_ba,
                                       double* acc, void* workspace, void* det_workspace, void* stream);
PVRAFT_API int64_t pvraft_chamfer_bwd_det_workspace_bytes(int S, int B, int N, int M);
PVRAFT_API int pvraft_flow_smooth_fwd(const float* f, const int32_t* nbr, int S, int B, int N, int k, double* acc, void* det_workspace,
                                      void* stream);
PVRAFT_API int64_t pvraft_flow_smooth_fwd_det_workspace_bytes(int S);
PVRAFT_API int pvraft_flow_smooth_bwd(const float* f, const int32_t* nbr, const float* g, int S, int B, int N, int k, float* d_f,
                                      void* det_workspace, void* stream);
PVRAFT_API int64_t pvraft_flow_smooth_bwd_det_workspace_bytes(int S, int N);

/* The Laplacian regularity term of the self-supervised loss (PointPWC-Net's third term): the local shape of W = P1 + flow
 * should match the local shape of P2 around the same place.  Same sample stacking as above (sample s pairs with batch entry
 * s % B); graphs are int32 local ids of k_lap neighbours that include the point itself (pvraft_knn_fwd, mode 0); squared
 * distances in the difference form of pvraft_chamfer_fwd.  Null pointers, S < 1, B < 1, S % B != 0, N < 1, M < 1, k_lap
 * outside 2..min(32, N) and k_int outside 1..min(8, M) return PVRAFT_ERR_BAD_ARG before any launch.
 *   pvraft_cloud_laplacian_fwd: x [B,N,3], nbr [B,N,k] (2 <= k <= min(32, N))
 *       -> out [B,N,3]: L(x)_i = sum_e (x[nbr[i,e]] - x_i) / (k - 1), fp32 summed in edge order (a self edge adds 0).  Every
 *          output is written once: no det_workspace.
 *   pvraft_cloud_laplacian_bwd: g_l [B,N,3] -> d_x [B,N,3] (ACCUMULATED, zeroed by the caller): c = g_l[i] / (k - 1),
 *       d_x[nbr[i,e]] += c for every edge with nbr[i,e] != i, d_x[i] -= c per such edge.
 *   pvraft_laplacian_fwd: w [S,N,3] (W), p2 [B,M,3], l2 [B,M,3] (pvraft_cloud_laplacian_fwd of p2 over its own graph),
 *       g1 [B,N,k_lap] (P1's graph)
 *       -> nn_idx [S,N,k_int] int32: the k_int nearest of w[s,i] in p2[s%B] ranked on (||w_i - p2_j||^2, j), nearest first
 *          (an unfilled slot, possible only with non-finite coordinates, reads -1);
 *          res [S,N,3]: Lhat_i - L(w)_i with Lhat_i = sum_r w_r l2[j_r] / sum_r w_r, w_r = 1 / (d_r + 1e-8) on the SQUARED
 *          distance d_r (fp32, nearest first), and L(w) over g1;
 *          acc [S] double (ZEROED by the caller) += sum_i ||res_i||^2, each point's term in double:  R_s = acc[s] / N.
 *          A brute-force search of S N M pairs.
 *   pvraft_laplacian_bwd: g [S] the DEVICE upstream gradient of R_s, the forward's nn_idx and res, neighbours held fixed;
 *       e_i = 2 g_s / N res_i ->
 *          d_w [S,N,3]: -e_i/(k_lap-1) at every neighbour j != i of g1(i) and +e_i/(k_lap-1) per such edge at i, plus at i
 *          sum_r (dLhat/dd_r . e_i) 2 (w_i - p2_{j_r}) with dLhat/dd_r = -(w_r / sum w)^2 sum_q w_q (l2_{j_r} - l2_{j_q});
 *          d_p2 [B,M,3] (or NULL): the negated distance terms at p2_{j_r};  d_l2 [B,M,3] (or NULL): (w_r / sum w) e_i at j_r.
 *          All ACCUMULATED, zeroed by the caller; d_l2 reaches p2 through pvraft_cloud_laplacian_bwd.
 * Accumulation: acc in double atomics, the gradients in fp32 atomics (order varies run to run); with a det_workspace all in
 * the fixed-point form ("Deterministic mode"). */
PVRAFT_API int pvraft_cloud_laplacian_fwd(const float* x, const int32_t* nbr, int B, int N, int k, float* out, void* stream);
PVRAFT_API int pvraft_cloud_laplacian_bwd(const float* g_l, const int32_t* nbr, int B, int N, int k, float* d_x, void* det_workspace,
                                          void* stream);
PVRAFT_API int64_t pvraft_cloud_laplacian_bwd_det_workspace_bytes(int B, int N);
PVRAFT_API int pvraft_laplacian_fwd(const float* w, const float* p2, const float* l2, const int32_t* g1, int S, int B, int N, int M, int k_lap,
                                    int k_int, int32_t* nn_idx, float* res, double* acc, void* det_workspace, void* stream);
PVRAFT_API int64_t pvraft_laplacian_fwd_det_workspace_bytes(int S);
/* The same pvraft_laplacian_fwd results (nn_idx and res bitwise; acc up to summation order) from a search on a uniform-grid
 * index of p2.  workspace: pvraft_grid_index_workspace_bytes(B, M) bytes, 16-byte aligned; det_workspace:
 * pvraft_laplacian_fwd_det_workspace_bytes(S) bytes or NULL. */
PVRAFT_API int pvraft_laplacian_grid_fwd(const float* w, const float* p2, const float* l2, const int32_t* g1, int S, int B, int N, int M,
                                         int k_lap, int k_int, int32_t* nn_idx, float* res, double* acc, void* workspace,
                                         void* det_workspace, void* stream);
PVRAFT_API int pvraft_laplacian_bwd(const float* w, const float* p2, const float* l2, const int32_t* g1, const int32_t* nn_idx, const float* res,
                                    const float* g, int S, int B, int N, int M, int k_lap, int k_int, float* d_w, float* d_p2, float* d_l2,
                                    void* det_workspace, void* stream);
PVRAFT_API int64_t pvraft_laplacian_bwd_det_workspace_bytes(int S, int B, int N, int M);

/* The forward-backward consistency of a pair of flows (UnFlow's term and occlusion test, for scene flow): W = P1 + f12 moved
 * by the reverse flow found there should land back on P1.  Same sample stacking as above (sample s pairs with batch entry
 * s % B of p2 and with prediction s of f21); the search and the interpolation are pvraft_laplacian_fwd's, bit for bit, with
 * the reverse flow as the interpolated field.  Null pointers, S < 1, B < 1, S % B != 0, N < 1, M < 1, k outside
 * 1..min(8, M), and alpha or beta negative or not finite return PVRAFT_ERR_BAD_ARG before any launch.
 *   pvraft_flow_consistency_fwd: w [S,N,3] (W = P1 + f12), f12 [S,N,3], p2 [B,M,3], f21 [S,M,3]
 *       -> nn_idx [S,N,k] int32: the k nearest of w[s,i] in p2[s%B] ranked on (||w_i - p2_j||^2, j), nearest first (an
 *          unfilled slot, possible only with non-finite coordinates, reads -1);
 *          res [S,N,3]: r_i = f12_i + bhat_i, bhat_i = sum_r w_r f21[s,j_r] / sum_r w_r, w_r = 1 / (d_r + 1e-8) on the SQUARED
 *          distance d_r (fp32, nearest first);
 *          ok [S,N] uint8: ||r_i||^2 < alpha (||f12_i||^2 + ||bhat_i||^2) + beta, each squared length in double;
 *          acc [S] double (ZEROED by the caller) += sum_i ||r_i||^2, each point's term in double:  F_s = acc[s] / N.
 *          A brute-force search of S N M pairs.
 *   pvraft_flow_consistency_bwd: g [S] the DEVICE upstream gradient of F_s, the forward's nn_idx and res, neighbours held
 *       fixed; e_i = 2 g_s / N r_i ->
 *          d_f12 [S,N,3] = e_i and d_w [S,N,3] = sum_r (dbhat/dd_r . e_i) 2 (w_i - p2_{j_r}), dbhat/dd_r = -(w_r / sum w)^2
 *          sum_q w_q (f21_{j_r} - f21_{j_q}): both WRITTEN, every element once;
 *          d_p2 [B,M,3] (or NULL): the negated distance terms at p2_{j_r};  d_f21 [S,M,3]: (w_r / sum w) e_i at j_r.  Both
 *          ACCUMULATED, zeroed by the caller.
 * Accumulation: acc in double atomics, d_p2 and d_f21 in fp32 atomics (order varies run to run); with a det_workspace in the
 * fixed-point form ("Deterministic mode"). */
PVRAFT_API int pvraft_flow_consistency_fwd(const float* w, const float* f12, const float* p2, const float* f21, int S, int B, int N, int M,
                                           int k, float alpha, float beta, int32_t* nn_idx, float* res, uint8_t* ok, double* acc,
                                           void* det_workspace, void* stream);
PVRAFT_API int64_t pvraft_flow_consistency_fwd_det_workspace_bytes(int S);
/* The same pvraft_flow_consistency_fwd results (nn_idx, res and ok bitwise; acc up to summation order) from a search on a
 * uniform-grid index of p2.  workspace: pvraft_grid_index_workspace_bytes(B, M) bytes, 16-byte aligned; det_workspace:
 * pvraft_flow_consistency_fwd_det_workspace_bytes(S) bytes or NULL. */
PVRAFT_API int pvraft_flow_consistency_grid_fwd(const float* w, const float* f12, const float* p2, const float* f21, int S, int B, int N,
                                                int M, int k, float alpha, float beta, int32_t* nn_idx, float* res, uint8_t* ok,
                                                double* acc, void* workspace, void* det_workspace, void* stream);
PVRAFT_API int pvraft_flow_consistency_bwd(const float* w, const float* p2, const float* f21, const int32_t* nn_idx, const float* res,
                                           const float* g, int S, int B, int N, int M, int k, float* d_w, float* d_f12, float* d_p2,
                                           float* d_f21, void* det_workspace, void* stream);
PVRAFT_API int64_t pvraft_flow_consistency_bwd_det_workspace_bytes(int S, int B, int M);

/* Flow propagation along a scan sequence (no counterpart in the reference, which estimates one pair at a time): carries a
 * flow defined on one cloud onto the points of another, the warm start of the next pair under a constant-velocity
 * assumption (pvraft_b200.stream.SceneFlowStream).
 *   xyz_prev [B,M,3], flow_prev [B,M,3] (the flow on xyz_prev's points), xyz [B,N,3]
 *   -> for every query q of xyz, the k nearest of the moved points W = xyz_prev + flow_prev (formed in the kernel, one fp32
 *      add per coordinate), ranked by ||q - W_j||^2 = (dx*dx + dy*dy) + dz*dz of the fp32 difference vector, rounded to
 *      nearest at every step, never contracted, on (distance, index): exact ties go to the lowest index.
 *      flow_out [B,N,3]: sum_j w_j flow_prev[j] / sum_j w_j with w_j = 1 / (sqrt_rn(d_j) + 1e-8), summed in fp32 nearest first;
 *      idx_out [B,N,k] int32 (or NULL): the neighbours, nearest first.
 * A brute-force search of B N M pairs.  No det_workspace: no value is accumulated with atomics, and every sum runs in a fixed
 * order inside one thread, so the result is bitwise reproducible as it is.  Null inputs or flow_out, B, M or N < 1, and k
 * outside 1..min(8, M) return PVRAFT_ERR_BAD_ARG before any launch. */
PVRAFT_API int pvraft_flow_propagate_fwd(const float* xyz_prev, const float* flow_prev, const float* xyz, int B, int M, int N, int k,
                                         float* flow_out, int32_t* idx_out, void* stream);
/* The same pvraft_flow_propagate_fwd results, bitwise, from a search on a uniform-grid index of W = xyz_prev + flow_prev
 * (built with flow_prev as its offset: the same fp32 add).  workspace: pvraft_grid_index_workspace_bytes(B, M) bytes,
 * 16-byte aligned.  No det_workspace, for the same reason. */
PVRAFT_API int pvraft_flow_propagate_grid_fwd(const float* xyz_prev, const float* flow_prev, const float* xyz, int B, int M, int N, int k,
                                              float* flow_out, int32_t* idx_out, void* workspace, void* stream);

/* Euclidean clustering (single linkage; no counterpart in the reference), the segments of pvraft_rigid_objects_fwd.  Integer
 * decisions only: the outputs are the same bits in every mode and from run to run, so there is no det_workspace.
 *   Edges: points i != j of one sample are adjacent when both take part -- mask[b,i] != 0 (every point with mask NULL) and
 *       all three coordinates finite -- and diff_sq(x_i, x_j) <= fl(radius * radius), diff_sq the fp32 difference form of
 *       the searches ((dx dx + dy dy) + dz dz, every operation rounded to nearest, none contracted); with flow != NULL also
 *       diff_sq(f_i, f_j) <= fl(flow_radius * flow_radius) (a non-finite flow then has no edge).
 *   Components: the connected components of that graph; a component's key is its smallest point id.  The result does not
 *       depend on the order of any atomic operation.
 *   Objects: the components of >= min_points points, ranked by size (descending), then by smallest id (ascending); the
 *       first max_objects are objects 0 .. num_objects[b] - 1.
 *   pvraft_euclidean_clusters_fwd: xyz [B,N,3], flow [B,N,3] or NULL, mask [B,N] uint8 or NULL -> labels [B,N] int32 (the
 *       object, -1 for none), num_objects [B] int32, sizes [B,max_objects] int32 (each object's number of points, 0 for an
 *       empty slot).  workspace: pvraft_euclidean_clusters_workspace_bytes(B, N) bytes, 16-byte aligned, no initialisation
 *       needed.  No host synchronisation.
 * Null required pointers, B < 1, N < 1, B N >= 2^31, a radius (or, with flow, a flow_radius) that is not finite and > 0 or
 * whose square overflows fp32, min_points < 1 and max_objects outside 1..256 return PVRAFT_ERR_BAD_ARG before any launch;
 * B > 65535 PVRAFT_ERR_UNSUPPORTED. */
PVRAFT_API int pvraft_euclidean_clusters_fwd(const float* xyz, const float* flow, const uint8_t* mask, int B, int N, float radius,
                                             float flow_radius, int min_points, int max_objects, int32_t* labels, int32_t* num_objects,
                                             int32_t* sizes, void* workspace, void* stream);
PVRAFT_API int64_t pvraft_euclidean_clusters_workspace_bytes(int B, int N);

/* A robust rigid fit of a flow (no counterpart in the reference): RANSAC over minimal samples and a Horn/Kabsch refit, such
 * that xyz1 R^T + t ~ xyz1 + flow on the inliers, once per SEGMENT.  Sample b has O segments: segment (b, o) is the points
 * with labels[b,i] == o (a value outside 0 .. O - 1 is in no segment); with labels NULL (only with O = 1) segment (b, 0) is
 * every point of the sample.  pvraft_b200.rigid_motion, the sensor's ego-motion, is O = 1 (labels[b,i] = 0 where its mask
 * allows the point, -1 elsewhere, or NULL without a mask); pvraft_b200.rigid_objects one segment per object, with the labels
 * pvraft_euclidean_clusters_fwd writes.  Every segment is fitted as the same call with B = 1, O = 1 and labels =
 * (labels[b] == o ? 0 : -1) fits it: below, "allowed" means a member of the segment.  y = x + f is formed in fp32 (one
 * rounded add per coordinate) wherever it appears.  No host synchronisation; every output element is written.
 *   Sampling: hypothesis h < H draws r = 0, 1, 2: j_r = splitmix64((seed << 32) | (h << 2) | r) mod n_allowed, an index into
 *       the segment's ascending list of allowed points, where splitmix64(k) = mix(k + 0x9e3779b97f4a7c15), mix(z) = z3 ^
 *       (z3 >> 31), z2 = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9, z3 = (z2 ^ (z2 >> 27)) * 0x94d049bb133111eb (uint64
 *       arithmetic).  The key leaves out the sample and the segment index: a batched call equals per-sample calls.  The
 *       triple is REJECTED (never redrawn) when n_allowed = 0, two j_r are equal, it is near-collinear: NOT |a x b|^2 >
 *       1e-6 |a|^2 |b|^2 (a = x1 - x0, b = x2 - x0; coincident points are rejected too), or one of its pairwise distances
 *       (0-1, 0-2, 1-2) changes by more than 2 threshold: NOT | ||x_i - x_j|| - ||y_i - y_j|| | <= 2 threshold.  Both tests
 *       in double on the fp32 coordinates, each operation rounded to nearest, none contracted (|u|^2 = (u0 u0 + u1 u1) +
 *       u2 u2, cross products as a1 b2 - a2 b1, ...).
 *   Minimal fit: Horn's closed form about the triple's centroids (c_x, c_y): the eigenvector of the largest eigenvalue of
 *       the 4x4 N(S), S = sum (x - c_x)(y - c_y)^T, by cyclic Jacobi sweeps in double; a proper rotation always.  The model
 *       (R, c_x, c_y) is stored in fp32.
 *   Score: count of allowed points with ||r||^2 <= threshold^2 (fp32 threshold * threshold), r = R (x - c_x) - (y - c_y),
 *       in fp32: d = x - c_x, e = y - c_y, r_k = ((R_k0 d_0 + R_k1 d_1) + R_k2 d_2) - e_k, ||r||^2 = (r_0^2 + r_1^2) + r_2^2,
 *       each operation rounded to nearest, none contracted.  Integer counts; the best hypothesis has the most inliers, the
 *       lowest h on ties.  The scoring takes (allowed points) x H residual tests, not O N H.
 *   Refit, `rounds` times: the inliers are the allowed points within the threshold (the same test) of the current model --
 *       the best hypothesis, then the previous round's (R, x-bar, y-bar) -- and get the unweighted Horn fit from their
 *       moments (n, sum dx, sum dy, sum dx dy^T) in double about the current model's (c_x, c_y); x-bar = c_x + sum dx / n,
 *       t = y-bar - R x-bar.  The last round's inliers are inliers_out.  The moments are summed per window of 256 point ids
 *       and the windows' partial sums added, so in the deterministic mode a segment's R, t, count, degenerate, state and
 *       inliers are the same bits as those of its B = 1, O = 1 call.
 *   Degenerate: n < 3, or lambda0 - lambda1 <= 1e-5 lambda0 (the top two eigenvalues of N(S): collinear or coincident
 *       inliers): R = I, t = y-bar - x-bar (0 with no inlier), degenerate = 1.  A segment none of whose hypotheses is
 *       accepted takes every allowed point as an inlier in every round and is degenerate; a segment with no member gets
 *       R = I, t = 0, count 0, degenerate 1.
 *   pvraft_rigid_objects_fwd: xyz1, flow [B,N,3], labels [B,N] int32 or NULL (O = 1) -> R [B,O,3,3] and t [B,O,3] fp32,
 *       inliers [B,N] uint8 (an inlier of its own segment's fit), count [B,O] int32, degenerate [B,O] uint8, state [B,O,32]
 *       double (pvraft_rigid_objects_bwd's input: eigenvectors at [4j, 4j+4), eigenvalues [16, 20) (the top first), x-bar
 *       [20, 23), y-bar [23, 26), n, degenerate); optional (NULL to skip): triples [B O,H,3] int32, the drawn point indices
 *       (-1 with no allowed point), hyp_count [B O,H] int32, the counts (-1 for a rejected triple).  workspace:
 *       pvraft_rigid_objects_workspace_bytes(B, N, O, H, rounds) bytes, 16-byte aligned, no initialisation needed;
 *       det_workspace: pvraft_rigid_objects_fwd_det_workspace_bytes(B, O, rounds) bytes or NULL ("Deterministic mode": the
 *       moments in fixed point, so R and t are the same bits from run to run).  The counts, the selection and the inlier
 *       sets are integer decisions and do not depend on the mode except through R and t.
 *   pvraft_rigid_objects_bwd: dR [B,O,3,3], dt [B,O,3] the DEVICE upstream gradients, the forward's labels, inliers and
 *       state, the inlier sets held fixed -> d_xyz1, d_flow [B,N,3], every element WRITTEN once (zero off the inliers): dt
 *       gives d y-bar += dt, d x-bar -= R^T dt, dR -= dt x-bar^T; dR -> dq through R(q); dq -> dN = sym(sum_{j>=1} v_j v_j^T
 *       dq v0^T / (lambda0 - lambda_j)); dN -> dS; per inlier dx_i = dS (y_i - y-bar) + d x-bar / n, dy_i = dS^T (x_i -
 *       x-bar) + d y-bar / n; d_flow = dy, d_xyz1 = dx + dy.  Degenerate segments propagate the translation only.  A point
 *       belongs to at most one segment, so there are no atomics: the result is bitwise reproducible as it is.
 * Null required pointers, labels NULL with O != 1, B < 1, N < 1, B N >= 2^31, O outside 1..256, H outside 1..4096, rounds
 * outside 1..8, a threshold that is not finite and > 0, and seed < 0 return PVRAFT_ERR_BAD_ARG before any launch; B O > 65535
 * PVRAFT_ERR_UNSUPPORTED. */
PVRAFT_API int pvraft_rigid_objects_fwd(const float* xyz1, const float* flow, const int32_t* labels, int B, int N, int O, float threshold,
                                        int H, int rounds, int seed, float* R, float* t, uint8_t* inliers, int32_t* count,
                                        uint8_t* degenerate, double* state, int32_t* triples, int32_t* hyp_count, void* workspace,
                                        void* det_workspace, void* stream);
PVRAFT_API int64_t pvraft_rigid_objects_workspace_bytes(int B, int N, int O, int H, int rounds);
PVRAFT_API int64_t pvraft_rigid_objects_fwd_det_workspace_bytes(int B, int O, int rounds);
PVRAFT_API int pvraft_rigid_objects_bwd(const float* xyz1, const float* flow, const int32_t* labels, const uint8_t* inliers,
                                        const double* state, const float* dR, const float* dt, int B, int N, int O, float* d_xyz1,
                                        float* d_flow, void* stream);

/* sizeof() of the argument structs as compiled into the library (0 = linear, 1 = corrfeat, 2 = gru, 3 = flowout,
 * 4 = tc_linear, 5 = knn_branch, 6 = update_chain; -1 otherwise): lets a foreign-language binding verify its struct layout
 * at load time. */
PVRAFT_API int pvraft_sizeof(int which);

/* [B,C,N] <-> [B,N,C] transposes used at the reference-layout seams of the Python modules. */
PVRAFT_API int pvraft_transpose_fwd(const float* in, int B, int R, int C, float* out, void* stream); /* [B,R,C] -> [B,C,R] */

#ifdef __cplusplus
}
#endif
#endif /* PVRAFT_B200_H */
