/*
 * b200sht -- C ABI of the H100-native (sm_90a) spherical-harmonic hot path (RealSHT / InverseRealSHT / SpectralConv).
 *
 * Nothing equivalent exists in the reference: NVIDIA/makani has no native code (SURVEY.md F2) and reaches this
 * arithmetic through the Python package torch-harmonics.  Each entry point below names the reference interface
 * it replaces (paths relative to /root/reference):
 *
 *   b200sht_plan_create          <- torch_harmonics.RealSHT.__init__ / InverseRealSHT.__init__ as constructed at
 *                                   makani/models/networks/sfnonet.py:792-805 (Legendre table + quadrature precompute)
 *   b200sht_sht_forward          <- RealSHT.forward            (call site makani/models/common/spectral_convolution.py:239)
 *   b200sht_sht_inverse          <- InverseRealSHT.forward     (call sites spectral_convolution.py:241,253)
 *   b200sht_sht_forward_adjoint  <- autograd backward of RealSHT.forward (rfft + einsum adjoints)
 *   b200sht_sht_inverse_adjoint  <- autograd backward of InverseRealSHT.forward
 *   b200sht_mix_forward/backward <- makani/models/common/contractions.py:19-54 (_contract_* einsums) and :62-151
 *   b200sht_spectral_conv_forward<- SpectralConv.forward       (spectral_convolution.py:213-264), one call
 *   b200sht_complex_relu_*       <- makani/models/common/activations.py:88-127 (ComplexReLU)
 *   b200sht_vsht_forward         <- torch_harmonics.RealVectorSHT.forward         (makani/utils/losses/base_loss.py:427-469 VortDivBaseLoss)
 *   b200sht_vsht_inverse         <- torch_harmonics.InverseRealVectorSHT.forward  (base_loss.py:427-469 and :518-565 GradientBaseLoss)
 *   b200sht_vsht_*_adjoint       <- autograd backward of the two vector transforms
 *   b200sht_disco_forward/adjoint<- the psi contraction of torch_harmonics.DiscreteContinuousConvS2 and its adjoint (fourcastnet3.py:117-252, :511-543)
 *   b200sht_resample_forward/adjoint <- torch_harmonics.ResampleS2(mode="bilinear") and its adjoint (fourcastnet3.py:356-358)
 *   b200sht_attention_forward/backward <- the attention of torch_harmonics.NeighborhoodAttentionS2 (not constructed by makani)
 *
 * Conventions
 *   - every function returns 0 on success, a negative b200sht_status otherwise; b200sht_last_error() gives text.
 *   - all data pointers are DEVICE pointers owned by the caller (e.g. the PyTorch caching allocator) unless a
 *     parameter is documented as host memory.  The library allocates only inside plans (Legendre table, FFT
 *     twiddles, TMA descriptors).
 *   - every launch takes the cudaStream_t to enqueue on (as void*), is asynchronous and never synchronises.
 *   - plans are immutable after creation and may be shared by concurrent calls on different streams.
 *   - no thread-local state except the last-error string.
 *
 * Internal ("packed") tensor formats -- opaque to callers that only use the *_sht_* / spectral_conv entry points,
 * documented in DESIGN.md section 3:
 *   latspec  float [mmax8][2][B*C][kp]          (after the longitude FFT;  kp = nlat rounded up to 8, mmax8 = mmax rounded up to 8)
 *   spec     float [lmax][mmax][2][B][cp]       (spectral coefficients;    cp = C rounded up to 4)
 */
#ifndef B200SHT_H
#define B200SHT_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  B200SHT_OK = 0,
  B200SHT_ERR_INVALID = -1,      /* bad argument (shape, dtype, null pointer)            */
  B200SHT_ERR_CUDA = -2,         /* a CUDA runtime/driver call failed                    */
  B200SHT_ERR_UNSUPPORTED = -3,  /* valid request this build cannot serve (e.g. FFT len) */
  B200SHT_ERR_NOMEM = -4
} b200sht_status;

typedef enum { B200SHT_F32 = 0, B200SHT_BF16 = 1 } b200sht_dtype;

/* arithmetic of the Legendre / channel-mix contractions */
typedef enum {
  B200SHT_PREC_FP32 = 0, /* fp32 FMA on CUDA cores (reference tests run with TF32 disabled)          */
  B200SHT_PREC_TF32 = 1, /* TF32 tensor-core MMA (mma.sync), fp32 accumulate (reference training: allow_tf32) */
  B200SHT_PREC_FP32X3 = 2 /* fp32 operands on the tensor cores: Legendre stages as 3 x TF32 (hi.hi + hi.lo + lo.hi into one fp32 accumulator),
                             longitude transform and channel mix as in FP32.  Element errors stay inside rtol 1e-5 (atol = rtol max|ref|), relative
                             L2 ~ 1e-6 .. 8e-6 growing with nlat (the tensor core truncates its fp32 accumulator on every add; the CUDA-core FP32 mode
                             rounds to nearest and stays at ~ 3e-7): ~1.7 x the speed of FP32 at 721 x 1440.  Uses a per-device scratch buffer for the
                             operand residuals: issue calls of this mode from one stream per device.                                          */
} b200sht_precision;

typedef enum {
  B200SHT_OP_DHCONV = 0,      /* weight [G][Ci][Co][L]        contractions.py:23  */
  B200SHT_OP_DIAGONAL = 1,    /* weight [G][Ci][Co][L][M]     contractions.py:19  */
  B200SHT_OP_SEP_DHCONV = 2,  /* weight [G][Ci][L]            contractions.py:31  */
  B200SHT_OP_SEP_DIAGONAL = 3,/* weight [G][Ci][L][M]         contractions.py:27  */
  B200SHT_OP_SHARED = 4,      /* weight [Ci][Co]              contractions.py:62  (compl_mul2d_fwd)     */
  B200SHT_OP_LDEP = 5         /* weight [L][Ci][Co]           contractions.py:106 (compl_exp_mul2d_fwd) */
} b200sht_mix_op;

/* or-ed into `op` (mix) / `mode` (ComplexReLU): the packed spec operands store every (l, m) entry (no block triangle) */
#define B200SHT_DENSE_FLAG 0x100

typedef struct b200sht_plan b200sht_plan;

const char* b200sht_last_error(void);
int b200sht_version(void);

/* ---------------------------------------------------------------------------------------------- plan */
/* cost/quad_w: HOST arrays [nlat]: cos(colatitude) in row order (row 0 = north) and quadrature weights on [-1,1].
 * The Legendre table P[m][l][k] (orthonormal, optional Condon-Shortley phase) is built on the device in fp64
 * and stored as fp32 [mmax][lmax][kp]. */
int b200sht_plan_create(b200sht_plan** plan, int nlat, int nlon, int lmax, int mmax,
                        const double* cost, const double* quad_w, int csphase, void* stream);
/* Extended creation for the h x w model-parallel (distributed) SHT and for the vector SHT:
 *   m_offset : the plan's orders are m_offset .. m_offset + mmax - 1 (this rank's shard of the orders)
 *   flags & B200SHT_PLAN_FFT_ONLY: no Legendre table: nlat is this rank's latitude count, quad_w its slice of the weights
 *   flags & B200SHT_PLAN_VECTOR:   vector-SHT plan.  Instead of P it holds, built on the device in fp64 and stored as fp32
 *                                  [mmax][lmax][kp] each (exact zeros for l < m, zero at l = 0):
 *                                    D[m][l][k] = dP_l^m(cos theta)/dtheta at theta_k,   Q[m][l][k] = m P_l^m(cos theta_k) / sin(theta_k)
 *                                  (P the orthonormal table of the scalar plan, Condon-Shortley phase when csphase).  Only the vector entry
 *                                  points (b200sht_vector_*, b200sht_vsht_*) and the longitude stages accept it.  With m_offset > 0 its
 *                                  local order m holds the columns of the global order m_offset + m, bit-identical to those of the plan of
 *                                  all orders: an order shard of the distributed vector transforms, served by the Legendre stages and the
 *                                  converters only (see the vector SHT section).  B200SHT_PLAN_VECTOR | B200SHT_PLAN_FFT_ONLY is refused. */
#define B200SHT_PLAN_FFT_ONLY 1
#define B200SHT_PLAN_VECTOR 2
int b200sht_plan_create_ex(b200sht_plan** plan, int nlat, int nlon, int lmax, int mmax, int m_offset, int flags,
                           const double* cost, const double* quad_w, int csphase, void* stream);
int b200sht_plan_destroy(b200sht_plan* plan);
/* what: 0 nlat, 1 nlon, 2 lmax, 3 mmax, 4 kp, 5 table bytes (both tables of a vector plan), 6 tensor-core path available (0/1; sm_90
 *       devices), 7 m_offset, 8 tensor-core longitude DFT available for this grid (0/1), 9 vector plan (0/1) */
int64_t b200sht_plan_query(const b200sht_plan* plan, int what);
/* device pointer to the fp32 table [mmax][lmax][kp] (for tests) */
const float* b200sht_plan_table(const b200sht_plan* plan);
/* copy the table into caller-owned device memory (mmax*lmax*kp floats; a vector plan: D then Q, 2*mmax*lmax*kp floats).
 * b200sht_plan_table of a vector plan points at its internal layout [mmax][2][lmax][kp] (D rows, then Q rows, of each order). */
int b200sht_plan_copy_table(const b200sht_plan* plan, float* dst, void* stream);

/* ------------------------------------------------------------------------------ packed-format sizes */
/* (for the buffers of C vector fields on a vector plan pass 2C: see the vector SHT section) */
int64_t b200sht_latspec_elems(const b200sht_plan* plan, int B, int C); /* floats in a latspec buffer */
int64_t b200sht_spec_elems(const b200sht_plan* plan, int B, int C);    /* floats in a spec buffer    */
int64_t b200sht_spec_elems_lm(int L, int M, int B, int C);

/* ------------------------------------------------------------------------------------ stage kernels */
/* Longitude analysis: real rows -> truncated half spectrum.
 *   X[m][p][r][k] = row_scale[k] * mode_scale[m] * sum_j x[r][k][j] exp(-2 pi i m j / nlon)
 * scale_mode 0: SHT forward     (row_scale = quad_w[k] * 2 pi / nlon, mode_scale = 1)
 * scale_mode 1: adjoint of irfft (row_scale = 1, mode_scale = 1 for m = 0 and Nyquist, 2 otherwise)
 * scale_mode | 2: TF32 precision: the output is a TF32 value (it is the operand of a TF32 GEMM) and, for nlon = 8 * N2 <= 1520 and
 *                 mmax <= 256, the transform itself runs on the tensor cores (radix-8 butterflies on the CUDA cores x a
 *                 [mmax/8 x nlon/16] DFT matrix as a TF32 GEMM, csrc/dft.cu) when also x is 16-byte aligned and, for fp32 rows,
 *                 nlon % 32 == 0 (bf16 rows: any such nlon); otherwise the CUDA-core FFT serves the call.  The CUDA-core FFT
 *                 rounds its output to the nearest TF32 value; the tensor-core DFT stores a bias-compensated truncation
 *                 (the value scaled by 1 + 2^-10/3, then its 13 low mantissa bits cleared), unbiased over a binade. */
int b200sht_fft_analysis(const b200sht_plan* plan, const void* x, int dtype, int B, int C,
                         float* latspec, int scale_mode, void* stream);
/* Longitude synthesis: truncated half spectrum -> real rows (+ optional per-channel bias, cast to dtype).
 * scale_mode 0: irfft(norm="forward") semantics (imaginary part of m=0 / Nyquist ignored)
 * scale_mode 1: adjoint of the scale_mode-0 analysis (row_scale = quad_w[k] 2 pi/nlon, modes m>0 halved)
 * In scale_mode 0 / 1 `latspec` must be 8-byte aligned (B200SHT_ERR_INVALID otherwise); `y` needs only the alignment of its dtype.
 * scale_mode | 2: `latspec` is in the TILED layout written by b200sht_legendre_synthesis_tiled and the transform runs on the tensor
 *                 cores (TF32; radix-8 butterflies on the CUDA cores x a [mmax/8 x nlon/16] DFT matrix as a TF32 GEMM, csrc/dft.cu).
 *                 Error unless b200sht_plan_query(plan, 8) == 1. */
int b200sht_fft_synthesis(const b200sht_plan* plan, const float* latspec, void* y, int dtype, int B, int C,
                          const float* bias, int scale_mode, void* stream);
/* Legendre analysis  spec[l][m][..] = sum_k P[m][l][k] latspec[m][..][k]   (l >= 32*floor(m/32)).  At every precision only the rows
 * k < nlat of latspec are read: its latitude padding [nlat, kp) may hold anything, NaN included. */
int b200sht_legendre_analysis(const b200sht_plan* plan, const float* latspec, float* spec, int B, int C,
                              int precision, void* stream);
/* Legendre synthesis latspec[m][..][k] = sum_l P[m][l][k] spec[l][m][..] */
int b200sht_legendre_synthesis(const b200sht_plan* plan, const float* spec, float* latspec, int B, int C,
                               int precision, void* stream);
/* Legendre synthesis (TF32) into the TILED latspec layout the tensor-core longitude DFT consumes:
 *   latspec[r][k / 8][plane][m / 8][m % 8][k % 8]   (orders padded with zeros to a multiple of 8; same size as the standard layout)
 * i.e. the 16 KB that one 8-row tile of the DFT kernel reads are contiguous and arrive as 128-byte TMA rows.  Pair it with
 * b200sht_fft_synthesis(..., scale_mode | 2).  Requires b200sht_plan_query(plan, 8) == 1. */
int b200sht_legendre_synthesis_tiled(const b200sht_plan* plan, const float* spec, float* latspec, int B, int C, void* stream);
/* packed spec [L][M][2][B][cp] <-> torch complex64 [B*C][L][M] (exact zeros written for l < m).  These and the
 * mix / ComplexReLU entry points below depend only on the mode counts (L, M), not on a grid, so they take no plan. */
int b200sht_spec_unpack(int L, int M, const float* spec, void* coeffs, int B, int C, void* stream);
int b200sht_spec_pack(int L, int M, const void* coeffs, float* spec, int B, int C, void* stream);
/* same with an order offset (orders m_offset + m) and/or dense storage (every (l, m) entry stored: used for l/m-sharded spectra) */
int b200sht_spec_unpack_ex(int L, int M, int m_offset, int dense, const float* spec, void* coeffs, int B, int C, void* stream);
int b200sht_spec_pack_ex(int L, int M, int m_offset, int dense, const void* coeffs, float* spec, int B, int C, void* stream);
/* latspec [mmax][2][B*C][kp] <-> complex64 [B*C][nlat][mmax]: the layout the distributed lat<->lon transposes exchange */
int b200sht_latspec_unpack(const b200sht_plan* plan, const float* latspec, void* coeffs, int B, int C, void* stream);
int b200sht_latspec_pack(const b200sht_plan* plan, const void* coeffs, float* latspec, int B, int C, void* stream);

/* ------------------------------------------------------------------------- torch-harmonics boundary */
/* bytes of scratch the four calls below need for (B, C) */
int64_t b200sht_sht_workspace_bytes(const b200sht_plan* plan, int B, int C);
/* x [B*C][nlat][nlon] (dtype) -> coeffs complex64 [B*C][lmax][mmax] */
int b200sht_sht_forward(const b200sht_plan* plan, const void* x, int dtype, int B, int C, void* coeffs,
                        void* workspace, int precision, void* stream);
/* coeffs complex64 [B*C][lmax][mmax] -> y [B*C][nlat][nlon] (dtype) */
int b200sht_sht_inverse(const b200sht_plan* plan, const void* coeffs, void* y, int dtype, int B, int C,
                        void* workspace, int precision, void* stream);
/* gradient of sht_forward w.r.t. x given dL/dcoeffs (PyTorch complex-gradient convention) */
int b200sht_sht_forward_adjoint(const b200sht_plan* plan, const void* gcoeffs, void* gx, int dtype, int B, int C,
                                void* workspace, int precision, void* stream);
/* gradient of sht_inverse w.r.t. coeffs given dL/dy */
int b200sht_sht_inverse_adjoint(const b200sht_plan* plan, const void* gy, int dtype, int B, int C, void* gcoeffs,
                                void* workspace, int precision, void* stream);

/* ------------------------------------------------------------------------------------- vector SHT */
/* torch_harmonics.RealVectorSHT / InverseRealVectorSHT (norm "ortho") on a vector plan.  A field of C vector channels is
 * x [B][C][2][nlat][nlon] (component 0 = colatitude theta, 1 = longitude phi; rows north to south); its coefficients are
 * complex64 [B][C][2][lmax][mmax] (0 = spheroidal S, 1 = toroidal T; exact zeros for l < m).  With X = 2 pi rfft(x, norm="forward")[:mmax]
 * and the quadrature weights w_k:
 *   S_lm = sum_k w_k (D X_theta - i Q X_phi) / (l (l+1)),   T_lm = sum_k w_k (-i Q X_theta - D X_phi) / (l (l+1)),   S_0m = T_0m = 0
 *   U_theta = irfft(sum_l D S + i Q T),   U_phi = irfft(sum_l i Q S - D T)   (n = nlon, norm "forward"; Im of m = 0 / Nyquist ignored)
 * so that ivsht([f_lm, 0]) = (df/dtheta, df/dphi / sin theta) and ivsht([0, g_lm]) = -r x grad g.
 * Stage formats: the 2C component rows (b, c, component) are read and written in place as the rows of a scalar latspec of 2C channels, and
 * the Legendre stages produce a STACKED spec [2][lmax][mmax][2][B][cp] (cp = 2C rounded up to 4, column 2c + component): the D
 * contractions, then the Q contractions (b200sht_spec_elems(plan, B, 2C) floats).  The +-i rotations and 1/(l(l+1)) happen in the
 * spec <-> coefficient converters.  Precision FP32 or TF32 (3 x TF32 is refused with B200SHT_ERR_UNSUPPORTED).
 * Order shards (a vector plan with m_offset > 0, the distributed vector transforms): b200sht_vector_legendre_analysis / _synthesis and
 * b200sht_vector_spec_pack / _unpack serve them, with mmax the shard's order count and "l < m" read as l < m_offset + m; their outputs are
 * the order slice of the plan of all orders.  b200sht_vector_legendre_synthesis_tiled and the one-call b200sht_vsht_* entries return
 * B200SHT_ERR_INVALID on them (b200sht_vsht_workspace_bytes returns -1): their longitude stage covers orders 0 .. mmax - 1. */
int b200sht_vector_legendre_analysis(const b200sht_plan* plan, const float* latspec, float* spec, int B, int C, int precision, void* stream);
int b200sht_vector_legendre_synthesis(const b200sht_plan* plan, const float* spec, float* latspec, int B, int C, int precision, void* stream);
/* TF32 into the tiled latspec layout of the tensor-core DFT (see b200sht_legendre_synthesis_tiled); needs b200sht_plan_query(plan, 8) == 1 */
int b200sht_vector_legendre_synthesis_tiled(const b200sht_plan* plan, const float* spec, float* latspec, int B, int C, void* stream);
/* stacked spec <-> coefficients [B][C][2][lmax][mmax].  unpack: S = f (D x_theta - i Q x_phi), T = f (-i Q x_theta - D x_phi);
 * pack: D_theta = f S, D_phi = -f T, Q_theta = i f T, Q_phi = i f S; f = 1 / (l (l+1)) (0 at l = 0) when scaled, else 1.
 * pack(scaled) is the adjoint of unpack(scaled).  pack writes every entry of the stacked spec. */
int b200sht_vector_spec_unpack(const b200sht_plan* plan, const float* spec, void* coeffs, int B, int C, int scaled, void* stream);
int b200sht_vector_spec_pack(const b200sht_plan* plan, const void* coeffs, float* spec, int B, int C, int scaled, void* stream);
/* One-call boundary, as b200sht_sht_* (workspace of b200sht_vsht_workspace_bytes; -1 for a scalar plan or an order shard):
 *   forward          x [B][C][2][nlat][nlon] (dtype) -> coeffs                        <- RealVectorSHT.forward
 *   inverse          coeffs -> y [B][C][2][nlat][nlon] (dtype)                        <- InverseRealVectorSHT.forward
 *   forward_adjoint  dL/dcoeffs -> dL/dx     inverse_adjoint  dL/dy -> dL/dcoeffs      <- their autograd backward (PyTorch complex-gradient convention) */
int64_t b200sht_vsht_workspace_bytes(const b200sht_plan* plan, int B, int C);
int b200sht_vsht_forward(const b200sht_plan* plan, const void* x, int dtype, int B, int C, void* coeffs, void* workspace, int precision, void* stream);
int b200sht_vsht_inverse(const b200sht_plan* plan, const void* coeffs, void* y, int dtype, int B, int C, void* workspace, int precision, void* stream);
int b200sht_vsht_forward_adjoint(const b200sht_plan* plan, const void* gcoeffs, void* gx, int dtype, int B, int C, void* workspace, int precision,
                                 void* stream);
int b200sht_vsht_inverse_adjoint(const b200sht_plan* plan, const void* gy, int dtype, int B, int C, void* gcoeffs, void* workspace, int precision,
                                 void* stream);

/* -------------------------------------------------------------------------------------- channel mix */
/* weight re-layout: native torch parameter (complex64, shapes per b200sht_mix_op) -> packed
 * float [L][G][Ci/G][2][cop] (real and imaginary planes; cop = Co/G rounded up to 4; l-stride 0 for OP_SHARED).  Only the dense
 * operators (DHCONV, SHARED, LDEP) use a packed weight; the others read the native layout. */
int64_t b200sht_mix_weight_elems(int op, int L, int M, int G, int Ci, int Co);
int b200sht_mix_weight_pack(int op, const void* w_native, float* w_packed, int L, int G, int Ci, int Co, int precision, void* stream);
int b200sht_mix_weight_unpack(int op, const float* w_packed, void* w_native, int L, int G, int Ci, int Co, void* stream);

/* y[l][m][.][b][o] = sum_i x[l][m][.][b][i] * w[...]   on packed spec tensors (x: C = Ci, y: C = Co).
 * w: packed weight for dense ops, native complex64 for DIAGONAL / SEP_* ops.
 * cbias (OP_SHARED / OP_LDEP only, may be null): complex64 [Co] added to every mode (compl_muladd2d_fwd). */
int b200sht_mix_forward(int L, int M, int op, const float* x, const void* w, const void* cbias,
                        float* y, int B, int G, int Ci, int Co, int precision, void* stream);
/* 1 when b200sht_mix_forward / _backward run this shape on the tensor cores at `precision`, 0 when they run the fp32 CUDA-core
 * kernels: B200SHT_PREC_TF32 needs a dense operator, a batch that divides 32 and 16-byte aligned group slices; anything else is
 * served in fp32 -- the caller should then pack the weight with B200SHT_PREC_FP32 (no TF32 rounding) and may want to tell the user. */
int b200sht_mix_uses_tensor_cores(int op, int B, int G, int Ci, int Co, int precision);
/* gx = dL/dx (may be null), gw = dL/dw in the same format as w (may be null; overwritten, not accumulated),
 * gcbias complex64 [Co] (may be null). */
int b200sht_mix_backward(int L, int M, int op, const float* x, const void* w, const float* gy,
                         float* gx, void* gw, void* gcbias, int B, int G, int Ci, int Co, int precision, void* stream);

/* ------------------------------------------------------------------------------------- ComplexReLU */
/* mode 0 real, 1 cartesian, 2 modulus, 3 halfplane (activations.py:88-127) on a packed spec tensor.
 * bias: float [C] (modes 2,3; null -> 0).  In-place allowed (y == x). */
int b200sht_complex_relu_forward(int L, int M, int mode, const float* x, const float* bias,
                                 float negative_slope, float* y, int B, int C, void* stream);
int b200sht_complex_relu_backward(int L, int M, int mode, const float* x, const float* bias,
                                  float negative_slope, const float* gy, float* gx, float* gbias, int B, int C,
                                  void* stream);

/* ------------------------------------------------------------------------------ SpectralConv, one call */
typedef struct {
  int B, Cin, Cout, G;
  int op;          /* b200sht_mix_op */
  int dtype;       /* activation dtype of x / y / residual */
  int precision;   /* b200sht_precision */
} b200sht_conv_desc;
int64_t b200sht_spectral_conv_workspace_bytes(const b200sht_plan* fwd, const b200sht_plan* inv, const b200sht_conv_desc* d);
/* y = iSHT(W . SHT(x)) (+bias); residual (may be null) = iSHT(SHT(x)).  w: packed for dense ops, native otherwise.
 * spec_x_saved (may be null): packed spec buffer that receives SHT(x) for the backward pass. */
int b200sht_spectral_conv_forward(const b200sht_plan* fwd, const b200sht_plan* inv, const b200sht_conv_desc* d,
                                  const void* x, const void* w, const float* bias, void* y, void* residual,
                                  float* spec_x_saved, void* workspace, void* stream);
/* gy, gresidual (may be null) -> gx, gw (same format as w), gbias float [Cout] (may be null) */
int b200sht_spectral_conv_backward(const b200sht_plan* fwd, const b200sht_plan* inv, const b200sht_conv_desc* d,
                                   const void* gy, const void* gresidual, const float* spec_x_saved, const void* w,
                                   void* gx, void* gw, float* gbias, void* workspace, void* stream);

/* same, plus (both optional): gw_native receives the weight gradient re-laid-out to the parameter's native complex64 layout (dense operators)
 * and wgrad_ready_event (a cudaEvent_t) is recorded on `stream` as soon as the weight / bias gradients are final, i.e. BEFORE the two stages
 * that produce gx -- a data-parallel gradient all-reduce waiting on it from another stream overlaps them.  (The reference reaches the same
 * overlap through DDP gradient hooks, makani/mpu/mappings.py:398-406 init_gradient_reduction_hooks.) */
int b200sht_spectral_conv_backward_ex(const b200sht_plan* fwd, const b200sht_plan* inv, const b200sht_conv_desc* d,
                                      const void* gy, const void* gresidual, const float* spec_x_saved, const void* w,
                                      void* gx, void* gw, float* gbias, void* workspace, void* gw_native, void* wgrad_ready_event,
                                      void* stream);

/* sum over batch and latitude of latspec[m=0][re][b][c][k]: d(loss)/d(bias) when latspec = fft_analysis(gy, mode 1) */
int b200sht_bias_grad(const b200sht_plan* plan, const float* latspec, float* gbias, int B, int C, void* stream);

/* host-buffer convenience (end-to-end path for FFI users): copies x (pinned or pageable HOST memory) to the
 * device, runs b200sht_spectral_conv_forward, copies y back.  Synchronises the stream before returning. */
int b200sht_spectral_conv_forward_host(const b200sht_plan* fwd, const b200sht_plan* inv, const b200sht_conv_desc* d,
                                       const void* x_host, const void* w_device, const float* bias_device,
                                       void* y_host, void* stream);

/* ------------------------------------------------------------------- debug / CPU-testable entry points
 * These run the SAME __host__ __device__ code as the kernels on the host, so the FFT plan / butterflies / pair
 * splitting and the Legendre recurrence are unit-tested without a GPU.  All pointers are HOST pointers. */
/* direction 0: rows a, b (float[N]) -> half spectra Xa, Xb (float[2*mmax], interleaved), unscaled rfft.
 * direction 1: half spectra (float[2*mmax]) -> rows (float[N]), irfft(norm="forward") semantics. */
int b200sht_debug_fft_host(int N, int mmax, int direction, const float* in_a, const float* in_b, float* out_a, float* out_b);
/* the tensor-core DFT's factorisation (radix-8 stage, twiddles, index maps: the same __host__ __device__ code as the kernels) with the
 * GEMM summed in double on the host.  direction 0: in float[N] -> out float[2*mmax] (interleaved); direction 1: the reverse.
 * scale_mode / row_scale as for b200sht_fft_analysis / _synthesis (row_scale = the row's quadrature factor). */
int b200sht_debug_dft_host(int N, int mmax, int direction, int scale_mode, float row_scale, const float* in, float* out);
/* wait-time profile of the tensor-core DFT kernels (environment B200SHT_DFT_PROF=1): 16 counters of SM clocks, accumulated over all launches since the
 * last call and cleared by it (slots: see csrc/dft.cu).  All zeros when the profile is off.  Synchronises the device. */
int b200sht_debug_dft_profile(uint64_t* counters16);
/* wait-time profile of the tensor-core GEMM engine (a library built with -DB200SHT_UMMA_PROFILE): 16 counters of SM clocks, accumulated over all
 * engine launches since the last call and cleared by it (slots: see csrc/umma.cu).  All zeros in the shipped build.  Synchronises the device. */
int b200sht_debug_umma_profile(uint64_t* counters16);
/* ------------------------------------------------------------------ pointwise tail of the SFNO block (SURVEY row N2) */
/* Replaces torch.nn.InstanceNorm2d(num_features, eps, affine) (+ the nn.GELU that follows it) as built at makani/models/networks/sfnonet.py:618-620 and
 * applied at :385-406, and the bias + GELU of the 1x1-convolution stacks (makani/models/common/layers.py:537-760).  x, y, dy, dx: [B][C][hw] contiguous, float or
 * bf16 (dtype); gamma / beta / bias: float [C] (null: 1 / 0); stats: float [B*C][2] (mean, rstd), written by forward, read by backward; sums: float [B*C][2]
 * written by backward: per row sum g and sum g * xhat -- dbeta[c] / dgamma[c] are their sums over the batch; workspace: b200sht_pointwise_workspace_floats floats.
 * gelu != 0 fuses y = gelu(norm(x)) (exact erf GELU).  Statistics are biased (1 / hw), as InstanceNorm uses them. */
int64_t b200sht_pointwise_workspace_floats(int B, int C, int64_t hw);
int b200sht_instance_norm_forward(const void* x, void* y, const float* gamma, const float* beta, float* stats, float* workspace, int dtype, int B, int C,
                                  int64_t hw, float eps, int gelu, void* stream);
int b200sht_instance_norm_backward(const void* x, const void* dy, void* dx, const float* gamma, const float* beta, const float* stats, float* sums,
                                   float* workspace, int dtype, int B, int C, int64_t hw, int gelu, void* stream);
/* y = gelu(x + bias[c]);  dx = dy * gelu'(x + bias[c]), row_sums: float [B*C][2] with sum dx in [.][0] (dbias[c] = its sum over the batch; may be null) */
int b200sht_bias_gelu_forward(const void* x, const float* bias, void* y, int dtype, int B, int C, int64_t hw, void* stream);
int b200sht_bias_gelu_backward(const void* x, const float* bias, const void* dy, void* dx, float* row_sums, float* workspace, int dtype, int B, int C, int64_t hw,
                               void* stream);

/* ------------------------------------------------------------------ quadrature-weighted instance norm on the sphere (SURVEY row N2)
 * Replaces makani's GeometricInstanceNormS2 (makani/models/common/layer_norm.py:30-152) and DistributedGeometricInstanceNormS2
 * (makani/mpu/layer_norm.py:173-253), staged so that the distributed class can gather the per-rank statistics between the stages; the serial class
 * calls the same stages with R = 1 and D = 1.  A row (b, c) of x is an H x W plane (the local shard), q: float [H] the latitude weights of its rows,
 * constant along longitude.  x, y, dy, dx: [B][C][H][W] contiguous, float or bf16 (dtype); gamma / beta: float [C] (null: 1 / 0); B*C <= 65535.
 *   mu = (1/D) sum q x,  var = (1/D) sum q (x - mu)^2,  r = (var + eps)^-1/2,  xhat = (x - mu) r,  y = [gelu](gamma xhat + beta)
 *   dx = gamma r (g - (q/D) (S1 + xhat S2 - corr S2)),  S1 = sum g, S2 = sum g xhat over the whole field (g = dy, or dy gelu'(z) when gelu != 0)
 * partials: double [B*C][3] per row (sum q, mean, M2), the fp64 Welford triple of this shard; sums: double [B*C][2] per row (S1, S2) of this shard;
 * stats: float [B*C][3] (mu, r, corr = r mu (D - S) / D, S the combined weight).  fp64 buffers and the workspace must be 8-byte aligned;
 * workspace: b200sht_geometric_norm_workspace_floats floats. */
int64_t b200sht_geometric_norm_workspace_floats(int B, int C, int64_t hw);
/* the fp64 triple (sum q, mean, M2) of every row of this shard, sums taken about the pivot x[row, 0] */
int b200sht_geometric_norm_partials(const void* x, const float* q, double* partials, float* workspace, int dtype, int B, int C, int H, int W, void* stream);
/* partials: double [R][rows][3], R ranks' triples, combined (Chan / Welford) in rank order; D > 0 the normaliser -> stats */
int b200sht_geometric_norm_finalize(const double* partials, int R, int rows, double D, float eps, float* stats, void* stream);
/* y = [gelu](gamma (x - mu) r + beta), written in the dtype of x */
int b200sht_geometric_norm_apply(const void* x, void* y, const float* gamma, const float* beta, const float* stats, int dtype, int B, int C, int H, int W,
                                 int gelu, void* stream);
/* per row of this shard, the unweighted fp64 sums (S1, S2) */
int b200sht_geometric_norm_backward_sums(const void* x, const void* dy, const float* gamma, const float* beta, const float* stats, double* sums,
                                         float* workspace, int dtype, int B, int C, int H, int W, int gelu, void* stream);
/* sums: double [R][rows][2], R ranks' (S1, S2) added in rank order -> dx by the formula above with the row's q[i] / D */
int b200sht_geometric_norm_backward_apply(const void* x, const void* dy, void* dx, const float* gamma, const float* beta, const float* stats, const double* sums,
                                          int R, const float* q, double D, int dtype, int B, int C, int H, int W, int gelu, void* stream);
/* sums: double [B][C][2] of this shard (backward_sums) -> dgamma[c] = sum_b S2, dbeta[c] = sum_b S1 (float [C]; either may be null) */
int b200sht_geometric_norm_param_grads(const double* sums, float* dgamma, float* dbeta, int B, int C, void* stream);

/* ------------------------------------------------------------------ DISCO convolution on the sphere (SURVEY row N1)
 * Replaces the two sparse contractions of torch_harmonics.DiscreteContinuousConvS2 (built at makani/models/networks/fourcastnet3.py:117-252,
 * :364-381, :511-543, snonet.py).  The filter tensor psi[k, t, i, j] (K kernel functions, output latitude t, input latitude i, input longitude
 * j, quadrature merged in) is restated in makani_b200/disco.py and DESIGN.md section 5:
 *   output point (colatitude theta_t, longitude 0), input point (theta_i, phi_j = 2 pi j / nlon_in);
 *   r = arccos(cos theta_t cos theta_i + sin theta_t sin theta_i cos phi_j),
 *   phi' = atan2(sin phi_j sin theta_i, cos theta_t sin theta_i cos phi_j - cos theta_i sin theta_t) in [0, 2 pi)   (YZY rotation by -theta_t);
 *   support r <= r_c = (1 + 1e-3) theta_cutoff; morlet: rho = r / r_c, x = rho sin phi', y = rho cos phi',
 *   psi_k = cos^2(pi rho / 2) h_n(x) h_m(y), n = k mod n1, m = k / n1, h_j(u) = sin(ceil(j/2) pi u) (j odd), cos(ceil(j/2) pi u) (j even);
 *   stored psi_hat = psi q_i / (d + 1e-9), q_i = 2 pi w_i / nlon_in, d per basis_norm_mode ("mean": mean over t of sum |psi| q, "individual":
 *   that sum at t, "support": sum q at t, "none": 1).
 * Contractions, with pscale = nlon_in / nlon_out (nlon_in % nlon_out == 0):
 *   forward  X[b,c,k,t,p] = sum_{i,j} psi_hat[k,t,i,j] x[b,c,i,(j + pscale p) mod nlon_in]            x: [B][C][nlat_in][nlon_in] fp32 or bf16
 *   adjoint  dx[b,c,i,j'] = sum_{k,t,p,j: (j + pscale p) mod nlon_in = j'} psi_hat[k,t,i,j] dX[b,c,k,t,p]   X, dX: [B][C][K][nlat_out][nlon_out] fp32
 * The channel contraction y = W X (+ bias) is a grouped GEMM left to the caller.
 *
 * b200sht_disco_plan_create: nnz entries (ker[n], lat_out[n], col_in[n] = i * nlon_in + j, vals[n]) in HOST memory, any order; entries with the
 *   same (k, t, col) are summed in fp64.  Both device layouts (by output latitude, sorted by (i, j); by input latitude, sorted by (t, j)) hold the
 *   values rounded to fp32.  Synchronises `stream` once, after the upload.  nlon_in and nlon_out at most 16384 (B200SHT_ERR_UNSUPPORTED).
 * b200sht_disco_plan_query: 0 nlat_in, 1 nlon_in, 2 nlat_out, 3 nlon_out, 4 K, 5 nnz, 6 support points (distinct (t, i, j)), 7 device bytes,
 *   8 pscale; -1 otherwise.
 * b200sht_disco_forward: writes every element of X; fp32 accumulation, each X element summed over its points in (i, j) order.
 * b200sht_disco_adjoint: writes every element of dx (dtype: fp32 or bf16, rounded once at the end); each dx element is summed by one thread in a
 *   fixed order, without atomics: results are bit-identical run to run.
 * B * C rows at most 65535 per call. */
typedef struct b200sht_disco_plan b200sht_disco_plan;
int b200sht_disco_plan_create(b200sht_disco_plan** plan, int nlat_in, int nlon_in, int nlat_out, int nlon_out, int K, int64_t nnz, const int* ker,
                              const int* lat_out, const int* col_in, const double* vals, void* stream);
int b200sht_disco_plan_destroy(b200sht_disco_plan* plan);
int64_t b200sht_disco_plan_query(const b200sht_disco_plan* plan, int what);
int b200sht_disco_forward(const b200sht_disco_plan* plan, const void* x, int dtype, int B, int C, float* X, void* stream);
int b200sht_disco_adjoint(const b200sht_disco_plan* plan, const float* dX, void* dx, int dtype, int B, int C, void* stream);

/* ------------------------------------------------------------------ neighbourhood attention on the sphere
 * The attention of torch_harmonics.NeighborhoodAttentionS2 (makani_b200/attention.py, DESIGN.md section 4.9; element-wise parity with
 * torch-harmonics is not pinned, its source is not available).  The neighbourhood is a DISCO plan with K = 1 whose value at (t, i, j) is the
 * quadrature weight w_i = 2 pi w_in[i] / nlon_in and whose support S(t) is that of b200sht_disco_plan_create's psi (r <= (1 + 1e-3) theta_cutoff
 * at longitude 0).  Within each (t, i) the support must be an arc of longitudes j in [-off, n - 1 - off] (mod nlon_in), n its point count and
 * off = (n - 1) / 2, or the whole ring; makani_b200.attention builds and checks such plans.  With s = nlon_in / nlon_out and H heads:
 *   N(t, p) = { (i, (j + s p) mod nlon_in) : (i, j) in S(t) },   l_n = scale <q_h(t, p), k_h(n)>
 *   y_h(t, p) = sum_{n in N(t,p)} w_i exp(l_n) v_h(n) / sum_{n in N(t,p)} w_i exp(l_n),   lse_h(t, p) = log sum_{n in N(t,p)} w_i exp(l_n)
 * Operands (fp32, device): q, dq [B][nlat_out nlon_out][heads ek], k, dk [B][nlat_in nlon_in][heads ek], v, dv [B][nlat_in nlon_in][heads ev],
 *   y, dy [B][nlat_out nlon_out][heads ev], lse, D [B][heads][nlat_out nlon_out]: point-major, head h at channels [h e, (h + 1) e).
 * b200sht_attention_forward: writes y and lse; online softmax per output point with a running max and sum in fp32.
 * b200sht_attention_backward: given dy, writes dq, dk, dv and D = <dy_h, y_h> per output point (scratch the caller provides):
 *   alpha_n = w_i exp(l_n - lse), dl_n = alpha_n (<dy_h, v_h(n)> - D), dq = scale sum_n dl_n k_h(n), dv_n = sum alpha dy, dk_n = scale sum dl q.
 *   dk and dv are gathers by input point without atomics: results are bit-identical run to run.  The backward recomputes the forward's
 *   logits bit for bit.
 * Head dims ek, ev in 1 .. 64 (any value; multiples of 4 with 16-byte aligned operands take the vector path), otherwise B200SHT_ERR_UNSUPPORTED.
 * B * heads at most 65535 per call. */
int b200sht_attention_forward(const b200sht_disco_plan* plan, const float* q, const float* k, const float* v, float* y, float* lse, int B, int heads,
                              int ek, int ev, float scale, void* stream);
int b200sht_attention_backward(const b200sht_disco_plan* plan, const float* q, const float* k, const float* v, const float* y, const float* lse,
                               const float* dy, float* dq, float* dk, float* dv, float* D, int B, int heads, int ek, int ev, float scale,
                               void* stream);

/* ------------------------------------------------------------------ bilinear resampling on the sphere
 * Replaces torch_harmonics.ResampleS2(mode="bilinear"), the upsampling of FCN3's DiscreteContinuousDecoder with upsample_sht=False
 * (makani/models/networks/fourcastnet3.py:356-358) and of SNO's decoder.  The tables are built on the host in fp64 (makani_b200/resample.py,
 * DESIGN.md section 4.8) and passed here rounded to fp32:
 *   lat_idx[t] = a, lat_w[t] = wt (t < nlat_out): output row t interpolates the expanded input rows a and a + 1; lon_left[p] = l, lon_right[p] = r,
 *   lon_w[p] = wp (p < nlon_out).  With expand_poles the expanded input has nlat_in + 2 rows: row 0 is the longitude mean of input row 0, row
 *   nlat_in + 1 the mean of input row nlat_in - 1, and row e otherwise input row e - 1; without it the expanded input is the input.
 *   forward  y[b,t,p] = lerp(lerp(X[b,a,l], X[b,a,r], wp), lerp(X[b,a+1,l], X[b,a+1,r], wp), wt),  lerp(u, v, w) = u + w (v - u) (w < 1/2),
 *            v - (v - u)(1 - w) otherwise, so w = 0 and w = 1 reproduce u and v exactly;     x: [planes][nlat_in][nlon_in], y: [planes][nlat_out][nlon_out]
 *   adjoint  dx = R^T dy, the weights of the adjoint being 1 - wt, wt, 1 - wp, wp (1 - w rounded once from fp64).  A pole pseudo-row adds
 *            (1 / nlon_in) sum_{t: a_t or a_t + 1 is the pseudo-row} w sum_p dy[b,t,p] to every element of input row 0 (nlat_in - 1).
 * All data fp32.
 *
 * b200sht_resample_plan_create: the tables in HOST memory; checks 0 <= a, a + 1 < nlat_in + 2 expand_poles and 0 <= l, r < nlon_in.  Builds the
 *   adjoint's two CSR lists (by expanded input row, t ascending; by input column, p ascending) and synchronises `stream` once, after the upload.
 *   nlon_in at most 8192 and nlon_out at most 16384 (B200SHT_ERR_UNSUPPORTED).
 * b200sht_resample_plan_query: 0 nlat_in, 1 nlon_in, 2 nlat_out, 3 nlon_out, 4 expand_poles, 5 device bytes; -1 otherwise.
 * b200sht_resample_forward: writes every element of y; a pole mean is one fp32 sum over the row in a fixed order, divided by nlon_in.
 * b200sht_resample_adjoint: writes every element of dx; each element is summed by one thread (the pole term by one warp) in a fixed order, without
 *   atomics: results are bit-identical run to run.
 * planes: up to 65535 per call (more where the row lengths let several planes share a CTA). */
typedef struct b200sht_resample_plan b200sht_resample_plan;
int b200sht_resample_plan_create(b200sht_resample_plan** plan, int nlat_in, int nlon_in, int nlat_out, int nlon_out, int expand_poles, const int* lat_idx,
                                 const float* lat_w, const int* lon_left, const int* lon_right, const float* lon_w, void* stream);
int b200sht_resample_plan_destroy(b200sht_resample_plan* plan);
int64_t b200sht_resample_plan_query(const b200sht_resample_plan* plan, int what);
int b200sht_resample_forward(const b200sht_resample_plan* plan, const float* x, float* y, int planes, void* stream);
int b200sht_resample_adjoint(const b200sht_resample_plan* plan, const float* dy, float* dx, int planes, void* stream);

/* Programmatic dependent launch between the tensor-core kernels of a call sequence (prologue of kernel i+1 under the tail of kernel i; environment
 * B200SHT_PDL sets the initial value, default on).  Returns the previous setting.  Results do not depend on it. */
int b200sht_debug_set_pdl(int on);
/* radices chosen for length N; returns the number of stages or a negative status */
int b200sht_debug_fft_plan(int N, int* radices, int max_radices);
/* table [mmax][lmax][nlat] (fp32) from cos(colatitude) cost[nlat] */
int b200sht_debug_table_host(int nlat, int lmax, int mmax, const double* cost, int csphase, float* table);
/* the vector plan's tables D and Q, each [mmax][lmax][nlat] (fp32), from cost[nlat] */
int b200sht_debug_vector_table_host(int nlat, int lmax, int mmax, const double* cost, int csphase, float* D, float* Q);

#ifdef __cplusplus
}
#endif
#endif /* B200SHT_H */
