/* allegro_b200 C ABI -- H100 (sm_90a) kernels for Allegro's per-edge hot path.
 *
 * The reference (mir-group/allegro v0.7.1) is pure Python; its "FFI" for this path is the
 * kernel plug-in point Contracter.forward(x1, x2, idxs, scatter_dim_size)
 * (allegro/nn/_strided/_contract.py:185-211, swapped by enable_TritonContracter :253-282 and
 * enable_CuEquivarianceContracter :284-310) plus the graph modules whose forward(data) the
 * fused pipeline replaces (allegro/nn/tensorembed.py:85-96, allegro/nn/_allegro.py:237-301,
 * allegro/nn/edgewise.py:40-60).  Each entry point below cites the reference lines it replaces.
 *
 * Conventions
 *  - plain C types only; every pointer is a DEVICE pointer unless its name ends in _host;
 *  - the caller owns every buffer (kernels never allocate); work is enqueued on `stream`
 *    (a cudaStream_t passed as void*) and is asynchronous;
 *  - return 0 on success, non-zero on error; ab2_last_error() gives the message
 *    (thread-local);
 *  - dtype: AB2_F64 / AB2_F32 / AB2_BF16 selects the storage type of activations ("TAct").
 *    Accumulation type ("TAcc") is double for AB2_F64, float otherwise.  Geometry, spherical
 *    harmonics, environment sums, energies and gradients w.r.t. them are always TAcc.
 *  - edges are sorted by centre ("CSR": row_ptr[N+1], int32); internal feature layout is
 *    component-major  V[E][d][U]  (channel u fastest), env weights  w[E][n_ir][U].
 */
#ifndef ALLEGRO_B200_H
#define ALLEGRO_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { AB2_F64 = 0, AB2_F32 = 1, AB2_BF16 = 2 };
enum { AB2_ACT_NONE = 0, AB2_ACT_SILU = 1, AB2_ACT_MUL_DSILU = 2 };
enum { AB2_EPI_NONE = 0, AB2_EPI_MUL_DSILU = 1 };
/* MLP nonlinearity of the _nl entry points (nequip ScalarMLPFunction `nonlinearity`).  With it the act / epi codes above
 * keep their meaning: AB2_ACT_SILU applies the nonlinearity phi, AB2_ACT_MUL_DSILU and AB2_EPI_MUL_DSILU multiply by phi'.
 *   AB2_NL_SILU  phi(x) = x sigma(x)
 *   AB2_NL_MISH  phi(x) = x tanh(softplus(x))
 *   AB2_NL_GELU  phi(x) = x Phi(x) = x erfc(-x / sqrt2) / 2   (the exact erf form, not the tanh approximation)
 * Every entry without the _nl suffix is its _nl twin with AB2_NL_SILU. */
enum { AB2_NL_SILU = 1, AB2_NL_MISH = 2, AB2_NL_GELU = 3 };

#define AB2_MAX_SEG 4
#define AB2_MAX_LMAX 4

const char* ab2_last_error(void);
int ab2_version(void);
/* 1 if a CUDA device with compute capability 9.0 is current, else 0 (no error). */
int ab2_device_ok(void);
/* Kernel-selection switches (for A/B tests and tuning; process-global, not thread-safe):
 *   "tp_fast"    1 shared-memory / register-tiled tensor product (default), 2 register-M variants, 0 shape-generic kernels
 *   "linear_tc"  1 wgmma tensor-core linear (default), 0 CUDA-core tile kernel
 *   "tp_variant" 1: 3 CTAs/SM (default), 0: 2 CTAs/SM for the shared-memory tensor-product kernel
 *   "tp_stream"  1 TMA-staged streaming tensor product where instantiated (default), 0 round-1 kernels;
 *                "tp_stream_te" edges per stage (0 = 8), "tp_stream_cps" cap on CTAs per SM (0 = occupancy limit),
 *                "tp_stream3" 1: three consumer warps per centre stream for the layer-0 backward (default), 0: two,
 *                "tp_stream_last" 1: 9 -> 1 (last layer) backward through the streaming kernel (default), 0: tp_smem + split,
 *                "tp_stream_gytile" 1: gY of the layer-0 backward reduced through a shared-memory tile (default), 0: shuffles
 *   "tp_baked64" 1 fp64 tensor-product kernels with the baked l_max = 3 table structure (default), 0 shape-generic kernels
 *   "env_stream" 1 streaming adjoint of the environment sum (default), 0 round-1 kernel
 *   "linear_tma" 1 TMA-producer variant of the tensor-core linear where eligible (default), 0 cp.async producers
 *   "env_split"  warps per (centre, channel chunk) in ab2_env_sum / ab2_env_bwd: 0 auto (default), 1, 2, 4
 *   "tc_debug"   stage knock-out mask of the wgmma linear (bit0 no stores, bit1 no loads, bit2 no MMA); results are
 *                wrong when non-zero -- for tools/exp_env.py only
 * Returns 1 (and sets ab2_last_error) for an unknown key. */
int ab2_set_option(const char* key, int value);

/* ---- operator level: the reference's own kernel plug-in point ----------------------- */

/* Contracter.forward, part 1 (_contract.py:195-204): gamma[n][u][j] += sf * x2[z][u][j] for
 * n = idxs[z] (reference "strided" layout [z][u][j], unsorted int64 idxs).  gamma must be
 * zeroed by the caller.  dtype AB2_F64 / AB2_F32. */
int ab2_op_scatter_env(int dtype, int64_t E, int64_t row /* = U*d2 */, double sf,
                       const void* x2, const int64_t* idxs, void* gamma, void* stream);

/* Contracter.forward, part 2 (_contract.py:205-251): out[z][u][k] =
 *   sum_nnz cgw[nnz][u] * x1[z][u][i_nnz] * gamma[idxs[z]][u][j_nnz]
 * with cgw[nnz][u] = w3j_value * weights[u, path]  (pre-contracted, _contract.py:218-219).
 * tab_ijk: int32 [nnz][3].  Also used for both backward products (caller permutes roles):
 *   mode 0: out[k] from (x1[i], g[j])      forward
 *   mode 1: gx1[i] from (gout[k], g[j])    (Triton "bwd1" table, _flashallegro.py:352-355)
 *   mode 2: gg[j]  from (x1[i], gout[k])   per-edge term, atomically added into
 *           ggamma[idxs[z]] (adjoint of the gather _contract.py:205); ggamma pre-zeroed. */
int ab2_op_contract(int dtype, int mode, int64_t E, int U, int d1, int d2, int dout, int nnz,
                    const int32_t* tab_ijk, const void* cgw, const void* a, const void* b,
                    const int64_t* idxs, void* out, void* stream);

/* Training support (the reference's `weights` are Parameters, _contract.py:170-177; its einsum path gets this product
 * from autograd, its Triton path is inference-only, _flashallegro.py:727):
 *   gcgw[n][u] += sum_z x1[z][u][i_n] * gamma[idxs[z]][u][j_n] * gout[z][u][k_n]      (gcgw pre-zeroed, atomics).
 * Together with modes 0-2 above every derivative of the trilinear form is one of these four products, which is how
 * allegro_b200.nn.Contracter provides weight gradients and double backward (forces in the loss). */
int ab2_op_contract_wgrad(int dtype, int64_t E, int U, int d1, int d2, int dout, int nnz,
                          const int32_t* tab_ijk, const void* x1, const void* gamma, const void* gout,
                          const int64_t* idxs, void* gcgw, void* stream);

/* Gather rows: out[z][:] = sf * src[idxs[z]][:]  (adjoint of the scatter; _contract.py:205). */
int ab2_op_gather_rows(int dtype, int64_t E, int64_t row, double sf, const void* src,
                       const int64_t* idxs, void* out, void* stream);

/* ---- fused pipeline (centre-sorted CSR edges, component-major layout) --------------- */

/* tensorembed.py:86,91-93: Y[z][0..d) = SH_{l<=lmax}(vec[z]/|vec[z]|), "component"
 * normalisation; vec, Y are TAcc.  (a1, a2) */
int ab2_sh_fwd(int acc_dtype, int lmax, int64_t E, const void* vec, void* Y, void* stream);
/* backward of the above: gvec[z] (+)= d Y/d vec ^T gY[z]   (SURVEY appendix B step 8). */
int ab2_sh_bwd(int acc_dtype, int lmax, int64_t E, const void* vec, const void* gY, void* gvec,
               int accumulate, void* stream);

/* Generic fused linear layer (nequip ScalarMLPFunction layer, _allegro.py:251,278;
 * tensorembed.py:88-89; allegro_models.py:231-241):
 *   Out[M][N] (split over <=4 column segments) (+)= epi( act(concat_k A_k)[M][K] @ W[K][N] )
 * act: AB2_ACT_SILU applies silu to A on load; AB2_ACT_MUL_DSILU multiplies segment s of A on
 * load by silu'(a_aux[s][m][k]) (a_aux_ptr_host[s] may be NULL = plain segment): the MLP backward's
 * g_pre = g_h * silu'(pre) formed inside the consuming GEMM's (prefetched) prologue.
 * epi: AB2_EPI_MUL_DSILU multiplies the result by silu'(aux[m][n]).  W is [K][N] row-major in TAct (alpha pre-folded on host).
 * A segments: (ptr, leading dim in elements, width); widths sum to K; outputs likewise to N. */
int ab2_linear(int dtype, int64_t M, int K, int N, int n_a, const void* const* a_ptr_host,
               const int64_t* a_ld_host, const int32_t* a_width_host,
               const void* const* a_aux_ptr_host /* nullable */, const int64_t* a_aux_ld_host,
               int act, const void* W,
               const void* W_packed /* nullable: image from ab2_linear_pack -> wgmma path */,
               int n_o, void* const* o_ptr_host, const int64_t* o_ld_host,
               const int32_t* o_width_host, const int32_t* o_accum_host, int epi, const void* aux,
               int64_t aux_ld, void* stream);
/* ab2_linear with the MLP nonlinearity `nonlin` (AB2_NL_*) in place of SiLU: act applies phi or multiplies by phi'(a_aux),
 * epi multiplies by phi'(aux).  fp32 / bf16 storage evaluate phi and phi' with fast fp32 intrinsics (gelu: erfcf), fp64
 * with the IEEE functions.  Returns 1 (and sets ab2_last_error) for an unknown nonlin. */
int ab2_linear_nl(int dtype, int64_t M, int K, int N, int n_a, const void* const* a_ptr_host,
                  const int64_t* a_ld_host, const int32_t* a_width_host,
                  const void* const* a_aux_ptr_host /* nullable */, const int64_t* a_aux_ld_host,
                  int act, const void* W, const void* W_packed /* nullable */,
                  int n_o, void* const* o_ptr_host, const int64_t* o_ld_host,
                  const int32_t* o_width_host, const int32_t* o_accum_host, int epi, const void* aux,
                  int64_t aux_ld, void* stream, int nonlin);

/* Tensor-core (wgmma) path of ab2_linear.  ab2_linear_packed_bytes returns the size of the
 * packed weight image (bf16 hi + lo parts in the GMMA canonical K-major core-matrix layout) or 0
 * if (dtype, K, N) is not eligible (fp64, K % 16 != 0, K > 512); ab2_linear_pack builds it on the
 * device from W[K][N].  Any N is accepted: outputs wider than 128 columns, or whose W image does not
 * fit the shared-memory budget (128 KB), run as column slices (one launch per slice, W slice resident).
 * With fp32 storage the kernel computes A_hi W_hi + A_lo W_hi + A_hi W_lo in bf16 MMAs with fp32
 * accumulation (~2^-16 relative). */
int64_t ab2_linear_packed_bytes(int dtype, int K, int N);
int ab2_linear_pack(int dtype, int K, int N, const void* W, void* packed, void* stream);

/* Two-layer SiLU MLP in one tensor-core kernel (the latent and readout MLPs, _allegro.py:278; allegro_models.py:231-241),
 * with the hidden layer kept on chip:
 *   backward == 0:  pre = A @ W1 (written, [M][H]),       Out (+)= silu(pre) @ W2
 *   backward != 0:  pre is read,                           Out (+)= ((A @ W1) * silu'(pre)) @ W2
 * A: n_a row segments (ptr, leading dim, width) whose widths sum to K; Out: n_o column segments summing to N, each with
 * its own accumulate flag.  W1 [K][H] and W2 [H][N] are given as ab2_linear_pack images.  For the MLP backward pass
 * A = Gout, W1 = W2_fwd^T, W2 = W1_fwd^T and Out = Gin.
 * Rank-1 backward (w1_row != NULL): K = 1, A is the single gradient column and w1_row the H fp32 entries of the 1 x H
 * matrix W1; the first stage is then an exact fp32 product (no packed W1).
 * Numerics: the same split-bf16 MMAs, k order and SiLU / silu' arithmetic as the two ab2_linear launches it replaces, so
 * the results are bitwise theirs, except in rank-1 mode, whose first stage is more accurate than the split MMA.
 * Returns AB2_NOT_ELIGIBLE (nothing enqueued, no error set) for what the kernel does not take: dtype other than AB2_F32,
 * A segments not multiples of 32 columns (except the rank-1 column) or not 16-byte aligned, H other than 32 or 64, N above
 * 256, or W1 + W2 + pipeline exceeding the shared memory of one SM.  The caller then runs the MLP as
 * two ab2_linear calls. */
#define AB2_NOT_ELIGIBLE (-1)
int ab2_mlp2(int dtype, int backward, int64_t M, int K, int H, int N, int n_a, const void* const* a_ptr_host,
             const int64_t* a_ld_host, const int32_t* a_width_host, const void* W1_packed, const void* W2_packed,
             const void* w1_row /* nullable: rank-1 backward */, void* pre, int64_t pre_ld, int n_o,
             void* const* o_ptr_host, const int64_t* o_ld_host, const int32_t* o_width_host,
             const int32_t* o_accum_host, void* stream);
/* ab2_mlp2 with the nonlinearity `nonlin` (AB2_NL_*) in place of SiLU: forward Out (+)= phi(pre) @ W2, backward
 * Out (+)= ((A @ W1) * phi'(pre)) @ W2.  The results are bitwise those of the two ab2_linear_nl launches it replaces (with
 * the rank-1 exception above).  Returns 1 (and sets ab2_last_error) for an unknown nonlin. */
int ab2_mlp2_nl(int dtype, int backward, int64_t M, int K, int H, int N, int n_a, const void* const* a_ptr_host,
                const int64_t* a_ld_host, const int32_t* a_width_host, const void* W1_packed, const void* W2_packed,
                const void* w1_row /* nullable: rank-1 backward */, void* pre, int64_t pre_ld, int n_o,
                void* const* o_ptr_host, const int64_t* o_ld_host, const int32_t* o_width_host,
                const int32_t* o_accum_host, void* stream, int nonlin);

/* Last latent MLP + readout MLP in one tensor-core kernel per direction (two-layer SiLU MLPs, hidden width H).  The
 * readout reads X[:, :P + S] and the last latent MLP reads [X[:, :P] | s] and writes x_L = X[:, P:P+S], with P = S L;
 * x_L and its gradient stay on chip.  W1_ro = [W1_ro_a ; W1_ro_b] is the readout's first layer split by rows at P, w2_ro
 * its H x 1 output layer (H fp32 values).
 *   backward == 0:  reads x = X[:, :P] and s [M][U]; writes pre_l = [x | s] @ W1_lat, xl = x_L = silu(pre_l) @ W2_lat,
 *                   pre_r = x @ W1_ro_a + x_L @ W1_ro_b and ez = Ez = silu(pre_r) @ w2_ro.
 *                   w_packed = {W1_lat [P+U][H], W2_lat [H][S], W1_ro_a [P][H], W1_ro_b [S][H]}.
 *   backward != 0:  reads ez = gEz [M][1], pre_l and pre_r; g_r = gEz w2_ro^T * silu'(pre_r),
 *                   g_h = ((g_r @ W1_ro^T[:, P:]) @ W2_lat^T) * silu'(pre_l); writes x = gX[:, :P] =
 *                   g_h @ W1_lat^T[:, :P] + g_r @ W1_ro^T[:, :P] and s = gs = g_h @ W1_lat^T[:, P:].  gX[:, P:] is not
 *                   formed.  xl is unused.  w_packed = {W1_ro^T [H][P+S], W2_lat^T [S][H], W1_lat^T [H][P+U]}.
 * All matrices are ab2_linear_pack images.  Numerics: pre_l, x_L, pre_r, gX[:, :P] and gs are bitwise those of the two
 * ab2_mlp2 calls this replaces (forward: last latent, then readout; backward: rank-1 readout, then last latent).  Ez is
 * an fp32 dot product of silu(pre_r) and w2_ro instead of the split-bf16 MMA, so it differs in the last bits.
 * Returns AB2_NOT_ELIGIBLE (nothing enqueued, no error set) for dtype other than AB2_F32, H or S other than 64, P or U
 * not multiples of 32, P + U above 512 (backward: above 256), operands not 16-byte aligned, a missing packed image, or a
 * shared-memory plan that does not fit one SM.  The caller then runs the two MLPs separately. */
int ab2_mlp2_readout(int dtype, int backward, int64_t M, int P, int S, int U, int H, void* x, int64_t x_ld, void* s, int64_t s_ld,
                     void* xl, int64_t xl_ld, void* pre_l, int64_t pre_l_ld, void* pre_r, int64_t pre_r_ld, void* ez, int64_t ez_ld,
                     const void* const* w_packed_host, const void* w2_ro, void* stream);
/* ab2_mlp2_readout with one nonlinearity `nonlin` (AB2_NL_*) for both MLPs in place of SiLU (silu / silu' above become
 * phi / phi').  The same numerics contract holds against two ab2_mlp2_nl calls.  Returns 1 (and sets ab2_last_error) for
 * an unknown nonlin; AB2_NOT_ELIGIBLE as above. */
int ab2_mlp2_readout_nl(int dtype, int backward, int64_t M, int P, int S, int U, int H, void* x, int64_t x_ld, void* s, int64_t s_ld,
                        void* xl, int64_t xl_ld, void* pre_l, int64_t pre_l_ld, void* pre_r, int64_t pre_r_ld, void* ez, int64_t ez_ld,
                        const void* const* w_packed_host, const void* w2_ro, void* stream, int nonlin);

/* _channels.py:44-57 + _contract.py:195-204 fused: gamma[c][j][u] =
 *   sf * sum_{z in row c} Y[z][j] * w[z][irrep(j)][u]      (a4, a7; deterministic, no atomics) */
int ab2_env_sum(int dtype, int lmax, int64_t N, int U, const int32_t* row_ptr, const void* Y,
                const void* w, int64_t w_ld, double sf, void* gamma, void* stream);

/* Adjoint of ab2_env_sum given ggamma[N][d][U]:
 *   gw[z][r][u] = sf * sum_{j in r} Y[z][j] ggamma[c][j][u]
 *   gY[z][j]   += sf * sum_u w[z][irrep(j)][u] ggamma[c][j][u]     (appendix B steps 3-4) */
int ab2_env_bwd(int dtype, int lmax, int64_t N, int64_t E, int U, const int32_t* row_ptr,
                const int32_t* ctr, const void* Y, const void* w, int64_t w_ld, const void* ggamma,
                double sf, void* gw, int64_t gw_ld, void* gY, void* stream);

/* _contract.py:205-251 for one layer on the fused layout (a8, a10):
 *   Vout[z][k][u] = sum_i Vin[z][i][u] * M_c[u][i][k],
 *   M_c[u][i][k]  = sum_nnz cgw[nnz][u] * gamma[c][j_nnz][u]      (built once per centre)
 * tab_ijk must be sorted by (i, k) (entries of one output target contiguous): the fast kernels
 * gather every M[i][k] from its table segment.
 * implicit_v0 != 0: Vin[z][i][u] = Y[z][i] * w0[z][irrep(i)][u] is formed on the fly
 * (tensorembed.py:95) and never stored. */
int ab2_tp_fwd(int dtype, int lmax, int64_t N, int64_t E, int U, int d_in, int d_out, int nnz,
               const int32_t* tab_ijk, const void* cgw, const int32_t* row_ptr, const int32_t* ctr,
               const void* gamma, const void* Vin, int implicit_v0, const void* Y, const void* w0,
               int64_t w0_ld, void* Vout, void* stream);

/* Backward of ab2_tp_fwd (appendix B steps 1-2): given gVout,
 *   gVin[z][i][u] = sum_k M_c[u][i][k] gVout[z][k][u]
 *   ggamma[c][j][u] = sum_nnz cgw * sum_{z in c} Vin[z][i][u] gVout[z][k][u]
 * implicit_v0: instead of gVin writes gw0[z][r][u] and accumulates into gY[z][i]. */
int ab2_tp_bwd(int dtype, int lmax, int64_t N, int64_t E, int U, int d_in, int d_out, int nnz,
               const int32_t* tab_ijk, const void* cgw, const int32_t* row_ptr, const int32_t* ctr,
               const void* gamma, const void* Vin, int implicit_v0, const void* Y, const void* w0,
               int64_t w0_ld, const void* gVout, void* gVin, void* gw0, int64_t gw0_ld, void* gY,
               void* ggamma, void* stream);

/* The two tensor products of a two-layer l_max = 2 model composed per centre, so that the layer-1 features V_1 and
 * their gradient are never formed (_allegro.py:237-301 with nothing between the layers on the tensor track).
 * Layer 0 is 9 x 9 -> 9 with implicit V_0, layer 1 is 9 x 9 -> 1; cgw0 [83][U] and cgw1 [9][U] are in the order of
 * the baked structures Tab9x9x9 / Tab9x9x1 (tp_tables_generated.cuh), which the caller checks on the host.  Per
 * channel u, with v0[i] = Y[z][i] w0[z][l(i)][u]:
 *   M0_c[i][k] = sum_{(i,j,k) in tab0} cgw0 gamma0[c][j],   M1_c[k] = sum_{(k,j,0) in tab1} cgw1 gamma1[c][j]
 *   A_c[i] = M0_c[i][0],   B_c[i] = sum_k M0_c[i][k] M1_c[k]
 * Forward:  last = 0: s[z][u] = sum_i A_c[i] v0[i]  (= V_1[z][0][u]);  last = 1: s[z][u] = sum_i B_c[i] v0[i]
 *           (= the layer-1 output);  gamma1 / cgw1 are only read when last = 1.
 * Backward, g1 = d/ds_1 and g2 = d/ds_2 as [E][U]:
 *   first = 0: ggamma[c][j] = gamma1's gradient = sum_{(k,j,0) in tab1} cgw1 sum_i M0_c[i][k] G_c[i],
 *              G_c[i] = sum_{z in c} g2[z] v0[i]   (reads Y, w0, g2; g1 / gw0 / gY unused)
 *   first = 1: gv0[i] = A_c[i] g1 + B_c[i] g2;  gw0[z][l][u] = sum_{i in l} Y[z][i] gv0[i];
 *              gY[z][i] += sum_u w0[z][l(i)][u] gv0[i];
 *              ggamma[c][j] = gamma0's gradient = sum_{(i,j,k) in tab0} cgw0 (delta_k0 H_c[i] + M1_c[k] G_c[i]),
 *              H_c[i] = sum_{z in c} g1[z] v0[i]
 * ggamma is written once per centre (zero for centres without edges), in a fixed order, no atomics.  All buffers are
 * fp32 and dense: Y / gY [E][9], w0 / gw0 [E][3U], s / g1 / g2 [E][U], gamma0 / gamma1 / ggamma [N][9][U].  Returns
 * AB2_NOT_ELIGIBLE (nothing enqueued, no error set) for dtype other than AB2_F32, U other than 32 or 64, E >= 2^31, or
 * a gamma / w0 / g1 / g2 base that is null or not 16-byte aligned. */
int ab2_tp_chain_fwd(int dtype, int last, int64_t N, int64_t E, int U, const int32_t* row_ptr, const int32_t* ctr,
                     const void* cgw0, const void* cgw1, const void* gamma0, const void* gamma1, const void* Y,
                     const void* w0, void* s, void* stream);
int ab2_tp_chain_bwd(int dtype, int first, int64_t N, int64_t E, int U, const int32_t* row_ptr, const int32_t* ctr,
                     const void* cgw0, const void* cgw1, const void* gamma0, const void* gamma1, const void* Y,
                     const void* w0, const void* g1, const void* g2, void* gw0, void* gY, void* ggamma, void* stream);

/* edgewise.py:40-60 (a12): Ei[c] = factor * sum_{z in row c} Ez[z]   (TAcc, deterministic). */
int ab2_edge_sum(int acc_dtype, int64_t N, const int32_t* row_ptr, const void* Ez, double factor,
                 void* Ei, void* stream);
/* adjoint: gEz[z] = factor * gEi[ctr[z]] */
int ab2_edge_sum_bwd(int acc_dtype, int64_t E, const int32_t* ctr, const void* gEi, double factor,
                     void* gEz, void* stream);

/* Force assembly (appendix B step 9): F[a] = sum_{z in CSR row a} g[z] - sum_{z: nbr[z]=a} g[z].
 * Both sums are segmented reductions in a fixed order (deterministic, no atomics, F need not be
 * zeroed): the neighbour side walks the TRANSPOSED CSR, col_ptr[n_total+1] / col_perm[E] = edge ids
 * grouped by neighbour atom (built once per neighbour list).  N = number of centres (owned atoms),
 * n_total = rows of F (owned + ghost atoms, allegro/_compile.py:41-61).  F: acc dtype. */
int ab2_force_scatter(int acc_dtype, int64_t N, int64_t n_total, int64_t E, const int32_t* row_ptr,
                      const int32_t* col_ptr, const int32_t* col_perm, const void* gvec, void* F,
                      void* stream);
/* ab2_force_scatter plus the centroid per-atom virial (Fan et al., PRB 92, 094301 (2015)) in the same walk:
 *   W[a][p][q] = - sum_{z : nbr[z] = a} vec[z][p] gvec[z][q]          W: [n_total][3][3], acc dtype
 * vec[z] = pos[nbr[z]] - pos[ctr[z]] (+ shift) and gvec[z] = dE/dvec[z].  In Allegro vec[z] reaches only the energy of
 * its centre, so gvec[z] = dE_ctr(z)/dvec[z] and W is exact.  W has 9 components and is NOT symmetric.
 * Sign: sum_a W[a] = -vec^T gvec = -dE/d(strain) before symmetrisation, the sign LAMMPS uses for its virial (sym of the
 * sum is the `virial` output of the Python layer).  Ghost rows (a >= N) carry the contributions their owners must
 * receive, like ghost forces.  F is bitwise ab2_force_scatter's for the same gvec; W is reduced in a fixed order (no
 * atomics, no zero-fill needed).  A pair style maps W[a] to LAMMPS' 9-component cvatom order
 *   cvatom[a] = { W[a][0][0], W[a][1][1], W[a][2][2], W[a][0][1], W[a][0][2], W[a][1][2], W[a][1][0], W[a][2][0], W[a][2][1] }
 * (xx, yy, zz, xy, xz, yz, yx, zx, zy).  vec may be null when E == 0. */
int ab2_force_virial_scatter(int acc_dtype, int64_t N, int64_t n_total, int64_t E, const int32_t* row_ptr,
                             const int32_t* col_ptr, const int32_t* col_perm, const void* vec, const void* gvec,
                             void* F, void* W, void* stream);

/* ---- upstream two-body scalar track + geometry (SURVEY section 8 row f1) ------------------ */

/* nequip with_edge_vectors_ (tensorembed.py:86): vec[z] = pos[nbr[z]] - pos[ctr[z]] (+ shift[z]),
 * computed in the positions' dtype (AB2_F64 / AB2_F32), stored in the accumulate dtype.
 * shift = edge_cell_shift @ cell, nullable. */
int ab2_edge_vec(int pos_dtype, int acc_dtype, int64_t E, const void* pos, const int32_t* ctr,
                 const int32_t* nbr, const void* shift, void* vec, void* stream);

/* EdgeLengthNormalizer + BesselEdgeLengthEncoding*PolynomialCutoff + ProductTypeEmbedding
 * (allegro_models.py:153-157, scalarembed.py:60-81, _edgeembed.py:68-85):
 *   x = |vec| / rmax_table[t_c][t_n];  B_n = sin(pi w_n x)/(pi x) * f_p(x);
 *   e0[z][c] = (c < S_rc/2 ? center_embed[t_c][c] : neighbor_embed[t_n][c - S_rc/2]) * sum_n B_n Wb[n][c]
 * Tables are in the accumulate dtype; e0 in the activation dtype. */
int ab2_radial_fwd(int dtype, int64_t E, int S_rc, int num_bessels, double p_cut, const void* vec,
                   const int32_t* ctr, const int32_t* nbr, const int32_t* types,
                   const void* rmax_table, int num_types, const void* bessel_w, const void* Wb,
                   const void* center_embed, const void* neighbor_embed, void* e0, void* stream);
/* adjoint: gvec[z] += (d e0 / d vec)^T g_e0[z] */
int ab2_radial_bwd(int dtype, int64_t E, int S_rc, int num_bessels, double p_cut, const void* vec,
                   const int32_t* ctr, const int32_t* nbr, const int32_t* types,
                   const void* rmax_table, int num_types, const void* bessel_w, const void* Wb,
                   const void* center_embed, const void* neighbor_embed, const void* g_e0,
                   void* gvec, void* stream);

/* ---- neighbour list on the device, directly in CSR (SURVEY section 8 row f2) --------------- */

/* Cell-list search on an orthorhombic box with per-axis periodicity.  The reference receives edge_index [2,E] int64
 * from nequip's data pipeline / LAMMPS (allegro/nn/_allegro.py:238, allegro/_compile.py:41-61); these three kernels
 * produce the centre-sorted CSR (row_ptr / nbr int32) and the per-edge shift VECTORS the path consumes, without the
 * int64 COO list.  Host-side geometry: box[3], origin[3] (doubles), pbc[3], ncell[3] with box/ncell >= r_max,
 * >= 3 cells on every periodic axis and fewer than 2^31 - 1 cells in all.  An open axis spans [origin, origin + box):
 * every position must lie inside it; one cell wider than r_max is valid for a layer thinner than the cutoff.  pos: [n][3] fp64 or fp32, raw (unwrapped) coordinates;
 *   r = pos[nbr] + shift - pos[centre]  holds for the raw positions.
 * Call order: ab2_nl_bin -> (host: order = stable argsort(cell_id), cell_start = prefix sum of the cell histogram)
 *             -> ab2_nl_count -> (host: row_ptr = prefix sum) -> ab2_nl_fill.
 * Centres are atoms [0, n_centres) (owned atoms first, ghosts after: only owned atoms get rows). */
int ab2_nl_bin(int pos_dtype, int64_t n, const void* pos, const double* box_host, const double* origin_host,
               const int32_t* pbc_host, const int32_t* ncell_host, double r_max, int32_t* cell_id, void* stream);
int ab2_nl_count(int pos_dtype, int64_t n_centres, const void* pos, const double* box_host,
                 const double* origin_host, const int32_t* pbc_host, const int32_t* ncell_host, double r_max,
                 const int32_t* cell_start, const int32_t* order, int32_t* counts, void* stream);
int ab2_nl_fill(int pos_dtype, int64_t n_centres, const void* pos, const double* box_host,
                const double* origin_host, const int32_t* pbc_host, const int32_t* ncell_host, double r_max,
                const int32_t* cell_start, const int32_t* order, const int32_t* row_ptr, int32_t* nbr,
                void* shift, void* stream);

/* The same search on a general lattice: triclinic or left-handed cells, periodic axes of any height (also below r_max),
 * open axes whose cell rows are replaced for binning.  Host-side geometry: rows[9] (row-major 3x3 binning rows a, b,
 * c, doubles; the inverse is computed inside), origin[3] (fractional, in units of the rows), pbc[3], ncell[3] bins per
 * axis and reach[3] bins walked either side of a centre's bin.  Atoms are binned by f = pos . rows^-1 - origin; on a
 * periodic axis img0 = floor(f) and the wrapped position is pos - img0 . rows; on an open axis every f must lie in
 * [0, 1).  With H_a = |det| / |row_p x row_q| the height of the cell along a and t_a = H_a / ncell[a] the bin thickness,
 * every axis needs t_a * reach[a] >= r_max (to 1 - 1e-12); the rows must be finite and non-singular, and there must be
 * fewer than 2^31 - 1 bins in all and fewer than 2^31 - 1 bins visited per centre.  Each call checks all of this
 * before it launches anything.  Wrap, bin and distance test run in fp64 for fp32 positions too; a row's shift
 * (im - img0[nbr] + img0[centre]) . rows is rounded once to the positions' dtype and is exactly 0 along axes with
 * pbc = 0, so  r = pos[nbr] + shift - pos[centre]  holds for the raw positions.  Rows come out in bin-walk order, fixed
 * for a given frame.  Call order, host steps and centres as for ab2_nl_*: ab2_nl_lattice_bin -> (order, cell_start)
 * -> ab2_nl_lattice_count -> (row_ptr) -> ab2_nl_lattice_fill. */
int ab2_nl_lattice_bin(int pos_dtype, int64_t n, const void* pos, const double* rows_host, const double* origin_host,
                       const int32_t* pbc_host, const int32_t* ncell_host, const int32_t* reach_host, double r_max,
                       int32_t* cell_id, void* stream);
int ab2_nl_lattice_count(int pos_dtype, int64_t n_centres, const void* pos, const double* rows_host,
                         const double* origin_host, const int32_t* pbc_host, const int32_t* ncell_host,
                         const int32_t* reach_host, double r_max, const int32_t* cell_start, const int32_t* order,
                         int32_t* counts, void* stream);
int ab2_nl_lattice_fill(int pos_dtype, int64_t n_centres, const void* pos, const double* rows_host,
                        const double* origin_host, const int32_t* pbc_host, const int32_t* ncell_host,
                        const int32_t* reach_host, double r_max, const int32_t* cell_start, const int32_t* order,
                        const int32_t* row_ptr, int32_t* nbr, void* shift, void* stream);

/* ---- batches of frames: many small frames concatenated into one graph ------------------------ */

/* All-pairs search for a batch of frames (nequip's batched data: `batch`, `num_atoms`, one cell per frame), for any
 * cell the all-pairs search of the reference data pipeline accepts: triclinic, narrower than r_max (several images per
 * axis, n_a = ceil(r_max / h_a) with h_a the cell height along axis a), mixed per-axis periodicity, or no periodic axis
 * at all (a molecule: no wrap, one image).  Each centre checks every atom of its own frame over the frame's image
 * range, so the work of frame b is O(N_b^2 * images): meant for small frames (the Python wrapper caps them).
 * Geometry, all device buffers: frame_ptr[n_frames+1] int32 (atoms of frame b are [frame_ptr[b], frame_ptr[b+1]),
 * frame_ptr[0] = 0, frame_ptr[n_frames] = n), cell / inv_cell [n_frames][3][3] (rows = lattice vectors; inv_cell its
 * inverse, any finite values for a frame with no periodic axis), pbc [n_frames][3] int32, nimg [n_frames][3] int32 the
 * images searched on each side of every periodic axis (ceil(r_max / h_a); ignored on open axes).  The kernels walk
 * prod(2 nimg_a + 1) images per pair as given: the caller bounds them (the Python wrapper _lib.nl_frames computes them
 * on the host with data.frames_geometry, which refuses near-singular cells and caps the product at
 * data.FRAMES_MAX_IMAGES).  pos: [n][3] fp64 or fp32
 * raw (unwrapped) coordinates; cell, inv_cell and shift in the same dtype.  Positions are wrapped along the periodic
 * axes in fractional coordinates (frac = pos @ inv_cell, image = floor(frac)) and the raw images folded back, so
 *   r = pos[nbr] + shift - pos[centre]  holds for the raw positions; shift = (integer image) @ cell.
 * Rows are ordered by neighbour index, then by image (x, y, z) lexicographically.  Every atom is a centre.
 * Call order: ab2_nl_frames_count -> (host: row_ptr = prefix sum of counts) -> ab2_nl_frames_fill. */
int ab2_nl_frames_count(int pos_dtype, int64_t n, int64_t n_frames, const int32_t* frame_ptr, const void* pos,
                        const void* cell, const void* inv_cell, const int32_t* pbc, const int32_t* nimg, double r_max,
                        int32_t* counts, void* stream);
int ab2_nl_frames_fill(int pos_dtype, int64_t n, int64_t n_frames, const int32_t* frame_ptr, const void* pos,
                       const void* cell, const void* inv_cell, const int32_t* pbc, const int32_t* nimg, double r_max,
                       const int32_t* row_ptr, int32_t* nbr, void* shift, void* stream);

/* Pruning of any centre-sorted list above (or a slab's local list) to per-edge-type list radii (the reference's
 * per_edge_type_cutoff, allegro_models.py:42,122,156).  Edge z of row i (neighbour j = nbr[z], shift s = shift[z]) is
 * kept iff
 *   d2 < cut2[types[i] * num_types + types[j]],   d2 = ((dx * dx + dy * dy) + dz * dz),   d_x = (pos[j][x] + s[x]) - pos[i][x]
 * every operation in fp64 with round-to-nearest and no contraction (fp32 positions and shifts convert exactly), so a
 * restatement in any language gets the same bits.  cut2 [num_types][num_types] fp64 device table of SQUARED radii,
 * directed: row = centre type, column = neighbour type.  An edge beyond its own cutoff r_ab contributes an exact zero to
 * the model (x = r / r_ab >= 1), so with cut2 = (rmax_table + skin)^2 the pruned list gives the same energies, forces and
 * virials as the list it came from.  Rows i in [0, n_centres) (row_ptr [n_centres + 1] int32, n_edges = row_ptr[n_centres]
 * < 2^31 - 1); neighbours index the n >= n_centres atoms of pos [n][3] (fp64 or fp32; shift [n_edges][3] in the same
 * dtype) and types [n] int32 in [0, num_types) (not checked here: the Python wrapper data.prune_csr checks them).
 *   ab2_nl_prune_count: counts[i] = kept edges of row i                                         (one warp per row)
 *   ab2_nl_prune_fill : the kept edges of row i at out_row_ptr[i], in their input order; out_nbr and out_shift are bitwise
 *                       copies of nbr and shift
 * Call order: ab2_nl_prune_count -> (host: out_row_ptr = prefix sum of counts) -> ab2_nl_prune_fill.  n_centres = 0 or
 * n_edges = 0 launches nothing and writes nothing (every count is 0). */
int ab2_nl_prune_count(int pos_dtype, int64_t n_centres, int64_t n_edges, int num_types, const void* pos, const int32_t* types,
                       const double* cut2, const int32_t* row_ptr, const int32_t* nbr, const void* shift, int32_t* counts,
                       void* stream);
int ab2_nl_prune_fill(int pos_dtype, int64_t n_centres, int64_t n_edges, int num_types, const void* pos, const int32_t* types,
                      const double* cut2, const int32_t* row_ptr, const int32_t* nbr, const void* shift,
                      const int32_t* out_row_ptr, int32_t* out_nbr, void* out_shift, void* stream);

/* Per-frame reductions (nequip's per-graph sums of a batch):
 *   ab2_frame_sum     out[b] = sum_{a in [frame_ptr[b], frame_ptr[b+1])} x[a]                 x [n], out [n_frames]
 *   ab2_frame_virial  W[b] = sum_{z in frame b} vec[z] (x) gvec[z]                 vec, gvec [E][3], W [n_frames][3][3]
 *                     frame b's edges are [row_ptr[frame_ptr[b]], row_ptr[frame_ptr[b+1]])   (centre-sorted CSR)
 * in the accumulate dtype (acc_dtype fp64 or fp32; summed in fp64 and rounded once).  Every frame is cut into fixed
 * chunks counted from its own start and the chunk sums are added in chunk order: deterministic, no atomics, independent
 * of the launch and of the other frames in the batch; an empty frame gives exactly 0.  scratch: fp64 device buffer of
 * at least ab2_frame_scratch_elems(n or E, n_frames) * width elements (width 1 for the sum, 9 for the virial). */
int64_t ab2_frame_scratch_elems(int64_t total, int64_t n_frames);
int ab2_frame_sum(int acc_dtype, int64_t n, int64_t n_frames, const int32_t* frame_ptr, const void* x, double* scratch,
                  int64_t scratch_elems, void* out, void* stream);
int ab2_frame_virial(int acc_dtype, int64_t E, int64_t n_frames, const int32_t* frame_ptr, const int32_t* row_ptr,
                     const void* vec, const void* gvec, double* scratch, int64_t scratch_elems, void* W, void* stream);
/* Potential part of the heat current of every frame, from per-atom energies and the centroid per-atom virial:
 *   J[b][p] = sum_{a in frame b} ( e_atom[a] vel[a][p] + sum_q W[a][p][q] vel[a][q] )
 * e_atom [n], vel [n][3], W [n][3][3] (ab2_force_virial_scatter), J [n_frames][3], all in the accumulate dtype; summed
 * in fp64 and rounded once, with the chunking of the reductions above (a frame's J does not depend on the launch or on
 * the other frames; an empty frame gives 0).  One frame: n_frames = 1, frame_ptr = {0, n}.  scratch: at least
 * ab2_frame_scratch_elems(n, n_frames) * 3 elements.  The kinetic term sum_a m_a |v_a|^2 v_a / 2 needs masses and is
 * the caller's. */
int ab2_frame_heat_current(int acc_dtype, int64_t n, int64_t n_frames, const int32_t* frame_ptr, const void* e_atom,
                           const void* vel, const void* W, double* scratch, int64_t scratch_elems, void* J, void* stream);

/* Radial embedding with per-type-pair matrices: out[z][c] = sum_n B_n(x_z) PQ[t_c * T + t_n][n][c], B_n as above
 * (num_bessels must be 8, S <= 128).  PQ: [T*T][8][S] in the accumulate dtype.  The product embedding above is
 * PQ = typeemb(t_c,t_n)[c] * Wb[n][c]; because everything up to the first nonlinearity is linear
 * (allegro/nn/_edgeembed.py:68-85, allegro_models.py:153-183) the host may fold the first scalar_embed_mlp layer in,
 * PQ = Wb diag(typeemb) W_1, and receive that layer's pre-activation directly.
 * bwd: gvec[z] += (d out / d vec)^T (g_out[z] * silu'(aux[z]))   (aux nullable = plain g_out). */
int ab2_radial_pq_fwd(int dtype, int64_t E, int S, int num_bessels, double p_cut, const void* vec,
                      const int32_t* ctr, const int32_t* nbr, const int32_t* types, const void* rmax_table,
                      int num_types, const void* bessel_w, const void* PQ, void* out, void* stream);
int ab2_radial_pq_bwd(int dtype, int64_t E, int S, int num_bessels, double p_cut, const void* vec,
                      const int32_t* ctr, const int32_t* nbr, const int32_t* types, const void* rmax_table,
                      int num_types, const void* bessel_w, const void* PQ, const void* g_out, const void* aux,
                      void* gvec, void* stream);
/* ab2_radial_pq_bwd with phi'(aux[z]) of the nonlinearity `nonlin` (AB2_NL_*) in place of silu'(aux[z]).  Returns 1 (and
 * sets ab2_last_error) for an unknown nonlin. */
int ab2_radial_pq_bwd_nl(int dtype, int64_t E, int S, int num_bessels, double p_cut, const void* vec,
                         const int32_t* ctr, const int32_t* nbr, const int32_t* types, const void* rmax_table,
                         int num_types, const void* bessel_w, const void* PQ, const void* g_out, const void* aux,
                         void* gvec, void* stream, int nonlin);

/* ZBL pair term (reference call site allegro/model/allegro_models.py:270-288; the module is nequip's
 * nequip.nn.pair_potential.ZBL = LAMMPS pair_style zbl, constants of pair_zbl_const.h):
 *   Ez[z] = qq * Z_i Z_j / r * phi((Z_i^0.23 + Z_j^0.23) r / 0.46850) * u(r / rmax_table[t_c][t_n]),
 *   phi(x) = 0.18175 e^{-3.19980x} + 0.50986 e^{-0.94229x} + 0.28022 e^{-0.40290x} + 0.02817 e^{-0.20162x},
 * u = polynomial cutoff of order p_cut, qq = qqr2e / 2 (each pair is two directed edges); and
 *   gvec[z] += dEz/dvec[z].
 * vec, Z [num_types], rmax_table [num_types^2], Ez [E], gvec [E][3] in the accumulate dtype; Ez or gvec may be null. */
int ab2_zbl(int acc_dtype, int64_t E, int num_types, double p_cut, double qq, const void* vec, const int32_t* ctr,
            const int32_t* nbr, const int32_t* types, const void* Z, const void* rmax_table, void* Ez, void* gvec,
            void* stream);

/* ---- ghost-atom halo exchange over NVLink peer memory (SURVEY section 8e) ------------------- */

/* One mailbox per rank (cudaMalloc'ed here so that it can be exported through CUDA IPC), mapped by its peers.
 * Per step: ab2_p2p_begin (bumps the step counter), ab2_p2p_push_rows into the neighbours' mailboxes (positions of
 * my boundary atoms / gradients of my ghosts), ab2_p2p_wait_unpack of what they pushed into mine, and
 * ab2_p2p_allreduce_energy -- kernels only (peer stores + system-scope release/acquire flags), so the whole step
 * including the halo replays from one CUDA graph with no NCCL call.  Waits are bounded (~2 s): a protocol error sets
 * the mailbox's error word (ab2_p2p_error) instead of hanging the GPU.  There is no reference counterpart (the
 * reference leaves domain decomposition to LAMMPS' MPI, allegro/_compile.py:41-61 only defines the ghost format). */
int64_t ab2_p2p_mailbox_bytes(int max_rows, int world);
int ab2_p2p_alloc(int64_t bytes, void** ptr);
int ab2_p2p_free(void* ptr);
int ab2_p2p_get_handle(void* ptr, void* handle64_host);
int ab2_p2p_open_handle(const void* handle64_host, void** ptr);
int ab2_p2p_close_handle(void* ptr);
int ab2_p2p_error(void* my_mailbox, int max_rows, int world, void* stream);
int ab2_p2p_begin(void* step_counter, void* stream);
int ab2_p2p_push_rows(int src_dtype, int kind, int side, const void* src, const int64_t* idx, int n, double shift_x,
                      void* peer_mailbox, int max_rows, int world, const void* step_counter, void* done_counter,
                      void* stream);
/* ab2_p2p_push_rows with a 3-component shift added to every row (positions of a triclinic cell, whose ghosts that cross
 * the periodic face of lattice row 0 move by that row); passed by value, so a captured graph replays it. */
int ab2_p2p_push_rows_v(int src_dtype, int kind, int side, const void* src, const int64_t* idx, int n, double shift_x, double shift_y,
                        double shift_z, void* peer_mailbox, int max_rows, int world, const void* step_counter, void* done_counter,
                        void* stream);
int ab2_p2p_wait_unpack(int dst_dtype, int kind, int side, void* my_mailbox, int max_rows, int world,
                        const void* step_counter, int n, void* dst, const int64_t* idx, int accumulate, void* stream);
int ab2_p2p_allreduce_energy(const void* e_local, int rank, int world, int max_rows, void* const* peers_dev,
                             void* my_mailbox, const void* step_counter, void* e_total, void* stream);

/* Extended mailbox for the stress, per-atom virial and heat current of a slab-decomposed step.  With
 * flags = AB2_P2P_EXT_VIRIAL, ab2_p2p_mailbox_bytes_ex sizes the base mailbox (same offsets, same error word, so every
 * call above works on it unchanged) followed by
 *   [parity][side] reverse rows of width 12, fp64: 3 gradient then 9 per-atom virial values W[a][p][q] (row-major),
 *   [parity][rank] a vector of up to AB2_P2P_VEC_MAX doubles,
 *   their flags;
 * flags = 0 gives exactly ab2_p2p_mailbox_bytes, unknown bits -1.  Every rank must allocate with the same flags: peers
 * compute offsets into each other's mailboxes from (max_rows, world, flags).
 * ab2_p2p_push_rows_w / ab2_p2p_wait_unpack_w are ab2_p2p_push_rows / ab2_p2p_wait_unpack (kind 1, accumulate) for the
 * width-12 rows: the push reads n gradient rows g_src[n][3] and n virial rows W_src[n][3][3] (both fp64 or both fp32;
 * the ghost rows, contiguous), the unpack adds them into g_dst[idx[i]] and W_dst[idx[i]] in one launch (idx entries
 * unique, null = row i).  A ghost's W row is what its owner must receive (ab2_force_virial_scatter), so after the two
 * unpacks (left neighbour's slot 0 first, then slot 1: fixed order) W_dst holds the owned atoms' full W.
 * ab2_p2p_allreduce_vec sums n_values (1..AB2_P2P_VEC_MAX) doubles over the ranks, in rank order: bitwise the same
 * result on every rank, and for n_values = 1 bitwise what ab2_p2p_allreduce_energy gives.  All waits are bounded and set
 * the mailbox's one error word (ab2_p2p_error). */
#define AB2_P2P_EXT_VIRIAL 1
#define AB2_P2P_VEC_MAX 16
int64_t ab2_p2p_mailbox_bytes_ex(int max_rows, int world, int flags);
int ab2_p2p_push_rows_w(int src_dtype, int side, const void* g_src, const void* W_src, int n, void* peer_mailbox,
                        int max_rows, int world, const void* step_counter, void* done_counter, void* stream);
int ab2_p2p_wait_unpack_w(int dst_dtype, int side, void* my_mailbox, int max_rows, int world,
                          const void* step_counter, int n, void* g_dst, void* W_dst, const int64_t* idx, void* stream);
int ab2_p2p_allreduce_vec(const void* v_local, int n_values, int rank, int world, int max_rows, void* const* peers_dev,
                          void* my_mailbox, const void* step_counter, void* v_total, void* stream);

/* Exchange plan of a 1-D slab decomposition along x, built on the device from one rank's atoms (slab rank of world,
 * each `width` wide, lo = rank * width, hi = lo + width).  ab2_slab_plan_count writes one class byte per atom into
 * cls[n] and per-block member counts into block_counts[ceil(n / 256)][4]; the caller turns the counts into exclusive
 * per-list prefix sums over the blocks (block_offsets, same shape), and ab2_slab_plan_fill writes each list k (null:
 * skipped) as int64 atom indices in ascending order, list k of block b starting at block_offsets[b][k].
 *   mode 0: wraps pos [n][3] (fp64 / fp32, in place) into [0, box[a]) on every axis, adding the boxes removed to
 *           image [n][3] int32, and classifies by s = clamp(floor(x / width), 0, world - 1): list 0 = stays (s == rank),
 *           list 1 = to the left neighbour, list 2 = to the right one (world 2: by the side of [lo, hi) the atom left
 *           by); column 3 counts refused atoms: bound for a non-adjacent slab, or with x before the wrap outside
 *           [lo - jump, hi + jump).  Refused atoms are in no list.
 *   mode 1: pos read only, image unused: list 0 = atoms with x < lo + r_list, list 1 = atoms with x >= hi - r_list
 *           (compared in fp64), list 2 empty.
 * n = 0 launches nothing.  Both launch on `stream`. */
int ab2_slab_plan_count(int pos_dtype, int mode, int64_t n, void* pos, int32_t* image, const double* box_host, int rank, int world,
                        double width, double jump, double r_list, uint8_t* cls, int32_t* block_counts, void* stream);
/* The same plan for any regular cell, cut along lattice row 0 in fractional coordinates s = pos . h^-1 (rows_host[9] =
 * the rows h_0, h_1, h_2; the inverse is computed here, and a non-finite, singular or near-coplanar cell is refused
 * before any launch).  Rank r owns s_0 in [lo, hi) = [r / world, (r + 1) / world).  Outputs as ab2_slab_plan_count;
 * ab2_slab_plan_fill takes them unchanged.
 *   mode 0: img_a = floor(s_a), pos <- pos - sum_a img_a h_a (fp64, rounded once to the positions' dtype), image += img;
 *           classified by clamp(floor(s_0 world), 0, world - 1) of the wrapped position; refused (column 3): the
 *           unwrapped s_0 outside [lo - jump, hi + jump) (jump in fractional units) or a non-adjacent slab.  world 2:
 *           left when the unwrapped s_0 < lo.
 *   mode 1: list 0 = s_0 < lo + r_list / H_0, list 1 = s_0 >= hi - r_list / H_0 (fp64; H_0 = |det h| / |h_1 x h_2|). */
int ab2_slab_plan_count_lattice(int pos_dtype, int mode, int64_t n, void* pos, int32_t* image, const double* rows_host, int rank, int world,
                                double jump, double r_list, uint8_t* cls, int32_t* block_counts, void* stream);
int ab2_slab_plan_fill(int64_t n, const uint8_t* cls, const int32_t* block_offsets, int64_t* list0, int64_t* list1, int64_t* list2,
                       void* stream);

/* layout helpers between the reference strided layout [z][u][i] and the internal [z][i][u] */
int ab2_transpose_ui(int dtype, int64_t E, int U, int d, const void* src, void* dst, int to_internal,
                     void* stream);

#ifdef __cplusplus
}
#endif
#endif
