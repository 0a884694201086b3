/*
 * spateo_b200.h — C ABI of the H100-native (sm_90a) morpho-align hot path (libspateo_b200.so).
 *
 * The reference (aristoteleo/spateo-release @ 9ce1a90) is pure Python: it has NO FFI for this path. The seam a
 * maintainer would bind is the array-backend seam `check_backend()/nx.*` (spateo/alignment/methods/utils.py:35-66)
 * under `Morpho_pairwise` (spateo/alignment/methods/morpho_class.py:54). Every entry point below replaces one math call
 * site of that class; the citation after each prototype is the reference code it replaces. INTEGRATION.md shows the
 * ctypes stub that binds them from the reference's side.
 *
 * Conventions: plain C types only; every pointer is a DEVICE pointer unless the name ends in `_host`; `stream` is a
 * cudaStream_t passed as void* (NULL = default stream); all functions return 0 on success or a cudaError_t / negative
 * SPB_E* code, and never synchronise the device unless documented. float = IEEE fp32, accumulators are fp64.
 *
 * Layout vocabulary (moving slice A = rows i, fixed slice B = columns j):
 *   ldx          row pitch: N_A rounded up to SPB_ROW_TILE. Per-row vectors are length ldx.
 *   xa / XAHat   [3][ldx] structure-of-arrays coordinates (unused dims = 0; pad rows i >= N_A hold 1e18).
 *   xb4          [N_B][4] fixed-slice coordinates (y0,y1,y2,0).
 *   GT           [N_B][ldx] expression-probability matrix g_ij stored COLUMN-OF-P-major (one contiguous row per
 *                fixed cell j; pad entries i >= N_A are 0). 4*N_A*N_B bytes: 40 GB at 100k x 100k.
 *   UT           [K][ldx] inducing-point kernel U^T.
 */
#ifndef SPATEO_B200_H
#define SPATEO_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SPB_ROW_TILE 512
#define SPB_COL_STAGE 8
#define SPB_COLCONST_FLOATS 20 /* per-column constant record of sweep 2 (see spb_em_params.colconst) */
#define SPB_MAX_K_FUSED 64 /* largest K solved by the in-library Jacobi kernel */
#define SPB_TRACE_STRIDE 8
#define SPB_COLMASK_WORDS 16 /* per-column bit mask over row blocks (sparse mode): up to 512 row blocks = 262,144 rows */
#define SPB_TRANSFER_PANEL 16 /* features per pass of the posterior-transfer kernels */

#define SPB_EINVAL (-2)
#define SPB_EUNSUPPORTED (-3)

/* dissimilarity metric / probability type codes (utils.py:900-941, :974-985) */
#define SPB_METRIC_KL 0
#define SPB_METRIC_EUC 1 /* "euc"/"euclidean": SQUARED distance (reference quirk) */
#define SPB_METRIC_COS 2
#define SPB_METRIC_SQRT_EUC 3 /* "square_euc": sqrt of the squared distance (reference quirk) */
#define SPB_METRIC_SYMKL 4    /* "sym_kl": operands are [Xn | log X] and [log Y | Yn]; e = (rowA + rowB - dot) / 2 */
#define SPB_PROB_GAUSS 0
#define SPB_PROB_COS 1
#define SPB_PROB_PROB 2

/* Scalar EM state, resident on the device (doubles; the reference keeps these as fp32 0-d arrays). */
typedef struct spb_scalars {
  double sigma2;          /* morpho_class.py:701,1426 */
  double sigma2_variance; /* annealed spatial variance factor (:705,1431) */
  double gamma;           /* inlier ratio (:724,1214) */
  double Sp;              /* (SVI: running average) sum of P (:1171-1185) */
  double Sp_spatial;
  double Sp_sigma2;
  double sigma2_related; /* (:1200) */
  double step;           /* SVI step size (:894) */
  double omega;          /* outlier mass of the current E-step (utils.py:1053) */
  double SpK;            /* un-averaged sum of K_NA of the current batch */
  double R[9];           /* row-major 3x3 (top-left DxD used) (:1374-1378) */
  double t[3];           /* (:1398-1402) */
  double dotKS;          /* sum_i K_NA_sigma2_i * SigmaDiag_i (:1427) */
  double sums[8];        /* scratch: Sp_spatial_new, Sp_sigma2_new, Sp_new, S2 */
  double visited;        /* (row block, column) tiles read by this iteration's sweeps, a tile counting (128-row quarters whose cost rows are read, colquarters) / 4 (all of them without culling) */
  float c_q;             /* -log2(e) / (2 sigma2) */
  float c_s;             /* c_q * sigma2_variance */
  int32_t nonrigid_flag; /* latched once iter > nonrigid_start_iter (:289-291) */
  int32_t iter;
} spb_scalars;

/* Everything one EM iteration touches. One field per line: spateo_release_b200/_capi.py parses this struct. */
typedef struct spb_em_params {
  int32_t NA;                  /* moving cells (rows) */
  int32_t NB;                  /* fixed cells (all columns) */
  int32_t NBb;                 /* columns per iteration: NB, or the SVI batch size */
  int32_t D;                   /* 2 or 3 */
  int32_t K;                   /* inducing points */
  int32_t ldx;                 /* row pitch (multiple of SPB_ROW_TILE) */
  int32_t svi;                 /* SVI_mode */
  int32_t nn_init;             /* coarse-init prior active */
  int32_t update_R;            /* morpho_class.py:1373 */
  int32_t nonrigid_start_iter; /* default 80 */
  int32_t seg1;                /* column segments of sweep 1 */
  int32_t seg2;                /* column segments of sweep 2 */
  int32_t nbb_pad;             /* pitch of the column-partial arrays */
  int32_t trace;               /* 1: record per-iteration scalars into trace_buf */
  int32_t cull;                /* 1: drop (row block, column) tiles whose every pair underflows to exactly 0 */
  int32_t g_on;                /* guidance pairs active (morpho_class.py:551-555) */
  int32_t g_nonrigid;          /* guidance_effect in ("nonrigid", "both") */
  int32_t g_rigid;             /* guidance_effect in ("rigid", "both") */
  int32_t g_NI;                /* number of guidance pairs */
  int32_t sparse_k;            /* > 0: sparse_calculation_mode with sparse_top_k = sparse_k (utils.py:1085-1094) */
  int32_t NB_total;            /* columns of the whole iteration when one call sees only a block of them (column-sharded pair: fixed cells of ALL ranks; column chunk: the iteration's NB or batch size); gamma update; 0 = NBb */
  int32_t gt_by_position;      /* 1: GT row j is the j-th column of THIS call (a cost chunk built for its columns), not fixed cell batch_idx[iter][j] */
  int32_t fold_add;            /* 1: spb_row_fold adds into rowstat[parity] instead of overwriting it (column chunks of one iteration, folded in order) */
  int32_t reserved1;
  double lambdaVF;
  double gamma_a;
  double gamma_b;
  double samples_s;            /* morpho_class.py:738-741 */
  double nn_init_weight;
  double sigma2_variance_decress;
  double sigma2_variance_end;
  double inl_SP;               /* sum inlier_P */
  double inl_Sa[3];            /* inlier_P^T inlier_A */
  double inl_Sb[3];            /* inlier_P^T inlier_B */
  double inl_Mab[9];           /* sum_n P_n a_n b_n^T */
  double pinv_eps;             /* machine epsilon of the reference's SigmaInv dtype: pinv cutoff = K * pinv_eps * max|ev| (scipy.linalg.pinv, utils.py:1435) */
  double g_weight;             /* guidance_weight */
  double g_meanXB;             /* X_BI.mean() over ALL elements (the reference adds this scalar to every axis) */
  double g_meanXA;             /* X_AI.mean() */
  const float* GT;             /* [NB][ldx] */
  const float* xa;             /* [3][ldx] rigidly-initialised normalised coords of A (coordsA) */
  const float* xb4;            /* [NB][4] */
  const float* UT;             /* [K][ldx] */
  const float* Gamma;          /* [K][K] GammaSparse */
  const float* kappa;          /* [ldx] */
  const int32_t* batch_idx;    /* [max_iter][NBb] SVI column indices per iteration, or NULL */
  float* alpha;                /* [ldx] */
  float* SigmaDiag;            /* [ldx] */
  float* lm;                   /* [ldx] log2(alpha * exp(-SigmaDiag/sigma2)) */
  float* mm;                   /* [ldx] alpha * exp(-SigmaDiag/sigma2) */
  float* VnA;                  /* [3][ldx] */
  float* RnA;                  /* [3][ldx] */
  float* XAHat;                /* [3][ldx] */
  float* K_NA;                 /* [ldx] */
  float* K_NA_spatial;         /* [ldx] */
  float* K_NA_sigma2;          /* [ldx] */
  float* PXB;                  /* [3][ldx] rows of P @ XB */
  float* PXB_term;             /* [3][ldx] (SVI running average) */
  float* K_NB;                 /* [NBb] */
  float* colgeom;              /* [nbb_pad][8] (y0,y0,y1,y1,y2,y2,0,0): this iteration's columns, duplicated for f32x2 */
  float* colconst;             /* [nbb_pad][SPB_COLCONST_FLOATS] (y0,y0,y1,y1, y2,y2,a,a, b,b,c,c, cy0,cy0,cy1,cy1, cy2,cy2,tau,tau); zero beyond NBb */
  float* colpart;              /* [ldx/ROW_TILE][4][nbb_pad] partial column sums of each row block, by position in its work list (sums 0 and 1 of the spatially dead columns are not stored: they are zero) */
  uint32_t* keepmask;          /* [ldx/ROW_TILE][(nbb_pad+31)/32] bit j of row rb: column j is on rb's work list, i.e. rb has column sums of j */
  uint32_t* livemask;          /* [ldx/ROW_TILE][(nbb_pad+31)/32] bit j of row rb: column j is on rb's work list before colsplit (spatially live) */
  int32_t* keepoff;            /* [ldx/ROW_TILE][(nbb_pad+31)/32][2] list position of the first spatially live / dead listed column of each 32-column word */
  float* rowpart;              /* [seg2][8][ldx] partial row statistics */
  float* bbox;                 /* [ldx/ROW_TILE][4][8] bounding box (lo0,lo1,lo2,hi0,hi1,hi2) of the XAHat of each 128-row quarter of each row block and the largest lm of the quarter (float 6) (valid rows only; a quarter without valid rows has lo > hi and lm -inf) */
  int32_t* collist;            /* [ldx/ROW_TILE][nbb_pad] per-row-block column work list */
  int32_t* colcount;           /* [ldx/ROW_TILE] list lengths */
  uint8_t* colquarters;        /* [ldx/ROW_TILE][nbb_pad] per list position: bit q set <=> rows 128q..128q+127 of the row block can hold a non-zero weight q = exp2(c_q d + lm) for that column (their cost rows are read) */
  uint8_t* colspatial;         /* [ldx/ROW_TILE][nbb_pad] per list position: bit q set <=> rows 128q..128q+127 of the row block can hold a non-zero spatial weight exp2(c_s d) for that column */
  int32_t* colsplit;           /* [ldx/ROW_TILE] list positions >= colsplit[rb] hold columns whose SPATIAL weights exp(-d/(2 sigma2/variance)) are exactly 0 for the whole row block (they only need the sigma2 / full posteriors) */
  uint32_t* colmask;           /* [nbb_pad][SPB_COLMASK_WORDS] sparse mode: row blocks that can hold a non-zero weight, or NULL */
  double* UtWU;                /* [K][K] accumulator */
  double* UtPXB;               /* [K][3] accumulator */
  double* SigmaInv;            /* [K][K] (SVI running average) */
  double* Sigma;               /* [K][K] pinv(SigmaInv) */
  double* Coff;                /* [K][3] */
  double* moments;             /* [32] rigid-update moment accumulator */
  double* jacobi_ws;           /* [1 + K*K] eigenbasis of the previous non-rigid solve ([0] = K once valid): Jacobi warm start, or NULL */
  const float* UT_hi;          /* [K][ldx] tf32 split of the row-centred UT (tensor-core K^T P K contraction); required when K > 32, NULL selects the fp64 kernel for K <= 32 */
  const float* UT_lo;          /* [K][ldx] */
  const float* UT_mean;        /* [K] row means of UT (spb_gram_center) */
  float* GB_hi;                /* [K+4][ldx] per-iteration B operand [K_NA o D ; PXB_term^T ; K_NA], hi part */
  float* GB_lo;                /* [K+4][ldx] */
  double* gram_sums;           /* [4] sum K_NA, sum_n PXB_term[e] */
  float* gram_scratch;         /* slice partials of the tensor-core contraction (spb_gram_tc_scratch_floats) */
  int64_t gram_scratch_floats;
  const double* g_XA;          /* [g_NI][3] normalised guidance points on the moving slice */
  const double* g_XB;          /* [g_NI][3] ... on the fixed slice */
  double* g_VA;                /* [g_NI][3] V_AI = U_I Coff */
  double* g_RA;                /* [g_NI][3] R_AI (iterated from zeros, morpho_class.py:1407-1408) */
  const double* g_UI;          /* [g_NI][K] kernel of the guidance points */
  const double* g_G1;          /* [K][K] U_I^T U_I */
  spb_scalars* sc;             /* device scalars */
  double* trace_buf;           /* [max_iter][SPB_TRACE_STRIDE] or NULL */
  double* red_scratch;         /* [red_scratch_doubles] block partials of the deterministic (ordered) grid reductions */
  int64_t red_scratch_doubles;
  uint32_t* red_counter;       /* [8] arrival tickets of those reductions (zero-initialised) */
  /* column-sharded pair (one slice pair over several GPUs, SURVEY 8(e)): every rank holds a block of fixed cells */
  /* (columns of P); sweep 1 is local, the per-row statistics of sweep 2 are summed over the ranks once per iteration */
  int32_t shard_rank;
  int32_t shard_world;         /* 0 / 1 = not sharded */
  double* rowstat;             /* [2][8][ldx] fp64 row statistics of THIS rank's columns, double-buffered by call parity */
  const uint64_t* peer_rowstat; /* device array [shard_world]: every rank's rowstat base mapped into this process (NVLink P2P), or NULL */
  uint64_t* shard_flags;       /* [shard_world] epochs written by the peers (this rank's own slot by itself) */
  const uint64_t* peer_flags;  /* device array [shard_world]: every rank's shard_flags base, P2P mapped */
} spb_em_params;

/* ---- library info ------------------------------------------------------------------------------------------- */
int spb_version(void);
/* number of kernels launched by this library since load (bench.py's gpu_launches) */
int64_t spb_launch_count(void);
/* sizeof the two structs as compiled (the ctypes mirror checks them at load time) */
int spb_sizeof_em_params(void);
int spb_sizeof_scalars(void);

/* ---- expression cost matrix: calc_distance + calc_probability (utils.py:647-788, :866-985) ------------------- */
/* KL pre-pass: Xn=(X+.01)/rowsum, xlogx=sum Xn log(Xn+1e-8); with is_fixed!=0 writes log(Xn+1e-8) instead, optionally
   centred by c_j = sum_g center_w[g] * (that row) which is returned in rowterm (the cost epilogue adds it back). */
int spb_kl_prepare_rows(const float* X, int64_t n, int64_t G, int64_t ldin, float* out, int64_t ldout, float* rowterm,
                        int32_t is_fixed, const float* center_w, void* stream); /* utils.py:683-695 */
/* row squared norms (euc) or row-normalisation (cos) */
int spb_rows_sqnorm(const float* X, int64_t n, int64_t G, int64_t ldin, float* rowterm, void* stream); /* utils.py:780 */
int spb_rows_normalize(const float* X, int64_t n, int64_t G, int64_t ldin, float* out, int64_t ldout, void* stream); /* utils.py:736-739 */
/* GT[j][i] (op)= prob(metric(A_i, B_j)); A:[NA][G] pitch lda, B:[NB][G] pitch ldb; accumulate!=0 multiplies into GT.
   wgmma tf32 with a 3xTF32 split: each operand is given as the hi/lo pair of spb_split_tf32, zero-padded to 32 features */
int spb_split_tf32(const float* x, float* hi, float* lo, int64_t n, void* stream);
int spb_gene_cost_tc(const float* A_hi, const float* A_lo, int64_t lda, const float* rowtermA, const float* B_hi,
                     const float* B_lo, int64_t ldb, const float* rowtermB, int64_t NA, int64_t NB, int64_t G, int32_t metric,
                     int32_t prob_type, float prob_param, int32_t accumulate, float* GT, int64_t ldx,
                     void* stream); /* utils.py:697,780-783,742 + :977-981 */
/* ---- K^T P K contraction on wgmma (3xTF32, fp32 accumulate per <= 4096-element slice, fp64 fold) ----------------------
   UtWU[k][l] = sum_n UT[k][n] w[n] UT[l][n]  (morpho_class.py:1266-1268; SparseVFC U^T P U, sparsevfc.py:189-198)
   UtX[k][e]  = sum_n UT[k][n] X[e][n], e < E <= 3  (morpho_class.py:1279)
   The tensor core's fp32 accumulator truncates, so the contraction runs on the row-centred kernel D = UT - mean (signed
   terms) and the rank-one corrections are added back in fp64:
     spb_gram_center  (once; UT is constant over the EM): mean[K], A_hi/A_lo = tf32 split of D            [K][ldn]
     spb_gram_prepare (every iteration): B_hi/B_lo rows k < K = w o D[k], rows K..K+E-1 = X[e], row K+E = w  [K+E+1][ldn]
                      and sums4 = (sum w, sum_n X[0], X[1], X[2]) in fp64
     spb_gram_tc      : the GEMM + fp64 reduction -> UtWU [K][K] (exactly symmetric), UtX [K][3]
   K + E + 1 <= 1024; scratch size from spb_gram_tc_scratch_floats. */
int spb_gram_tc_scratch_floats(int32_t K, int32_t E, int64_t N, int64_t* floats);
int spb_gram_center(const float* UT, int64_t ldn, int64_t N, int32_t K, float* mean, float* A_hi, float* A_lo, void* stream);
int spb_gram_prepare(const float* UT, int64_t ldn, int64_t N, int32_t K, const float* mean, const float* w, const float* X,
                     int64_t ldxx, int32_t E, float* B_hi, float* B_lo, double* sums4, void* stream);
int spb_gram_tc(const float* A_hi, const float* A_lo, const float* B_hi, const float* B_lo, int64_t ldn, int64_t N, int32_t K,
                int32_t E, const float* mean, const double* sums4, float* scratch, int64_t scratch_floats, double* UtWU,
                double* UtX, void* stream);
/* dst[r][0..width) = src[idx[r]][0..width) for r < n, in 4-byte words (pitches in words): the fixed-side operands of the
   columns of one iteration chunk (tf32 hi / lo, row terms, labels). 16-byte accesses when width, pitches and bases allow. */
int spb_gather_rows(const void* src, int64_t ld_src, int64_t width, const int32_t* idx, int64_t n, void* dst, int64_t ld_dst,
                    void* stream);
/* label layer: GT[j][i] (op)= LT[labA_i][labB_j] */
int spb_label_cost(const int32_t* labA, const int32_t* labB, const float* LT, int32_t nB_labels, int64_t NA, int64_t NB,
                   int32_t accumulate, float* GT, int64_t ldx, void* stream); /* utils.py:830 */

/* ---- E-step: calc_distance(euc) + get_P_core + row/col sums, P never materialised ---------------------------- */
int spb_gather_cols(const spb_em_params* p, int32_t iter, void* stream);   /* morpho_class.py:1149 */
/* row-block bounding boxes + per-block column work lists (exact zero-tile culling when p->cull) — new, no reference line */
int spb_estep_col_lists(const spb_em_params* p, void* stream);
int spb_estep_sweep1(const spb_em_params* p, int32_t iter, void* stream); /* utils.py:1049-1059,1063-1073,1080-1083 (column sums) */
int spb_col_finalize(const spb_em_params* p, void* stream);               /* utils.py:1053-1055 + denominators */
int spb_estep_sweep2(const spb_em_params* p, int32_t iter, void* stream); /* utils.py:1059-1083, morpho_class.py:1171-1176,1270,1357 */
int spb_row_finalize(const spb_em_params* p, void* stream);
/* column-sharded pair: (1) fold this rank's segment partials into rowstat[parity] (fp64); (2a) after the caller summed
   rowstat[parity] over the ranks (e.g. ncclAllReduce), finish the row statistics from it; or (2b) ONE kernel that signals
   the peers, waits for their epoch flags and sums their rowstat[parity] straight over NVLink peer memory in rank order
   (bit-identical on every rank) before finishing — no separate collective. epoch must increase by one per call on every rank. */
int spb_row_fold(const spb_em_params* p, int32_t parity, void* stream); /* p->fold_add: add instead of overwrite */
int spb_row_stats_finalize(const spb_em_params* p, int32_t parity, void* stream);
int spb_row_stats_p2p(const spb_em_params* p, int32_t parity, uint64_t epoch, void* stream);
/* dense P [NA][NBb] (row-major, pitch ldp) of the state left by the last E-step */
/* sparse_calculation_mode (p->sparse_k > 0): per-column top-k threshold tau_j of the full posterior by an exact radix
   select (one CTA per column), written to colconst[j][18..19]; K_NB_j becomes the kept mass. Call between
   spb_col_finalize and spb_estep_sweep2 (spb_em_iteration does). */
int spb_estep_col_select(const spb_em_params* p, int32_t iter, void* stream); /* utils.py:1085-1094,1369-1404 */
/* COO entries of the sparse posterior of the last E-step: rows[NBb][sparse_k], vals[NBb][sparse_k] (unordered inside a
   column; columns with fewer than sparse_k non-zero entries are filled with explicit zeros like the reference's sort) */
int spb_sparse_P_emit(const spb_em_params* p, int32_t iter, int32_t* rows, float* vals, void* stream); /* utils.py:1385-1392,1506-1510 */
/* Row / column maxima of the posterior of the last E-step without forming it: rowbest[NA], colbest[NBb] hold
   (float bits of P) << 32 | (0xffffffff - argmax index) — lowest index on ties; either pointer may be NULL.
   In sparse mode entries below a column's top-k threshold count as absent (0), as in the reference's sparse pi.
   colmap[NBb] (int32, device; NULL = the identity): the output column index of every column of the E-step, -1 for a column
   that is not part of the posterior (the row maxima skip it). The row keys carry colmap[j] instead of j, so a
   column-sharded pair passes its block's global column indices and merges the ranks' rowbest with a 64-bit maximum
   (keys of non-negative values are below 2^63). colbest is unchanged (row indices). */
int spb_posterior_argmax_mapped(const spb_em_params* p, int32_t iter, const int32_t* colmap, uint64_t* rowbest,
                                uint64_t* colbest, void* stream); /* spateo/alignment/utils.py:157-191 (get_optimal_mapping_relationship) */
int spb_materialize_P(const spb_em_params* p, int32_t iter, float* P, int64_t ldp, void* stream); /* utils.py:1083 */
/* Posterior transfer of the last E-step without forming P (sparse mode: the entries w >= tau_j, as sweep 2 keeps them).
   Both visit the tiles and quarters of the E-step's work lists, SPB_TRANSFER_PANEL features per pass, no float atomics.
   rows: out[f][i] (fp64, [ldf][ldx], processing order) = (P @ F_B)[i][f] for f < F; F_B is [rows of xb4][ldf] (fixed
         cells, ldf a multiple of SPB_TRANSFER_PANEL, pad features zero); part: [seg2][SPB_TRANSFER_PANEL][ldx] floats.
         The segment partials are folded in fp64 in segment order; p->fold_add adds into out (column chunks, in order).
   cols: out[j][f] (fp32, pitch ldo) = (P^T @ F_A)[j][f] for the NBb columns of the E-step; F_A is [roundup(F,
         SPB_TRANSFER_PANEL)][ldx] in processing order (pad rows and features zero); part: [ldx/ROW_TILE][SPB_TRANSFER_PANEL]
         [nbb_pad] floats, by list position; the row blocks are summed in fp64 in row-block order. */
int spb_posterior_transfer_rows(const spb_em_params* p, int32_t iter, const float* FB, int64_t ldf, int32_t F, float* part,
                                double* out, void* stream);
int spb_posterior_transfer_cols(const spb_em_params* p, int32_t iter, const float* FA, int32_t F, float* part, float* out,
                                int64_t ldo, void* stream);

/* ---- M-step pieces ---------------------------------------------------------------------------------------------- */
int spb_iter_begin(const spb_em_params* p, int32_t iter, void* stream);      /* morpho_class.py:894 + zeroing */
int spb_update_gamma_alpha(const spb_em_params* p, void* stream);            /* morpho_class.py:1178-1252 */
int spb_nonrigid_accumulate(const spb_em_params* p, void* stream);           /* morpho_class.py:1266-1279 */
int spb_nonrigid_solve(const spb_em_params* p, void* stream);                /* morpho_class.py:1273-1291 (K<=64) */
int spb_nonrigid_blend(const spb_em_params* p, void* stream);                /* SigmaInv assembly only (K>64 path) */
int spb_field_apply(const spb_em_params* p, void* stream);                   /* morpho_class.py:1293-1298 */
/* the same from a factor of Sigma: Sigma = G G^T, G [K][ldg] with only the first *rank (device int32) columns non-zero; K * rank
   work per moving cell instead of K^2 (large inducing sets, where the eigen-solve runs outside spb_nonrigid_solve) */
int spb_field_apply_lowrank(const spb_em_params* p, const double* G, int32_t ldg, const int32_t* rank, void* stream); /* morpho_class.py:1293-1298 */
int spb_rigid_moments(const spb_em_params* p, void* stream);                 /* morpho_class.py:1312-1318,1356-1357,1427 */
int spb_rigid_solve(const spb_em_params* p, int32_t iter, void* stream);     /* morpho_class.py:1320-1402,1426-1435 */
int spb_row_update(const spb_em_params* p, void* stream);                    /* morpho_class.py:1404,293,1087 */
/* full iteration = all of the above in reference order; needs K <= SPB_MAX_K_FUSED (else call the pieces) */
int spb_em_iteration(const spb_em_params* p, int32_t iter, void* stream);    /* morpho_class.py:280-294 */
/* same launch sequence with the non-rigid phase chosen by the caller; iter < 0: the iteration index is the device counter
   spb_scalars.iter + 1 (SVI batch, step size, the iter < 100 sigma2 floor and the trace row all follow it), so ONE captured
   CUDA graph of this call replays every iteration of a phase */
int spb_em_iteration_ex(const spb_em_params* p, int32_t iter, int32_t nonrigid, void* stream);
/* one-time per-device kernel attributes of the non-rigid phase (lets the phase be graph-captured before its first eager launch) */
int spb_nonrigid_warm(void);
/* closing similarity from the last E-step's statistics: out = optimal_R[9], optimal_t[3] (device doubles) */
int spb_optimal_rigid(const spb_em_params* p, double* out12, void* stream);  /* morpho_class.py:1451-1468 */

/* ---- Gaussian-kernel vector field ------------------------------------------------------------------------------ */
/* UT[k][i] = exp(-beta |x_i - z_k|^2);  x:[3][ldx] SoA, z:[K][3] */
int spb_rbf_kernel_T(const float* x, int64_t n, int64_t ldx, const float* z, int32_t K, float beta, float* UT,
                     void* stream); /* utils.py:1132-1158 */
/* out[i][:] = sum_k exp(-beta|q_i - z_k|^2) Coff[k][:] for query points q:[n][D] row-major (fp64 in/out) */
int spb_field_eval(const double* q, int64_t n, int32_t D, const double* z, const double* Coff, int32_t K, double beta,
                   double* out, void* stream); /* transform.py:93,103; gaussian_process.py:109,117 */

/* Descriptor of a fitted field (the vecfld dict of morpho_class.py:1499-1528, host side; passed by value).
   velocity_divisor: 10000 for the Gaussian-process field (gaussian_process.py:127 divides the displacement by 10000 and the
   derived quantities of GPVectorField.py inherit that scale); 1 for a plain RBF field v(x) = K(x, X_ctrl) C (the SparseVFC
   field of sparsevfc.py:189-198, evaluated with nonrigid_only = 1, unit scales, zero means). */
typedef struct spb_field_desc {
  int32_t D;
  int32_t K;
  int32_t nonrigid_only;
  int32_t curvature_formula;
  double beta;
  double scale_transformed;
  double scale_fixed;
  double mean_transformed[3];
  double mean_fixed[3];
  double R[9];
  double t[3];
  double velocity_divisor;
} spb_field_desc;
int spb_sizeof_field_desc(void);
/* Differential geometry of the field at n raw query points X:[n][D] (device doubles), one pass, any output may be NULL:
   V[n][D] velocity (x_new - x)/velocity_divisor, J[n][D][D] analytical Jacobian, acc[n] / acc_mat[n][D] = J v, curvature
   (formula 1 or 2; curv_mat only for 2), curl ([n] in 2-D, [n][3] in 3-D), torsion[n][3] (3-D only), div[n], det[n].
   z, Coff: [K][D] device doubles; f is a HOST pointer. */
int spb_field_geometry(const spb_field_desc* f, const double* X, int64_t n, const double* z, const double* Coff,
                       double* V, double* J, double* acc, double* acc_mat, double* curv, double* curv_mat, double* curl,
                       double* torsion, double* div, double* det,
                       void* stream); /* GPVectorField.py:12-125,143-190; gaussian_process.py:102-127 */

/* Trajectories dx/dt = v(x) of n cells through the field f from X0:[n][D] (device doubles), one thread per cell, fp64:
   scipy.integrate.solve_ivp(v, (0, t_end), x0, method="RK45", max_step, rtol, atol, t_eval=np.linspace(0, t_end, n_out))
   with dynamo's terminal event np.all(abs(v(x)) < 1e-5) - 1 (morphopath, trajectory.py:11-61, hands the field to
   dynamo's fate). The sign of t_end is the direction. out[n][n_out][D]: the dense-output samples at the grid times; the
   samples after a cell's stop hold its state at the stop. t_stop[n]: stop time; steps[n][2]: accepted, rejected steps;
   status[n]: 0 reached t_end, 1 stopped by the event, -1 failed (100 (n_out - 1) accepted steps, or a step below
   scipy's minimum). z, Coff: [K][D] device doubles; f is a HOST pointer. No host synchronisation. */
int spb_field_integrate(const spb_field_desc* f, const double* X0, int64_t n, const double* z, const double* Coff,
                        double t_end, int32_t n_out, double rtol, double atol, double max_step, double* out,
                        double* t_stop, int32_t* steps, int32_t* status, void* stream); /* trajectory.py:11-61 */

/* ---- coarse rigid initialisation ---------------------------------------------------------------------------------- */
/* voxel_data: members of every grid-point ball (radius voxel_size / 2; overlapping) and voxel means. coords [N][D] in
   float (is_f64 = 0) or double, ax0/ax1/ax2 the np.arange axes in the same dtype (device), lo3 / step3 HOST doubles used
   only to bracket the candidate grid points; flat voxel index follows np.meshgrid('xy') + reshape(-1, D).
   spb_voxel_count: counts[nvox] += 1 per member (zero it first). spb_voxel_accumulate: means[new_id[v]][:] +=
   exp[i][:] / counts[v] (fp64 atomics, zero it first). */
int spb_voxel_count(const void* coords, int32_t is_f64, int64_t N, int32_t D, const void* ax0, int32_t n0, const void* ax1,
                    int32_t n1, const void* ax2, int32_t n2, double radius, const double* lo3, const double* step3,
                    int32_t* counts, void* stream); /* utils.py:1311-1330 */
int spb_voxel_accumulate(const void* coords, int32_t is_f64, int64_t N, int32_t D, const void* ax0, int32_t n0,
                         const void* ax1, int32_t n1, const void* ax2, int32_t n2, double radius, const double* lo3,
                         const double* step3, const int32_t* counts, const int32_t* new_id, const float* exp, int64_t ldg,
                         int32_t G, double* means, int64_t ldm, void* stream); /* utils.py:1326-1333 */
/* annealed robust Procrustes over matched pairs, 100 iterations on the device; x, y: [N][3] doubles, dist normalised,
   P in = exp(-dist), out = closing posterior; state: 512 B scratch; out16 = R[9], t[3], sigma2, gamma (device doubles) */
int spb_inlier_from_nn(const double* x, const double* y, const double* dist, int64_t N, int32_t D, double area, double dmin,
                       double sigma2_init, double sumP_init, double* P, double* resid, void* state, double* out16,
                       void* stream); /* utils.py:1220-1280 */

/* ---- SparseVFC building blocks (replaces third-party dynamo scVectorField.SparseVFC; parity unpinned) ---------- */
/* UtWU[K][K] = U^T diag(w) U and UtX[K][3] = U^T X3 (fp64 accumulation; outputs are zeroed first) */
int spb_weighted_gram(const float* UT, int64_t ldx, int64_t N, int32_t K, const float* w, const float* X3,
                      double* UtWU, double* UtX, void* stream); /* morpho_class.py:1266-1279; sparsevfc.py:189 (M-step) */
/* V = U C, P_i inlier posterior (clamped at minP); Pf / PY3 are the fp32 weight and P*Y ([3][ldn]) for the gram call;
   sums5 = {sum Ppre r, sum Ppre, sum P r, sum P, #{Ppre > theta}} */
int spb_vfc_estep(const float* UT, int64_t ldn, int64_t N, int32_t M, int32_t D, const double* C, const double* Y,
                  double sigma2, double gamma, double a, double minP, double theta, double* P, double* V, float* Pf,
                  float* PY3, double* sums5, void* stream); /* sparsevfc.py:189-198 (dynamo get_P) */

/* ---- host-buffer convenience (H2D/D2H inside; used for the end-to-end measurement) ------------------------------ */
int spb_field_eval_host(const double* q_host, int64_t n, int32_t D, const double* z_host, const double* Coff_host,
                        int32_t K, double beta, double* out_host); /* transform.py:61-116 */

#ifdef __cplusplus
}
#endif
#endif /* SPATEO_B200_H */
