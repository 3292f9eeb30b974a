// forward.cuh -- declarations shared by forward_kernels.cu / vbn_kernels.cu / dne_api.cu
#pragma once
#include "common.cuh"

struct SlotArgs {
    const float* theta;        // [n_theta, P]
    const float* noise;        // slab
    const int64_t* noise_idx;  // [n_slots]
    const float* scale;        // [n_slots]
    const int32_t* theta_idx;  // nullable
    const uint8_t* active;     // nullable
    int64_t P;
};

struct LayerEpi {
    int64_t off_b, off_beta, off_gamma;
    int act, bn, bn_off, vbn_len;
    const float* vbn;          // [n_slots, vbn_len]
};

// source of a streamed weight matrix for the GEMV kernels: the noise slab (per-slot element offset) or the theta
// matrix (per-slot parent row)
struct GemvSrc {
    const float* base;        // noise slab, or theta matrix
    const int64_t* idx64;     // per-slot element offset (noise index) ...
    const int32_t* idx32;     // ... or per-slot row (theta_idx) times `mul`
    int64_t mul, off;         // off = layer weight offset inside the flat vector
};

extern int g_dne_gemv_bulk;
extern int g_dne_fold_theta;
extern int g_dne_gemv_ctas_per_sm;
int dne_launch_member_gemm_tc(const SlotArgs& sa, int64_t off_w, int64_t off_b, const float* X, int64_t x_slot_stride, int M,
                              int K, int N, float* out, int64_t out_slot_stride, int n_slots, cudaStream_t st);
// Union GEMV (gemv_bulk.cu): the table is cut into blocks of DNE_GEMV_BLOCK_ROWS rows of N floats, each covered block is
// streamed once per launch through a cp.async.bulk ring and applied to every group whose slice intersects it.  Each group
// writes dne_gemv_pieces(K) partials [group][piece][G][N].  Returns DNE_ERR_UNSUP if the shape is not covered.
constexpr int DNE_GEMV_BLOCK_ROWS = 256;
int dne_gemv_pieces(int K);
int dne_launch_gemv_union(const SlotArgs& sa, const GemvSrc& src, int G, const float* X, int64_t x_slot_stride, int K,
                          int N, int n_pieces, int n_slots, float* part, int sm_count, cudaStream_t st,
                          const float* fold_theta = nullptr, int fold_n_split = 0);

struct DensePlan {
    bool decomposed;
    int n_split, k_per_split;     // theta GEMM split-K
    // n_chunks: partials per group (dne_gemv_pieces); rows_per_chunk: K rows per partial of the SIMT GEMV
    int G, Gt, rows_per_chunk, n_chunks, rw;     // Gt: theta group size (0 = shared theta GEMM)
    size_t part_theta_floats, part_noise_floats;
};

extern int g_dne_conv_tc;
int dne_launch_conv_layer_tc(const SlotArgs& sa, const dne_layer_desc& L, const LayerEpi& epi, bool in_u8,
                             const void* in, int64_t in_slot_stride, int64_t in_img_stride, float* out,
                             int64_t out_slot_stride, int64_t out_img_stride, int n_slots, int n_img,
                             cudaStream_t st);
int dne_launch_conv_layer_simt(const SlotArgs& sa, const dne_layer_desc& L, const LayerEpi& epi, bool in_u8,
                               const void* in, int64_t in_slot_stride, int64_t in_img_stride, float* out,
                               int64_t out_slot_stride, int64_t out_img_stride, int n_slots, int n_img,
                               cudaStream_t st);

DensePlan dne_plan_dense(const dne_layer_desc& L, int n_slots, int paired, bool shared_theta, int sm_count);

int dne_launch_conv_layer(const SlotArgs& sa, const dne_layer_desc& L, const LayerEpi& epi, bool in_u8,
                          const void* in, int64_t in_slot_stride, int64_t in_img_stride, float* out,
                          int64_t out_slot_stride, int64_t out_img_stride, int n_slots, int n_img,
                          cudaStream_t st);

// the output head fused behind a decomposed dense layer (dense_combine_head_kernel)
struct DenseHead {
    const dne_layer_desc* L;
    LayerEpi epi;
    float* out;                // logits [n_slots, out_slot_stride]
    int64_t out_slot_stride;
    int32_t* actions;          // nullable
};
bool dne_head_fusable(const dne_layer_desc& L, const DensePlan& p, const dne_layer_desc& head, const DensePlan& hp);
// TMA-fed shared-theta GEMM (theta_gemm_tma.cu): both operands pre-arranged in the wgmma canonical layout, split hi / lo
struct TgmOperands {
    const float* Xc;           // [m tile][k quad][hi|lo][128][4], written by the producing conv epilogue
    const float* Wc;           // [n tile][k quad][hi|lo][128][4], written by dne_theta_prepare
};
size_t dne_tgm_xc_bytes(int n_slots, int K);
size_t dne_tgm_wc_bytes(int K, int N);
bool dne_tgm_supported(int K, int N, int k_per_split);
int dne_launch_theta_prep(const float* W, int K, int N, float* Wc, cudaStream_t st);
int dne_launch_theta_gemm_tma(const float* Xc, const float* Wc, int M, int K, int N, int k_per_split, int n_split, float* part,
                              cudaStream_t st);
int dne_launch_dense_layer(const dne_ctx* ctx, const SlotArgs& sa, const dne_layer_desc& L, const LayerEpi& epi,
                           const DensePlan& p, const float* X, int64_t x_slot_stride, float* out,
                           int64_t out_slot_stride, int32_t* actions, float* part_theta, float* part_noise,
                           int n_slots, cudaStream_t st, const DenseHead* head = nullptr, const TgmOperands* tgm = nullptr);

void dne_launch_ob_norm(const float* obs, const float* mean, const float* stdv, int64_t total, int dim, float* out,
                        cudaStream_t st);

// episode_kernels.cu: whole episodes of the DNE_EPISODE_* discrete-action tasks on the device (dne_discrete_episodes,
// dne_cartpole_episodes); dne_discrete_time_limit is 0 for an unknown task
int dne_discrete_time_limit(int env);
bool dne_discrete_net_supported(int env, const dne_net_desc* net, const char** why);
int dne_launch_discrete_episodes(int env, const dne_net_desc* net, const float* theta, const float* noise,
                                 const int64_t* noise_idx, const float* scale, const int32_t* theta_idx, int n_members,
                                 const double* init_state, int max_steps, float* returns, int32_t* lengths,
                                 double* final_state, cudaStream_t st);
// episode_kernels.cu: whole Pendulum-v1 episodes on the device (dne_pendulum_episodes)
bool dne_pendulum_net_supported(const dne_net_desc* net, const char** why);
int dne_launch_pendulum_episodes(const dne_net_desc* net, const float* theta, const float* noise, const int64_t* noise_idx,
                                 const float* scale, const int32_t* theta_idx, int n_members, const double* init_state,
                                 int max_steps, const float* ob_mean, const float* ob_std, const float* ac_noise,
                                 float* returns, float* signreturns, int32_t* lengths, double* final_state, double* ob_sum,
                                 double* ob_sumsq, cudaStream_t st);
// episode_kernels.cu: whole hard-maze episodes on the device (dne_maze_episodes); `maze` already checked
bool dne_maze_net_supported(const dne_net_desc* net, const char** why);
int dne_launch_maze_episodes(const dne_maze_desc* maze, const dne_net_desc* net, const float* theta, const float* noise,
                             const int64_t* noise_idx, const float* scale, const int32_t* theta_idx, int n_members,
                             const double* init_state, int max_steps, const float* ob_mean, const float* ob_std,
                             const float* ac_noise, float* returns, float* signreturns, int32_t* lengths,
                             double* final_state, double* ob_sum, double* ob_sumsq, cudaStream_t st);
// episode_kernels.cu: the same episodes with one member per thread-block cluster (dne_*_cluster_episodes).  `cluster` is
// 0 (automatic) or 2, 4, 8 (already checked); the geometry is int[4] = (cluster size, threads per CTA, shared bytes per
// CTA, members resident on the device).  DNE_ERR_UNSUP sets `why`, as does a failed launch (DNE_ERR_CUDA).
bool dne_pendulum_cluster_net_supported(const dne_net_desc* net, const char** why);
bool dne_maze_cluster_net_supported(const dne_net_desc* net, const char** why);
int dne_pendulum_cluster_geometry(const dne_net_desc* net, int cluster, int* geometry, const char** why);
int dne_maze_cluster_geometry(const dne_net_desc* net, int cluster, int* geometry, const char** why);
int dne_launch_pendulum_cluster_episodes(const dne_net_desc* net, const float* theta, const float* noise,
                                         const int64_t* noise_idx, const float* scale, const int32_t* theta_idx,
                                         int n_members, const double* init_state, int max_steps, const float* ob_mean,
                                         const float* ob_std, const float* ac_noise, float* returns, float* signreturns,
                                         int32_t* lengths, double* final_state, double* ob_sum, double* ob_sumsq,
                                         int cluster, const char** why, cudaStream_t st);
int dne_launch_maze_cluster_episodes(const dne_maze_desc* maze, const dne_net_desc* net, const float* theta,
                                     const float* noise, const int64_t* noise_idx, const float* scale,
                                     const int32_t* theta_idx, int n_members, const double* init_state, int max_steps,
                                     const float* ob_mean, const float* ob_std, const float* ac_noise, float* returns,
                                     float* signreturns, int32_t* lengths, double* final_state, double* ob_sum,
                                     double* ob_sumsq, int cluster, const char** why, cudaStream_t st);
// episode_kernels.cu: the same episodes with a discretised head of `nb` bins per action dimension (dne_*_binned_episodes);
// `bins` is the host table [N_OUT][nb] (non-null, checked).  `cluster` 0 runs the single-CTA kernel when the member fits
// one CTA and the automatic cluster size otherwise; 2, 4, 8 force the cluster kernel at that size.
bool dne_pendulum_binned_net_supported(const dne_net_desc* net, int nb, const char** why);
bool dne_maze_binned_net_supported(const dne_net_desc* net, int nb, const char** why);
int dne_launch_pendulum_binned_episodes(const dne_net_desc* net, const float* theta, const float* noise,
                                        const int64_t* noise_idx, const float* scale, const int32_t* theta_idx,
                                        int n_members, const double* init_state, int max_steps, const float* ob_mean,
                                        const float* ob_std, const float* ac_noise, float* returns, float* signreturns,
                                        int32_t* lengths, double* final_state, double* ob_sum, double* ob_sumsq,
                                        const float* bins, int nb, int cluster, const char** why, cudaStream_t st);
int dne_launch_maze_binned_episodes(const dne_maze_desc* maze, const dne_net_desc* net, const float* theta,
                                    const float* noise, const int64_t* noise_idx, const float* scale,
                                    const int32_t* theta_idx, int n_members, const double* init_state, int max_steps,
                                    const float* ob_mean, const float* ob_std, const float* ac_noise, float* returns,
                                    float* signreturns, int32_t* lengths, double* final_state, double* ob_sum,
                                    double* ob_sumsq, const float* bins, int nb, int cluster, const char** why,
                                    cudaStream_t st);

int dne_launch_theta_gemm_tc(const float* X, int M, int K, int N, const float* W, int k_per_split, int n_split,
                             float* part, cudaStream_t st);

// conv_s2d.cu: shifted-window implicit-GEMM convolutions (wgmma, A operand by TMA), dne_set_option("conv_tc", 2) [default]
bool dne_s2d_supported(const dne_layer_desc& L, bool in_u8);
size_t dne_s2d_image_bytes(const dne_layer_desc& L);
int dne_launch_conv_layer_s2d(const SlotArgs& sa, const dne_layer_desc& L, const LayerEpi& epi, bool in_u8, const void* in,
                              int64_t in_slot_stride, float* out, int64_t out_slot_stride, const dne_layer_desc* next,
                              int n_slots, int sm_count, cudaStream_t st, float* xc = nullptr, int vdiv = 1, int in_mod = 0);
void dne_s2d_image_geom(const dne_layer_desc& L, int* nS, int* nPADB, int* nW, int* nPIXP, int* nHP);
