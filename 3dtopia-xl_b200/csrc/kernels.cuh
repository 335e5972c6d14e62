// Internal launchers shared by the translation units of libtpx_b200, grouped by defining file.  A launcher whose only caller is
// its C entry point is part of that entry (defined beside its kernels) and is not declared here.
#pragma once
#include "gemm_tc.cuh"

namespace tpx {

// elementwise.cu
int launch_ln_modulate(float* x, int rows, int D, float eps, const __half* shift, const __half* scale, int mod_bstride, int rows_per_batch,
                       int mod_batches, __half* out, const __half* pre_gate, const __half* pre_const, int pre_row0, cudaStream_t st);
enum { GEMV_IN_TIMESTEP = 0, GEMV_IN_F32 = 1, GEMV_IN_F16 = 2 };
enum { GEMV_OUT_F32 = 0, GEMV_OUT_F32_SILU = 1, GEMV_OUT_F16 = 2, GEMV_OUT_F32_AND_SILU16 = 3 };
int launch_gemv(int in_mode, int out_mode, const __half* W, const __half* bias, const void* in, const long long* t, int B, int J, int K, void* out,
                __half* out2, int out_ld, cudaStream_t st);
int launch_x_embed(const float* x, const __half* W, const __half* bias, int rows, int Cin, int D, float* out, long long dup_offset, cudaStream_t st);
int launch_cfg_combine(const __half* both, long long n_half, float s, __half* out, cudaStream_t st);
int launch_to_half(const void* src, int src_dtype, __half* dst, long long n, cudaStream_t st);
int launch_from_half(const __half* src, void* dst, int dst_dtype, long long n, cudaStream_t st);
int launch_fill_rows_half(const __half* vec, __half* dst, long long rows, int K, cudaStream_t st);

// attention.cu :  q [B,H,Nq,DhP], k/v [B,H,Nk,DhP] fp16 (zero padded beyond Dh) -> out [B,Nq,H*Dh] fp16
int launch_attention(const __half* q, const __half* k, const __half* v, __half* out, int B, int H, int Nq, int Nk, int Dh, int DhP, float scale,
                     cudaStream_t st);

// attention_tc.cu : wgmma version for Dh = 72 or 64 (80-wide tiles); vT is V transposed [B,H,80,NkPad]
int launch_attention_tc(const __half* q, const __half* k, const __half* vT, __half* out, int B, int H, int Nq, int Nk, int NkPad, int Dh, float scale,
                        cudaStream_t st);

// gemm_tc.cu : cached 2-D TMA descriptor over a row-major fp16 matrix (swizzle = box_cols * 2 bytes: 128/64/32)
int make_tensor_map_2d(const void* ptr, long long rows, long long cols, long long ld, int box_rows, int box_cols, CUtensorMap* out);
int make_tensor_map_nd(const void* ptr, int rank, const long long* dims, const long long* strides_bytes, const int* box, int swizzle_bytes, CUtensorMap* out,
                       int l2_promotion_bytes = 256);

// conv_halo.cu : 3x3x3 / pad 1 convolution on [P,8,8,8,C] volumes with the input block (+halo) staged ONCE per output tile
int launch_conv3_halo(const __half* x, const __half* W, const __half* bias, const __half* resid, float alpha, __half* out, float* out32, int n_valid, int P,
                      int C, int Cout, int epi, cudaStream_t st);
bool conv3_halo_supported(int S, int C, int Cout, int epi);

// vae_kernels.cu
int launch_vae_conv_in(const void* z, int z_dtype, const __half* w_pq, const __half* b_pq, const __half* W, const __half* bias, int P, int C,
                       __half* out, cudaStream_t st);
int launch_groupnorm_silu(const __half* x, const __half* gamma, const __half* beta, int P, int S3, int C, int groups, float eps, int apply_silu,
                          __half* out, cudaStream_t st);
int launch_pack_conv3(const void* src, int dtype, __half* dst, int Cout, int Cin, int transposed, cudaStream_t st);
int launch_pack_convt2(const void* src, int dtype, __half* dst, int Cin, int Cout, cudaStream_t st);
int launch_vae_enc_conv_in(const void* x, int x_dtype, const __half* W, const __half* bias, int P, __half* out, cudaStream_t st);
int launch_space_to_depth2(const __half* in, __half* out, int P, int C, cudaStream_t st);
int launch_pack_conv3_s2d(const void* src, int dtype, __half* dst, int Cout, int Cin, cudaStream_t st);

}  // namespace tpx
