// h264_kernels.h — launchers of the encoder stages (each returns the number of kernels launched)
#pragma once
#include <cuda_runtime.h>
namespace b2v {
struct FrameCtx;
int launch_intra(const FrameCtx& f, cudaStream_t st);    // IDR: one block per slice (h264_intra.cu)
int launch_inter(const FrameCtx& f, cudaStream_t st);    // P: motion search + residual (h264_inter.cu)
cudaError_t inter_search_grid(int* blocks);
int launch_coarse(const FrameCtx& f, cudaStream_t st);   // B2V_FLAG_WIDE_MOTION: decimated luma and anchor groups' coarse vectors (h264_inter.cu)              // blocks of k_inter_search resident at once on the current device
int launch_ltr_mark(const FrameCtx& f, cudaStream_t st);   // B2V_FLAG_LONG_TERM_REF: the marking decision and the long-term copy (h264_inter.cu)
int launch_scene_cut(const FrameCtx& f, cudaStream_t st);   // B2V_FLAG_SCENE_CUT: the decision, then the intra coding of a cut picture (h264_intra.cu)
int launch_cavlc(const FrameCtx& f, cudaStream_t st);    // per-macroblock CAVLC bit strings (h264_entropy.cu)
int launch_size_cap(const FrameCtx& f, cudaStream_t st);      // B2V_FLAG_SIZE_CAP, P pictures: the count, the decision, the recode (h264_cap.cu)
int launch_requant(const FrameCtx& f, cudaStream_t st);       // B2V_FLAG_SIZE_CAP: k_requant (h264_inter.cu)
int launch_cavlc_recode(const FrameCtx& f, cudaStream_t st);  // B2V_FLAG_SIZE_CAP: CAVLC again after k_requant (h264_entropy.cu)
int launch_slice_build(const FrameCtx& f, cudaStream_t st);     // k_slice_build: scan + copy + emulation-prevention count; its last block runs the rate-control step (h264_entropy.cu)
int launch_pack_cap(const FrameCtx& f, long long au_cap, cudaStream_t st);   // emulation prevention + AU assembly
}  // namespace b2v
