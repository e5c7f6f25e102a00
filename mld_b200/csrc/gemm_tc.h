// wgmma (Hopper warpgroup MMA) split-fp16 GEMM with fused epilogues - interface.
#pragma once
#include "ops.cuh"

struct TcCtx;
TcCtx* tc_create(int device);
void tc_destroy(TcCtx* c);
// can this GEMM run on the tensor-core kernel (shape / alignment constraints)?
bool tc_gemm_supported(const TcCtx* c, const GemmArgs& g);
// ... with the residual + LayerNorm epilogue fused (the tile must cover a full 256-wide row)?
bool tc_gemm_ln_supported(const TcCtx* c, const GemmArgs& g, const LnArgs& l);
// enqueue; ln == nullptr for the plain epilogue.  false: tensor-map encoding failed, nothing was
// launched and mldb_last_error() says why.
bool tc_gemm(TcCtx* c, const GemmArgs& g, const LnArgs* ln, cudaStream_t st);
// FFN block linear1 + GELU + linear2 + residual + LayerNorm as one launch (hidden stays in registers)
bool tc_ffn_supported(const TcCtx* c, const GemmArgs& g1, const GemmArgs& g2, const LnArgs& l2);
// scratch / flags: TC_FFN_SCRATCH_BYTES / TC_FFN_FLAG_BYTES of device memory owned by the caller, one pair per stream
// that may run tc_ffn concurrently (flags zeroed once); nullptr = no hidden-dimension split of leftover tiles
constexpr size_t TC_FFN_SCRATCH_BYTES = (size_t)160 * 128 * 256 * 4, TC_FFN_FLAG_BYTES = 160 * 4;
bool tc_ffn(TcCtx* c, const GemmArgs& g1, const GemmArgs& g2, const LnArgs& l2, float* scratch, int* flags, cudaStream_t st);
int tc_set_ffn_split(TcCtx* c, int on);
int tc_set_ffn_fused(TcCtx* c, int on);   // returns the previous setting
