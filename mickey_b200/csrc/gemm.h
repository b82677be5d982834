// Host-callable interface of the GEMM family (see gemm_tc.cuh for the kernel).
#pragma once
#include "common.cuh"

namespace mk {

struct GemmOperand {       // a row-major fp16 matrix [rows, cols] with leading dimension ld (elements)
  const void* ptr;
  long long rows, cols, ld;
};

// GEMM_IMPL_DEFAULT and GEMM_IMPL_TC run the wgmma kernel; GEMM_IMPL_SIMT runs the SIMT debug kernel.
// GEMM_IMPL_TC_PAIRED / _UNPAIRED run the persistent kernel with or without two-CTA pairs on every grid whose epilogue
// it serves (other epilogues run as GEMM_IMPL_TC), whatever the grid size: a test or a benchmark can set the two side
// by side.  The default picks the paired kernel for grids of more than 8 tiles per SM.
enum GemmImpl : int { GEMM_IMPL_DEFAULT = 0, GEMM_IMPL_TC = 1, GEMM_IMPL_SIMT = 2, GEMM_IMPL_TC_PAIRED = 3, GEMM_IMPL_TC_UNPAIRED = 4 };

int make_tensor_map_f16(CUtensorMap* map, const void* ptr, long long rows, long long cols, long long ld_elems, int box_rows);
// Uncached TMA load map of a row-major fp16 or fp32 [rows, cols] operand with leading dimension ld_elems: box = 128 bytes
// of columns x box_rows rows, 128-byte swizzle, zero fill.  The base and the row pitch must be 16-byte aligned.
int encode_tensor_map_2d(CUtensorMap* map, CUtensorMapDataType dtype, const void* ptr, long long rows, long long cols,
                         long long ld_elems, int box_rows);
// TMA store map of a contiguous fp16 [groups, rows, cols] tensor (box 64 columns x box_rows rows, 128-byte swizzle)
int make_tensor_map_out_f16(CUtensorMap* map, void* ptr, long long groups, long long rows, long long cols, int box_rows);
int sm_count();            // SMs of the current device
int launch_gemm(int epi, const GemmOperand& A, const GemmOperand& B, const GemmParams& p, cudaStream_t stream,
                int impl = GEMM_IMPL_DEFAULT);
const char* last_error();

}  // namespace mk
