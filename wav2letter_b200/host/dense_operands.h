// dense_operands.h — how fp32 activations and weights become w2l_gemm operands in a precision (W2L_PRECISION_*), written
// once for the trainer's Linear layers and large-channel convolutions (fl_compat.cpp) and the streaming acoustic model
// (stream_capi.cpp), so both compute the same bits.  Operand rows are TMA rows (16 bytes: 4 floats, 8 bf16); other rows
// and all bf16 operands are copies into memory the caller supplies, sized by the *Bytes queries.  Not part of the C ABI.
#pragma once
#include <cstddef>

namespace w2l {
namespace dense {

// kind W2L_GEMM_*, rows of ld elements; mnMajor: a weight's rows read as W itself (b_mn_major), not as K-major rows
struct Operand {
  int kind = 0;
  const void* ptr = nullptr;
  int ld = 0;
  bool mnMajor = false;
};

int rowKind(int precision);               // the precision's kind of row operands: TF32, F32X3, BF16 or FP16
long long padRow(int kind, long long n);  // n padded to whole TMA rows of the kind

// contiguous rows of `cols` floats as rows of padRow(kind, cols) entries behind `zeroRows` zero rows: the source itself
// when it already is that (fp32, 16-byte aligned), else a zero-padded fp32 or a bf16 copy in dst.  rowBytes: the bytes
// of that copy, 0 when the source serves (a null src: the copy's size).
size_t rowBytes(int kind, long long rows, int cols, const float* src, int zeroRows = 0);
Operand rows(void* stream, int kind, long long rows, int cols, const float* src, void* dst, int zeroRows = 0);

// W [nout][nin] as the forward's B with rows of len >= nin entries: TF32 its rows or a zero-padded copy, BF16 a bf16
// copy, F32 the tf32 hi / lo planes [2][nout][len] (kind F32X3_SPLIT_B)
size_t weightBytes(int precision, int nout, int nin, int len, const float* w);
Operand weight(void* stream, int precision, int nout, int nin, int len, const float* w, void* dst);
// W as the data gradient's B (dx [M][cols] = dy W, cols <= the forward's len): TF32 / BF16 the forward's operand read
// as W; F32 the planes of W^T split from W (through a zero-padded copy when cols > nin).  The GEMM takes the plane
// stride from N, so the planes have exactly `cols` rows.
size_t weightTBytes(const Operand& fwd, int nout, int nin, int cols);
Operand weightT(void* stream, const Operand& fwd, int nout, int nin, int cols, const float* w, void* dst);

// C = act(A B^T + bias) with the rest of w2l_gemm's epilogue: A K-major rows, B a weight operand, in B's kind
int gemm(void* stream, int M, int N, int K, const Operand& A, const Operand& B, float* C, int ldc, const float* bias = nullptr, int act = 0,
         int accumulate = 0, const float* aux = nullptr, int ld_aux = 0, int aux_mode = 0, float aux_scale = 1.f, float dropout_p = 0.f,
         unsigned long long seed = 0, int allow_overlap = 0);

}  // namespace dense
}  // namespace w2l
