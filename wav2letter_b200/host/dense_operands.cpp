// dense_operands.cpp — the operands of the dense-layer GEMMs in a precision (dense_operands.h).
#include "dense_operands.h"

#include <cuda_runtime.h>

#include <cstdint>
#include <stdexcept>
#include <string>

#include "w2l_b200.h"

namespace w2l {
void check(int rc);

namespace dense {
namespace {
void cuda(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string("dense operand: ") + what + ": " + cudaGetErrorString(e));
}
bool is16(int kind) { return kind == W2L_GEMM_BF16 || kind == W2L_GEMM_FP16; }
size_t elemBytes(int kind) { return is16(kind) ? 2 : 4; }
bool servesInPlace(int kind, int cols, long long len, const float* src, int zeroRows) {
  return !is16(kind) && zeroRows == 0 && len == cols && src && (reinterpret_cast<uintptr_t>(src) & 15) == 0;
}
size_t copyBytes(int kind, long long rows, int cols, long long len, const float* src, int zeroRows) {
  return servesInPlace(kind, cols, len, src, zeroRows) ? 0 : elemBytes(kind) * (size_t)(zeroRows + rows) * (size_t)len;
}
// rows of `cols` floats as rows of len >= cols entries behind zeroRows zero rows
Operand rowsOf(void* stream, int kind, long long rows, int cols, long long len, const float* src, void* dst, int zeroRows) {
  if (servesInPlace(kind, cols, len, src, zeroRows)) return {kind, src, (int)len};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t pitch = elemBytes(kind) * (size_t)len;
  char* body = static_cast<char*>(dst) + (size_t)zeroRows * pitch;
  const bool half = is16(kind), padCols = !half && len > cols;  // the 16-bit casts write their own pad columns
  if (zeroRows || padCols) cuda(cudaMemsetAsync(dst, 0, (size_t)(zeroRows + (padCols ? rows : 0)) * pitch, st), "zero padding");
  if (half && len == cols)
    check(kind == W2L_GEMM_FP16 ? w2l_cast_fp16(st, rows * cols, src, body) : w2l_cast_bf16(st, rows * cols, src, body));
  else if (half)
    check(kind == W2L_GEMM_FP16 ? w2l_cast_fp16_rows(st, rows, cols, cols, (int)len, src, body)
                                : w2l_cast_bf16_rows(st, rows, cols, cols, (int)len, src, body));
  else if (len == cols)
    cuda(cudaMemcpyAsync(body, src, sizeof(float) * (size_t)rows * cols, cudaMemcpyDeviceToDevice, st), "copy");
  else
    cuda(cudaMemcpy2DAsync(body, pitch, src, sizeof(float) * cols, sizeof(float) * cols, (size_t)rows, cudaMemcpyDeviceToDevice, st), "padded copy");
  return {kind, dst, (int)len};
}
}  // namespace

int rowKind(int precision) {
  switch (precision) {
    case W2L_PRECISION_BF16: return W2L_GEMM_BF16;
    case W2L_PRECISION_FP16: return W2L_GEMM_FP16;
    case W2L_PRECISION_F32: return W2L_GEMM_F32X3;
    default: return W2L_GEMM_TF32;
  }
}
long long padRow(int kind, long long n) {
  const long long a = is16(kind) ? 8 : 4;
  return (n + a - 1) / a * a;
}

size_t rowBytes(int kind, long long rows, int cols, const float* src, int zeroRows) {
  return copyBytes(kind, rows, cols, padRow(kind, cols), src, zeroRows);
}
Operand rows(void* stream, int kind, long long rows, int cols, const float* src, void* dst, int zeroRows) {
  return rowsOf(stream, kind, rows, cols, padRow(kind, cols), src, dst, zeroRows);
}

size_t weightBytes(int precision, int nout, int nin, int len, const float* w) {
  const int kind = rowKind(precision);
  if (kind == W2L_GEMM_F32X3) return sizeof(float) * 2 * (size_t)nout * len;
  return copyBytes(kind, nout, nin, len, w, 0);
}
Operand weight(void* stream, int precision, int nout, int nin, int len, const float* w, void* dst) {
  const int kind = rowKind(precision);
  if (kind != W2L_GEMM_F32X3) return rowsOf(stream, kind, nout, nin, len, w, dst, 0);
  check(w2l_split_tf32(stream, 0, nout, nin, nin, len, w, static_cast<float*>(dst)));
  return {W2L_GEMM_F32X3_SPLIT_B, dst, len};
}

size_t weightTBytes(const Operand& fwd, int nout, int nin, int cols) {
  if (fwd.kind != W2L_GEMM_F32X3_SPLIT_B) return 0;
  const size_t padded = cols > nin ? copyBytes(W2L_GEMM_F32X3, nout, nin, padRow(W2L_GEMM_F32X3, cols), nullptr, 0) : 0;
  return sizeof(float) * 2 * (size_t)cols * padRow(W2L_GEMM_F32X3, nout) + padded;
}
Operand weightT(void* stream, const Operand& fwd, int nout, int nin, int cols, const float* w, void* dst) {
  if (fwd.kind != W2L_GEMM_F32X3_SPLIT_B) return {fwd.kind, fwd.ptr, fwd.ld, true};
  const int ld = (int)padRow(W2L_GEMM_F32X3, nout);
  float* planes = static_cast<float*>(dst);
  Operand src{W2L_GEMM_F32X3, w, nin};
  if (cols > nin) src = rowsOf(stream, W2L_GEMM_F32X3, nout, nin, padRow(W2L_GEMM_F32X3, cols), w, planes + 2 * (size_t)cols * ld, 0);
  check(w2l_split_tf32(stream, 1, nout, cols, src.ld, ld, static_cast<const float*>(src.ptr), planes));
  return {W2L_GEMM_F32X3_SPLIT_B, planes, ld};
}

int gemm(void* stream, int M, int N, int K, const Operand& A, const Operand& B, float* C, int ldc, const float* bias, int act, int accumulate,
         const float* aux, int ld_aux, int aux_mode, float aux_scale, float dropout_p, unsigned long long seed, int allow_overlap) {
  return w2l_gemm(stream, B.kind, 0, B.mnMajor ? 1 : 0, M, N, K, A.ptr, A.ld, B.ptr, B.ld, C, ldc, 0, bias, act, accumulate, aux, ld_aux, 0, aux_mode,
                  aux_scale, dropout_p, seed, allow_overlap);
}

}  // namespace dense
}  // namespace w2l
