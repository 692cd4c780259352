// Grow-only device workspace of the small per-call GEMMs (tracker cosine costs, ReID distance matrices, camera-pair
// costs): raw fp32 rows, fp16 operand planes, products, row norms, int32 tables, a gate, the operands' range flag and the
// GEMM plans cached per padded shape.  Allocating the buffers and encoding the tensor maps on every call costs more than the GEMM itself.
#pragma once
#include <map>
#include <vector>

#include "engine_core.h"

namespace b2 {

// What one call needs, in elements.
struct GemmNeed {
  size_t a = 0, b = 0;          // raw fp32 inputs uploaded from the host
  size_t Sp = 0, Np = 0, Dp = 0;   // padded GEMM rows, columns and depth
  size_t out = 0;               // fp32 results
  size_t ints = 0;              // int32 tables (segment offsets)
  size_t gate = 0;              // bytes
};

struct GemmWs {
  int num_sms = 0;
  cudaStream_t stream = nullptr;
  bool transient = false;   // owned by one call: sized exactly, released with the object
  GemmNeed cap;
  float *d_a = nullptr, *d_b = nullptr, *d_dots = nullptr, *d_out = nullptr, *d_bias = nullptr, *d_na2 = nullptr,
        *d_nb2 = nullptr;
  int* d_int = nullptr;
  uint8_t* d_gate = nullptr;
  unsigned int* d_range = nullptr;   // ORed by rows_to_planes when a finite input rounds to an fp16 inf
  __half *a_hi = nullptr, *a_lo = nullptr, *b_hi = nullptr, *b_lo = nullptr;
  std::map<std::vector<int>, PlanPtr> plans;   // key: Sp, Np, Dp, split

  GemmWs() = default;
  GemmWs(const GemmWs&) = delete;
  GemmWs& operator=(const GemmWs&) = delete;
  ~GemmWs();   // the per-device workspaces live as long as the process (no CUDA calls at exit)
  // Makes every buffer hold at least `need` (on `device`) and clears the range flag.  Growing reallocates all buffers
  // (the plans hold their addresses) at twice the size that overflowed, zero-filled.  Operand rows beyond a call's data,
  // up to the plan's padded shape, then hold leftovers of earlier calls -- NaN or inf too, when those calls had such
  // inputs.  A GEMM output element depends on one operand row of each side only, so those rows only produce products
  // nobody reads.
  int reserve(int device, const GemmNeed& need);
  // d_dots [Sp][Np] = (a planes [Sp][Dp]) x (b planes [Np][Dp])^T on the stream
  int gemm(int Sp, int Np, int Dp, bool split);
  // Copies n results from d_out to the host `out`, waits for the stream and fails (naming `who`) when an operand
  // conversion of the call set the range flag.
  int download(float* out, size_t n, const char* who);

 private:
  void release();
};

}  // namespace b2
