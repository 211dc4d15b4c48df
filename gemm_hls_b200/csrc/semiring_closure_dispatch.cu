// Run-time (dtype, map, reduce) -> compile-time instantiation of the closure kernels (mm_kernel_enqueue_closure).
// Float Min / Max take the FMNMX operators unless MM_FLAG_EXACT is set, exactly as launch_semiring chooses.
#include "common.cuh"
#include "semiring_closure_kernel.cuh"

namespace mm {

namespace {

template <typename T>
int by_map(int map_op, int reduce_op, void *d, unsigned n, unsigned batch, cudaStream_t s) {
  switch (map_op) {
    case MM_OP_MULTIPLY: return launch_semiring_closure_for<T, MM_OP_MULTIPLY>(reduce_op, d, n, batch, s);
    case MM_OP_ADD: return launch_semiring_closure_for<T, MM_OP_ADD>(reduce_op, d, n, batch, s);
    case MM_OP_MIN: return launch_semiring_closure_for<T, MM_OP_MIN>(reduce_op, d, n, batch, s);
    case MM_OP_MAX: return launch_semiring_closure_for<T, MM_OP_MAX>(reduce_op, d, n, batch, s);
    case MM_OP_AND: return launch_semiring_closure_for<T, MM_OP_AND>(reduce_op, d, n, batch, s);
  }
  return -1;
}

int by_map_float(int map_op, int reduce_op, void *d, unsigned n, unsigned batch, cudaStream_t s) {
  switch (map_op) {
    case MM_OP_MIN_FAST: return launch_semiring_closure_for<float, MM_OP_MIN_FAST>(reduce_op, d, n, batch, s);
    case MM_OP_MAX_FAST: return launch_semiring_closure_for<float, MM_OP_MAX_FAST>(reduce_op, d, n, batch, s);
  }
  return by_map<float>(map_op, reduce_op, d, n, batch, s);
}

}  // namespace

int launch_semiring_closure(int dtype, int map_op, int reduce_op, int flags, void *d, unsigned n, unsigned batch,
                            cudaStream_t s) {
  int rc = -1;
  switch (dtype) {
    case MM_DTYPE_HALF: rc = by_map<__half>(map_op, reduce_op, d, n, batch, s); break;
    case MM_DTYPE_FLOAT: {
      auto fast = [&](int op) {
        if (flags & MM_FLAG_EXACT) return op;
        return op == MM_OP_MIN ? int(MM_OP_MIN_FAST) : (op == MM_OP_MAX ? int(MM_OP_MAX_FAST) : op);
      };
      rc = by_map_float(fast(map_op), fast(reduce_op), d, n, batch, s);
      break;
    }
    case MM_DTYPE_DOUBLE: rc = by_map<double>(map_op, reduce_op, d, n, batch, s); break;
    case MM_DTYPE_INT32: rc = by_map<int>(map_op, reduce_op, d, n, batch, s); break;
    case MM_DTYPE_UINT32: rc = by_map<unsigned>(map_op, reduce_op, d, n, batch, s); break;
    case MM_DTYPE_UINT8: rc = by_map<unsigned char>(map_op, reduce_op, d, n, batch, s); break;
    case MM_DTYPE_BFLOAT16: rc = by_map<__nv_bfloat16>(map_op, reduce_op, d, n, batch, s); break;
    default: return fail(MM_ERR_INVALID, "unknown data type");
  }
  if (rc < 0) return fail(MM_ERR_INVALID, "unknown map operator, or a reduce without a closure");
  if (rc != 0) return fail(MM_ERR_CUDA, std::string("closure kernel launch: ") + cudaGetErrorString(static_cast<cudaError_t>(rc)));
  return MM_OK;
}

}  // namespace mm
