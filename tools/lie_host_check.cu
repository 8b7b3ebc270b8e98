// Host-side driver of the lietorch_backends operators: runs one of the 19 operators for SO3 (1), RxSO3 (2), SE3 (3)
// or Sim3 (4) on the HOST through the very functions the CUDA kernels of lie.cu call (lie_ops.cuh, lie_scaled.cuh, all
// __host__ __device__), so the math can be checked without a GPU.  Built and driven by tests/test_lie_scaled_host_cpu.py
// and tests/test_lie_edges_host_cpu.py.
//   usage: lie_host_check <group> <op> <n> <w0> <w1> <w2> <wo0> <wo1> <f32|f64> <in.bin> <out.bin>
//   in.bin  = in0[n*w0] in1[n*w1] in2[n*w2]   out.bin = out0[n*wo0] out1[n*wo1]        (scalars of the given type)
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "lie_ops.cuh"
#include "lie_scaled.cuh"

using namespace dpvo;
using namespace dpvo::lie;

template <typename S, int OP>
static void so3_se3_op(int group, const LieArgs& A) {
  for (long long i = 0; i < A.n; ++i) {
    if (group == 3) se3_op<S, OP>(A, i);
    else so3_op<S, OP>(A, i);
  }
}

// the operator code as a template argument, as lie_launch does for the kernels
template <typename S, int OP = 0>
static void so3_se3_dispatch(int group, int op, const LieArgs& A) {
  if constexpr (OP <= OP_JINV) {
    if (op == OP) so3_se3_op<S, OP>(group, A);
    else so3_se3_dispatch<S, OP + 1>(group, op, A);
  }
}

template <typename S>
static int run(int group, int op, long long n, const int* w, const char* in, const char* out) {
  std::vector<S> i0(n * w[0] + 1), i1(n * w[1] + 1), i2(n * w[2] + 1), o0(n * w[3] + 1), o1(n * w[4] + 1);
  FILE* f = fopen(in, "rb");
  if (!f) return 2;
  if (fread(i0.data(), sizeof(S), n * w[0], f) != (size_t)(n * w[0])) return 3;
  if (fread(i1.data(), sizeof(S), n * w[1], f) != (size_t)(n * w[1])) return 3;
  if (fread(i2.data(), sizeof(S), n * w[2], f) != (size_t)(n * w[2])) return 3;
  fclose(f);
  if (group == 1 || group == 3) {
    so3_se3_dispatch<S>(group, op, LieArgs{i0.data(), i1.data(), i2.data(), o0.data(), o1.data(), n});
  } else {
    for (long long i = 0; i < n; ++i) {
      if (group == 2) scaled_group_op<RxSO3g<S>, S>(op, i0.data(), i1.data(), i2.data(), o0.data(), o1.data(), i);
      else scaled_group_op<Sim3g<S>, S>(op, i0.data(), i1.data(), i2.data(), o0.data(), o1.data(), i);
    }
  }
  f = fopen(out, "wb");
  if (!f) return 4;
  fwrite(o0.data(), sizeof(S), n * w[3], f);
  fwrite(o1.data(), sizeof(S), n * w[4], f);
  fclose(f);
  return 0;
}

int main(int argc, char** argv) {
  if (argc != 12) { fprintf(stderr, "bad usage\n"); return 1; }
  const int group = atoi(argv[1]), op = atoi(argv[2]);
  const long long n = atoll(argv[3]);
  int w[5];
  for (int k = 0; k < 5; ++k) w[k] = atoi(argv[4 + k]);
  if (group < 1 || group > 4 || op < 0 || op > OP_JINV) return 1;
  return strcmp(argv[9], "f32") == 0 ? run<float>(group, op, n, w, argv[10], argv[11]) : run<double>(group, op, n, w, argv[10], argv[11]);
}
