// Torch-extension shims over the C-ABI of include/dpvo_b200.h.
//
// One translation unit defines five Python modules; the build copies the resulting shared object
// to cuda_corr*.so, cuda_ba*.so, lietorch_backends*.so, dpvo_b200_ext*.so and dpvo_b200_camera*.so:
//   cuda_corr          same pybind surface as dpvo/altcorr/correlation.cpp:57-62
//   cuda_ba            same as dpvo/fastba/ba.cpp:183-188
//   lietorch_backends  same as dpvo/lietorch/src/lietorch.cpp:286-316
//   dpvo_b200_ext      the fused entry points that have no counterpart in the reference
//   dpvo_b200_camera   the camera-image preparation in front of the encoders (undistort.cu)
// The shims only adapt torch::Tensor -> (pointer, sizes, strides, current CUDA stream), allocate
// outputs and raise RuntimeError on a non-zero status.  There is no CPU path: a CPU tensor is an
// error, not a fallback.
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <algorithm>
#include <vector>

#include "../../include/dpvo_b200.h"

namespace {

using torch::Tensor;

void check(int rc, const char* what) {
  if (rc != DPVO_OK) {
    TORCH_CHECK(false, what, " failed (status ", rc, "): ", dpvo_last_error());
  }
}

int dt(const Tensor& t) {
  switch (t.scalar_type()) {
    case at::kHalf: return DPVO_F16;
    case at::kBFloat16: return DPVO_BF16;
    case at::kFloat: return DPVO_F32;
    case at::kDouble: return DPVO_F64;
    default: TORCH_CHECK(false, "dpvo_b200: unsupported dtype ", t.scalar_type());
  }
  return -1;
}

const char* dtype_name(at::ScalarType st) {
  switch (st) {
    case at::kHalf: return "float16";
    case at::kFloat: return "float32";
    case at::kDouble: return "float64";
    case at::kByte: return "uint8";
    case at::kInt: return "int32";
    case at::kLong: return "int64";
    default: return c10::toString(st);
  }
}

// The tensor contract of every entry point.  Each tensor argument, outputs and workspaces the caller passes included,
// goes through one of these before the op allocates on the device or calls the library: it must be a CUDA tensor on
// the device of the op's anchor tensor, the one its CUDAGuard selects.  A host tensor or one on another GPU is an error
// here and never reaches a kernel.  Messages start with the op's name.
constexpr at::ScalarType kAny = at::ScalarType::Undefined;
struct Args {
  const char* op;
  c10::Device dev;
  Args(const char* op, const Tensor& anchor, const char* what) : op(op), dev(anchor.device()) {
    TORCH_CHECK(anchor.is_cuda(), op, ": ", what, " must be a CUDA tensor (this build has no CPU path)");
  }
  // any layout, of dtype st unless st is kAny
  Tensor on(const Tensor& t, const char* what, at::ScalarType st = kAny) const {
    TORCH_CHECK(t.is_cuda() && t.device() == dev, op, ": ", what, " must be a CUDA tensor on ", dev, " (this build has no CPU path)");
    TORCH_CHECK(st == kAny || t.scalar_type() == st, op, ": ", what, " must be ", dtype_name(st), ", not ", dtype_name(t.scalar_type()));
    return t;
  }
  // on(), contiguous, and of n elements unless n < 0
  Tensor need(const Tensor& t, const char* what, at::ScalarType st = kAny, int64_t n = -1) const {
    on(t, what, st);
    TORCH_CHECK(t.is_contiguous(), op, ": ", what, " must be contiguous");
    TORCH_CHECK(n < 0 || t.numel() == n, op, ": ", what, " must have ", n, " elements, not ", t.numel());
    return t;
  }
  // on(), then converted to st (unless kAny) and made contiguous
  Tensor as(const Tensor& t, const char* what, at::ScalarType st = kAny) const {
    on(t, what);
    return (st == kAny ? t : t.to(st)).contiguous();
  }
  // optional arguments: an undefined tensor when absent
  Tensor on(const c10::optional<Tensor>& t, const char* what, at::ScalarType st = kAny) const { return t ? on(*t, what, st) : Tensor(); }
  Tensor need(const c10::optional<Tensor>& t, const char* what, at::ScalarType st = kAny, int64_t n = -1) const {
    return t ? need(*t, what, st, n) : Tensor();
  }
  Tensor as(const c10::optional<Tensor>& t, const char* what, at::ScalarType st = kAny) const { return t ? as(*t, what, st) : Tensor(); }
};

void* stream() { return (void*)at::cuda::getCurrentCUDAStream().stream(); }

std::vector<int64_t> strides5(const Tensor& t) {
  TORCH_CHECK(t.dim() == 5, "dpvo_b200: expected a 5-d tensor");
  return {t.stride(0), t.stride(1), t.stride(2), t.stride(3), t.stride(4)};
}

Tensor byte_ws(int64_t bytes, const Tensor& like) {
  return torch::empty({bytes}, like.options().dtype(at::kByte));
}

// ------------------------------------------------------------------------------ cuda_corr
std::vector<Tensor> corr_forward(Tensor fmap1, Tensor fmap2, Tensor coords, Tensor ii, Tensor jj, int radius) {
  const Args arg("cuda_corr.forward", fmap1, "fmap1");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.on(fmap2, "fmap2", fmap1.scalar_type());
  coords = arg.as(coords, "coords", at::kFloat); ii = arg.as(ii, "ii", at::kLong); jj = arg.as(jj, "jj", at::kLong);
  TORCH_CHECK(fmap1.dim() == 5 && fmap2.dim() == 5 && coords.dim() == 5, "corr: expected 5-d inputs");
  const int B = coords.size(0), M = coords.size(1), P = coords.size(3);
  const int C = fmap1.size(2), O = 2 * radius + 1;
  TORCH_CHECK(coords.size(2) == 2 && coords.size(4) == P, "corr: coords must be [B,M,2,P,P]");
  TORCH_CHECK(fmap1.size(3) == P && fmap1.size(4) == P && fmap2.size(2) == C, "corr: feature shapes do not match");
  TORCH_CHECK(ii.numel() == M && jj.numel() == M, "corr: index length mismatch");
  Tensor out = torch::empty({B, M, O, O, P, P}, fmap1.options());
  auto s1 = strides5(fmap1), s2 = strides5(fmap2);
  check(dpvo_corr_forward(fmap1.data_ptr(), s1.data(), fmap2.data_ptr(), s2.data(), coords.data_ptr<float>(),
                          ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), out.data_ptr(), 1, dt(fmap1), B, M, C, P,
                          (int)fmap1.size(1), (int)fmap2.size(1), (int)fmap2.size(3), (int)fmap2.size(4), radius, stream()),
        "cuda_corr.forward");
  return {out};
}

std::vector<Tensor> corr_backward(Tensor fmap1, Tensor fmap2, Tensor coords, Tensor ii, Tensor jj, Tensor grad, int radius) {
  const Args arg("cuda_corr.backward", fmap1, "fmap1");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.on(fmap2, "fmap2");
  coords = arg.as(coords, "coords", at::kFloat); ii = arg.as(ii, "ii", at::kLong); jj = arg.as(jj, "jj", at::kLong);
  grad = arg.as(grad, "grad");
  const int B = coords.size(0), M = coords.size(1), P = coords.size(3), C = fmap1.size(2);
  Tensor g1 = torch::zeros_like(fmap1);
  Tensor g2 = torch::zeros_like(fmap2);
  auto s1 = strides5(fmap1), s2 = strides5(fmap2), gs1 = strides5(g1), gs2 = strides5(g2);
  check(dpvo_corr_backward(fmap1.data_ptr(), s1.data(), fmap2.data_ptr(), s2.data(), coords.data_ptr<float>(),
                           ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), grad.data_ptr(), dt(grad),
                           g1.data_ptr(), gs1.data(), g2.data_ptr(), gs2.data(), dt(fmap1), B, M, C, P, (int)fmap1.size(1),
                           (int)fmap2.size(1), (int)fmap2.size(3), (int)fmap2.size(4), radius, stream()),
        "cuda_corr.backward");
  return {g1, g2};
}

std::vector<Tensor> patchify_forward(Tensor net, Tensor coords, int radius) {
  const Args arg("cuda_corr.patchify_forward", net, "net");
  c10::cuda::CUDAGuard guard(arg.dev);
  coords = arg.as(coords, "coords", at::kFloat);
  TORCH_CHECK(net.dim() == 4 && coords.dim() == 3 && coords.size(2) == 2, "patchify: net [B,C,H,W], coords [B,M,2]");
  const int B = coords.size(0), M = coords.size(1), C = net.size(1), D = 2 * radius + 2;
  Tensor patches = torch::empty({B, M, C, D, D}, net.options());
  std::vector<int64_t> s = {net.stride(0), net.stride(1), net.stride(2), net.stride(3)};
  check(dpvo_patchify_forward(net.data_ptr(), s.data(), coords.data_ptr<float>(), patches.data_ptr(), dt(net),
                              B, M, C, (int)net.size(2), (int)net.size(3), radius, stream()),
        "cuda_corr.patchify_forward");
  return {patches};
}

std::vector<Tensor> patchify_backward(Tensor net, Tensor coords, Tensor gradient, int radius) {
  const Args arg("cuda_corr.patchify_backward", net, "net");
  c10::cuda::CUDAGuard guard(arg.dev);
  coords = arg.as(coords, "coords", at::kFloat);
  gradient = arg.as(gradient, "gradient", net.scalar_type());
  const int B = coords.size(0), M = coords.size(1), C = net.size(1);
  Tensor g = torch::zeros(net.sizes(), net.options());
  check(dpvo_patchify_backward(gradient.data_ptr(), coords.data_ptr<float>(), g.data_ptr(), dt(net), B, M, C,
                               (int)net.size(2), (int)net.size(3), radius, stream()),
        "cuda_corr.patchify_backward");
  return {g};
}

// -------------------------------------------------------------------------------- cuda_ba
std::vector<Tensor> group_edges(Tensor key_a, c10::optional<Tensor> key_b, c10::optional<Tensor> sec);
std::vector<Tensor> ba_forward(Tensor poses, Tensor patches, Tensor intrinsics, Tensor target, Tensor weight,
                               Tensor lmbda, Tensor ii, Tensor jj, Tensor kk, int PPF, int t0, int t1,
                               int iterations, bool eff_impl) {
  // poses and patches are updated in place
  const Args arg("cuda_ba.forward", poses, "poses");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.need(poses, "poses", at::kFloat); arg.need(patches, "patches", at::kFloat);
  const int P = patches.size(-1);
  intrinsics = arg.as(intrinsics, "intrinsics", at::kFloat).view({-1, 4});
  target = arg.as(target, "target", at::kFloat).view({-1, 2});
  weight = arg.as(weight, "weight", at::kFloat).view({-1, 2});
  lmbda = arg.as(lmbda, "lmbda", at::kFloat).view({-1});
  ii = arg.as(ii, "ii", at::kLong); jj = arg.as(jj, "jj", at::kLong); kk = arg.as(kk, "kk", at::kLong);
  const int64_t E = ii.numel();
  TORCH_CHECK(jj.numel() == E && kk.numel() == E && target.size(0) == E && weight.size(0) == E, "cuda_ba.forward: edge arrays disagree in length");
  const int64_t n_poses = poses.numel() / 7, n_patches = patches.numel() / (3 * P * P);
  const int N = t1 - t0;
  if (N > 0 && E > 0 && iterations > 0 && (eff_impl || N > 32)) {
    // wide windows / global BA (dpvo.py:312-326): block-sparse Schur complement per source frame (ba_wide.cu), dense
    // Cholesky of the 6N x 6N system by the library -- ba_cuda.cu:547-549 does the same -- then back-substitution
    TORCH_CHECK(PPF > 0, "cuda_ba.forward: patches per frame must be positive");
    std::vector<Tensor> g = group_edges(ii, jj, c10::nullopt);
    Tensor S = torch::empty({6 * N, 6 * N}, poses.options()), y = torch::empty({6 * N}, poses.options());
    Tensor status = torch::zeros({1}, poses.options().dtype(at::kInt));
    for (int it = 0; it < iterations; ++it) {
      check(dpvo_ba_wide_system(poses.data_ptr<float>(), patches.data_ptr<float>(), intrinsics.data_ptr<float>(), target.data_ptr<float>(),
                                weight.data_ptr<float>(), lmbda.data_ptr<float>(), ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(),
                                kk.data_ptr<int64_t>(), E, P, PPF, t0, t1, g[0].data_ptr<int>(), g[2].data_ptr<int>(), g[3].data_ptr<int64_t>(),
                                g[4].data_ptr<int64_t>(), g[5].data_ptr<int>(), S.data_ptr<float>(), y.data_ptr<float>(), status.data_ptr<int>(),
                                stream()),
            "cuda_ba.forward (wide)");
      Tensor L = std::get<0>(at::linalg_cholesky_ex(S));
      Tensor dX = at::cholesky_solve(y.view({6 * N, 1}), L).contiguous();
      check(dpvo_ba_wide_update(poses.data_ptr<float>(), patches.data_ptr<float>(), intrinsics.data_ptr<float>(), target.data_ptr<float>(),
                                weight.data_ptr<float>(), lmbda.data_ptr<float>(), ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(),
                                kk.data_ptr<int64_t>(), E, P, PPF, t0, t1, g[0].data_ptr<int>(), g[2].data_ptr<int>(), g[3].data_ptr<int64_t>(),
                                g[4].data_ptr<int64_t>(), g[5].data_ptr<int>(), dX.data_ptr<float>(), status.data_ptr<int>(), stream()),
            "cuda_ba.forward (wide)");
    }
    const int st = status.item<int>();
    TORCH_CHECK(st == 0, st == 1 ? "cuda_ba.forward (wide): a frame is observed from more frames than the on-chip product holds"
                                 : "cuda_ba.forward (wide): patch ids must be frame * PPF + slot (as dpvo/fastba/block_e.cu assumes)");
    return {};
  }
  const int64_t wsb = dpvo_ba_workspace_bytes(E, t1 - t0);
  Tensor ws = byte_ws(wsb, poses);
  check(dpvo_ba_forward(poses.data_ptr<float>(), patches.data_ptr<float>(), intrinsics.data_ptr<float>(),
                        target.data_ptr<float>(), weight.data_ptr<float>(), lmbda.data_ptr<float>(),
                        ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), kk.data_ptr<int64_t>(), E, n_poses, n_patches, P,
                        t0, t1, iterations, ws.data_ptr(), wsb, stream()),
        "cuda_ba.forward");
  return {};
}

std::vector<Tensor> ba_neighbors(Tensor ii, Tensor jj) {
  const Args arg("cuda_ba.neighbors", ii, "ii");
  c10::cuda::CUDAGuard guard(arg.dev);
  ii = arg.as(ii, "ii", at::kLong); jj = arg.as(jj, "jj", at::kLong);
  const int64_t E = ii.numel();
  TORCH_CHECK(jj.numel() == E, "cuda_ba.neighbors: length mismatch");
  Tensor ix = torch::empty({E}, ii.options()), jx = torch::empty({E}, ii.options());
  const int64_t wsb = dpvo_neighbors_workspace_bytes(E);
  Tensor ws = byte_ws(wsb, ii);
  check(dpvo_neighbors(ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), E, ix.data_ptr<int64_t>(), jx.data_ptr<int64_t>(),
                       ws.data_ptr(), wsb, stream()),
        "cuda_ba.neighbors");
  return {ix, jx};
}

Tensor reproject_impl(Tensor poses, Tensor patches, Tensor intrinsics, Tensor ii, Tensor jj, Tensor kk, int clamp, const char* op) {
  const Args arg(op, poses, "poses");
  c10::cuda::CUDAGuard guard(arg.dev);
  const int P = patches.size(-1);
  poses = arg.as(poses, "poses", at::kFloat); patches = arg.as(patches, "patches", at::kFloat);
  intrinsics = arg.as(intrinsics, "intrinsics", at::kFloat);
  ii = arg.as(ii, "ii", at::kLong); jj = arg.as(jj, "jj", at::kLong); kk = arg.as(kk, "kk", at::kLong);
  const int64_t E = ii.numel();
  Tensor coords = torch::empty({1, E, 2, P, P}, poses.options());
  check(dpvo_reproject(poses.data_ptr<float>(), patches.data_ptr<float>(), intrinsics.data_ptr<float>(),
                       ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), kk.data_ptr<int64_t>(), coords.data_ptr<float>(), E, P,
                       clamp, stream()),
        op);
  return coords;
}
Tensor ba_reproject(Tensor poses, Tensor patches, Tensor intrinsics, Tensor ii, Tensor jj, Tensor kk) {
  return reproject_impl(poses, patches, intrinsics, ii, jj, kk, 0, "cuda_ba.reproject");
}

// cuda_ba.solve_system (ba.cpp:120-180): pose-graph Gauss-Newton step of the loop-closure back end.  The normal
// equations are assembled on the device in fp64 (the reference: Eigen sparse, fp64, on the CPU); the leading
// 7*freen block is solved by a dense Cholesky and the remaining poses get a zero step (ba.cpp:101-118).
std::vector<Tensor> ba_solve_system(Tensor J_Ginv_i, Tensor J_Ginv_j, Tensor ii, Tensor jj, Tensor res, float ep, float lm, int freen) {
  const Args arg("cuda_ba.solve_system", res, "res");
  c10::cuda::CUDAGuard guard(arg.dev);
  J_Ginv_i = arg.as(J_Ginv_i, "J_Ginv_i", at::kFloat); J_Ginv_j = arg.as(J_Ginv_j, "J_Ginv_j", at::kFloat);
  ii = arg.as(ii, "ii", at::kLong); jj = arg.as(jj, "jj", at::kLong);
  Tensor r32 = arg.as(res, "res", at::kFloat).view({-1, 7});
  const int64_t r = r32.size(0);
  TORCH_CHECK(J_Ginv_i.numel() == r * 49 && J_Ginv_j.numel() == r * 49 && ii.numel() == r && jj.numel() == r, "cuda_ba.solve_system: shape mismatch");
  TORCH_CHECK(r > 0, "cuda_ba.solve_system: no residuals");
  TORCH_CHECK(!(ii == jj).any().item<bool>(), "cuda_ba.solve_system: an edge connects a pose to itself");      // ba.cpp:152 exits
  const int64_t n = std::max(ii.max().item<int64_t>(), jj.max().item<int64_t>()) + 1;
  auto od = res.options().dtype(at::kDouble);
  Tensor A = torch::empty({n * 7, n * 7}, od), b = torch::empty({n * 7}, od);
  check(dpvo_posegraph_system(J_Ginv_i.data_ptr<float>(), J_Ginv_j.data_ptr<float>(), ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(),
                              r32.data_ptr<float>(), r, n, (double)ep, (double)lm, A.data_ptr<double>(), b.data_ptr<double>(), stream()),
        "cuda_ba.solve_system");
  const int64_t f = freen < 0 ? n * 7 : std::min<int64_t>((int64_t)freen * 7, n * 7);
  Tensor delta = torch::zeros({n * 7}, od);
  if (f > 0) {
    Tensor L = std::get<0>(at::linalg_cholesky_ex(A.slice(0, 0, f).slice(1, 0, f).contiguous()));
    delta.slice(0, 0, f).copy_(at::cholesky_solve(b.slice(0, 0, f).view({f, 1}), L).view({f}));
  }
  return {delta.to(at::kFloat).view({n, 7})};
}

// ------------------------------------------------------------------------ lietorch_backends
int emb_dim(int g) { return g == DPVO_SO3 ? 4 : g == DPVO_RXSO3 ? 5 : g == DPVO_SE3 ? 7 : 8; }
int tan_dim(int g) { return g == DPVO_SO3 ? 3 : g == DPVO_RXSO3 ? 4 : g == DPVO_SE3 ? 6 : 7; }

typedef int (*un_fn)(int, int, const void*, void*, int64_t, void*);
typedef int (*bin_fn)(int, int, const void*, const void*, void*, int64_t, void*);
typedef int (*unb_fn)(int, int, const void*, const void*, void*, int64_t, void*);
typedef int (*binb_fn)(int, int, const void*, const void*, const void*, void*, void*, int64_t, void*);

Tensor lie_unary(un_fn f, int g, Tensor x, int out_dim, const char* name) {
  const Args arg(name, x, "x");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.need(x, "x");
  Tensor y = torch::empty({x.size(0), out_dim}, x.options());
  check(f(g, dt(x), x.data_ptr(), y.data_ptr(), x.size(0), stream()), name);
  return y;
}
Tensor lie_binary(bin_fn f, int g, Tensor x, Tensor y, int out_dim, const char* name) {
  const Args arg(name, x, "x");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.need(x, "x"); arg.need(y, "y", x.scalar_type());
  TORCH_CHECK(x.size(0) == y.size(0), name, ": operand mismatch");
  Tensor z = torch::empty({x.size(0), out_dim}, x.options());
  check(f(g, dt(x), x.data_ptr(), y.data_ptr(), z.data_ptr(), x.size(0), stream()), name);
  return z;
}
std::vector<Tensor> lie_unary_bwd(unb_fn f, int g, Tensor grad, Tensor x, const char* name) {
  const Args arg(name, x, "x");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.need(x, "x");
  grad = arg.need(grad, "grad").to(x.scalar_type());
  Tensor dx = torch::empty(x.sizes(), x.options());
  check(f(g, dt(x), grad.data_ptr(), x.data_ptr(), dx.data_ptr(), x.size(0), stream()), name);
  return {dx};
}
std::vector<Tensor> lie_binary_bwd(binb_fn f, int g, Tensor grad, Tensor x, Tensor y, const char* name) {
  const Args arg(name, x, "x");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.need(x, "x"); arg.need(y, "y");
  grad = arg.need(grad, "grad").to(x.scalar_type());
  Tensor dx = torch::empty(x.sizes(), x.options()), dy = torch::empty(y.sizes(), y.options());
  check(f(g, dt(x), grad.data_ptr(), x.data_ptr(), y.data_ptr(), dx.data_ptr(), dy.data_ptr(), x.size(0), stream()), name);
  return {dx, dy};
}

Tensor l_expm(int g, Tensor a) { return lie_unary(dpvo_lie_exp, g, a, emb_dim(g), "lietorch_backends.expm"); }
std::vector<Tensor> l_expm_b(int g, Tensor grad, Tensor a) { return lie_unary_bwd(dpvo_lie_exp_backward, g, grad, a, "lietorch_backends.expm_backward"); }
Tensor l_logm(int g, Tensor X) { return lie_unary(dpvo_lie_log, g, X, tan_dim(g), "lietorch_backends.logm"); }
std::vector<Tensor> l_logm_b(int g, Tensor grad, Tensor X) { return lie_unary_bwd(dpvo_lie_log_backward, g, grad, X, "lietorch_backends.logm_backward"); }
Tensor l_inv(int g, Tensor X) { return lie_unary(dpvo_lie_inv, g, X, emb_dim(g), "lietorch_backends.inv"); }
std::vector<Tensor> l_inv_b(int g, Tensor grad, Tensor X) { return lie_unary_bwd(dpvo_lie_inv_backward, g, grad, X, "lietorch_backends.inv_backward"); }
Tensor l_mul(int g, Tensor X, Tensor Y) { return lie_binary(dpvo_lie_mul, g, X, Y, emb_dim(g), "lietorch_backends.mul"); }
std::vector<Tensor> l_mul_b(int g, Tensor grad, Tensor X, Tensor Y) { return lie_binary_bwd(dpvo_lie_mul_backward, g, grad, X, Y, "lietorch_backends.mul_backward"); }
Tensor l_adj(int g, Tensor X, Tensor a) { return lie_binary(dpvo_lie_adj, g, X, a, tan_dim(g), "lietorch_backends.adj"); }
std::vector<Tensor> l_adj_b(int g, Tensor grad, Tensor X, Tensor a) { return lie_binary_bwd(dpvo_lie_adj_backward, g, grad, X, a, "lietorch_backends.adj_backward"); }
Tensor l_adjT(int g, Tensor X, Tensor a) { return lie_binary(dpvo_lie_adjT, g, X, a, tan_dim(g), "lietorch_backends.adjT"); }
std::vector<Tensor> l_adjT_b(int g, Tensor grad, Tensor X, Tensor a) { return lie_binary_bwd(dpvo_lie_adjT_backward, g, grad, X, a, "lietorch_backends.adjT_backward"); }
Tensor l_act(int g, Tensor X, Tensor p) { return lie_binary(dpvo_lie_act, g, X, p, 3, "lietorch_backends.act"); }
std::vector<Tensor> l_act_b(int g, Tensor grad, Tensor X, Tensor p) { return lie_binary_bwd(dpvo_lie_act_backward, g, grad, X, p, "lietorch_backends.act_backward"); }
Tensor l_act4(int g, Tensor X, Tensor p) { return lie_binary(dpvo_lie_act4, g, X, p, 4, "lietorch_backends.act4"); }
std::vector<Tensor> l_act4_b(int g, Tensor grad, Tensor X, Tensor p) { return lie_binary_bwd(dpvo_lie_act4_backward, g, grad, X, p, "lietorch_backends.act4_backward"); }
Tensor l_as_matrix(int g, Tensor X) {
  const Args arg("lietorch_backends.as_matrix", X, "X");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.need(X, "X");
  Tensor T = torch::empty({X.size(0), 4, 4}, X.options());
  check(dpvo_lie_as_matrix(g, dt(X), X.data_ptr(), T.data_ptr(), X.size(0), stream()), "lietorch_backends.as_matrix");
  return T;
}
Tensor l_projector(int g, Tensor X) {
  const Args arg("lietorch_backends.projector", X, "X");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.need(X, "X");
  const int n = emb_dim(g);
  Tensor Pm = torch::empty({X.size(0), n, n}, X.options());
  check(dpvo_lie_projector(g, dt(X), X.data_ptr(), Pm.data_ptr(), X.size(0), stream()), "lietorch_backends.projector");
  return Pm;
}
Tensor l_jinv(int g, Tensor X, Tensor a) { return lie_binary(dpvo_lie_jinv, g, X, a, tan_dim(g), "lietorch_backends.Jinv"); }

// ------------------------------------------------------------------------- dpvo_b200_ext
// DPVO.corr (dpvo.py:200-207) in one launch: returns [1, E, 882]-compatible [B,M,O,O,P,P,2]
Tensor corr_pyramid2(Tensor fmap1, Tensor fmap2_l0, Tensor fmap2_l1, Tensor coords, Tensor ii, Tensor jj, int radius, double div, int64_t pad_to,
                     c10::optional<Tensor> out_buf) {
  const Args arg("dpvo_b200_ext.corr_pyramid2", fmap1, "fmap1");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.on(fmap2_l0, "fmap2_l0"); arg.on(fmap2_l1, "fmap2_l1");
  coords = arg.as(coords, "coords", at::kFloat); ii = arg.as(ii, "ii", at::kLong); jj = arg.as(jj, "jj", at::kLong);
  const int B = coords.size(0), M = coords.size(1), P = coords.size(3), C = fmap1.size(2), O = 2 * radius + 1;
  const int64_t feat = (int64_t)O * O * P * P * 2;
  const int64_t row = pad_to > feat ? pad_to : feat;
  // padded rows ([B, M, row], zero tail) feed the wgmma dense layer directly; unpadded keep the 7-d view
  // out_buf: a caller-owned [B, M, row] buffer whose padding columns are already zero (reused every update)
  Tensor out = arg.need(out_buf, "out", fmap1.scalar_type());
  if (!out.defined()) out = (row == feat) ? torch::empty({B, M, O, O, P, P, 2}, fmap1.options()) : torch::zeros({B, M, row}, fmap1.options());
  TORCH_CHECK(out.numel() == (int64_t)B * M * row, "corr_pyramid2: out buffer must be [B, M, ", row, "]");
  auto s1 = strides5(fmap1), s20 = strides5(fmap2_l0), s21 = strides5(fmap2_l1);
  const int64_t wsb = dpvo_corr_pyramid2_workspace_bytes(M);
  Tensor ws = torch::empty({wsb}, torch::dtype(torch::kUInt8).device(fmap1.device()));
  check(dpvo_corr_forward_pyramid2(fmap1.data_ptr(), s1.data(), fmap2_l0.data_ptr(), s20.data(), (int)fmap2_l0.size(3),
                                   (int)fmap2_l0.size(4), fmap2_l1.data_ptr(), s21.data(), (int)fmap2_l1.size(3),
                                   (int)fmap2_l1.size(4), (float)div, coords.data_ptr<float>(), ii.data_ptr<int64_t>(),
                                   jj.data_ptr<int64_t>(), out.data_ptr(), row, dt(fmap1), B, M, C, P, (int)fmap1.size(1),
                                   (int)fmap2_l0.size(1), radius, ws.data_ptr(), wsb, stream()),
        "dpvo_b200_ext.corr_pyramid2");
  return out;
}

// returns (order, group_of, group_start, key_a, key_b, n_groups) -- all device tensors
std::vector<Tensor> group_edges(Tensor key_a, c10::optional<Tensor> key_b, c10::optional<Tensor> sec) {
  const Args arg("dpvo_b200_ext.group_edges", key_a, "key_a");
  c10::cuda::CUDAGuard guard(arg.dev);
  key_a = arg.as(key_a, "key_a", at::kLong);
  const int64_t E = key_a.numel();
  Tensor kb = arg.as(key_b, "key_b", at::kLong), sc = arg.as(sec, "sec", at::kLong);
  auto oi = key_a.options().dtype(at::kInt);
  Tensor order = torch::empty({E}, oi), gof = torch::empty({E}, oi), gstart = torch::empty({E + 1}, oi);
  Tensor ka = torch::empty({E}, key_a.options()), kbo = torch::empty({E}, key_a.options()), ng = torch::empty({1}, oi);
  const int64_t wsb = dpvo_group_workspace_bytes(E);
  Tensor ws = byte_ws(wsb, key_a);
  check(dpvo_group_edges(key_a.data_ptr<int64_t>(), kb.defined() ? kb.data_ptr<int64_t>() : nullptr,
                         sc.defined() ? sc.data_ptr<int64_t>() : nullptr, E, order.data_ptr<int>(), gof.data_ptr<int>(),
                         gstart.data_ptr<int>(), ka.data_ptr<int64_t>(), kbo.data_ptr<int64_t>(), ng.data_ptr<int>(),
                         ws.data_ptr(), wsb, stream()),
        "dpvo_b200_ext.group_edges");
  return {order, gof, gstart, ka, kbo, ng};
}

// both groupings of an update in one launch; returns the two 6-tuples of group_edges concatenated
std::vector<Tensor> group_edges_pair(Tensor a0, c10::optional<Tensor> b0, c10::optional<Tensor> s0, Tensor a1, c10::optional<Tensor> b1,
                                     c10::optional<Tensor> s1) {
  const Args arg("dpvo_b200_ext.group_edges_pair", a0, "key_a0");
  c10::cuda::CUDAGuard guard(arg.dev);
  a0 = arg.as(a0, "key_a0", at::kLong); a1 = arg.as(a1, "key_a1", at::kLong);
  const int64_t E = a0.numel();
  TORCH_CHECK(a1.numel() == E, "group_edges_pair: both problems group the same edges");
  Tensor kb[2] = {arg.as(b0, "key_b0", at::kLong), arg.as(b1, "key_b1", at::kLong)};
  Tensor sc[2] = {arg.as(s0, "sec0", at::kLong), arg.as(s1, "sec1", at::kLong)};
  auto oi = a0.options().dtype(at::kInt);
  const int64_t wsb = dpvo_group_workspace_bytes(E);
  std::vector<Tensor> out;
  Tensor ws[2];
  for (int q = 0; q < 2; ++q) {
    out.push_back(torch::empty({E}, oi)); out.push_back(torch::empty({E}, oi)); out.push_back(torch::empty({E + 1}, oi));
    out.push_back(torch::empty({E}, a0.options())); out.push_back(torch::empty({E}, a0.options())); out.push_back(torch::empty({1}, oi));
    ws[q] = byte_ws(wsb, a0);
  }
  auto P = [](const Tensor& t) -> const int64_t* { return t.defined() ? t.data_ptr<int64_t>() : nullptr; };
  check(dpvo_group_edges_pair(a0.data_ptr<int64_t>(), P(kb[0]), P(sc[0]), out[0].data_ptr<int>(), out[1].data_ptr<int>(), out[2].data_ptr<int>(),
                              out[3].data_ptr<int64_t>(), out[4].data_ptr<int64_t>(), out[5].data_ptr<int>(), ws[0].data_ptr(),
                              a1.data_ptr<int64_t>(), P(kb[1]), P(sc[1]), out[6].data_ptr<int>(), out[7].data_ptr<int>(), out[8].data_ptr<int>(),
                              out[9].data_ptr<int64_t>(), out[10].data_ptr<int64_t>(), out[11].data_ptr<int>(), ws[1].data_ptr(),
                              E, wsb, stream()),
        "dpvo_b200_ext.group_edges_pair");
  return out;
}

// the operands of ba_forward_grouped / _batched: poses and patches are updated in place, the rest converted as read
void ba_args(const Args& arg, const Tensor& poses, const Tensor& patches, Tensor& intrinsics, Tensor& target, Tensor& weight,
             Tensor& lmbda, Tensor& ii, Tensor& jj, Tensor& kk, const Tensor& k_order, const Tensor& k_start, const Tensor& k_key,
             const Tensor& k_n, const Tensor& p_order, const Tensor& p_start, const Tensor& p_key_i, const Tensor& p_key_j,
             const Tensor& p_n) {
  arg.need(poses, "poses", at::kFloat); arg.need(patches, "patches", at::kFloat);
  intrinsics = arg.as(intrinsics, "intrinsics", at::kFloat); target = arg.as(target, "target", at::kFloat);
  weight = arg.as(weight, "weight", at::kFloat); lmbda = arg.as(lmbda, "lmbda", at::kFloat);
  ii = arg.as(ii, "ii", at::kLong); jj = arg.as(jj, "jj", at::kLong); kk = arg.as(kk, "kk", at::kLong);
  arg.need(k_order, "k_order", at::kInt); arg.need(k_start, "k_start", at::kInt); arg.need(k_key, "k_key", at::kLong);
  arg.need(k_n, "k_n", at::kInt); arg.need(p_order, "p_order", at::kInt); arg.need(p_start, "p_start", at::kInt);
  arg.need(p_key_i, "p_key_i", at::kLong); arg.need(p_key_j, "p_key_j", at::kLong); arg.need(p_n, "p_n", at::kInt);
}

// fastba.BA on groupings built once per update (order, group_start, key_a[, key_b], n of EdgeGroups)
void ba_forward_grouped(Tensor poses, Tensor patches, Tensor intrinsics, Tensor target, Tensor weight, Tensor lmbda,
                        Tensor ii, Tensor jj, Tensor kk, int t0, int t1, int iterations,
                        Tensor k_order, Tensor k_start, Tensor k_key, Tensor k_n,
                        Tensor p_order, Tensor p_start, Tensor p_key_i, Tensor p_key_j, Tensor p_n) {
  const Args arg("dpvo_b200_ext.ba_forward_grouped", poses, "poses");
  c10::cuda::CUDAGuard guard(arg.dev);
  ba_args(arg, poses, patches, intrinsics, target, weight, lmbda, ii, jj, kk, k_order, k_start, k_key, k_n, p_order, p_start,
          p_key_i, p_key_j, p_n);
  const int P = patches.size(-1);
  const int64_t E = ii.numel();
  const int64_t wsb = dpvo_ba_grouped_workspace_bytes(E, t1 - t0);
  Tensor ws = byte_ws(wsb, poses);
  check(dpvo_ba_forward_grouped(poses.data_ptr<float>(), patches.data_ptr<float>(), intrinsics.data_ptr<float>(),
                                target.data_ptr<float>(), weight.data_ptr<float>(), lmbda.data_ptr<float>(),
                                ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), kk.data_ptr<int64_t>(), E, P, t0, t1, iterations,
                                k_order.data_ptr<int>(), k_start.data_ptr<int>(), k_key.data_ptr<int64_t>(), k_n.data_ptr<int>(),
                                p_order.data_ptr<int>(), p_start.data_ptr<int>(), p_key_i.data_ptr<int64_t>(),
                                p_key_j.data_ptr<int64_t>(), p_n.data_ptr<int>(), ws.data_ptr(), wsb, stream()),
        "dpvo_b200_ext.ba_forward_grouped");
}

// B streams' sliding windows in one reduce and one solve launch per iteration; t0 / t1 are global frame numbers
void ba_forward_batched(Tensor poses, Tensor patches, Tensor intrinsics, Tensor target, Tensor weight, Tensor lmbda,
                        Tensor ii, Tensor jj, Tensor kk, int64_t frames_per_stream, std::vector<int> t0, std::vector<int> t1,
                        int iterations, Tensor k_order, Tensor k_start, Tensor k_key, Tensor k_n,
                        Tensor p_order, Tensor p_start, Tensor p_key_i, Tensor p_key_j, Tensor p_n) {
  const Args arg("dpvo_b200_ext.ba_forward_batched", poses, "poses");
  c10::cuda::CUDAGuard guard(arg.dev);
  ba_args(arg, poses, patches, intrinsics, target, weight, lmbda, ii, jj, kk, k_order, k_start, k_key, k_n, p_order, p_start,
          p_key_i, p_key_j, p_n);
  TORCH_CHECK(t0.size() == t1.size() && !t0.empty(), "ba_forward_batched: t0 and t1 need one entry per stream");
  const int B = (int)t0.size();
  const int64_t n_frames = poses.numel() / 7, n_patches = patches.numel() / (3 * patches.size(-1) * patches.size(-1));
  TORCH_CHECK(frames_per_stream > 0 && n_frames == B * frames_per_stream && n_patches % n_frames == 0,
              "ba_forward_batched: poses hold ", n_frames, " frames and patches ", n_patches, ", not ", B, " streams of ",
              frames_per_stream, " frames with the same number of patches each");
  TORCH_CHECK(intrinsics.numel() == 4 * n_frames, "ba_forward_batched: intrinsics need one row per frame");
  const int P = patches.size(-1);
  const int64_t E = ii.numel();
  int max_n = 0;
  for (int b = 0; b < B; ++b) max_n = std::max(max_n, t1[b] - t0[b]);
  const int64_t wsb = dpvo_ba_batched_workspace_bytes(E, B, max_n);
  Tensor ws = byte_ws(wsb, poses);
  check(dpvo_ba_forward_batched(poses.data_ptr<float>(), patches.data_ptr<float>(), intrinsics.data_ptr<float>(),
                                target.data_ptr<float>(), weight.data_ptr<float>(), lmbda.data_ptr<float>(),
                                ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), kk.data_ptr<int64_t>(), E, P, B,
                                (int)frames_per_stream, (int)(n_patches / n_frames), t0.data(), t1.data(), iterations,
                                k_order.data_ptr<int>(), k_start.data_ptr<int>(), k_key.data_ptr<int64_t>(), k_n.data_ptr<int>(),
                                p_order.data_ptr<int>(), p_start.data_ptr<int>(), p_key_i.data_ptr<int64_t>(),
                                p_key_j.data_ptr<int64_t>(), p_n.data_ptr<int>(), ws.data_ptr(), wsb, stream()),
        "dpvo_b200_ext.ba_forward_batched");
}

int64_t ba_batched_workspace_bytes(int64_t E, int64_t B, int64_t max_free_poses) {
  return dpvo_ba_batched_workspace_bytes(E, (int)B, (int)max_free_poses);
}

Tensor reproject_clamped(Tensor poses, Tensor patches, Tensor intrinsics, Tensor ii, Tensor jj, Tensor kk) {
  return reproject_impl(poses, patches, intrinsics, ii, jj, kk, 1, "dpvo_b200_ext.reproject_clamped");
}


// ---- update-operator building blocks (include/dpvo_b200.h, "Update operator building blocks")
int dt16or32(const Tensor& t) {
  TORCH_CHECK(t.scalar_type() == at::kHalf || t.scalar_type() == at::kFloat, "dpvo_b200: expected float16 or float32");
  return dt(t);
}

std::vector<Tensor> add_layernorm(Tensor a, c10::optional<Tensor> b, c10::optional<Tensor> c, Tensor gamma, Tensor beta,
                                  double eps, bool relu, bool want32, bool want16, c10::optional<Tensor> b_index, bool inplace32,
                                  c10::optional<Tensor> c_scale) {
  const Args arg("dpvo_b200_ext.add_layernorm", a, "a");
  c10::cuda::CUDAGuard guard(arg.dev);
  const int dim = a.size(-1);
  const int64_t rows = a.numel() / dim;
  a = arg.as(a, "a");
  Tensor bb = arg.as(b, "b"), cc = arg.as(c, "c"), bidx = arg.as(b_index, "b_index", at::kLong);
  gamma = arg.as(gamma, "gamma", at::kFloat); beta = arg.as(beta, "beta", at::kFloat);
  Tensor csc = arg.on(c_scale, "c_scale", at::kHalf);
  int dts[3] = {dt16or32(a), 0, 0};
  if (bidx.defined()) TORCH_CHECK(bidx.numel() == rows, "add_layernorm: b_index length");
  if (bb.defined()) { dts[1] = dt16or32(bb); TORCH_CHECK(bidx.defined() || bb.numel() == a.numel(), "add_layernorm: shape mismatch"); }
  if (cc.defined()) { dts[2] = dt16or32(cc); TORCH_CHECK(cc.numel() == a.numel(), "add_layernorm: shape mismatch"); }
  int64_t ld_cs = 0;
  if (csc.defined()) {
    csc = csc.reshape({-1, dim});
    TORCH_CHECK(csc.stride(1) == 1 && csc.size(0) == rows && cc.defined(), "add_layernorm: c_scale must be fp16 [rows, dim] next to operand c");
    ld_cs = csc.stride(0);
  }
  Tensor y32, y16;
  // inplace32: the fp32 result overwrites operand a (rows are read completely before they are written), so a
  // recurrent state can live in one buffer -- which also makes the whole update capturable in a CUDA graph
  if (inplace32) TORCH_CHECK(want32 && a.scalar_type() == at::kFloat, "add_layernorm: inplace32 needs an fp32 operand a and want32");
  if (want32) y32 = inplace32 ? a : torch::empty(a.sizes(), a.options().dtype(at::kFloat));
  if (want16) y16 = torch::empty(a.sizes(), a.options().dtype(at::kHalf));
  check(dpvo_add_layernorm(a.data_ptr(), bb.defined() ? bb.data_ptr() : nullptr, cc.defined() ? cc.data_ptr() : nullptr, dts,
                           bidx.defined() ? bidx.data_ptr<int64_t>() : nullptr, csc.defined() ? csc.data_ptr() : nullptr, ld_cs,
                           gamma.data_ptr<float>(), beta.data_ptr<float>(), (float)eps, want32 ? y32.data_ptr() : nullptr,
                           want16 ? y16.data_ptr() : nullptr, relu ? 1 : 0, rows, dim, stream()),
        "dpvo_b200_ext.add_layernorm");
  return {y32, y16};
}

Tensor gather_rows_masked(Tensor x, Tensor idx, bool half_out) {
  const Args arg("dpvo_b200_ext.gather_rows_masked", x, "x");
  c10::cuda::CUDAGuard guard(arg.dev);
  x = arg.as(x, "x"); idx = arg.as(idx, "idx", at::kLong);
  const int dim = x.size(-1);
  const int64_t rows = idx.numel();
  Tensor y = torch::empty({1, rows, dim}, x.options().dtype(half_out ? at::kHalf : at::kFloat));
  check(dpvo_gather_rows_masked(x.data_ptr(), dt16or32(x), idx.data_ptr<int64_t>(), y.data_ptr(), dt(y), rows, dim, stream()),
        "dpvo_b200_ext.gather_rows_masked");
  return y;
}

Tensor residual_add_(Tensor net32, Tensor u, c10::optional<Tensor> group_of, bool want16) {
  const Args arg("dpvo_b200_ext.residual_add_", net32, "net");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.need(net32, "net", at::kFloat);
  u = arg.as(u, "u");
  Tensor gof = arg.as(group_of, "group_of", at::kInt), n16;
  const int dim = net32.size(-1);
  const int64_t rows = net32.numel() / dim;
  if (gof.defined()) { TORCH_CHECK(gof.numel() == rows, "residual_add_: group_of length"); }
  else TORCH_CHECK(u.numel() == net32.numel(), "residual_add_: shape mismatch");
  if (want16) n16 = torch::empty(net32.sizes(), net32.options().dtype(at::kHalf));
  check(dpvo_residual_add(net32.data_ptr(), u.data_ptr(), dt16or32(u), gof.defined() ? gof.data_ptr<int>() : nullptr,
                          want16 ? n16.data_ptr() : nullptr, rows, dim, stream()),
        "dpvo_b200_ext.residual_add_");
  return n16;
}

// fp16( net32 + u[group_of] ) without updating net32
Tensor residual_sum16(Tensor net32, Tensor u, c10::optional<Tensor> group_of) {
  const Args arg("dpvo_b200_ext.residual_sum16", net32, "net");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.need(net32, "net", at::kFloat);
  u = arg.as(u, "u");
  Tensor gof = arg.as(group_of, "group_of", at::kInt);
  const int dim = net32.size(-1);
  const int64_t rows = net32.numel() / dim;
  if (gof.defined()) { TORCH_CHECK(gof.numel() == rows, "residual_sum16: group_of length"); }
  else TORCH_CHECK(u.numel() == net32.numel(), "residual_sum16: shape mismatch");
  Tensor n16 = torch::empty(net32.sizes(), net32.options().dtype(at::kHalf));
  check(dpvo_residual_sum16(net32.data_ptr(), u.data_ptr(), dt16or32(u), gof.defined() ? gof.data_ptr<int>() : nullptr, n16.data_ptr(), rows, dim, stream()),
        "dpvo_b200_ext.residual_sum16");
  return n16;
}

std::vector<Tensor> gated_residual(Tensor x32, Tensor gate16, Tensor res16, bool want_relu16) {
  const Args arg("dpvo_b200_ext.gated_residual", x32, "x");
  c10::cuda::CUDAGuard guard(arg.dev);
  x32 = arg.on(x32, "x", at::kFloat).contiguous();
  gate16 = arg.on(gate16, "gate", at::kHalf).contiguous(); res16 = arg.on(res16, "res", at::kHalf).contiguous();
  const int dim = x32.size(-1);
  const int64_t rows = x32.numel() / dim;
  Tensor y = torch::empty_like(x32), r16;
  if (want_relu16) r16 = torch::empty(x32.sizes(), x32.options().dtype(at::kHalf));
  check(dpvo_gated_residual(x32.data_ptr(), gate16.data_ptr(), res16.data_ptr(), y.data_ptr(),
                            want_relu16 ? r16.data_ptr() : nullptr, rows, dim, stream()),
        "dpvo_b200_ext.gated_residual");
  return {y, r16};
}

// fg: [.., E, 2*dim] fp16 = [f | g] (one GEMM with the f and g weights stacked)
Tensor softagg_reduce(Tensor fg, Tensor order, Tensor group_start, Tensor n_groups, int64_t max_groups) {
  const Args arg("dpvo_b200_ext.softagg_reduce", fg, "fg");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.need(fg, "fg", at::kHalf);
  TORCH_CHECK(fg.size(-1) % 2 == 0, "softagg_reduce: expects [E, 2*dim]");
  const int dim = fg.size(-1) / 2;
  const int64_t E = fg.numel() / fg.size(-1);
  arg.need(order, "order (one entry per row of fg)", at::kInt, E);
  arg.need(group_start, "group_start", at::kInt);
  arg.need(n_groups, "n_groups", at::kInt, 1);
  TORCH_CHECK(group_start.numel() >= max_groups + 1, "softagg_reduce: group_start must have at least max_groups + 1 entries");
  TORCH_CHECK(max_groups >= 0 && max_groups <= E, "softagg_reduce: max_groups must be in [0, E]");
  Tensor y = torch::empty({1, max_groups, dim}, fg.options());   // rows past the group count are zeroed by the kernel itself
  const at::Half* base = fg.data_ptr<at::Half>();
  check(dpvo_softagg_reduce(base, base + dim, 2 * dim, order.data_ptr<int>(), group_start.data_ptr<int>(),
                            n_groups.data_ptr<int>(), max_groups, y.data_ptr(), dim, stream()),
        "dpvo_b200_ext.softagg_reduce");
  return y;
}

// x: [.., E, dim] fp16; w [2*dim, dim] fp16 / bias [2*dim] fp32 with the f and g rows interleaved by 96-channel slice
Tensor softagg_fused(Tensor x, Tensor order, Tensor group_of, Tensor group_start, Tensor n_groups, int64_t max_groups, Tensor w,
                     Tensor bias, c10::optional<Tensor> workspace) {
  const Args arg("dpvo_b200_ext.softagg_fused", x, "x");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.on(x, "x", at::kHalf);
  TORCH_CHECK(x.stride(-1) == 1, "softagg_fused: x must have contiguous rows");
  const int dim = x.size(-1);
  Tensor x2 = x.dim() == 2 ? x : x.reshape({-1, dim});
  const int64_t E = x2.size(0);
  arg.need(w, "w", at::kHalf);
  TORCH_CHECK(w.dim() == 2 && w.size(0) == 2 * dim && w.size(1) == dim, "softagg_fused: w must be float16 [2*dim, dim]");
  arg.need(bias, "bias [2*dim]", at::kFloat, 2 * dim);
  arg.need(order, "order (one entry per row of x)", at::kInt, E);
  arg.need(group_of, "group_of (one entry per row of x)", at::kInt, E);
  arg.need(group_start, "group_start", at::kInt);
  arg.need(n_groups, "n_groups", at::kInt, 1);
  Tensor ws = arg.need(workspace, "workspace");
  TORCH_CHECK(group_start.numel() >= max_groups + 1, "softagg_fused: group_start must have at least max_groups + 1 entries");
  TORCH_CHECK(max_groups >= 0 && max_groups <= E, "softagg_fused: max_groups must be in [0, E]");
  const int64_t wsb = dpvo_softagg_fused_workspace_bytes(E);
  if (!ws.defined()) ws = byte_ws(wsb, x);
  TORCH_CHECK((int64_t)(ws.numel() * ws.element_size()) >= wsb, "softagg_fused: workspace too small");
  Tensor y = torch::empty({1, max_groups, dim}, x.options());   // rows past the group count are zeroed by the op itself
  check(dpvo_softagg_fused(x2.data_ptr(), x2.stride(0), order.data_ptr<int>(), group_of.data_ptr<int>(), group_start.data_ptr<int>(),
                           n_groups.data_ptr<int>(), w.data_ptr(), bias.data_ptr<float>(), E, max_groups, y.data_ptr(),
                           ws.data_ptr(), wsb, dim, stream()),
        "dpvo_b200_ext.softagg_fused");
  return y;
}

int64_t softagg_fused_workspace_bytes(int64_t E) { return dpvo_softagg_fused_workspace_bytes(E); }

// Y = epilogue(X @ W^T + bias) on wgmma; X [.., rows, K] fp16 (row stride may exceed K), W [N, K] fp16
Tensor linear_f16(Tensor x, Tensor w, c10::optional<Tensor> bias, int64_t epilogue, c10::optional<Tensor> res,
                  c10::optional<Tensor> gate, c10::optional<Tensor> gather, bool out_f32, c10::optional<Tensor> out,
                  c10::optional<Tensor> out16) {
  const Args arg("dpvo_b200_ext.linear_f16", x, "x");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.on(x, "x", at::kHalf); arg.on(w, "w", at::kHalf);
  Tensor gi = arg.as(gather, "gather", at::kLong), b = arg.as(bias, "bias", at::kFloat), r = arg.on(res, "res");
  Tensor g = arg.on(gate, "gate", at::kHalf);
  Tensor y = arg.need(out, "out", out_f32 ? at::kFloat : at::kHalf), y16 = arg.need(out16, "out16", at::kHalf);
  TORCH_CHECK(x.stride(-1) == 1 && w.dim() == 2 && w.stride(1) == 1, "linear_f16: K must be contiguous");
  const int K = w.size(1), N = w.size(0);
  TORCH_CHECK(x.size(-1) == K, "linear_f16: X has ", x.size(-1), " columns, W expects ", K);
  Tensor x2 = x.dim() == 2 ? x : x.reshape({-1, K});
  TORCH_CHECK(x2.stride(1) == 1, "linear_f16: X rows must be dense");
  const int64_t rows = gi.defined() ? gi.numel() : x2.size(0);
  int res_dt = DPVO_F32; int64_t ldres = 0, ldgate = 0;
  if (r.defined()) { r = r.reshape({-1, N}); TORCH_CHECK(r.stride(1) == 1 && r.size(0) == rows, "linear_f16: res shape"); res_dt = dt16or32(r); ldres = r.stride(0); }
  if (g.defined()) { g = g.reshape({-1, N}); TORCH_CHECK(g.stride(1) == 1 && g.size(0) == rows, "linear_f16: gate shape"); ldgate = g.stride(0); }
  if (!y.defined()) y = torch::empty({1, rows, N}, x.options().dtype(out_f32 ? at::kFloat : at::kHalf));
  TORCH_CHECK(y.numel() == rows * N, "linear_f16: out tensor");
  if (y16.defined()) TORCH_CHECK(y16.numel() == rows * N, "linear_f16: out16 tensor");
  check(dpvo_linear_f16(x2.data_ptr(), x2.stride(0), gi.defined() ? gi.data_ptr<int64_t>() : nullptr, w.data_ptr(), w.stride(0),
                        b.defined() ? b.data_ptr<float>() : nullptr, r.defined() ? r.data_ptr() : nullptr, res_dt, ldres,
                        g.defined() ? g.data_ptr() : nullptr, ldgate, y.data_ptr(), out_f32 ? DPVO_F32 : DPVO_F16, N,
                        y16.defined() ? y16.data_ptr() : nullptr, N, rows, N, K, (int)epilogue, stream()),
        "dpvo_b200_ext.linear_f16");
  return y;
}

std::vector<Tensor> neighbors_from_groups(Tensor order, Tensor group_of) {
  const Args arg("dpvo_b200_ext.neighbors_from_groups", order, "order");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.need(order, "order", at::kInt); arg.need(group_of, "group_of", at::kInt);
  const int64_t E = order.numel();
  auto ol = order.options().dtype(at::kLong);
  Tensor ix = torch::empty({E}, ol), jx = torch::empty({E}, ol);
  check(dpvo_neighbors_from_groups(order.data_ptr<int>(), group_of.data_ptr<int>(), E, ix.data_ptr<int64_t>(),
                                   jx.data_ptr<int64_t>(), stream()),
        "dpvo_b200_ext.neighbors_from_groups");
  return {ix, jx};
}

std::vector<Tensor> update_heads(Tensor net32, Tensor W4, Tensor b4, c10::optional<Tensor> coords, c10::optional<Tensor> gate,
                                 c10::optional<Tensor> res) {
  const Args arg("dpvo_b200_ext.update_heads", net32, "net");
  c10::cuda::CUDAGuard guard(arg.dev);
  TORCH_CHECK(gate.has_value() == res.has_value(), "update_heads: gate and res come together");
  // the gated form updates net in place
  net32 = gate.has_value() ? arg.need(net32, "net", at::kFloat) : arg.on(net32, "net", at::kFloat).contiguous();
  W4 = arg.as(W4, "W4", at::kFloat); b4 = arg.as(b4, "b4", at::kFloat);
  Tensor cd = arg.as(coords, "coords", at::kFloat), g2 = arg.on(gate, "gate", at::kHalf), r2 = arg.on(res, "res", at::kHalf);
  const int dim = net32.size(-1);
  const int64_t rows = net32.numel() / dim;
  TORCH_CHECK(W4.numel() == 4 * dim && b4.numel() == 4, "update_heads: W4 [4,dim], b4 [4]");
  int P = 1;
  if (cd.defined()) { P = cd.size(-1); TORCH_CHECK(cd.numel() == rows * 2 * P * P, "update_heads: coords must be [rows,2,P,P]"); }
  int64_t ldg = 0, ldr = 0;
  if (g2.defined()) {
    g2 = g2.reshape({-1, dim}); r2 = r2.reshape({-1, dim});
    TORCH_CHECK(g2.stride(1) == 1 && r2.stride(1) == 1 && g2.size(0) == rows && r2.size(0) == rows, "update_heads: gate / res must be fp16 [rows, dim]");
    ldg = g2.stride(0); ldr = r2.stride(0);
  }
  Tensor delta = torch::empty({1, rows, 2}, net32.options()), weight = torch::empty({1, rows, 2}, net32.options());
  check(dpvo_update_heads(net32.data_ptr(), g2.defined() ? g2.data_ptr() : nullptr, ldg, r2.defined() ? r2.data_ptr() : nullptr, ldr,
                          W4.data_ptr<float>(), b4.data_ptr<float>(), cd.defined() ? cd.data_ptr<float>() : nullptr, P,
                          delta.data_ptr<float>(),
                          weight.data_ptr<float>(), rows, dim, stream()),
        "dpvo_b200_ext.update_heads");
  return {delta, weight};
}

// ---- fused layer chains of the update operator (include/dpvo_b200.h, "fused layer chains")
Tensor update_corr_norm(Tensor corr16, Tensor W0, Tensor W25, Tensor params, Tensor net32, Tensor inp16, c10::optional<Tensor> inp_index,
                        c10::optional<Tensor> net16_out) {
  const Args arg("dpvo_b200_ext.update_corr_norm", net32, "net32");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.on(corr16, "corr16", at::kHalf); arg.need(W0, "W0", at::kHalf); arg.need(W25, "W25", at::kHalf);
  arg.need(params, "params", at::kFloat); arg.need(net32, "net32", at::kFloat); arg.need(inp16, "inp16", at::kHalf);
  Tensor idx = arg.as(inp_index, "inp_index", at::kLong), n16 = arg.need(net16_out, "net16_out", at::kHalf);
  const int64_t E = net32.numel() / 384;
  Tensor c2 = corr16.reshape({-1, corr16.size(-1)});
  TORCH_CHECK(c2.stride(1) == 1 && c2.size(0) == E && c2.size(1) == 896, "update_corr_norm: corr must be fp16 [E, 896] (zero padded)");
  TORCH_CHECK(net32.size(-1) == 384 && W0.numel() == 384 * 896 && W25.numel() == 768 * 384 && params.numel() == 7 * 384 && inp16.size(-1) == 384, "update_corr_norm: shapes");
  if (idx.defined()) { TORCH_CHECK(idx.numel() == E, "update_corr_norm: inp_index length"); }
  else TORCH_CHECK(inp16.numel() == E * 384, "update_corr_norm: inp must have one row per edge when no index is given");
  if (!n16.defined()) n16 = torch::empty({1, E, 384}, net32.options().dtype(at::kHalf));
  TORCH_CHECK(n16.numel() == E * 384, "update_corr_norm: net16_out shape");
  check(dpvo_update_corr_norm(c2.data_ptr(), c2.stride(0), W0.data_ptr(), W25.data_ptr(), params.data_ptr<float>(), net32.data_ptr<float>(),
                              inp16.data_ptr(), idx.defined() ? idx.data_ptr<int64_t>() : nullptr, n16.data_ptr(), E, stream()),
        "dpvo_b200_ext.update_corr_norm");
  return n16;
}

Tensor update_neighbor_mlp(Tensor net16_in, Tensor index, Tensor Wab, Tensor params, Tensor net32, c10::optional<Tensor> net16_out) {
  const Args arg("dpvo_b200_ext.update_neighbor_mlp", net32, "net32");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.need(net16_in, "net16_in", at::kHalf); arg.need(Wab, "Wab", at::kHalf); arg.need(params, "params", at::kFloat);
  arg.need(net32, "net32", at::kFloat);
  index = arg.as(index, "index", at::kLong);
  Tensor n16 = arg.need(net16_out, "net16_out", at::kHalf);
  const int64_t E = net32.numel() / 384;
  TORCH_CHECK(net32.size(-1) == 384 && net16_in.numel() == E * 384 && index.numel() == E && Wab.numel() == 768 * 384 && params.numel() == 2 * 384, "update_neighbor_mlp: shapes");
  if (!n16.defined()) n16 = torch::empty({1, E, 384}, net32.options().dtype(at::kHalf));
  TORCH_CHECK(n16.numel() == E * 384, "update_neighbor_mlp: net16_out shape");
  check(dpvo_update_neighbor_mlp(net16_in.data_ptr(), index.data_ptr<int64_t>(), Wab.data_ptr(), params.data_ptr<float>(), net32.data_ptr<float>(),
                                 n16.data_ptr(), E, stream()),
        "dpvo_b200_ext.update_neighbor_mlp");
  return n16;
}

std::vector<Tensor> update_gru_heads(Tensor net32, c10::optional<Tensor> hij16, c10::optional<Tensor> group_of, Tensor W6, Tensor params,
                                     c10::optional<Tensor> coords, c10::optional<Tensor> workspace, c10::optional<Tensor> hkk16, c10::optional<Tensor> group_kk,
                                     c10::optional<Tensor> delta_out, c10::optional<Tensor> weight_out) {
  const Args arg("dpvo_b200_ext.update_gru_heads", net32, "net32");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.need(net32, "net32", at::kFloat); arg.need(W6, "W6", at::kHalf); arg.need(params, "params", at::kFloat);
  Tensor hij = arg.need(hij16, "hij16", at::kHalf), gof = arg.as(group_of, "group_of", at::kInt);
  Tensor hkk = arg.need(hkk16, "hkk16", at::kHalf), gkk = arg.as(group_kk, "group_kk", at::kInt);
  Tensor cd = arg.as(coords, "coords", at::kFloat), ws = arg.need(workspace, "workspace");
  Tensor delta = arg.need(delta_out, "delta_out", at::kFloat), weight = arg.need(weight_out, "weight_out", at::kFloat);
  const int64_t E = net32.numel() / 384;
  TORCH_CHECK(net32.size(-1) == 384 && W6.numel() == 6 * 384 * 384 && params.numel() == 14 * 384 + 4, "update_gru_heads: shapes");
  TORCH_CHECK(hij.defined() == gof.defined() && hkk.defined() == gkk.defined(), "update_gru_heads: group rows and group ids come together");
  if (hij.defined()) TORCH_CHECK(hij.size(-1) == 384 && gof.numel() == E, "update_gru_heads: group operand shapes");
  if (hkk.defined()) TORCH_CHECK(hkk.size(-1) == 384 && gkk.numel() == E, "update_gru_heads: group operand shapes");
  int P = 1;
  if (cd.defined()) { P = cd.size(-1); TORCH_CHECK(cd.numel() == E * 2 * P * P, "update_gru_heads: coords must be [E,2,P,P]"); }
  const int64_t wsb = dpvo_update_gru_workspace_bytes();
  if (!ws.defined()) ws = byte_ws(wsb, net32);
  TORCH_CHECK((int64_t)(ws.numel() * ws.element_size()) >= wsb, "update_gru_heads: workspace too small");
  if (!delta.defined()) delta = torch::empty({1, E, 2}, net32.options());
  if (!weight.defined()) weight = torch::empty({1, E, 2}, net32.options());
  TORCH_CHECK(delta.numel() == E * 2 && weight.numel() == E * 2, "update_gru_heads: delta_out / weight_out must hold [E, 2]");
  check(dpvo_update_gru_heads(net32.data_ptr<float>(), hij.defined() ? hij.data_ptr() : nullptr, gof.defined() ? gof.data_ptr<int>() : nullptr,
                              hkk.defined() ? hkk.data_ptr() : nullptr, gkk.defined() ? gkk.data_ptr<int>() : nullptr, W6.data_ptr(), params.data_ptr<float>(), cd.defined() ? cd.data_ptr<float>() : nullptr, P,
                              delta.data_ptr<float>(), weight.data_ptr<float>(), ws.data_ptr(), E, stream()),
        "dpvo_b200_ext.update_gru_heads");
  return {delta, weight};
}
int64_t update_gru_workspace_bytes() { return dpvo_update_gru_workspace_bytes(); }

// ---- device-resident patch-graph bookkeeping (include/dpvo_b200.h)
// the fixed-capacity edge store: ii / jj / kk int64 and active uint8, one entry per slot
static void edge_store(const Args& arg, const Tensor& ii, const Tensor& jj, const Tensor& kk, const Tensor& active) {
  arg.need(ii, "ii", at::kLong); arg.need(jj, "jj", at::kLong, ii.numel()); arg.need(kk, "kk", at::kLong, ii.numel());
  arg.need(active, "active", at::kByte, ii.numel());
}
void pgraph_remove(Tensor ii, Tensor jj, Tensor kk, Tensor active, int64_t rule, Tensor frame, int64_t param, c10::optional<Tensor> enable,
                   int64_t dummy_frame, int64_t dummy_patch, int64_t M, Tensor n_active) {
  const Args arg("dpvo_b200_ext.pgraph_remove", ii, "ii");
  c10::cuda::CUDAGuard guard(arg.dev);
  edge_store(arg, ii, jj, kk, active);
  arg.need(frame, "frame", at::kLong, 1); arg.need(n_active, "n_active", at::kInt, 1);
  Tensor e = arg.need(enable, "enable", at::kInt, 1);
  const int32_t* en = e.defined() ? e.data_ptr<int>() : nullptr;
  check(dpvo_pgraph_remove(ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), kk.data_ptr<int64_t>(), active.data_ptr<uint8_t>(), ii.numel(), (int)rule,
                           frame.data_ptr<int64_t>(), param, en, dummy_frame, dummy_patch, (int)M, n_active.data_ptr<int>(), stream()),
        "dpvo_b200_ext.pgraph_remove");
}
Tensor pgraph_append(Tensor ii, Tensor jj, Tensor kk, Tensor active, Tensor new_ii, Tensor new_jj, Tensor new_kk, c10::optional<Tensor> enable,
                     c10::optional<Tensor> state, Tensor n_active, Tensor overflow) {
  const Args arg("dpvo_b200_ext.pgraph_append", ii, "ii");
  c10::cuda::CUDAGuard guard(arg.dev);
  edge_store(arg, ii, jj, kk, active);
  new_ii = arg.as(new_ii, "new_ii", at::kLong); new_jj = arg.as(new_jj, "new_jj", at::kLong); new_kk = arg.as(new_kk, "new_kk", at::kLong);
  arg.need(n_active, "n_active", at::kInt, 1); arg.need(overflow, "overflow", at::kInt, 1);
  Tensor e = arg.need(enable, "enable", at::kInt, 1), s = arg.need(state, "state [cap, 384]", at::kFloat, ii.numel() * 384);
  const int64_t n_new = new_ii.numel();
  TORCH_CHECK(new_jj.numel() == n_new && new_kk.numel() == n_new, "pgraph_append: new edge lists differ in length");
  const int32_t* en = e.defined() ? e.data_ptr<int>() : nullptr;
  float* st = s.defined() ? s.data_ptr<float>() : nullptr;
  Tensor slots = torch::empty({n_new}, ii.options().dtype(at::kInt));
  check(dpvo_pgraph_append(ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), kk.data_ptr<int64_t>(), active.data_ptr<uint8_t>(), ii.numel(),
                           new_ii.data_ptr<int64_t>(), new_jj.data_ptr<int64_t>(), new_kk.data_ptr<int64_t>(), n_new, en, st, slots.data_ptr<int>(),
                           n_active.data_ptr<int>(), overflow.data_ptr<int>(), stream()),
        "dpvo_b200_ext.pgraph_append");
  return slots;
}
std::vector<Tensor> pgraph_new_edges(Tensor n_dev, int64_t M, int64_t r) {
  const Args arg("dpvo_b200_ext.pgraph_new_edges", n_dev, "n");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.need(n_dev, "n", at::kLong, 1);
  const int64_t total = M * (2 * r - 1);
  Tensor ii = torch::empty({total}, n_dev.options()), jj = torch::empty({total}, n_dev.options()), kk = torch::empty({total}, n_dev.options());
  check(dpvo_pgraph_new_edges(n_dev.data_ptr<int64_t>(), (int)M, (int)r, ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), kk.data_ptr<int64_t>(), stream()),
        "dpvo_b200_ext.pgraph_new_edges");
  return {ii, jj, kk};
}

// ---- proximity loop closure (include/dpvo_b200.h, csrc/loop.cu)
Tensor loop_scores(Tensor poses, Tensor patches, Tensor intrinsics, Tensor n_dev, Tensor last_ba, int64_t M, int64_t removal,
                   int64_t max_age, int64_t freq, int64_t kf_index) {
  const Args arg("dpvo_b200_ext.loop_scores", poses, "poses");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.need(poses, "poses", at::kFloat); arg.need(patches, "patches", at::kFloat); arg.need(intrinsics, "intrinsics", at::kFloat);
  arg.need(n_dev, "n", at::kLong, 1); arg.need(last_ba, "last_global_ba", at::kLong, 1);
  TORCH_CHECK(patches.numel() % 27 == 0 && patches.size(-1) == 3, "loop_scores: patches are [K, 3, 3, 3]");
  const int64_t S = dpvo_loop_candidates((int)max_age, (int)freq, (int)kf_index);
  Tensor scores = torch::empty({std::max<int64_t>(S, 1)}, poses.options());
  check(dpvo_loop_scores(poses.data_ptr<float>(), patches.data_ptr<float>(), intrinsics.data_ptr<float>(), n_dev.data_ptr<int64_t>(),
                         last_ba.data_ptr<int64_t>(), (int)M, (int)removal, (int)max_age, (int)freq, (int)kf_index, scores.data_ptr<float>(),
                         stream()),
        "dpvo_b200_ext.loop_scores");
  return scores;
}
void loop_select(Tensor scores, Tensor n_dev, Tensor last_ba, int64_t M, int64_t removal, int64_t max_age, int64_t freq, int64_t kf_index,
                 double thresh, Tensor pairs, Tensor n_pairs, Tensor ii, Tensor jj, Tensor kk, Tensor active, c10::optional<Tensor> state,
                 Tensor n_active, Tensor overflow) {
  const Args arg("dpvo_b200_ext.loop_select", scores, "scores");
  c10::cuda::CUDAGuard guard(arg.dev);
  const int64_t S = dpvo_loop_candidates((int)max_age, (int)freq, (int)kf_index);
  arg.need(scores, "scores (the [J * max_age] output of loop_scores)", at::kFloat, S);
  arg.need(n_dev, "n", at::kLong, 1); arg.need(last_ba, "last_global_ba", at::kLong, 1); arg.need(n_pairs, "n_pairs", at::kInt, 1);
  arg.need(n_active, "n_active", at::kInt, 1); arg.need(overflow, "overflow", at::kInt, 1);
  arg.need(pairs, "pairs", at::kLong);
  TORCH_CHECK(pairs.dim() == 2 && pairs.size(1) == 2, "loop_select: pairs is a device int64 [max_pairs, 2]");
  edge_store(arg, ii, jj, kk, active);
  Tensor s = arg.need(state, "state (the [region, 384] recurrent state of the loop region)", at::kFloat, ii.numel() * 384);
  float* st = s.defined() ? s.data_ptr<float>() : nullptr;
  check(dpvo_loop_select(scores.data_ptr<float>(), n_dev.data_ptr<int64_t>(), last_ba.data_ptr<int64_t>(), (int)M, (int)removal, (int)max_age,
                         (int)freq, (int)kf_index, (float)thresh, (int)pairs.size(0), pairs.data_ptr<int64_t>(), n_pairs.data_ptr<int>(),
                         ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), kk.data_ptr<int64_t>(), active.data_ptr<uint8_t>(), ii.numel(), st,
                         n_active.data_ptr<int>(), overflow.data_ptr<int>(), stream()),
        "dpvo_b200_ext.loop_select");
}
void pgraph_remove_store(Tensor ii, Tensor jj, Tensor kk, Tensor active, Tensor target, Tensor weight, Tensor n_dev, int64_t removal,
                         int64_t opt_window, c10::optional<Tensor> enable, int64_t dummy_frame, int64_t dummy_patch, int64_t M, Tensor n_active,
                         Tensor s_ii, Tensor s_jj, Tensor s_kk, Tensor s_target, Tensor s_weight, Tensor s_count, Tensor s_overflow) {
  const Args arg("dpvo_b200_ext.pgraph_remove_store", ii, "ii");
  c10::cuda::CUDAGuard guard(arg.dev);
  edge_store(arg, ii, jj, kk, active);
  const int64_t cap = ii.numel(), sc = s_ii.numel();
  arg.need(target, "target [cap, 2]", at::kFloat, cap * 2); arg.need(weight, "weight [cap, 2]", at::kFloat, cap * 2);
  arg.need(s_ii, "s_ii", at::kLong); arg.need(s_jj, "s_jj", at::kLong, sc); arg.need(s_kk, "s_kk", at::kLong, sc);
  arg.need(s_target, "s_target [store, 2]", at::kFloat, sc * 2); arg.need(s_weight, "s_weight [store, 2]", at::kFloat, sc * 2);
  arg.need(n_dev, "n", at::kLong, 1); arg.need(n_active, "n_active", at::kInt, 1);
  arg.need(s_count, "s_count", at::kInt, 1); arg.need(s_overflow, "s_overflow", at::kInt, 1);
  Tensor e = arg.need(enable, "enable", at::kInt, 1);
  const int32_t* en = e.defined() ? e.data_ptr<int>() : nullptr;
  check(dpvo_pgraph_remove_store(ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), kk.data_ptr<int64_t>(), active.data_ptr<uint8_t>(),
                                 target.data_ptr<float>(), weight.data_ptr<float>(), cap, n_dev.data_ptr<int64_t>(), (int)removal, (int)opt_window,
                                 en, dummy_frame, dummy_patch, (int)M, n_active.data_ptr<int>(), s_ii.data_ptr<int64_t>(), s_jj.data_ptr<int64_t>(),
                                 s_kk.data_ptr<int64_t>(), s_target.data_ptr<float>(), s_weight.data_ptr<float>(), sc, s_count.data_ptr<int>(),
                                 s_overflow.data_ptr<int>(), stream()),
        "dpvo_b200_ext.pgraph_remove_store");
}
void loop_flags(Tensor ii, Tensor active, int64_t normal, int64_t n, int64_t removal, c10::optional<Tensor> s_count, Tensor flags) {
  const Args arg("dpvo_b200_ext.loop_flags", ii, "ii");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.need(ii, "ii", at::kLong); arg.need(active, "active", at::kByte, ii.numel()); arg.need(flags, "flags", at::kLong, 4);
  Tensor c = arg.need(s_count, "s_count", at::kInt, 1);
  const int32_t* sc = c.defined() ? c.data_ptr<int>() : nullptr;
  check(dpvo_loop_flags(ii.data_ptr<int64_t>(), active.data_ptr<uint8_t>(), ii.numel(), normal, n, (int)removal, sc, flags.data_ptr<int64_t>(), stream()),
        "dpvo_b200_ext.loop_flags");
}
void loop_normalize(Tensor poses, Tensor patches, int64_t n, int64_t M, c10::optional<Tensor> delta) {
  const Args arg("dpvo_b200_ext.loop_normalize", poses, "poses");
  c10::cuda::CUDAGuard guard(arg.dev);
  arg.need(poses, "poses", at::kFloat); arg.need(patches, "patches", at::kFloat);
  Tensor d = arg.need(delta, "delta", at::kFloat);
  TORCH_CHECK(patches.dim() >= 3 && patches.size(-3) == 3, "loop_normalize: poses [N, 7] and patches [K, 3, P, P]");
  const int64_t P = patches.size(-1);
  TORCH_CHECK(n >= 0 && poses.numel() >= 7 * n && patches.numel() >= n * M * 3 * P * P, "loop_normalize: n = ", n, " frames exceed the buffers");
  if (!d.defined()) {
    check(dpvo_loop_normalize(poses.data_ptr<float>(), patches.data_ptr<float>(), n, (int)M, (int)P, stream()), "dpvo_b200_ext.loop_normalize");
    return;
  }
  TORCH_CHECK(d.numel() % 7 == 0, "loop_normalize: delta is a [T, 7] table of relative poses");
  check(dpvo_loop_normalize_deltas(poses.data_ptr<float>(), patches.data_ptr<float>(), n, (int)M, (int)P, d.data_ptr<float>(),
                                   d.numel() / 7, stream()),
        "dpvo_b200_ext.loop_normalize");
}

// ---- keyframe culling (include/dpvo_b200.h, csrc/keyframe.cu)
void keyframe_motion(Tensor poses, Tensor patches, Tensor intrinsics, int64_t F, Tensor ii, Tensor jj, Tensor kk, Tensor active,
                     Tensor n, Tensor tstamp, Tensor delta, Tensor delta_src, int64_t ki, double thresh, Tensor flag, Tensor k, Tensor m,
                     Tensor overflow) {
  const Args arg("dpvo_b200_ext.keyframe_motion", poses, "poses");
  c10::cuda::CUDAGuard guard(arg.dev);
  const int64_t B = n.numel();
  TORCH_CHECK(B >= 1 && F >= 2, "keyframe_motion: one frame count per stream and at least 2 frame slots");
  arg.need(poses, "poses [B F, 7]", at::kFloat, B * F * 7); arg.need(intrinsics, "intrinsics [B F, 4]", at::kFloat, B * F * 4);
  arg.need(patches, "patches", at::kFloat);
  TORCH_CHECK(patches.numel() % (B * F * 27) == 0 && patches.size(-1) == 3, "keyframe_motion: patches are [B F M, 3, 3, 3]");
  edge_store(arg, ii, jj, kk, active);
  TORCH_CHECK(ii.numel() % B == 0, "keyframe_motion: the edge store holds one slice of slots per stream");
  arg.need(n, "n", at::kLong); arg.need(tstamp, "tstamp [B, F]", at::kLong, B * F);
  arg.need(delta_src, "delta_src", at::kLong);
  TORCH_CHECK(delta_src.numel() % B == 0, "keyframe_motion: delta_src is [B, T]");
  const int64_t T = delta_src.numel() / B;
  arg.need(delta, "delta [B, T, 7]", at::kFloat, B * T * 7);
  arg.need(flag, "flag", at::kInt, B); arg.need(overflow, "overflow", at::kInt, B); arg.need(k, "k", at::kLong, B);
  arg.need(m, "m", at::kDouble, B);
  const int64_t wsb = dpvo_keyframe_motion_workspace_bytes((int)B);
  Tensor ws = torch::empty({wsb}, poses.options().dtype(at::kByte));
  check(dpvo_keyframe_motion(poses.data_ptr<float>(), patches.data_ptr<float>(), intrinsics.data_ptr<float>(), F, (int)B,
                             ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), kk.data_ptr<int64_t>(), active.data_ptr<uint8_t>(), ii.numel() / B,
                             n.data_ptr<int64_t>(), tstamp.data_ptr<int64_t>(), delta.data_ptr<float>(), delta_src.data_ptr<int64_t>(), T, (int)ki,
                             thresh, flag.data_ptr<int>(), k.data_ptr<int64_t>(), m.data_ptr<double>(), overflow.data_ptr<int>(), ws.data_ptr(),
                             wsb, stream()),
        "dpvo_b200_ext.keyframe_motion");
}
// each buffer is a dense tensor whose outermost dimension in memory holds B * rows slots of equal size, in order
void keyframe_shift(std::vector<Tensor> bufs, std::vector<int64_t> rows, int64_t F, int64_t ki, Tensor flag, Tensor k) {
  const Args arg("dpvo_b200_ext.keyframe_shift", flag, "flag");
  c10::cuda::CUDAGuard guard(arg.dev);
  const int64_t B = flag.numel();
  arg.need(flag, "flag", at::kInt); arg.need(k, "k", at::kLong, B);
  for (const Tensor& t : bufs) arg.on(t, "every buffer");
  TORCH_CHECK(B >= 1, "keyframe_shift: flag is a device int32 [B]");
  TORCH_CHECK(bufs.size() == rows.size(), "keyframe_shift: one slot count per buffer");
  std::vector<void*> bases;
  std::vector<int64_t> rb, rw;
  for (size_t q = 0; q < bufs.size(); ++q) {
    const Tensor& t = bufs[q];
    TORCH_CHECK(t.numel() > 0 && t.is_non_overlapping_and_dense(), "keyframe_shift: buffer ", q, " must be a dense CUDA tensor");
    // dense: the memory order is row-major over the dimensions sorted by stride, so the slots are contiguous blocks
    // when the leading dimensions of that order hold a multiple of B * rows blocks
    std::vector<int> dims;
    for (int i = 0; i < t.dim(); ++i) if (t.size(i) > 1) dims.push_back(i);
    std::stable_sort(dims.begin(), dims.end(), [&](int a, int b) { return t.stride(a) > t.stride(b); });
    bool ok = false;
    int64_t lead = 1;
    for (int d : dims) { lead *= t.size(d); if (rows[q] > 0 && lead % (B * rows[q]) == 0) { ok = true; break; } }
    TORCH_CHECK(ok, "keyframe_shift: buffer ", q, " does not hold ", B, " x ", rows[q], " slots in its leading dimensions");
    bases.push_back(t.data_ptr());
    rb.push_back(t.numel() * (int64_t)t.element_size() / (B * rows[q]));
    rw.push_back(rows[q]);
  }
  check(dpvo_keyframe_shift_bytes(bases.data(), rb.data(), rw.data(), (int)bases.size(), F, (int)B, (int)ki, flag.data_ptr<int>(),
                                  k.data_ptr<int64_t>(), stream()),
        "dpvo_b200_ext.keyframe_shift");
}
void keyframe_count(int64_t mode, Tensor n, Tensor tstamp, int64_t F, Tensor counter, Tensor delta, Tensor delta_src, Tensor overflow) {
  const Args arg("dpvo_b200_ext.keyframe_count", counter, "counter");
  c10::cuda::CUDAGuard guard(arg.dev);
  const int64_t B = counter.numel();
  arg.need(counter, "counter", at::kLong); arg.need(n, "n", at::kLong, B); arg.need(tstamp, "tstamp [B, F]", at::kLong, B * F);
  arg.need(delta_src, "delta_src", at::kLong);
  TORCH_CHECK(delta_src.numel() % B == 0, "keyframe_count: delta_src is [B, T]");
  const int64_t T = delta_src.numel() / B;
  arg.need(delta, "delta [B, T, 7]", at::kFloat, B * T * 7); arg.need(overflow, "overflow", at::kInt, B);
  check(dpvo_keyframe_count((int)mode, n.data_ptr<int64_t>(), tstamp.data_ptr<int64_t>(), F, (int)B, counter.data_ptr<int64_t>(),
                            delta.data_ptr<float>(), delta_src.data_ptr<int64_t>(), T, overflow.data_ptr<int>(), stream()),
        "dpvo_b200_ext.keyframe_count");
}
Tensor keyframe_trajectory(Tensor poses, Tensor tstamp, Tensor n, int64_t F, Tensor delta, Tensor delta_src, Tensor counter, Tensor error) {
  const Args arg("dpvo_b200_ext.keyframe_trajectory", poses, "poses");
  c10::cuda::CUDAGuard guard(arg.dev);
  const int64_t B = n.numel();
  arg.need(n, "n", at::kLong); arg.need(poses, "poses [B F, 7]", at::kFloat, B * F * 7);
  arg.need(tstamp, "tstamp [B, F]", at::kLong, B * F); arg.need(counter, "counter", at::kLong, B);
  arg.need(delta_src, "delta_src", at::kLong);
  TORCH_CHECK(delta_src.numel() % B == 0, "keyframe_trajectory: delta_src is [B, T]");
  const int64_t T = delta_src.numel() / B;
  arg.need(delta, "delta [B, T, 7]", at::kFloat, B * T * 7); arg.need(error, "error", at::kInt, B);
  Tensor map = torch::empty({B, T}, poses.options().dtype(at::kInt));
  Tensor out = torch::empty({B, T, 7}, poses.options());
  check(dpvo_keyframe_trajectory(poses.data_ptr<float>(), tstamp.data_ptr<int64_t>(), n.data_ptr<int64_t>(), F, (int)B, delta.data_ptr<float>(),
                                 delta_src.data_ptr<int64_t>(), T, counter.data_ptr<int64_t>(), map.data_ptr<int>(), out.data_ptr<float>(),
                                 error.data_ptr<int>(), stream()),
        "dpvo_b200_ext.keyframe_trajectory");
  return out;
}

// ------------------------------------------------------------------------------ frame encoders
struct EncShape { int ks, s, cin, cout; };
const EncShape kEncShapes[] = {{7, 2, 3, 32}, {3, 1, 32, 32}, {3, 2, 32, 64}, {1, 2, 32, 64}, {3, 1, 64, 64}, {1, 1, 64, 128}, {1, 1, 64, 384}};

// one layer of one encoder; returns (y [Ho, Wo, cout], stats [2, cout] or None, joined [H, W, cin] or None, pool or None)
std::vector<c10::optional<Tensor>> encoder_conv(int64_t shape, Tensor x, Tensor w, Tensor bias, c10::optional<Tensor> x_stats, bool x_relu,
                                                c10::optional<Tensor> skip, c10::optional<Tensor> skip_stats, bool skip_relu,
                                                bool want_joined, bool want_stats, bool want_pool, double scale) {
  TORCH_CHECK(shape >= 0 && shape < 7, "encoder_conv: unknown shape ", shape);
  const EncShape sh = kEncShapes[shape];
  const bool stem = shape == DPVO_ENC_STEM;
  const Args arg("dpvo_b200_ext.encoder_conv", x, "x");
  const c10::cuda::CUDAGuard guard(arg.dev);
  int H, W;
  dpvo_encoder_conv_io io{};
  if (stem) {
    arg.on(x, "x (the stem's image)", at::kByte);
    TORCH_CHECK(x.dim() == 3 && x.size(0) == 3, "encoder_conv: the stem takes a uint8 image [3, H, W]");
    H = (int)x.size(1); W = (int)x.size(2);
    io.x_strides[0] = x.stride(0); io.x_strides[1] = x.stride(1); io.x_strides[2] = x.stride(2);
  } else {
    arg.need(x, "x", at::kHalf);
    TORCH_CHECK(x.dim() == 3 && x.size(2) == sh.cin, "encoder_conv: x must be NHWC [H, W, ", sh.cin, "]");
    H = (int)x.size(0); W = (int)x.size(1);
  }
  const int Ho = (H + 2 * (sh.ks / 2) - sh.ks) / sh.s + 1, Wo = (W + 2 * (sh.ks / 2) - sh.ks) / sh.s + 1;
  arg.need(w, "w", at::kHalf);
  const int64_t taps = stem ? 1 : sh.ks * sh.ks, kc = stem ? 20 : sh.cin / 8;
  TORCH_CHECK(w.numel() == taps * kc * sh.cout * 8, "encoder_conv: w must hold the packed layer (", taps * kc * sh.cout * 8, " halves)");
  arg.need(bias, "bias", at::kFloat, sh.cout);
  Tensor xs = arg.need(x_stats, "x_stats", at::kFloat, 2 * sh.cin), sk = arg.need(skip, "skip", at::kHalf);
  Tensor ss = arg.need(skip_stats, "skip_stats", at::kFloat, 2 * sh.cin);
  if (sk.defined()) TORCH_CHECK(sk.sizes() == x.sizes(), "encoder_conv: skip must match x");
  auto opt16 = x.options().dtype(at::kHalf);
  Tensor y = torch::empty({Ho, Wo, sh.cout}, opt16);
  c10::optional<Tensor> st, jn, pl;
  if (want_stats) st = torch::empty({2, sh.cout}, x.options().dtype(at::kFloat));
  if (want_joined) jn = torch::empty({H, W, sh.cin}, opt16);
  if (want_pool) pl = torch::empty({Ho / 4, Wo / 4, sh.cout}, opt16);
  io.x = x.data_ptr(); io.x_stats = xs.defined() ? xs.data_ptr<float>() : nullptr; io.x_relu = x_relu;
  io.skip = sk.defined() ? sk.data_ptr() : nullptr; io.skip_stats = ss.defined() ? ss.data_ptr<float>() : nullptr; io.skip_relu = skip_relu;
  io.joined = jn ? jn->data_ptr() : nullptr;
  io.w = w.data_ptr(); io.bias = bias.data_ptr<float>();
  io.y = y.data_ptr(); io.y_sy = (int64_t)Wo * sh.cout; io.y_sx = sh.cout;
  io.pool = pl ? pl->data_ptr() : nullptr; io.pool_sy = (int64_t)(Wo / 4) * sh.cout; io.pool_sx = sh.cout;
  io.stats = st ? st->data_ptr<float>() : nullptr; io.scale = (float)scale;
  const int64_t wsb = dpvo_encoder_conv_workspace_bytes((int)shape, H, W);
  Tensor ws = byte_ws(wsb, x);
  check(dpvo_encoder_conv((int)shape, H, W, 1, &io, ws.data_ptr(), wsb, stream()), "dpvo_b200_ext.encoder_conv");
  return {y, st, jn, pl};
}

// the tensors both encode entry points take (images and rings, or one image and its slots); returns the colors or an
// undefined tensor
Tensor encode_args(const Args& arg, const Tensor& image, const Tensor& w16, const Tensor& b32, const Tensor& coords, const Tensor& fmap1,
                   const Tensor& fmap2, const Tensor& gmap, const Tensor& imap, const Tensor& patches, const Tensor& workspace,
                   const c10::optional<Tensor>& colors) {
  arg.on(image, "image", at::kByte); arg.need(w16, "w16", at::kHalf); arg.need(b32, "b32 [2, 11, 384]", at::kFloat, 2 * 11 * 384);
  arg.need(coords, "coords", at::kFloat); arg.on(fmap1, "fmap1", at::kHalf); arg.on(fmap2, "fmap2", at::kHalf);
  arg.on(gmap, "gmap", at::kHalf); arg.on(imap, "imap", at::kHalf); arg.need(patches, "patches", at::kFloat);
  arg.need(workspace, "workspace");
  return arg.need(colors, "colors", at::kByte);
}

// the viewer colours of the patch rows: rows x 3 bytes ([M, 3], or [F, M, 3])
uint8_t* color_rows(const Tensor& c, int64_t rows, const char* op) {
  if (!c.defined()) return nullptr;
  TORCH_CHECK(c.dim() >= 2 && c.size(-1) == 3 && c.numel() == rows * 3, op, ": colors must be ", rows, " rows of 3 bytes");
  return c.data_ptr<uint8_t>();
}

void encode_frame(Tensor image, Tensor w16, Tensor b32, Tensor coords, Tensor fmap1, Tensor fmap2, Tensor gmap, Tensor imap,
                  Tensor patches, Tensor workspace, c10::optional<Tensor> colors) {
  const Args arg("dpvo_b200_ext.encode_frame", image, "image");
  const c10::cuda::CUDAGuard guard(arg.dev);
  const Tensor clr = encode_args(arg, image, w16, b32, coords, fmap1, fmap2, gmap, imap, patches, workspace, colors);
  TORCH_CHECK(image.dim() == 3 && image.size(0) == 3, "encode_frame: image must be uint8 [3, H, W]");
  const int H = (int)image.size(1), W = (int)image.size(2);
  const int h = ((H - 1) / 2 + 1 - 1) / 2 + 1, w = ((W - 1) / 2 + 1 - 1) / 2 + 1;
  TORCH_CHECK(coords.dim() == 2 && coords.size(1) == 2, "encode_frame: coords must be contiguous float32 [M, 2]");
  const int64_t M = coords.size(0);
  TORCH_CHECK(fmap1.dim() == 3 && fmap1.size(2) == 128 && fmap1.stride(2) == 1, "encode_frame: fmap1 must be a channels-last float16 slot [h, w, 128]");
  TORCH_CHECK(fmap1.size(0) == h && fmap1.size(1) == w, "encode_frame: a ", H, "x", W, " image encodes to ", h, "x", w,
              ", the fmap1 slot is ", fmap1.size(0), "x", fmap1.size(1));
  TORCH_CHECK(fmap2.dim() == 3 && fmap2.size(0) == h / 4 && fmap2.size(1) == w / 4 && fmap2.size(2) == 128 && fmap2.stride(2) == 1,
              "encode_frame: fmap2 must be a channels-last float16 slot [h/4, w/4, 128]");
  TORCH_CHECK(gmap.dim() == 4 && gmap.size(0) == M && gmap.size(1) == 3 && gmap.size(2) == 3 && gmap.size(3) == 128 && gmap.stride(3) == 1,
              "encode_frame: gmap must be a channels-last float16 slot [M, 3, 3, 128]");
  TORCH_CHECK(imap.dim() == 2 && imap.size(0) == M && imap.size(1) == 384 && imap.stride(1) == 1, "encode_frame: imap must be float16 [M, 384] with contiguous rows");
  TORCH_CHECK(patches.numel() == M * 27, "encode_frame: patches must be contiguous float32 [M, 3, 3, 3]");
  if (clr.defined()) {
    uint8_t* cp = color_rows(clr, M, "encode_frame");
    const int64_t row0 = 0;
    check(dpvo_encode_frames_colors(image.data_ptr<uint8_t>(), 0, image.stride(0), image.stride(1), image.stride(2), 1, H, W,
                                    w16.data_ptr(), b32.data_ptr<float>(), coords.data_ptr<float>(), (int)M,
                                    fmap1.data_ptr(), 0, fmap1.stride(0), fmap1.stride(1), fmap2.data_ptr(), 0, fmap2.stride(0),
                                    fmap2.stride(1), 1, gmap.data_ptr(), gmap.stride(0), gmap.stride(1), gmap.stride(2), imap.data_ptr(),
                                    imap.stride(0), M, patches.data_ptr<float>(), M, &row0, &row0, &row0, nullptr, cp,
                                    workspace.data_ptr(), workspace.numel() * workspace.element_size(), stream()),
          "dpvo_b200_ext.encode_frame");
    return;
  }
  check(dpvo_encode_frame(image.data_ptr<uint8_t>(), image.stride(0), image.stride(1), image.stride(2), H, W, w16.data_ptr(), b32.data_ptr<float>(),
                          coords.data_ptr<float>(), (int)M, fmap1.data_ptr(), fmap1.stride(0), fmap1.stride(1), fmap2.data_ptr(), fmap2.stride(0),
                          fmap2.stride(1), gmap.data_ptr(), gmap.stride(0), gmap.stride(1), gmap.stride(2), imap.data_ptr(), imap.stride(0),
                          patches.data_ptr<float>(), workspace.data_ptr(), workspace.numel() * workspace.element_size(), stream()),
        "dpvo_b200_ext.encode_frame");
}

int64_t encode_frame_workspace_bytes(int64_t H, int64_t W) { return dpvo_encode_frame_workspace_bytes((int)H, (int)W); }

// B images [B, 3, H, W] (any strides) into rows of whole rings: fmap1 [R, h, w, 128], fmap2 [R, h/4, w/4, 128], gmap
// [Rg, 3, 3, 128] (channels-last), imap [Rg, 384], patches [Rp, 3, 3, 3]; image b into frame row frame_rows[b], patch-feature
// rows feat_rows[b] + [0, M) and patch rows patch_rows[b] + [0, M).  The library checks the rows.
void encode_frames(Tensor images, Tensor w16, Tensor b32, Tensor coords, Tensor fmap1, Tensor fmap2, Tensor gmap, Tensor imap,
                   Tensor patches, std::vector<int64_t> frame_rows, std::vector<int64_t> feat_rows, std::vector<int64_t> patch_rows,
                   c10::optional<Tensor> depth, Tensor workspace, c10::optional<Tensor> colors) {
  const Args arg("dpvo_b200_ext.encode_frames", images, "images");
  const c10::cuda::CUDAGuard guard(arg.dev);
  const Tensor clr = encode_args(arg, images, w16, b32, coords, fmap1, fmap2, gmap, imap, patches, workspace, colors);
  const Tensor dep = arg.need(depth, "depth", at::kFloat);
  TORCH_CHECK(images.dim() == 4 && images.size(1) == 3, "encode_frames: images must be uint8 [B, 3, H, W]");
  const int64_t B = images.size(0);
  const int H = (int)images.size(2), W = (int)images.size(3);
  const int h = ((H - 1) / 2 + 1 - 1) / 2 + 1, w = ((W - 1) / 2 + 1 - 1) / 2 + 1;
  TORCH_CHECK(coords.dim() == 3 && coords.size(0) == B && coords.size(2) == 2, "encode_frames: coords must be contiguous float32 [B, M, 2] with B = ", B);
  const int64_t M = coords.size(1);
  TORCH_CHECK(fmap1.dim() == 4 && fmap1.size(3) == 128 && fmap1.stride(3) == 1, "encode_frames: fmap1 must be a channels-last float16 ring [R, h, w, 128]");
  TORCH_CHECK(fmap1.size(1) == h && fmap1.size(2) == w, "encode_frames: a ", H, "x", W, " image encodes to ", h, "x", w,
              ", the fmap1 ring holds ", fmap1.size(1), "x", fmap1.size(2));
  TORCH_CHECK(fmap2.dim() == 4 && fmap2.size(0) == fmap1.size(0) && fmap2.size(1) == h / 4 && fmap2.size(2) == w / 4 && fmap2.size(3) == 128 &&
              fmap2.stride(3) == 1, "encode_frames: fmap2 must be a channels-last float16 ring [R, h/4, w/4, 128] with fmap1's R");
  TORCH_CHECK(gmap.dim() == 4 && gmap.size(1) == 3 && gmap.size(2) == 3 && gmap.size(3) == 128 && gmap.stride(3) == 1,
              "encode_frames: gmap must be a channels-last float16 ring [Rg, 3, 3, 128]");
  TORCH_CHECK(imap.dim() == 2 && imap.size(0) == gmap.size(0) && imap.size(1) == 384 && imap.stride(1) == 1,
              "encode_frames: imap must be float16 [Rg, 384] with contiguous rows and gmap's Rg");
  TORCH_CHECK(patches.dim() == 4 && patches.size(1) == 3 && patches.size(2) == 3 && patches.size(3) == 3,
              "encode_frames: patches must be contiguous float32 [Rp, 3, 3, 3]");
  TORCH_CHECK((int64_t)frame_rows.size() == B && (int64_t)feat_rows.size() == B && (int64_t)patch_rows.size() == B,
              "encode_frames: one frame row, one patch-feature row and one patch row per image (", B, " images)");
  if (dep.defined()) TORCH_CHECK(dep.dim() == 2 && dep.size(0) == B && dep.size(1) == M, "encode_frames: depth must be float32 [B, M]");
  const float* dp = dep.defined() ? dep.data_ptr<float>() : nullptr;
  if (clr.defined()) {
    uint8_t* cp = color_rows(clr, patches.size(0), "encode_frames");
    check(dpvo_encode_frames_colors(images.data_ptr<uint8_t>(), images.stride(0), images.stride(1), images.stride(2), images.stride(3),
                                    (int)B, H, W, w16.data_ptr(), b32.data_ptr<float>(), coords.data_ptr<float>(), (int)M,
                                    fmap1.data_ptr(), fmap1.stride(0), fmap1.stride(1), fmap1.stride(2),
                                    fmap2.data_ptr(), fmap2.stride(0), fmap2.stride(1), fmap2.stride(2), fmap1.size(0),
                                    gmap.data_ptr(), gmap.stride(0), gmap.stride(1), gmap.stride(2), imap.data_ptr(), imap.stride(0),
                                    gmap.size(0), patches.data_ptr<float>(), patches.size(0), frame_rows.data(), feat_rows.data(),
                                    patch_rows.data(), dp, cp, workspace.data_ptr(), workspace.numel() * workspace.element_size(), stream()),
          "dpvo_b200_ext.encode_frames");
    return;
  }
  check(dpvo_encode_frames(images.data_ptr<uint8_t>(), images.stride(0), images.stride(1), images.stride(2), images.stride(3), (int)B, H, W,
                           w16.data_ptr(), b32.data_ptr<float>(), coords.data_ptr<float>(), (int)M,
                           fmap1.data_ptr(), fmap1.stride(0), fmap1.stride(1), fmap1.stride(2),
                           fmap2.data_ptr(), fmap2.stride(0), fmap2.stride(1), fmap2.stride(2), fmap1.size(0),
                           gmap.data_ptr(), gmap.stride(0), gmap.stride(1), gmap.stride(2), imap.data_ptr(), imap.stride(0), gmap.size(0),
                           patches.data_ptr<float>(), patches.size(0), frame_rows.data(), feat_rows.data(), patch_rows.data(), dp,
                           workspace.data_ptr(), workspace.numel() * workspace.element_size(), stream()),
        "dpvo_b200_ext.encode_frames");
}

int64_t encode_frames_workspace_bytes(int64_t B, int64_t H, int64_t W) {
  return dpvo_encode_frames_workspace_bytes((int)B, (int)H, (int)W);
}

// ------------------------------------------------------------------------------ camera-image preparation
// images uint8 [B, 3, H, W] (any strides) -> the window rows [y0, y0 + Ho) x columns [x0, x0 + Wo) of each undistorted
// (and, with half, halved) image, into out uint8 [B, Ho, Wo, 3] (any strides).  cameras: B rows of 9 float64 values
// (fx fy cx cy k1 k2 p1 p2 k3), passed by value.  The library checks the values and the window.
void undistort_frames(Tensor images, std::vector<double> cameras, bool half, int64_t y0, int64_t x0, Tensor out) {
  const Args arg("dpvo_b200_ext.undistort_frames", images, "images");
  const c10::cuda::CUDAGuard guard(arg.dev);
  arg.on(images, "images", at::kByte); arg.on(out, "out", at::kByte);
  TORCH_CHECK(images.dim() == 4 && images.size(1) == 3, "undistort_frames: images must be uint8 [B, 3, H, W]");
  const int64_t B = images.size(0);
  TORCH_CHECK(out.dim() == 4 && out.size(0) == B && out.size(3) == 3, "undistort_frames: out must be uint8 [B, Ho, Wo, 3] with B = ", B);
  TORCH_CHECK((int64_t)cameras.size() == 9 * B, "undistort_frames: 9 camera values (fx fy cx cy k1 k2 p1 p2 k3) per image, ", B,
              " images, ", cameras.size(), " values");
  TORCH_CHECK(images.size(2) <= INT32_MAX && images.size(3) <= INT32_MAX && out.size(1) <= INT32_MAX && out.size(2) <= INT32_MAX &&
              y0 >= INT32_MIN && y0 <= INT32_MAX && x0 >= INT32_MIN && x0 <= INT32_MAX, "undistort_frames: sizes beyond 32-bit");
  std::vector<dpvo_camera> cams((size_t)B);
  for (int64_t b = 0; b < B; ++b) {
    const double* c = cameras.data() + 9 * b;
    cams[b] = dpvo_camera{c[0], c[1], c[2], c[3], c[4], c[5], c[6], c[7], c[8]};
  }
  check(dpvo_undistort_frames(images.data_ptr<uint8_t>(), images.stride(0), images.stride(1), images.stride(2), images.stride(3), (int)B,
                              (int)images.size(2), (int)images.size(3), cams.data(), half ? 1 : 0, (int)y0, (int)x0, (int)out.size(1),
                              (int)out.size(2), out.data_ptr<uint8_t>(), out.stride(0), out.stride(1), out.stride(2), out.stride(3), stream()),
        "dpvo_b200_ext.undistort_frames");
}

// ------------------------------------------------------------------------------ map
// points [B F M, 3] rows [b F M, b F M + n[b] M) of every stream b = 0 .. len(n) - 1, from poses [B F, 7], patches
// [B F M, 3, 3, 3] and intrinsics [B F, 4]
void point_cloud(Tensor poses, Tensor patches, Tensor intrinsics, int64_t F, std::vector<int64_t> n, Tensor points) {
  const Args arg("dpvo_b200_ext.point_cloud", poses, "poses");
  c10::cuda::CUDAGuard guard(arg.dev);
  const int64_t B = (int64_t)n.size();
  TORCH_CHECK(B >= 1 && F >= 1, "point_cloud: one frame count per stream and F >= 1 needed");
  arg.need(poses, "poses [B F, 7]", at::kFloat, B * F * 7); arg.need(intrinsics, "intrinsics [B F, 4]", at::kFloat, B * F * 4);
  arg.need(patches, "patches", at::kFloat);
  TORCH_CHECK(patches.numel() % (B * F * 27) == 0 && patches.numel() > 0, "point_cloud: patches are [B F M, 3, 3, 3]");
  const int64_t M = patches.numel() / (B * F * 27);
  arg.need(points, "points [B F M, 3]", at::kFloat, B * F * M * 3);
  check(dpvo_point_cloud(poses.data_ptr<float>(), patches.data_ptr<float>(), intrinsics.data_ptr<float>(), F, (int)M, (int)B, n.data(),
                         points.data_ptr<float>(), stream()),
        "dpvo_b200_ext.point_cloud");
}

int64_t launch_count() { return dpvo_launch_count(); }
std::string version() { return dpvo_version(); }

}  // namespace

PYBIND11_MODULE(cuda_corr, m) {
  m.def("forward", &corr_forward, "CORR forward");
  m.def("backward", &corr_backward, "CORR backward");
  m.def("patchify_forward", &patchify_forward, "PATCHIFY forward");
  m.def("patchify_backward", &patchify_backward, "PATCHIFY backward");
}

PYBIND11_MODULE(cuda_ba, m) {
  m.def("forward", &ba_forward, "BA forward operator");
  m.def("neighbors", &ba_neighbors, "temporal neighbor indices");
  m.def("reproject", &ba_reproject, "fused reprojection");
  m.def("solve_system", &ba_solve_system, "pose-graph normal equations + solve (loop closure back end)");
}

PYBIND11_MODULE(lietorch_backends, m) {
  m.def("expm", &l_expm, "exp map forward");
  m.def("expm_backward", &l_expm_b, "exp map backward");
  m.def("logm", &l_logm, "log map forward");
  m.def("logm_backward", &l_logm_b, "log map backward");
  m.def("inv", &l_inv, "inverse operator");
  m.def("inv_backward", &l_inv_b, "inverse operator backward");
  m.def("mul", &l_mul, "group operator");
  m.def("mul_backward", &l_mul_b, "group operator backward");
  m.def("adj", &l_adj, "adjoint operator");
  m.def("adj_backward", &l_adj_b, "adjoint operator backward");
  m.def("adjT", &l_adjT, "transposed adjoint operator");
  m.def("adjT_backward", &l_adjT_b, "transposed adjoint operator backward");
  m.def("act", &l_act, "action on point");
  m.def("act_backward", &l_act_b, "action on point backward");
  m.def("act4", &l_act4, "action on homogeneous point");
  m.def("act4_backward", &l_act4_b, "action on homogeneous point backward");
  m.def("as_matrix", &l_as_matrix, "convert to matrix");
  m.def("projector", &l_projector, "orthogonal projection matrix");
  m.def("Jinv", &l_jinv, "left inverse jacobian operator");
}

PYBIND11_MODULE(dpvo_b200_ext, m) {
  m.def("corr_pyramid2", &corr_pyramid2, "two-level fused correlation", py::arg("fmap1"), py::arg("fmap2_l0"), py::arg("fmap2_l1"),
        py::arg("coords"), py::arg("ii"), py::arg("jj"), py::arg("radius"), py::arg("div"), py::arg("pad_to") = 0, py::arg("out") = py::none());
  m.def("group_edges_pair", &group_edges_pair, "two device edge groupings in one launch", py::arg("key_a0"), py::arg("key_b0"), py::arg("sec0"),
        py::arg("key_a1"), py::arg("key_b1"), py::arg("sec1"));
  m.def("group_edges", &group_edges, "device edge grouping", py::arg("key_a"), py::arg("key_b") = py::none(),
        py::arg("sec") = py::none());
  m.def("ba_forward_grouped", &ba_forward_grouped, "fastba.BA on prebuilt edge groupings");
  m.def("ba_forward_batched", &ba_forward_batched, "fastba.BA over B streams' windows on prebuilt edge groupings");
  m.def("ba_batched_workspace_bytes", &ba_batched_workspace_bytes, "scratch bytes of ba_forward_batched (current device)",
        py::arg("E"), py::arg("B"), py::arg("max_free_poses"));
  m.def("reproject_clamped", &reproject_clamped, "pops.transform-compatible fused reprojection");
  m.def("add_layernorm", &add_layernorm, "fused add + LayerNorm (+ReLU)", py::arg("a"), py::arg("b"), py::arg("c"), py::arg("gamma"),
        py::arg("beta"), py::arg("eps"), py::arg("relu"), py::arg("want32"), py::arg("want16"), py::arg("b_index") = py::none(), py::arg("inplace32") = false, py::arg("c_scale") = py::none());
  m.def("gather_rows_masked", &gather_rows_masked, "masked row gather");
  m.def("residual_add_", &residual_add_, "in-place residual add with optional row indirection");
  m.def("residual_sum16", &residual_sum16, "fp16(net + u[group]) without updating net", py::arg("net32"), py::arg("u"), py::arg("group_of") = py::none());
  m.def("gated_residual", &gated_residual, "x + sigmoid(g) * r");
  m.def("softagg_reduce", &softagg_reduce, "segment softmax-weighted sum");
  m.def("softagg_fused", &softagg_fused, "SoftAgg f|g layer fused with its segment softmax-weighted sum", py::arg("x"), py::arg("order"),
        py::arg("group_of"), py::arg("group_start"), py::arg("n_groups"), py::arg("max_groups"), py::arg("w"), py::arg("bias"),
        py::arg("workspace") = py::none());
  m.def("softagg_fused_workspace_bytes", &softagg_fused_workspace_bytes, "scratch bytes of softagg_fused for E rows");
  m.def("update_heads", &update_heads, "delta / weight heads (optionally emitting the BA target)", py::arg("net32"), py::arg("W4"),
        py::arg("b4"), py::arg("coords") = py::none(), py::arg("gate") = py::none(), py::arg("res") = py::none());
  m.def("linear_f16", &linear_f16, "wgmma dense layer", py::arg("x"), py::arg("w"), py::arg("bias") = py::none(),
        py::arg("epilogue") = 0, py::arg("res") = py::none(), py::arg("gate") = py::none(), py::arg("gather") = py::none(),
        py::arg("out_f32") = false, py::arg("out") = py::none(), py::arg("out16") = py::none());
  m.def("update_corr_norm", &update_corr_norm, "fused corr MLP + context add + LayerNorm (net.py:76-77)", py::arg("corr16"), py::arg("W0"), py::arg("W25"),
        py::arg("params"), py::arg("net32"), py::arg("inp16"), py::arg("inp_index") = py::none(), py::arg("net16_out") = py::none());
  m.def("update_neighbor_mlp", &update_neighbor_mlp, "fused masked neighbour gather + 2-layer MLP + residual (net.py:83-85)", py::arg("net16_in"), py::arg("index"),
        py::arg("Wab"), py::arg("params"), py::arg("net32"), py::arg("net16_out") = py::none());
  m.def("update_gru_heads", &update_gru_heads, "fused group add + GRU + heads (net.py:88-92)", py::arg("net32"), py::arg("hij16"), py::arg("group_of"),
        py::arg("W6"), py::arg("params"), py::arg("coords") = py::none(), py::arg("workspace") = py::none(), py::arg("hkk16") = py::none(), py::arg("group_kk") = py::none(),
        py::arg("delta_out") = py::none(), py::arg("weight_out") = py::none());
  m.def("update_gru_workspace_bytes", &update_gru_workspace_bytes, "scratch bytes of update_gru_heads (current device)");
  m.def("pgraph_remove", &pgraph_remove, "park edges by rule on the fixed-capacity edge store", py::arg("ii"), py::arg("jj"), py::arg("kk"), py::arg("active"),
        py::arg("rule"), py::arg("frame"), py::arg("param"), py::arg("enable"), py::arg("dummy_frame"), py::arg("dummy_patch"), py::arg("M"), py::arg("n_active"));
  m.def("pgraph_append", &pgraph_append, "fill parked slots with new edges", py::arg("ii"), py::arg("jj"), py::arg("kk"), py::arg("active"), py::arg("new_ii"),
        py::arg("new_jj"), py::arg("new_kk"), py::arg("enable"), py::arg("state"), py::arg("n_active"), py::arg("overflow"));
  m.def("pgraph_new_edges", &pgraph_new_edges, "steady-state forward + backward edges of the newest frame");
  m.def("loop_scores", &loop_scores, "loop-candidate flow scores of every (old frame, recent frame) pair");
  m.def("loop_select", &loop_select, "greedy loop-pair selection and emission of the loop edges", py::arg("scores"), py::arg("n"),
        py::arg("last_global_ba"), py::arg("M"), py::arg("removal"), py::arg("max_age"), py::arg("freq"), py::arg("kf_index"), py::arg("thresh"),
        py::arg("pairs"), py::arg("n_pairs"), py::arg("ii"), py::arg("jj"), py::arg("kk"), py::arg("active"), py::arg("state"),
        py::arg("n_active"), py::arg("overflow"));
  m.def("pgraph_remove_store", &pgraph_remove_store, "window removal with the loop exception, removed edges kept in the inactive store");
  m.def("loop_flags", &loop_flags, "loop-edge / long-range flags, minimum active ii and inactive count in one record");
  m.def("loop_normalize", &loop_normalize, "PatchGraph.normalize on the device (and the keyframe delta table's translations)",
        py::arg("poses"), py::arg("patches"), py::arg("n"), py::arg("M"), py::arg("delta") = py::none());
  m.def("keyframe_motion", &keyframe_motion, "keyframe motion test, delta record and frame-count decrement of B streams");
  m.def("keyframe_shift", &keyframe_shift, "the KI - 1 slot copies of a culled keyframe over every per-frame buffer and ring");
  m.def("keyframe_count", &keyframe_count, "add_frame (mode 0) / skip_frame (mode 1) timestamp bookkeeping of B streams");
  m.def("keyframe_trajectory", &keyframe_trajectory, "one inverted pose per timestamp through the live keyframes and delta chains");
  m.def("neighbors_from_groups", &neighbors_from_groups, "temporal neighbours from a kk/jj grouping");
  m.def("encoder_conv", &encoder_conv, "one frame-encoder convolution (tensor cores, fused norm / join prologue)", py::arg("shape"),
        py::arg("x"), py::arg("w"), py::arg("bias"), py::arg("x_stats") = py::none(), py::arg("x_relu") = false, py::arg("skip") = py::none(),
        py::arg("skip_stats") = py::none(), py::arg("skip_relu") = false, py::arg("want_joined") = false, py::arg("want_stats") = false,
        py::arg("want_pool") = false, py::arg("scale") = 1.0);
  m.def("encode_frame", &encode_frame, "both frame encoders: uint8 image -> fmap1, fmap2, gmap, imap, patches slots", py::arg("image"),
        py::arg("w16"), py::arg("b32"), py::arg("coords"), py::arg("fmap1"), py::arg("fmap2"), py::arg("gmap"), py::arg("imap"),
        py::arg("patches"), py::arg("workspace"), py::arg("colors") = py::none());
  m.def("encode_frame_workspace_bytes", &encode_frame_workspace_bytes, "scratch bytes of encode_frame for an H x W image");
  m.def("encode_frames", &encode_frames, "both frame encoders over B images in one pass, into rows of the rings", py::arg("images"),
        py::arg("w16"), py::arg("b32"), py::arg("coords"), py::arg("fmap1"), py::arg("fmap2"), py::arg("gmap"), py::arg("imap"),
        py::arg("patches"), py::arg("frame_rows"), py::arg("feat_rows"), py::arg("patch_rows"), py::arg("depth"),
        py::arg("workspace"), py::arg("colors") = py::none());
  m.def("point_cloud", &point_cloud, "the world points of every patch centre of frames [0, n) of each stream (dpvo.py:358-360)",
        py::arg("poses"), py::arg("patches"), py::arg("intrinsics"), py::arg("F"), py::arg("n"), py::arg("points"));
  m.def("encode_frames_workspace_bytes", &encode_frames_workspace_bytes, "scratch bytes of encode_frames for B H x W images");
  m.def("launch_count", &launch_count, "kernel launches issued by libdpvo_b200 so far");
  m.def("version", &version, "library version string");
}

PYBIND11_MODULE(dpvo_b200_camera, m) {
  m.def("undistort_frames", &undistort_frames, "cv2.undistort (+ half-size INTER_AREA resize) and a crop window of B uint8 images",
        py::arg("images"), py::arg("cameras"), py::arg("half"), py::arg("y0"), py::arg("x0"), py::arg("out"));
}
