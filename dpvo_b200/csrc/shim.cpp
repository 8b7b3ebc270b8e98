// Torch-extension shims over the C-ABI of include/dpvo_b200.h.
//
// One translation unit defines four Python modules; the build copies the resulting shared object
// to cuda_corr*.so, cuda_ba*.so, lietorch_backends*.so and dpvo_b200_ext*.so:
//   cuda_corr          same pybind surface as dpvo/altcorr/correlation.cpp:57-62
//   cuda_ba            same as dpvo/fastba/ba.cpp:183-188
//   lietorch_backends  same as dpvo/lietorch/src/lietorch.cpp:286-316
//   dpvo_b200_ext      the fused entry points that have no counterpart in the reference
// The shims only adapt torch::Tensor -> (pointer, sizes, strides, current CUDA stream), allocate
// outputs and raise RuntimeError on a non-zero status.  There is no CPU path: a CPU tensor is an
// error, not a fallback.
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
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

void need_cuda(const Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda(), "dpvo_b200: ", name, " must be a CUDA tensor (this build has no CPU path)");
}

void* stream() { return (void*)at::cuda::getCurrentCUDAStream().stream(); }

Tensor i64c(const Tensor& t) { return t.to(at::kLong).contiguous(); }
Tensor f32c(const Tensor& t) { return t.to(at::kFloat).contiguous(); }

std::vector<int64_t> strides5(const Tensor& t) {
  TORCH_CHECK(t.dim() == 5, "dpvo_b200: expected a 5-d tensor");
  return {t.stride(0), t.stride(1), t.stride(2), t.stride(3), t.stride(4)};
}

Tensor byte_ws(int64_t bytes, const Tensor& like) {
  return torch::empty({bytes}, like.options().dtype(at::kByte));
}

// ------------------------------------------------------------------------------ cuda_corr
std::vector<Tensor> corr_forward(Tensor fmap1, Tensor fmap2, Tensor coords, Tensor ii, Tensor jj, int radius) {
  need_cuda(fmap1, "fmap1"); need_cuda(fmap2, "fmap2"); need_cuda(coords, "coords");
  c10::cuda::CUDAGuard guard(fmap1.device());
  TORCH_CHECK(fmap1.scalar_type() == fmap2.scalar_type(), "corr: fmap1/fmap2 dtype mismatch");
  TORCH_CHECK(fmap1.dim() == 5 && fmap2.dim() == 5 && coords.dim() == 5, "corr: expected 5-d inputs");
  coords = f32c(coords); ii = i64c(ii); jj = i64c(jj);
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
  need_cuda(fmap1, "fmap1"); need_cuda(fmap2, "fmap2"); need_cuda(grad, "corr_grad");
  c10::cuda::CUDAGuard guard(fmap1.device());
  coords = f32c(coords); ii = i64c(ii); jj = i64c(jj);
  grad = grad.contiguous();
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
  need_cuda(net, "net"); need_cuda(coords, "coords");
  c10::cuda::CUDAGuard guard(net.device());
  TORCH_CHECK(net.dim() == 4 && coords.dim() == 3 && coords.size(2) == 2, "patchify: net [B,C,H,W], coords [B,M,2]");
  coords = f32c(coords);
  const int B = coords.size(0), M = coords.size(1), C = net.size(1), D = 2 * radius + 2;
  Tensor patches = torch::empty({B, M, C, D, D}, net.options());
  std::vector<int64_t> s = {net.stride(0), net.stride(1), net.stride(2), net.stride(3)};
  check(dpvo_patchify_forward(net.data_ptr(), s.data(), coords.data_ptr<float>(), patches.data_ptr(), dt(net),
                              B, M, C, (int)net.size(2), (int)net.size(3), radius, stream()),
        "cuda_corr.patchify_forward");
  return {patches};
}

std::vector<Tensor> patchify_backward(Tensor net, Tensor coords, Tensor gradient, int radius) {
  need_cuda(net, "net"); need_cuda(gradient, "gradient");
  c10::cuda::CUDAGuard guard(net.device());
  coords = f32c(coords);
  gradient = gradient.to(net.scalar_type()).contiguous();
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
  need_cuda(poses, "poses"); need_cuda(patches, "patches");
  c10::cuda::CUDAGuard guard(poses.device());
  TORCH_CHECK(poses.is_contiguous() && patches.is_contiguous(), "cuda_ba.forward updates poses/patches in place: they must be contiguous");
  TORCH_CHECK(poses.scalar_type() == at::kFloat && patches.scalar_type() == at::kFloat, "cuda_ba.forward: poses/patches must be float32");
  const int P = patches.size(-1);
  intrinsics = f32c(intrinsics).view({-1, 4});
  target = f32c(target).view({-1, 2});
  weight = f32c(weight).view({-1, 2});
  lmbda = f32c(lmbda).view({-1});
  ii = i64c(ii); jj = i64c(jj); kk = i64c(kk);
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
  need_cuda(ii, "ii"); need_cuda(jj, "jj");
  c10::cuda::CUDAGuard guard(ii.device());
  ii = i64c(ii); jj = i64c(jj);
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

Tensor reproject_impl(Tensor poses, Tensor patches, Tensor intrinsics, Tensor ii, Tensor jj, Tensor kk, int clamp) {
  need_cuda(poses, "poses"); need_cuda(patches, "patches");
  c10::cuda::CUDAGuard guard(poses.device());
  const int P = patches.size(-1);
  poses = f32c(poses); patches = f32c(patches); intrinsics = f32c(intrinsics);
  ii = i64c(ii); jj = i64c(jj); kk = i64c(kk);
  const int64_t E = ii.numel();
  Tensor coords = torch::empty({1, E, 2, P, P}, poses.options());
  check(dpvo_reproject(poses.data_ptr<float>(), patches.data_ptr<float>(), intrinsics.data_ptr<float>(),
                       ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), kk.data_ptr<int64_t>(), coords.data_ptr<float>(), E, P,
                       clamp, stream()),
        "cuda_ba.reproject");
  return coords;
}
Tensor ba_reproject(Tensor poses, Tensor patches, Tensor intrinsics, Tensor ii, Tensor jj, Tensor kk) {
  return reproject_impl(poses, patches, intrinsics, ii, jj, kk, 0);
}

// cuda_ba.solve_system (ba.cpp:120-180): pose-graph Gauss-Newton step of the loop-closure back end.  The normal
// equations are assembled on the device in fp64 (the reference: Eigen sparse, fp64, on the CPU); the leading
// 7*freen block is solved by a dense Cholesky and the remaining poses get a zero step (ba.cpp:101-118).
std::vector<Tensor> ba_solve_system(Tensor J_Ginv_i, Tensor J_Ginv_j, Tensor ii, Tensor jj, Tensor res, float ep, float lm, int freen) {
  need_cuda(res, "res");
  c10::cuda::CUDAGuard guard(res.device());
  J_Ginv_i = f32c(J_Ginv_i.to(res.device())); J_Ginv_j = f32c(J_Ginv_j.to(res.device()));
  ii = i64c(ii.to(res.device())); jj = i64c(jj.to(res.device()));
  Tensor r32 = f32c(res).view({-1, 7});
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
#define CHECK_CONTIGUOUS(x) TORCH_CHECK(x.is_contiguous(), #x " must be contiguous")

int emb_dim(int g) { return g == DPVO_SO3 ? 4 : g == DPVO_RXSO3 ? 5 : g == DPVO_SE3 ? 7 : 8; }
int tan_dim(int g) { return g == DPVO_SO3 ? 3 : g == DPVO_RXSO3 ? 4 : g == DPVO_SE3 ? 6 : 7; }

typedef int (*un_fn)(int, int, const void*, void*, int64_t, void*);
typedef int (*bin_fn)(int, int, const void*, const void*, void*, int64_t, void*);
typedef int (*unb_fn)(int, int, const void*, const void*, void*, int64_t, void*);
typedef int (*binb_fn)(int, int, const void*, const void*, const void*, void*, void*, int64_t, void*);

Tensor lie_unary(un_fn f, int g, Tensor x, int out_dim, const char* name) {
  CHECK_CONTIGUOUS(x); need_cuda(x, name);
  c10::cuda::CUDAGuard guard(x.device());
  Tensor y = torch::empty({x.size(0), out_dim}, x.options());
  check(f(g, dt(x), x.data_ptr(), y.data_ptr(), x.size(0), stream()), name);
  return y;
}
Tensor lie_binary(bin_fn f, int g, Tensor x, Tensor y, int out_dim, const char* name) {
  CHECK_CONTIGUOUS(x); CHECK_CONTIGUOUS(y); need_cuda(x, name);
  c10::cuda::CUDAGuard guard(x.device());
  TORCH_CHECK(x.scalar_type() == y.scalar_type() && x.size(0) == y.size(0), name, ": operand mismatch");
  Tensor z = torch::empty({x.size(0), out_dim}, x.options());
  check(f(g, dt(x), x.data_ptr(), y.data_ptr(), z.data_ptr(), x.size(0), stream()), name);
  return z;
}
std::vector<Tensor> lie_unary_bwd(unb_fn f, int g, Tensor grad, Tensor x, const char* name) {
  CHECK_CONTIGUOUS(x); CHECK_CONTIGUOUS(grad); need_cuda(x, name);
  c10::cuda::CUDAGuard guard(x.device());
  grad = grad.to(x.scalar_type());
  Tensor dx = torch::empty(x.sizes(), x.options());
  check(f(g, dt(x), grad.data_ptr(), x.data_ptr(), dx.data_ptr(), x.size(0), stream()), name);
  return {dx};
}
std::vector<Tensor> lie_binary_bwd(binb_fn f, int g, Tensor grad, Tensor x, Tensor y, const char* name) {
  CHECK_CONTIGUOUS(x); CHECK_CONTIGUOUS(y); CHECK_CONTIGUOUS(grad); need_cuda(x, name);
  c10::cuda::CUDAGuard guard(x.device());
  grad = grad.to(x.scalar_type());
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
  CHECK_CONTIGUOUS(X); need_cuda(X, "X");
  c10::cuda::CUDAGuard guard(X.device());
  Tensor T = torch::empty({X.size(0), 4, 4}, X.options());
  check(dpvo_lie_as_matrix(g, dt(X), X.data_ptr(), T.data_ptr(), X.size(0), stream()), "lietorch_backends.as_matrix");
  return T;
}
Tensor l_projector(int g, Tensor X) {
  CHECK_CONTIGUOUS(X); need_cuda(X, "X");
  c10::cuda::CUDAGuard guard(X.device());
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
  need_cuda(fmap1, "fmap1");
  c10::cuda::CUDAGuard guard(fmap1.device());
  coords = f32c(coords); ii = i64c(ii); jj = i64c(jj);
  const int B = coords.size(0), M = coords.size(1), P = coords.size(3), C = fmap1.size(2), O = 2 * radius + 1;
  const int64_t feat = (int64_t)O * O * P * P * 2;
  const int64_t row = pad_to > feat ? pad_to : feat;
  // padded rows ([B, M, row], zero tail) feed the wgmma dense layer directly; unpadded keep the 7-d view
  // out_buf: a caller-owned [B, M, row] buffer whose padding columns are already zero (reused every update)
  Tensor out;
  if (out_buf.has_value()) {
    out = *out_buf;
    TORCH_CHECK(out.is_contiguous() && out.scalar_type() == fmap1.scalar_type() && out.numel() == (int64_t)B * M * row, "corr_pyramid2: out buffer must be contiguous [B, M, ", row, "]");
  } else {
    out = (row == feat) ? torch::empty({B, M, O, O, P, P, 2}, fmap1.options()) : torch::zeros({B, M, row}, fmap1.options());
  }
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
  need_cuda(key_a, "key_a");
  c10::cuda::CUDAGuard guard(key_a.device());
  key_a = i64c(key_a);
  const int64_t E = key_a.numel();
  Tensor kb, sc;
  if (key_b.has_value()) kb = i64c(*key_b);
  if (sec.has_value()) sc = i64c(*sec);
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
  need_cuda(a0, "key_a0");
  c10::cuda::CUDAGuard guard(a0.device());
  a0 = i64c(a0); a1 = i64c(a1);
  const int64_t E = a0.numel();
  TORCH_CHECK(a1.numel() == E, "group_edges_pair: both problems group the same edges");
  Tensor kb[2], sc[2];
  if (b0.has_value()) kb[0] = i64c(*b0);
  if (s0.has_value()) sc[0] = i64c(*s0);
  if (b1.has_value()) kb[1] = i64c(*b1);
  if (s1.has_value()) sc[1] = i64c(*s1);
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

// fastba.BA on groupings built once per update (order, group_start, key_a[, key_b], n of EdgeGroups)
void ba_forward_grouped(Tensor poses, Tensor patches, Tensor intrinsics, Tensor target, Tensor weight, Tensor lmbda,
                        Tensor ii, Tensor jj, Tensor kk, int t0, int t1, int iterations,
                        Tensor k_order, Tensor k_start, Tensor k_key, Tensor k_n,
                        Tensor p_order, Tensor p_start, Tensor p_key_i, Tensor p_key_j, Tensor p_n) {
  need_cuda(poses, "poses"); need_cuda(patches, "patches");
  c10::cuda::CUDAGuard guard(poses.device());
  TORCH_CHECK(poses.is_contiguous() && patches.is_contiguous(), "ba_forward_grouped updates poses/patches in place: they must be contiguous");
  TORCH_CHECK(poses.scalar_type() == at::kFloat && patches.scalar_type() == at::kFloat, "ba_forward_grouped: poses/patches must be float32");
  const int P = patches.size(-1);
  intrinsics = f32c(intrinsics); target = f32c(target); weight = f32c(weight); lmbda = f32c(lmbda);
  ii = i64c(ii); jj = i64c(jj); kk = i64c(kk);
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

Tensor reproject_clamped(Tensor poses, Tensor patches, Tensor intrinsics, Tensor ii, Tensor jj, Tensor kk) {
  return reproject_impl(poses, patches, intrinsics, ii, jj, kk, 1);
}


// ---- update-operator building blocks (include/dpvo_b200.h, "Update operator building blocks")
int dt16or32(const Tensor& t) {
  TORCH_CHECK(t.scalar_type() == at::kHalf || t.scalar_type() == at::kFloat, "dpvo_b200: expected float16 or float32");
  return dt(t);
}

std::vector<Tensor> add_layernorm(Tensor a, c10::optional<Tensor> b, c10::optional<Tensor> c, Tensor gamma, Tensor beta,
                                  double eps, bool relu, bool want32, bool want16, c10::optional<Tensor> b_index, bool inplace32,
                                  c10::optional<Tensor> c_scale) {
  need_cuda(a, "a");
  c10::cuda::CUDAGuard guard(a.device());
  const int dim = a.size(-1);
  const int64_t rows = a.numel() / dim;
  a = a.contiguous();
  Tensor bb, cc;
  int dts[3] = {dt16or32(a), 0, 0};
  Tensor bidx;
  if (b_index.has_value()) { bidx = i64c(*b_index); TORCH_CHECK(bidx.numel() == rows, "add_layernorm: b_index length"); }
  if (b.has_value()) { bb = b->contiguous(); dts[1] = dt16or32(bb); TORCH_CHECK(bidx.defined() || bb.numel() == a.numel(), "add_layernorm: shape mismatch"); }
  if (c.has_value()) { cc = c->contiguous(); dts[2] = dt16or32(cc); TORCH_CHECK(cc.numel() == a.numel(), "add_layernorm: shape mismatch"); }
  gamma = f32c(gamma); beta = f32c(beta);
  Tensor csc; int64_t ld_cs = 0;
  if (c_scale.has_value()) {
    csc = c_scale->reshape({-1, dim});
    TORCH_CHECK(csc.scalar_type() == at::kHalf && csc.stride(1) == 1 && csc.size(0) == rows && cc.defined(), "add_layernorm: c_scale must be fp16 [rows, dim] next to operand c");
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
  need_cuda(x, "x");
  c10::cuda::CUDAGuard guard(x.device());
  x = x.contiguous(); idx = i64c(idx);
  const int dim = x.size(-1);
  const int64_t rows = idx.numel();
  Tensor y = torch::empty({1, rows, dim}, x.options().dtype(half_out ? at::kHalf : at::kFloat));
  check(dpvo_gather_rows_masked(x.data_ptr(), dt16or32(x), idx.data_ptr<int64_t>(), y.data_ptr(), dt(y), rows, dim, stream()),
        "dpvo_b200_ext.gather_rows_masked");
  return y;
}

Tensor residual_add_(Tensor net32, Tensor u, c10::optional<Tensor> group_of, bool want16) {
  need_cuda(net32, "net");
  c10::cuda::CUDAGuard guard(net32.device());
  TORCH_CHECK(net32.is_contiguous() && net32.scalar_type() == at::kFloat, "residual_add_: net must be contiguous float32");
  u = u.contiguous();
  const int dim = net32.size(-1);
  const int64_t rows = net32.numel() / dim;
  Tensor gof, n16;
  if (group_of.has_value()) { gof = group_of->to(at::kInt).contiguous(); TORCH_CHECK(gof.numel() == rows, "residual_add_: group_of length"); }
  else TORCH_CHECK(u.numel() == net32.numel(), "residual_add_: shape mismatch");
  if (want16) n16 = torch::empty(net32.sizes(), net32.options().dtype(at::kHalf));
  check(dpvo_residual_add(net32.data_ptr(), u.data_ptr(), dt16or32(u), gof.defined() ? gof.data_ptr<int>() : nullptr,
                          want16 ? n16.data_ptr() : nullptr, rows, dim, stream()),
        "dpvo_b200_ext.residual_add_");
  return n16;
}

// fp16( net32 + u[group_of] ) without updating net32
Tensor residual_sum16(Tensor net32, Tensor u, c10::optional<Tensor> group_of) {
  need_cuda(net32, "net");
  c10::cuda::CUDAGuard guard(net32.device());
  TORCH_CHECK(net32.is_contiguous() && net32.scalar_type() == at::kFloat, "residual_sum16: net must be contiguous float32");
  u = u.contiguous();
  const int dim = net32.size(-1);
  const int64_t rows = net32.numel() / dim;
  Tensor gof;
  if (group_of.has_value()) { gof = group_of->to(at::kInt).contiguous(); TORCH_CHECK(gof.numel() == rows, "residual_sum16: group_of length"); }
  else TORCH_CHECK(u.numel() == net32.numel(), "residual_sum16: shape mismatch");
  Tensor n16 = torch::empty(net32.sizes(), net32.options().dtype(at::kHalf));
  check(dpvo_residual_sum16(net32.data_ptr(), u.data_ptr(), dt16or32(u), gof.defined() ? gof.data_ptr<int>() : nullptr, n16.data_ptr(), rows, dim, stream()),
        "dpvo_b200_ext.residual_sum16");
  return n16;
}

std::vector<Tensor> gated_residual(Tensor x32, Tensor gate16, Tensor res16, bool want_relu16) {
  need_cuda(x32, "x");
  c10::cuda::CUDAGuard guard(x32.device());
  TORCH_CHECK(x32.scalar_type() == at::kFloat && gate16.scalar_type() == at::kHalf && res16.scalar_type() == at::kHalf,
              "gated_residual: expects (float32, float16, float16)");
  x32 = x32.contiguous(); gate16 = gate16.contiguous(); res16 = res16.contiguous();
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
  need_cuda(fg, "fg");
  c10::cuda::CUDAGuard guard(fg.device());
  TORCH_CHECK(fg.scalar_type() == at::kHalf && fg.is_contiguous() && fg.size(-1) % 2 == 0, "softagg_reduce: expects contiguous float16 [E, 2*dim]");
  const int dim = fg.size(-1) / 2;
  const int64_t E = fg.numel() / fg.size(-1);
  TORCH_CHECK(order.is_cuda() && order.scalar_type() == at::kInt && order.is_contiguous() && order.numel() == E,
              "softagg_reduce: order must be a contiguous int32 CUDA tensor with one entry per row of fg");
  TORCH_CHECK(group_start.is_cuda() && group_start.scalar_type() == at::kInt && group_start.is_contiguous() && group_start.numel() >= max_groups + 1,
              "softagg_reduce: group_start must be int32 with at least max_groups + 1 entries");
  TORCH_CHECK(n_groups.is_cuda() && n_groups.scalar_type() == at::kInt && n_groups.numel() == 1, "softagg_reduce: n_groups must be a device int32 scalar");
  TORCH_CHECK(max_groups >= 0 && max_groups <= E, "softagg_reduce: max_groups must be in [0, E]");
  Tensor y = torch::empty({1, max_groups, dim}, fg.options());   // rows past the group count are zeroed by the kernel itself
  const at::Half* base = fg.data_ptr<at::Half>();
  check(dpvo_softagg_reduce(base, base + dim, 2 * dim, order.data_ptr<int>(), group_start.data_ptr<int>(),
                            n_groups.data_ptr<int>(), max_groups, y.data_ptr(), dim, stream()),
        "dpvo_b200_ext.softagg_reduce");
  return y;
}

// Y = epilogue(X @ W^T + bias) on wgmma; X [.., rows, K] fp16 (row stride may exceed K), W [N, K] fp16
Tensor linear_f16(Tensor x, Tensor w, c10::optional<Tensor> bias, int64_t epilogue, c10::optional<Tensor> res,
                  c10::optional<Tensor> gate, c10::optional<Tensor> gather, bool out_f32, c10::optional<Tensor> out,
                  c10::optional<Tensor> out16) {
  need_cuda(x, "x");
  c10::cuda::CUDAGuard guard(x.device());
  TORCH_CHECK(x.scalar_type() == at::kHalf && w.scalar_type() == at::kHalf, "linear_f16: fp16 operands expected");
  TORCH_CHECK(x.stride(-1) == 1 && w.dim() == 2 && w.stride(1) == 1, "linear_f16: K must be contiguous");
  const int K = w.size(1), N = w.size(0);
  TORCH_CHECK(x.size(-1) == K, "linear_f16: X has ", x.size(-1), " columns, W expects ", K);
  Tensor x2 = x.dim() == 2 ? x : x.reshape({-1, K});
  TORCH_CHECK(x2.stride(1) == 1, "linear_f16: X rows must be dense");
  Tensor gi, b, r, g;
  int64_t rows = x2.size(0);
  if (gather.has_value()) { gi = i64c(*gather); rows = gi.numel(); }
  if (bias.has_value()) b = f32c(*bias);
  int res_dt = DPVO_F32; int64_t ldres = 0, ldgate = 0;
  if (res.has_value()) { r = res->reshape({-1, N}); TORCH_CHECK(r.stride(1) == 1 && r.size(0) == rows, "linear_f16: res shape"); res_dt = dt16or32(r); ldres = r.stride(0); }
  if (gate.has_value()) { g = gate->reshape({-1, N}); TORCH_CHECK(g.scalar_type() == at::kHalf && g.stride(1) == 1 && g.size(0) == rows, "linear_f16: gate shape"); ldgate = g.stride(0); }
  Tensor y = out.has_value() ? *out : torch::empty({1, rows, N}, x.options().dtype(out_f32 ? at::kFloat : at::kHalf));
  TORCH_CHECK(y.is_contiguous() && y.numel() == rows * N && y.scalar_type() == (out_f32 ? at::kFloat : at::kHalf), "linear_f16: out tensor");
  Tensor y16;
  if (out16.has_value()) { y16 = *out16; TORCH_CHECK(y16.is_contiguous() && y16.numel() == rows * N && y16.scalar_type() == at::kHalf, "linear_f16: out16 tensor"); }
  check(dpvo_linear_f16(x2.data_ptr(), x2.stride(0), gi.defined() ? gi.data_ptr<int64_t>() : nullptr, w.data_ptr(), w.stride(0),
                        b.defined() ? b.data_ptr<float>() : nullptr, r.defined() ? r.data_ptr() : nullptr, res_dt, ldres,
                        g.defined() ? g.data_ptr() : nullptr, ldgate, y.data_ptr(), out_f32 ? DPVO_F32 : DPVO_F16, N,
                        y16.defined() ? y16.data_ptr() : nullptr, N, rows, N, K, (int)epilogue, stream()),
        "dpvo_b200_ext.linear_f16");
  return y;
}

std::vector<Tensor> neighbors_from_groups(Tensor order, Tensor group_of) {
  need_cuda(order, "order");
  c10::cuda::CUDAGuard guard(order.device());
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
  need_cuda(net32, "net");
  c10::cuda::CUDAGuard guard(net32.device());
  TORCH_CHECK(net32.scalar_type() == at::kFloat, "update_heads: net must be float32");
  TORCH_CHECK(gate.has_value() == res.has_value(), "update_heads: gate and res come together");
  TORCH_CHECK(!gate.has_value() || net32.is_contiguous(), "update_heads: the gated form updates net in place and needs it contiguous");
  net32 = net32.contiguous(); W4 = f32c(W4); b4 = f32c(b4);
  const int dim = net32.size(-1);
  const int64_t rows = net32.numel() / dim;
  TORCH_CHECK(W4.numel() == 4 * dim && b4.numel() == 4, "update_heads: W4 [4,dim], b4 [4]");
  Tensor delta = torch::empty({1, rows, 2}, net32.options()), weight = torch::empty({1, rows, 2}, net32.options());
  Tensor cd; int P = 1;
  if (coords.has_value()) { cd = f32c(*coords); P = cd.size(-1); TORCH_CHECK(cd.numel() == rows * 2 * P * P, "update_heads: coords must be [rows,2,P,P]"); }
  Tensor g2, r2; int64_t ldg = 0, ldr = 0;
  if (gate.has_value()) {
    g2 = gate->reshape({-1, dim}); r2 = res->reshape({-1, dim});
    TORCH_CHECK(g2.scalar_type() == at::kHalf && r2.scalar_type() == at::kHalf && g2.stride(1) == 1 && r2.stride(1) == 1 && g2.size(0) == rows && r2.size(0) == rows,
                "update_heads: gate / res must be fp16 [rows, dim]");
    ldg = g2.stride(0); ldr = r2.stride(0);
  }
  check(dpvo_update_heads(net32.data_ptr(), g2.defined() ? g2.data_ptr() : nullptr, ldg, r2.defined() ? r2.data_ptr() : nullptr, ldr,
                          W4.data_ptr<float>(), b4.data_ptr<float>(), cd.defined() ? cd.data_ptr<float>() : nullptr, P,
                          delta.data_ptr<float>(),
                          weight.data_ptr<float>(), rows, dim, stream()),
        "dpvo_b200_ext.update_heads");
  return {delta, weight};
}

// ---- fused layer chains of the update operator (include/dpvo_b200.h, "fused layer chains")
static void chain_check(const Tensor& t, at::ScalarType st, const char* what) {
  TORCH_CHECK(t.is_cuda() && t.is_contiguous() && t.scalar_type() == st, "dpvo_b200 update chain: ", what, " must be a contiguous CUDA tensor of the expected dtype");
}
Tensor update_corr_norm(Tensor corr16, Tensor W0, Tensor W25, Tensor params, Tensor net32, Tensor inp16, c10::optional<Tensor> inp_index,
                        c10::optional<Tensor> net16_out) {
  need_cuda(net32, "net");
  c10::cuda::CUDAGuard guard(net32.device());
  chain_check(W0, at::kHalf, "W0"); chain_check(W25, at::kHalf, "W25"); chain_check(params, at::kFloat, "params");
  chain_check(net32, at::kFloat, "net32"); chain_check(inp16, at::kHalf, "inp16");
  const int64_t E = net32.numel() / 384;
  Tensor c2 = corr16.reshape({-1, corr16.size(-1)});
  TORCH_CHECK(c2.scalar_type() == at::kHalf && c2.stride(1) == 1 && c2.size(0) == E && c2.size(1) == 896, "update_corr_norm: corr must be fp16 [E, 896] (zero padded)");
  TORCH_CHECK(net32.size(-1) == 384 && W0.numel() == 384 * 896 && W25.numel() == 768 * 384 && params.numel() == 7 * 384 && inp16.size(-1) == 384, "update_corr_norm: shapes");
  Tensor idx;
  if (inp_index.has_value()) { idx = i64c(*inp_index); TORCH_CHECK(idx.numel() == E, "update_corr_norm: inp_index length"); }
  else TORCH_CHECK(inp16.numel() == E * 384, "update_corr_norm: inp must have one row per edge when no index is given");
  Tensor n16 = net16_out.has_value() ? *net16_out : torch::empty({1, E, 384}, net32.options().dtype(at::kHalf));
  chain_check(n16, at::kHalf, "net16_out");
  TORCH_CHECK(n16.numel() == E * 384, "update_corr_norm: net16_out shape");
  check(dpvo_update_corr_norm(c2.data_ptr(), c2.stride(0), W0.data_ptr(), W25.data_ptr(), params.data_ptr<float>(), net32.data_ptr<float>(),
                              inp16.data_ptr(), idx.defined() ? idx.data_ptr<int64_t>() : nullptr, n16.data_ptr(), E, stream()),
        "dpvo_b200_ext.update_corr_norm");
  return n16;
}

Tensor update_neighbor_mlp(Tensor net16_in, Tensor index, Tensor Wab, Tensor params, Tensor net32, c10::optional<Tensor> net16_out) {
  need_cuda(net32, "net");
  c10::cuda::CUDAGuard guard(net32.device());
  chain_check(net16_in, at::kHalf, "net16_in"); chain_check(Wab, at::kHalf, "Wab"); chain_check(params, at::kFloat, "params"); chain_check(net32, at::kFloat, "net32");
  const int64_t E = net32.numel() / 384;
  index = i64c(index);
  TORCH_CHECK(net32.size(-1) == 384 && net16_in.numel() == E * 384 && index.numel() == E && Wab.numel() == 768 * 384 && params.numel() == 2 * 384, "update_neighbor_mlp: shapes");
  Tensor n16 = net16_out.has_value() ? *net16_out : torch::empty({1, E, 384}, net32.options().dtype(at::kHalf));
  chain_check(n16, at::kHalf, "net16_out");
  TORCH_CHECK(n16.numel() == E * 384, "update_neighbor_mlp: net16_out shape");
  check(dpvo_update_neighbor_mlp(net16_in.data_ptr(), index.data_ptr<int64_t>(), Wab.data_ptr(), params.data_ptr<float>(), net32.data_ptr<float>(),
                                 n16.data_ptr(), E, stream()),
        "dpvo_b200_ext.update_neighbor_mlp");
  return n16;
}

std::vector<Tensor> update_gru_heads(Tensor net32, c10::optional<Tensor> hij16, c10::optional<Tensor> group_of, Tensor W6, Tensor params,
                                     c10::optional<Tensor> coords, c10::optional<Tensor> workspace, c10::optional<Tensor> hkk16, c10::optional<Tensor> group_kk) {
  need_cuda(net32, "net");
  c10::cuda::CUDAGuard guard(net32.device());
  chain_check(net32, at::kFloat, "net32"); chain_check(W6, at::kHalf, "W6"); chain_check(params, at::kFloat, "params");
  const int64_t E = net32.numel() / 384;
  TORCH_CHECK(net32.size(-1) == 384 && W6.numel() == 6 * 384 * 384 && params.numel() == 14 * 384 + 4, "update_gru_heads: shapes");
  TORCH_CHECK(hij16.has_value() == group_of.has_value(), "update_gru_heads: group rows and group ids come together");
  Tensor hij, gof;
  if (hij16.has_value()) {
    hij = *hij16; gof = group_of->to(at::kInt).contiguous();
    chain_check(hij, at::kHalf, "hij16");
    TORCH_CHECK(hij.size(-1) == 384 && gof.numel() == E, "update_gru_heads: group operand shapes");
  }
  TORCH_CHECK(hkk16.has_value() == group_kk.has_value(), "update_gru_heads: group rows and group ids come together");
  Tensor hkk, gkk;
  if (hkk16.has_value()) {
    hkk = *hkk16; gkk = group_kk->to(at::kInt).contiguous();
    chain_check(hkk, at::kHalf, "hkk16");
    TORCH_CHECK(hkk.size(-1) == 384 && gkk.numel() == E, "update_gru_heads: group operand shapes");
  }
  Tensor cd; int P = 1;
  if (coords.has_value()) { cd = f32c(*coords); P = cd.size(-1); TORCH_CHECK(cd.numel() == E * 2 * P * P, "update_gru_heads: coords must be [E,2,P,P]"); }
  const int64_t wsb = dpvo_update_gru_workspace_bytes();
  Tensor ws = workspace.has_value() ? *workspace : byte_ws(wsb, net32);
  TORCH_CHECK(ws.is_cuda() && ws.is_contiguous() && (int64_t)(ws.numel() * ws.element_size()) >= wsb, "update_gru_heads: workspace too small");
  Tensor delta = torch::empty({1, E, 2}, net32.options()), weight = torch::empty({1, E, 2}, net32.options());
  check(dpvo_update_gru_heads(net32.data_ptr<float>(), hij.defined() ? hij.data_ptr() : nullptr, gof.defined() ? gof.data_ptr<int>() : nullptr,
                              hkk.defined() ? hkk.data_ptr() : nullptr, gkk.defined() ? gkk.data_ptr<int>() : nullptr, W6.data_ptr(), params.data_ptr<float>(), cd.defined() ? cd.data_ptr<float>() : nullptr, P,
                              delta.data_ptr<float>(), weight.data_ptr<float>(), ws.data_ptr(), E, stream()),
        "dpvo_b200_ext.update_gru_heads");
  return {delta, weight};
}
int64_t update_gru_workspace_bytes() { return dpvo_update_gru_workspace_bytes(); }

// ---- device-resident patch-graph bookkeeping (include/dpvo_b200.h)
static void pg_check(const Tensor& ii, const Tensor& jj, const Tensor& kk, const Tensor& active) {
  TORCH_CHECK(ii.is_cuda() && ii.scalar_type() == at::kLong && ii.is_contiguous() && jj.scalar_type() == at::kLong && jj.is_contiguous() &&
              kk.scalar_type() == at::kLong && kk.is_contiguous() && active.scalar_type() == at::kByte && active.is_contiguous() &&
              jj.numel() == ii.numel() && kk.numel() == ii.numel() && active.numel() == ii.numel(), "pgraph: ii / jj / kk int64 and active uint8, one entry per slot");
}
void pgraph_remove(Tensor ii, Tensor jj, Tensor kk, Tensor active, int64_t rule, Tensor frame, int64_t param, c10::optional<Tensor> enable,
                   int64_t dummy_frame, int64_t dummy_patch, int64_t M, Tensor n_active) {
  need_cuda(ii, "ii");
  c10::cuda::CUDAGuard guard(ii.device());
  pg_check(ii, jj, kk, active);
  TORCH_CHECK(frame.is_cuda() && frame.scalar_type() == at::kLong && frame.numel() == 1 && n_active.is_cuda() && n_active.scalar_type() == at::kInt && n_active.numel() == 1,
              "pgraph_remove: frame is a device int64 scalar, n_active a device int32 scalar");
  const int32_t* en = nullptr;
  if (enable.has_value()) { TORCH_CHECK(enable->is_cuda() && enable->scalar_type() == at::kInt && enable->numel() == 1, "pgraph_remove: enable is a device int32 scalar"); en = enable->data_ptr<int>(); }
  check(dpvo_pgraph_remove(ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), kk.data_ptr<int64_t>(), active.data_ptr<uint8_t>(), ii.numel(), (int)rule,
                           frame.data_ptr<int64_t>(), param, en, dummy_frame, dummy_patch, (int)M, n_active.data_ptr<int>(), stream()),
        "dpvo_b200_ext.pgraph_remove");
}
Tensor pgraph_append(Tensor ii, Tensor jj, Tensor kk, Tensor active, Tensor new_ii, Tensor new_jj, Tensor new_kk, c10::optional<Tensor> enable,
                     c10::optional<Tensor> state, Tensor n_active, Tensor overflow) {
  need_cuda(ii, "ii");
  c10::cuda::CUDAGuard guard(ii.device());
  pg_check(ii, jj, kk, active);
  new_ii = i64c(new_ii); new_jj = i64c(new_jj); new_kk = i64c(new_kk);
  const int64_t n_new = new_ii.numel();
  TORCH_CHECK(new_jj.numel() == n_new && new_kk.numel() == n_new, "pgraph_append: new edge lists differ in length");
  TORCH_CHECK(n_active.is_cuda() && n_active.scalar_type() == at::kInt && n_active.numel() == 1 && overflow.is_cuda() && overflow.scalar_type() == at::kInt && overflow.numel() == 1,
              "pgraph_append: n_active / overflow are device int32 scalars");
  const int32_t* en = nullptr;
  if (enable.has_value()) { TORCH_CHECK(enable->is_cuda() && enable->scalar_type() == at::kInt && enable->numel() == 1, "pgraph_append: enable is a device int32 scalar"); en = enable->data_ptr<int>(); }
  Tensor slots = torch::empty({n_new}, ii.options().dtype(at::kInt));
  float* st = nullptr;
  if (state.has_value()) {
    TORCH_CHECK(state->is_cuda() && state->scalar_type() == at::kFloat && state->is_contiguous() && state->numel() == ii.numel() * 384,
                "pgraph_append: state must be the contiguous fp32 [cap, 384] recurrent state");
    st = state->data_ptr<float>();
  }
  check(dpvo_pgraph_append(ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), kk.data_ptr<int64_t>(), active.data_ptr<uint8_t>(), ii.numel(),
                           new_ii.data_ptr<int64_t>(), new_jj.data_ptr<int64_t>(), new_kk.data_ptr<int64_t>(), n_new, en, st, slots.data_ptr<int>(),
                           n_active.data_ptr<int>(), overflow.data_ptr<int>(), stream()),
        "dpvo_b200_ext.pgraph_append");
  return slots;
}
std::vector<Tensor> pgraph_new_edges(Tensor n_dev, int64_t M, int64_t r) {
  need_cuda(n_dev, "n");
  c10::cuda::CUDAGuard guard(n_dev.device());
  TORCH_CHECK(n_dev.scalar_type() == at::kLong && n_dev.numel() == 1, "pgraph_new_edges: n is a device int64 scalar");
  const int64_t total = M * (2 * r - 1);
  Tensor ii = torch::empty({total}, n_dev.options()), jj = torch::empty({total}, n_dev.options()), kk = torch::empty({total}, n_dev.options());
  check(dpvo_pgraph_new_edges(n_dev.data_ptr<int64_t>(), (int)M, (int)r, ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), kk.data_ptr<int64_t>(), stream()),
        "dpvo_b200_ext.pgraph_new_edges");
  return {ii, jj, kk};
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
  m.def("reproject_clamped", &reproject_clamped, "pops.transform-compatible fused reprojection");
  m.def("add_layernorm", &add_layernorm, "fused add + LayerNorm (+ReLU)", py::arg("a"), py::arg("b"), py::arg("c"), py::arg("gamma"),
        py::arg("beta"), py::arg("eps"), py::arg("relu"), py::arg("want32"), py::arg("want16"), py::arg("b_index") = py::none(), py::arg("inplace32") = false, py::arg("c_scale") = py::none());
  m.def("gather_rows_masked", &gather_rows_masked, "masked row gather");
  m.def("residual_add_", &residual_add_, "in-place residual add with optional row indirection");
  m.def("residual_sum16", &residual_sum16, "fp16(net + u[group]) without updating net", py::arg("net32"), py::arg("u"), py::arg("group_of") = py::none());
  m.def("gated_residual", &gated_residual, "x + sigmoid(g) * r");
  m.def("softagg_reduce", &softagg_reduce, "segment softmax-weighted sum");
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
        py::arg("W6"), py::arg("params"), py::arg("coords") = py::none(), py::arg("workspace") = py::none(), py::arg("hkk16") = py::none(), py::arg("group_kk") = py::none());
  m.def("update_gru_workspace_bytes", &update_gru_workspace_bytes, "scratch bytes of update_gru_heads");
  m.def("pgraph_remove", &pgraph_remove, "park edges by rule on the fixed-capacity edge store", py::arg("ii"), py::arg("jj"), py::arg("kk"), py::arg("active"),
        py::arg("rule"), py::arg("frame"), py::arg("param"), py::arg("enable"), py::arg("dummy_frame"), py::arg("dummy_patch"), py::arg("M"), py::arg("n_active"));
  m.def("pgraph_append", &pgraph_append, "fill parked slots with new edges", py::arg("ii"), py::arg("jj"), py::arg("kk"), py::arg("active"), py::arg("new_ii"),
        py::arg("new_jj"), py::arg("new_kk"), py::arg("enable"), py::arg("state"), py::arg("n_active"), py::arg("overflow"));
  m.def("pgraph_new_edges", &pgraph_new_edges, "steady-state forward + backward edges of the newest frame");
  m.def("neighbors_from_groups", &neighbors_from_groups, "temporal neighbours from a kk/jj grouping");
  m.def("launch_count", &launch_count, "kernel launches issued by libdpvo_b200 so far");
  m.def("version", &version, "library version string");
}
