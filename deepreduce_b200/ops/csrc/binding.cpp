// pybind11 / ATen bindings for the sm_90a kernels + the C++ runtime pieces
// (bucket engine context, background launch thread, IPC arena).
// The reference's native layer is TensorFlow CPU op glue (tensorflow/bloom_filter_compression.cc,
// integer_compression.cc, logger.cc); its PyTorch path has no native code and runs strictly after backward with
// torch.cuda.synchronize() between stages (pytorch/deepreduce.py:71,86,120,140,256,278).  Here the runtime is native:
// `Engine` owns the kernel parameter block of one bucket, `Scheduler` is the background thread that launches bucket
// kernels behind a CUDA event while backward is still running.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <torch/extension.h>

#include <condition_variable>
#include <deque>
#include <mutex>
#include <thread>

#include "ops.h"

namespace py = pybind11;
using dr::EngineParams;

#define CHECK_CUDA_T(x) TORCH_CHECK((x).is_cuda() && (x).is_contiguous(), #x " must be a contiguous CUDA tensor")

static cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

static void check_last(const char* what) {
  cudaError_t e = cudaGetLastError();
  TORCH_CHECK(e == cudaSuccess, what, ": ", cudaGetErrorString(e));
}

// ---------------------------------------------------------------------------
// per-tensor ops
// ---------------------------------------------------------------------------
static torch::Tensor bloom_insert(torch::Tensor idx, int64_t k, int64_t m_bits, int64_t seed) {
  CHECK_CUDA_T(idx);
  TORCH_CHECK(idx.scalar_type() == torch::kInt64, "idx must be int64");
  c10::cuda::CUDAGuard g(idx.device());
  const int64_t n_words = (m_bits + 31) / 32;
  auto words = torch::zeros({n_words}, idx.options().dtype(torch::kInt32));
  dr::launch_bloom_insert(idx.data_ptr<int64_t>(), idx.numel(), (uint32_t*)words.data_ptr<int32_t>(), (uint32_t)k,
                          (uint32_t)m_bits, (uint32_t)seed, cur_stream());
  check_last("bloom_insert");
  return words;
}

// limit < 0 -> all positives (p0)
static torch::Tensor bloom_select(torch::Tensor words, int64_t d, int64_t limit, int64_t k, int64_t m_bits, int64_t seed) {
  CHECK_CUDA_T(words);
  c10::cuda::CUDAGuard g(words.device());
  const int64_t n_tiles = (d + dr::kTile - 1) / dr::kTile;
  auto opts32 = words.options().dtype(torch::kInt32);
  auto counts = torch::empty({n_tiles}, opts32);
  auto excl = torch::empty({n_tiles + 1}, opts32);
  const uint32_t* f = (const uint32_t*)words.data_ptr<int32_t>();
  dr::launch_bloom_count(f, (uint32_t)d, (uint32_t)k, (uint32_t)m_bits, (uint32_t)seed,
                         (uint32_t*)counts.data_ptr<int32_t>(), (uint32_t*)excl.data_ptr<int32_t>(), cur_stream());
  const int64_t total = excl[n_tiles].item<int32_t>();      // the GRACE-compatible path is synchronous by contract
  const int64_t n_out = (limit < 0) ? total : std::min<int64_t>(limit, total);
  auto out = torch::empty({n_out}, words.options().dtype(torch::kInt64));
  if (n_out > 0)
    dr::launch_bloom_emit(f, (uint32_t)d, (uint32_t)k, (uint32_t)m_bits, (uint32_t)seed,
                          (const uint32_t*)excl.data_ptr<int32_t>(), out.data_ptr<int64_t>(), (uint32_t)n_out, cur_stream());
  check_last("bloom_select");
  return out;
}

static std::vector<torch::Tensor> qsgd_encode(torch::Tensor vals, int64_t q, int64_t bucket, int64_t seed) {
  CHECK_CUDA_T(vals);
  c10::cuda::CUDAGuard g(vals.device());
  auto v = vals.to(torch::kFloat32).contiguous();
  const int64_t K = v.numel();
  const bool i16 = q >= 128;
  auto lvl = torch::empty({K}, v.options().dtype(i16 ? torch::kInt16 : torch::kInt8));
  auto norms = torch::empty({(K + bucket - 1) / bucket}, v.options());
  dr::launch_qsgd_encode(v.data_ptr<float>(), K, (int)bucket, (int)q, (uint32_t)seed, lvl.data_ptr(), i16,
                         norms.data_ptr<float>(), cur_stream());
  check_last("qsgd_encode");
  return {lvl, norms};
}

static torch::Tensor qsgd_decode(torch::Tensor lvl, torch::Tensor norms, int64_t q, int64_t bucket) {
  CHECK_CUDA_T(lvl); CHECK_CUDA_T(norms);
  c10::cuda::CUDAGuard g(lvl.device());
  const bool i16 = lvl.scalar_type() == torch::kInt16;
  auto out = torch::empty({lvl.numel()}, norms.options());
  dr::launch_qsgd_decode(lvl.data_ptr(), i16, norms.data_ptr<float>(), lvl.numel(), (int)bucket, (int)q,
                         out.data_ptr<float>(), cur_stream());
  check_last("qsgd_decode");
  return out;
}

static torch::Tensor pack_bits(torch::Tensor vals, int64_t bits) {
  CHECK_CUDA_T(vals);
  c10::cuda::CUDAGuard g(vals.device());
  auto v = vals.to(torch::kInt64).contiguous();
  const int64_t n = v.numel();
  const int64_t n_bytes = (n * bits + 7) / 8, n_words = (n * bits + 31) / 32;
  auto out = torch::empty({n_words}, v.options().dtype(torch::kInt32));
  dr::launch_pack_bits(v.data_ptr<int64_t>(), n, (int)bits, (uint32_t*)out.data_ptr<int32_t>(), n_words, cur_stream());
  check_last("pack_bits");
  return out.view(torch::kUInt8).slice(0, 0, n_bytes);
}

static torch::Tensor unpack_bits(torch::Tensor buf, int64_t n, int64_t bits) {
  CHECK_CUDA_T(buf);
  c10::cuda::CUDAGuard g(buf.device());
  const int64_t n_words = (n * bits + 31) / 32;
  auto padded = torch::zeros({n_words * 4}, buf.options().dtype(torch::kUInt8));
  padded.slice(0, 0, buf.numel()).copy_(buf);
  auto out = torch::empty({n}, buf.options().dtype(torch::kInt64));
  dr::launch_unpack_bits((const uint32_t*)padded.data_ptr<uint8_t>(), n_words, n, (int)bits, out.data_ptr<int64_t>(),
                         cur_stream());
  check_last("unpack_bits");
  return out;
}

static torch::Tensor polyfit_fit(torch::Tensor y, torch::Tensor seg_off, torch::Tensor seg_len, int64_t degree, int64_t max_seg) {
  CHECK_CUDA_T(y); CHECK_CUDA_T(seg_off); CHECK_CUDA_T(seg_len);
  c10::cuda::CUDAGuard g(y.device());
  auto coeffs = torch::zeros({max_seg * (degree + 1)}, y.options());
  dr::launch_polyfit_fit(y.data_ptr<float>(), seg_off.data_ptr<int>(), seg_len.data_ptr<int>(), (int)seg_len.numel(),
                         (int)degree, coeffs.data_ptr<float>(), cur_stream());
  check_last("polyfit_fit");
  return coeffs;
}

static torch::Tensor polyfit_eval(torch::Tensor coeffs, torch::Tensor seg_off, torch::Tensor seg_len, int64_t degree, int64_t total) {
  CHECK_CUDA_T(coeffs);
  c10::cuda::CUDAGuard g(coeffs.device());
  auto out = torch::empty({total}, coeffs.options());
  dr::launch_polyfit_eval(coeffs.data_ptr<float>(), seg_off.data_ptr<int>(), seg_len.data_ptr<int>(),
                          (int)seg_len.numel(), (int)degree, total, out.data_ptr<float>(), cur_stream());
  check_last("polyfit_eval");
  return out;
}

// sets in visit order (CSR over member RANKS); returns the chosen flags of the positives, bit-packed
static torch::Tensor conflict_sets_pick(torch::Tensor set_off, torch::Tensor members, torch::Tensor last, int64_t n_pos, int64_t K,
                                        int64_t pseed) {
  CHECK_CUDA_T(set_off); CHECK_CUDA_T(members); CHECK_CUDA_T(last);
  c10::cuda::CUDAGuard g(set_off.device());
  auto out = torch::zeros({(n_pos + 31) / 32}, set_off.options().dtype(torch::kInt32));
  cudaError_t e = dr::launch_conflict_sets_pick((const uint32_t*)set_off.data_ptr<int32_t>(), (const uint32_t*)members.data_ptr<int32_t>(),
                                                (uint32_t*)last.data_ptr<int32_t>(), (uint32_t)(set_off.numel() - 1), (uint32_t)n_pos,
                                                (uint32_t)K, (uint32_t)pseed, (uint32_t*)out.data_ptr<int32_t>(), cur_stream());
  TORCH_CHECK(e == cudaSuccess, "conflict_sets_pick: ", cudaGetErrorString(e));
  return out;
}

static torch::Tensor dexp_fit(torch::Tensor y) {
  CHECK_CUDA_T(y);
  c10::cuda::CUDAGuard g(y.device());
  auto v = y.to(torch::kFloat32).contiguous();
  auto out = torch::zeros({4}, v.options().dtype(torch::kFloat64));
  dr::launch_dexp_fit(v.data_ptr<float>(), v.numel(), out.data_ptr<double>(), cur_stream());
  check_last("dexp_fit");
  return out;
}

static torch::Tensor delta_bp128_encode(torch::Tensor idx) {
  CHECK_CUDA_T(idx);
  c10::cuda::CUDAGuard g(idx.device());
  const int64_t n = idx.numel();
  const int64_t nb = (n + 127) / 128;
  auto widths = torch::zeros({nb}, idx.options().dtype(torch::kInt32));
  dr::launch_bp128_widths(idx.data_ptr<int64_t>(), n, (uint32_t*)widths.data_ptr<int32_t>(), cur_stream());
  auto sizes = widths.to(torch::kInt64) * 4 + 1;
  auto incl = sizes.cumsum(0);
  auto off = (incl - sizes).contiguous();
  const int64_t total = nb ? incl[nb - 1].item<int64_t>() : 0;
  auto out = torch::zeros({total}, idx.options().dtype(torch::kInt32));
  dr::launch_bp128_pack(idx.data_ptr<int64_t>(), n, (const uint32_t*)widths.data_ptr<int32_t>(), off.data_ptr<int64_t>(),
                        (uint32_t*)out.data_ptr<int32_t>(), cur_stream());
  check_last("delta_bp128_encode");
  return out;
}

static torch::Tensor delta_bp128_decode(torch::Tensor payload, int64_t n) {
  CHECK_CUDA_T(payload);
  c10::cuda::CUDAGuard g(payload.device());
  const int64_t nb = (n + 127) / 128;
  auto off = torch::empty({nb + 1}, payload.options().dtype(torch::kInt64));
  auto deltas = torch::empty({n}, payload.options().dtype(torch::kInt64));
  dr::launch_bp128_unpack((const uint32_t*)payload.data_ptr<int32_t>(), n, off.data_ptr<int64_t>(),
                          deltas.data_ptr<int64_t>(), cur_stream());
  check_last("delta_bp128_decode");
  return deltas.cumsum(0);
}

// sorted unique indices -> runs [z0, o0, z1, o1, ..., (tail zeros)]
static torch::Tensor rle_runs(torch::Tensor idx, int64_t d) {
  CHECK_CUDA_T(idx);
  c10::cuda::CUDAGuard g(idx.device());
  const int64_t n = idx.numel();
  auto o64 = idx.options().dtype(torch::kInt64);
  if (n == 0) return torch::full({1}, d, o64);
  const int64_t nb = (n + 1023) / 1024;
  auto counts = torch::empty({nb}, idx.options().dtype(torch::kInt32));
  auto excl = torch::empty({nb + 1}, idx.options().dtype(torch::kInt32));
  dr::launch_rle_count(idx.data_ptr<int64_t>(), n, (uint32_t*)counts.data_ptr<int32_t>(), (uint32_t*)excl.data_ptr<int32_t>(),
                       cur_stream());
  const int64_t n_runs = excl[nb].item<int32_t>();
  auto start_pos = torch::empty({n_runs}, o64), end_pos = torch::empty({n_runs}, o64);
  auto runs = torch::zeros({2 * n_runs + 1}, o64);
  dr::launch_rle_runs(idx.data_ptr<int64_t>(), n, (const uint32_t*)excl.data_ptr<int32_t>(), start_pos.data_ptr<int64_t>(),
                      end_pos.data_ptr<int64_t>(), n_runs, d, runs.data_ptr<int64_t>(), cur_stream());
  check_last("rle_runs");
  const int64_t last = idx[n - 1].item<int64_t>();
  return (d - 1 - last > 0) ? runs : runs.slice(0, 0, 2 * n_runs);
}

static torch::Tensor rle_indices(torch::Tensor runs) {
  CHECK_CUDA_T(runs);
  c10::cuda::CUDAGuard g(runs.device());
  const int64_t n_pairs = runs.numel() / 2;
  auto o64 = runs.options().dtype(torch::kInt64);
  if (n_pairs == 0) return torch::empty({0}, o64);
  auto pairs = runs.slice(0, 0, 2 * n_pairs).to(torch::kInt64).view({n_pairs, 2});
  auto z = pairs.select(1, 0), o = pairs.select(1, 1);
  auto csum = (z + o).cumsum(0);
  auto run_start = (csum - o).contiguous();
  auto ones_incl = o.cumsum(0);
  auto ones_excl = (ones_incl - o).contiguous();
  const int64_t total = ones_incl[n_pairs - 1].item<int64_t>();
  auto out = torch::empty({total}, o64);
  dr::launch_rle_expand(ones_excl.data_ptr<int64_t>(), run_start.data_ptr<int64_t>(), n_pairs, total, out.data_ptr<int64_t>(),
                        cur_stream());
  check_last("rle_indices");
  return out;
}

static torch::Tensor u8_to_nhwc_norm(torch::Tensor in, std::vector<double> mean, std::vector<double> stdv) {
  CHECK_CUDA_T(in);
  TORCH_CHECK(in.scalar_type() == torch::kUInt8 && in.size(-1) == 3, "expect uint8 [...,3] NHWC");
  c10::cuda::CUDAGuard g(in.device());
  in = in.contiguous();
  // the kernel reads 4 pixels as three 32-bit words: a batch slice of images with an odd byte count (x[1:] of
  // 225x225x3 images) starts off a 4-byte boundary, so such an input goes through a fresh (aligned) copy first
  if (reinterpret_cast<uintptr_t>(in.data_ptr()) % 4 != 0) in = in.clone(at::MemoryFormat::Contiguous);
  auto out = torch::empty(in.sizes(), in.options().dtype(torch::kBFloat16));
  float m[3] = {(float)mean[0], (float)mean[1], (float)mean[2]};
  float s[3] = {(float)(1.0 / stdv[0]), (float)(1.0 / stdv[1]), (float)(1.0 / stdv[2])};
  dr::launch_u8_to_nhwc_norm(in.data_ptr<uint8_t>(), out.data_ptr(), in.numel() / 3, m, s, cur_stream());
  check_last("u8_to_nhwc_norm");
  return out;
}

// ---------------------------------------------------------------------------
// training BatchNorm (+ ReLU, + residual add) on channels_last bf16 (bn.cu)
// ---------------------------------------------------------------------------
// torch's own channels-last Welford statistics, the instantiation native_batch_norm runs for bf16 input (exported by
// libtorch_cuda).  bn_stats falls back to it where bn.cu's mirror of its tree does not apply.
namespace at::native {
struct Var;
template <typename scalar_t, typename VarTransform>
void batch_norm_stats_channels_last_cuda_template(const at::Tensor& out_mean, const at::Tensor& out_invstd,
                                                   const at::Tensor& input, double epsilon);
}  // namespace at::native

static void check_bn_input(const torch::Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == torch::kBFloat16 && x.dim() == 4 && x.stride(1) == 1 &&
                  x.is_contiguous(at::MemoryFormat::ChannelsLast),
              "bn: x must be a channels_last bf16 CUDA tensor");
  TORCH_CHECK(x.size(1) % 8 == 0 && x.size(1) <= 8192, "bn: channels must be a multiple of 8, at most 8192");
  TORCH_CHECK(x.numel() < std::numeric_limits<int32_t>::max(), "bn: tensor too large for 32-bit indexing");
}

static void check_chan(const torch::Tensor& t, int64_t C, const char* what) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == torch::kFloat32 && t.is_contiguous() && t.numel() == C, "bn: ", what,
              " must be a contiguous float32 CUDA tensor of C elements");
}

// -> (save_mean, save_invstd); updates running_mean / running_var in place like native_batch_norm(training=True).
// bn.cu's statistics pass reproduces torch's channels-last Welford tree, so the results are bitwise torch's.  torch's
// kernel (+ bn.cu's running-stats update) runs instead with torch_kernel, for A/B comparisons, and for a tree with more
// virtual threads than rows, which flexible_launch_configs does not produce but the mirror does not cover.
static std::vector<torch::Tensor> bn_stats(torch::Tensor x, torch::Tensor running_mean, torch::Tensor running_var,
                                           double momentum, double eps, bool torch_kernel) {
  check_bn_input(x);
  const int64_t C = x.size(1);
  check_chan(running_mean, C, "running_mean");
  check_chan(running_var, C, "running_var");
  const int64_t N = x.numel() / C;
  TORCH_CHECK(N > 1, "bn: expected more than 1 value per channel when training");
  c10::cuda::CUDAGuard g(x.device());
  auto opts = x.options().dtype(torch::kFloat32);
  auto mean = torch::empty({C}, opts), invstd = torch::empty({C}, opts);
  const float bessel = static_cast<float>(static_cast<double>(N) / static_cast<double>(N - 1));
  int block_y = 0, grid_y = 0;
  dr::bn_row_tree(N, (int)C, &block_y, &grid_y);
  cudaError_t e;
  if (!torch_kernel && (int64_t)block_y * grid_y <= N) {
    auto staging = grid_y > 1 ? torch::empty({(2 * C + 1) * grid_y}, opts) : torch::Tensor();
    const dr::BnStats s{x.data_ptr(), mean.data_ptr<float>(), invstd.data_ptr<float>(), running_mean.data_ptr<float>(),
                        running_var.data_ptr<float>(), grid_y > 1 ? staging.data_ptr<float>() : nullptr,
                        (float)momentum, bessel, (float)eps};
    e = dr::launch_bn_stats(s, N, (int)C, cur_stream());
  } else {
    at::native::batch_norm_stats_channels_last_cuda_template<c10::BFloat16, at::native::Var>(mean, invstd, x, eps);
    e = dr::launch_bn_update_stats(mean.data_ptr<float>(), invstd.data_ptr<float>(), running_mean.data_ptr<float>(),
                                   running_var.data_ptr<float>(), (int)C, (float)momentum, bessel, (float)eps,
                                   cur_stream());
  }
  TORCH_CHECK(e == cudaSuccess, "bn_stats: ", cudaGetErrorString(e));
  return {mean, invstd};
}

static dr::BnParams bn_params(const std::vector<torch::Tensor>& p, int64_t C) {
  TORCH_CHECK(p.size() == 4, "bn: expected (mean, invstd, weight, bias)");
  const char* names[4] = {"mean", "invstd", "weight", "bias"};
  for (int i = 0; i < 4; ++i) check_chan(p[i], C, names[i]);
  return {p[0].data_ptr<float>(), p[1].data_ptr<float>(), p[2].data_ptr<float>(), p[3].data_ptr<float>()};
}

static void check_like_x(const torch::Tensor& t, const torch::Tensor& x, const char* what) {
  TORCH_CHECK(t.sizes() == x.sizes() && t.strides() == x.strides() && t.scalar_type() == torch::kBFloat16 &&
                  t.device() == x.device(),
              "bn: ", what, " must match x in shape, layout, dtype and device");
}

// mode 0: relu(bn(x)); 1: relu(bn(x) + z); 2: relu(bn(x) + bn_z(z)).  p / pz = (mean, invstd, weight, bias).
// -> (out, mask): mask is uint8 [N*H*W, C/8], bit i of byte g set where out[..., 8g + i] is not <= 0.
static std::vector<torch::Tensor> bn_apply(int64_t mode, torch::Tensor x, std::vector<torch::Tensor> p,
                                           c10::optional<torch::Tensor> z, std::vector<torch::Tensor> pz) {
  check_bn_input(x);
  const int64_t C = x.size(1);
  const dr::BnParams px = bn_params(p, C);
  dr::BnParams pzz{};
  const void* zp = nullptr;
  if (mode != 0) {
    TORCH_CHECK(z.has_value(), "bn: mode ", mode, " needs z");
    check_like_x(*z, x, "z");
    zp = z->data_ptr();
    if (mode == 2) pzz = bn_params(pz, C);
  }
  c10::cuda::CUDAGuard g(x.device());
  const int64_t rows = x.numel() / C;
  auto out = torch::empty_like(x);
  auto mask = torch::empty({rows, C / 8}, x.options().dtype(torch::kUInt8));
  cudaError_t e = dr::launch_bn_apply((int)mode, x.data_ptr(), px, zp, pzz, out.data_ptr(), mask.data_ptr(), rows,
                                      (int)C, cur_stream());
  TORCH_CHECK(e == cudaSuccess, "bn_apply: ", cudaGetErrorString(e));
  return {out, mask};
}

// maxpool(relu(bn(x))) for the one pool this is specialised to: kernel 3, stride 2, padding 1, dilation 1, floor mode.
// p = (mean, invstd, weight, bias).  -> (pooled, codes): pooled is channels_last (N, C, Ho, Wo) with
// Ho = (H - 1) / 2 + 1, bitwise max_pool2d(relu(bn(x))); codes is uint8 [N*Ho*Wo, C], one byte per pooled element:
// bits 0-6 the winner's slot in its 3x3 window, bit 7 the winner's ReLU mask.
static std::vector<torch::Tensor> bn_apply_pool(torch::Tensor x, std::vector<torch::Tensor> p, int64_t kernel_size,
                                                int64_t stride, int64_t padding, int64_t dilation, bool ceil_mode) {
  TORCH_CHECK(kernel_size == 3 && stride == 2 && padding == 1 && dilation == 1 && !ceil_mode,
              "bn_apply_pool: only kernel 3, stride 2, padding 1, dilation 1, floor mode");
  check_bn_input(x);
  const int64_t N = x.size(0), C = x.size(1), H = x.size(2), W = x.size(3);
  const dr::BnParams px = bn_params(p, C);
  c10::cuda::CUDAGuard g(x.device());
  const dr::PoolGeom pg{(int)H, (int)W, (int)((H - 1) / 2 + 1), (int)((W - 1) / 2 + 1)};
  auto out = torch::empty({N, C, pg.Ho, pg.Wo}, x.options().memory_format(at::MemoryFormat::ChannelsLast));
  auto codes = torch::empty({N * pg.Ho * pg.Wo, C}, x.options().dtype(torch::kUInt8));
  cudaError_t e = dr::launch_bn_apply_pool(x.data_ptr(), px, out.data_ptr(), codes.data_ptr(), (int)N, pg, (int)C,
                                           cur_stream());
  TORCH_CHECK(e == cudaSuccess, "bn_apply_pool: ", cudaGetErrorString(e));
  return {out, codes};
}

static dr::BnParams bn_bwd_params(const std::vector<torch::Tensor>& p, int64_t C) {
  TORCH_CHECK(p.size() == 3, "bn_backward: expected (mean, invstd, weight)");
  const char* names[3] = {"mean", "invstd", "weight"};
  for (int i = 0; i < 3; ++i) check_chan(p[i], C, names[i]);
  return {p[0].data_ptr<float>(), p[1].data_ptr<float>(), p[2].data_ptr<float>(), nullptr};
}

// Backward of bn_apply(mode) from the output gradient go and bn_apply's mask; p / pz = (mean, invstd, weight).
// The gradient of the ReLU input is g = mask ? go : 0.  Returns
//   mode 0: (dx, dw, db);  1: (dx, dw, db, g) (g is the gradient of z);  2: (dx, dw, db, dz, dw_z, db_z).
// Bitwise native_batch_norm_backward(threshold_backward(go, out, 0), ...) of torch's channels-last kernels.
// Mode 3 is the backward of bn_apply_pool: go is the pooled gradient (N, C, Ho, Wo) and mask the codes; go reaches
// the ReLU output as max_pool2d_with_indices_backward gives it.  Returns (dx, dw, db).
// go2 (modes 1-3): a second gradient of the output, checked like go.  The output then feeds two consumers, and the
// kernels use the bf16 sum go + go2 (fp32 sum, rounded once: autograd's add) wherever they would use go.
static std::vector<torch::Tensor> bn_backward(int64_t mode, torch::Tensor go, torch::Tensor mask, torch::Tensor x,
                                              std::vector<torch::Tensor> p, c10::optional<torch::Tensor> z,
                                              std::vector<torch::Tensor> pz, c10::optional<torch::Tensor> go2) {
  TORCH_CHECK(mode >= 0 && mode <= 3, "bn_backward: mode must be 0, 1, 2 or 3");
  TORCH_CHECK(!go2.has_value() || mode != 0, "bn_backward: mode 0 takes no go2");
  check_bn_input(x);
  const int64_t C = x.size(1), rows = x.numel() / C;
  dr::PoolGeom pg{(int)x.size(2), (int)x.size(3), (int)((x.size(2) - 1) / 2 + 1), (int)((x.size(3) - 1) / 2 + 1)};
  const std::vector<int64_t> go_shape =
      mode == 3 ? std::vector<int64_t>{x.size(0), C, pg.Ho, pg.Wo} : x.sizes().vec();
  for (const torch::Tensor* t : {&go, go2.has_value() ? &*go2 : &go})
    TORCH_CHECK(t->sizes() == go_shape && t->scalar_type() == torch::kBFloat16 && t->device() == x.device() &&
                    t->is_contiguous(at::MemoryFormat::ChannelsLast),
                "bn_backward: go and go2 must be channels_last bf16 tensors on x's device, of x's shape (mode 3: the "
                "pooled shape)");
  const int64_t mask_numel = mode == 3 ? go.numel() : rows * (C / 8);
  TORCH_CHECK(mask.is_cuda() && mask.scalar_type() == torch::kUInt8 && mask.is_contiguous() &&
                  mask.numel() == mask_numel && mask.device() == x.device(),
              "bn_backward: mask must be bn_apply's mask (mode 3: bn_apply_pool's codes) for x");
  c10::cuda::CUDAGuard guard(x.device());
  int block_y = 0, grid_y = 0;
  dr::bn_row_tree(rows, (int)C, &block_y, &grid_y);
  // every virtual thread of torch's tree owns at least one row, so no slot of its block tree is left unwritten
  TORCH_CHECK((int64_t)block_y * grid_y <= rows, "bn_backward: reduction tree wider than the rows");
  const int n_sums = mode == 2 ? 3 : 2;
  auto f32 = x.options().dtype(torch::kFloat32);
  auto sums = torch::empty({n_sums, C}, f32);
  auto staging = grid_y > 1 ? torch::empty({n_sums, grid_y, C}, f32) : torch::Tensor();
  auto dx = torch::empty_like(x), dw = torch::empty({C}, f32), db = torch::empty({C}, f32);
  dr::BnBwd b{};
  b.go = go.data_ptr(); b.go2 = go2.has_value() ? go2->data_ptr() : nullptr; b.mask = mask.data_ptr<uint8_t>(); b.x = x.data_ptr();
  b.px = bn_bwd_params(p, C);
  b.dx = dx.data_ptr(); b.sums = sums.data_ptr<float>(); b.staging = grid_y > 1 ? staging.data_ptr<float>() : nullptr;
  b.dw = dw.data_ptr<float>(); b.db = db.data_ptr<float>();
  b.pool = pg;
  std::vector<torch::Tensor> res{dx, dw, db};
  torch::Tensor g;
  if (mode == 1 || mode == 3) {
    g = torch::empty_like(x);
    b.g = g.data_ptr();
    if (mode == 1) res.push_back(g);     // mode 3: the gathered, masked pooled gradient, read by both passes
  } else if (mode == 2) {
    TORCH_CHECK(z.has_value(), "bn_backward: mode 2 needs z");
    check_like_x(*z, x, "z");
    b.z = z->data_ptr();
    b.pz = bn_bwd_params(pz, C);
    auto dz = torch::empty_like(x), dwz = torch::empty({C}, f32), dbz = torch::empty({C}, f32);
    b.dz = dz.data_ptr(); b.dwz = dwz.data_ptr<float>(); b.dbz = dbz.data_ptr<float>();
    res.insert(res.end(), {dz, dwz, dbz});
  }
  cudaError_t e = dr::launch_bn_backward((int)mode, b, rows, (int)C, cur_stream());
  TORCH_CHECK(e == cudaSuccess, "bn_backward: ", cudaGetErrorString(e));
  return res;
}

// ---------------------------------------------------------------------------
// engine context
// ---------------------------------------------------------------------------
struct Engine {
  EngineParams P{};
  int grid = 0;
  int grid_cap = 0;            // > 0: launch at most this many CTAs (overlapped buckets leave SMs to backward)
  int blocks_per_sm = 2;
  int dyn_smem = 64 * 1024;
  int device = 0;

  Engine(int64_t tensors, int64_t tiles, int64_t n_tensors, int64_t n_tiles, int64_t slot_words,
         int64_t payload_words, int64_t grad, int64_t resid, int64_t hist, int64_t hist_total, int64_t sel,
         int64_t tile_count, int64_t barrier, int64_t status, std::vector<int64_t> arenas, int rank, int world) {
    TORCH_CHECK(world <= dr::kMaxWorld && (int)arenas.size() == world, "bad world/arenas");
    P.tensors = reinterpret_cast<const dr::TensorDesc*>(tensors);
    P.tiles = reinterpret_cast<const dr::TileInfo*>(tiles);
    P.n_tensors = (uint32_t)n_tensors; P.n_tiles = (uint32_t)n_tiles;
    P.slot_words = (uint32_t)slot_words; P.payload_words = (uint32_t)payload_words;
    P.grad = reinterpret_cast<float*>(grad); P.resid = reinterpret_cast<float*>(resid);
    P.hist = reinterpret_cast<uint32_t*>(hist); P.hist_total = reinterpret_cast<uint32_t*>(hist_total);
    P.sel = reinterpret_cast<dr::SelState*>(sel);
    P.tile_count = reinterpret_cast<uint32_t*>(tile_count);
    P.barrier = reinterpret_cast<uint32_t*>(barrier); P.status = reinterpret_cast<uint32_t*>(status);
    for (int i = 0; i < world; ++i) P.arena[i] = reinterpret_cast<uint32_t*>(arenas[i]);
    P.rank = rank; P.world = world;
    P.beta = 1.f; P.gamma = 1.f; P.scale = 1.f / world; P.seed = dr::kDefaultSeed; P.policy = 0; P.use_history = 1;
    P.spin_limit = 20u * 1000u * 1000u;
    P.filter_smem_words = (uint32_t)(dyn_smem / 4);
    P.use_tma = 1; P.hist_shift = 23;
    P.shard = 0; P.s2_words = 0; P.s2_cap = 0; P.has_rle = 0; P.mc_arena = nullptr;
    P.peer_timeout_ms = 120000u; P.fault = 0; P.debug_times = nullptr; P.cost_prefix = nullptr; P.deterministic = 0; P.cuts = nullptr; P.cuts_grid = 0;
    cudaGetDevice(&device);
  }

  void configure(double beta, double gamma, double scale, int64_t seed, int policy, int use_history, int64_t spin_limit,
                 int bps, int64_t filter_smem_bytes, int use_tma, int hist_shift) {
    P.beta = (float)beta; P.gamma = (float)gamma; P.scale = (float)scale; P.seed = (uint32_t)seed;
    P.policy = policy; P.use_history = use_history; P.spin_limit = (uint32_t)spin_limit;
    blocks_per_sm = bps; grid = 0;
    dyn_smem = (int)filter_smem_bytes; P.filter_smem_words = (uint32_t)(dyn_smem / 4);
    P.use_tma = use_tma; P.hist_shift = (uint32_t)hist_shift;
  }

  void set_poly(int64_t tensors, int64_t n_poly, int64_t tasks, int64_t n_tasks, int64_t bins, int64_t bucket_val,
                int64_t bucket_pos, int64_t expand_buf, int64_t poly_total) {
    P.poly_tensors = reinterpret_cast<const uint32_t*>(tensors); P.n_poly = (uint32_t)n_poly;
    P.poly_tasks = reinterpret_cast<const uint32_t*>(tasks); P.n_poly_tasks = (uint32_t)n_tasks;
    P.poly_bins = reinterpret_cast<uint32_t*>(bins); P.bucket_val = reinterpret_cast<float*>(bucket_val);
    P.bucket_pos = reinterpret_cast<uint32_t*>(bucket_pos); P.expand_buf = reinterpret_cast<float*>(expand_buf);
    P.poly_total = (uint32_t)poly_total;
  }

  void set_has_rle(int v) { P.has_rle = v; }
  // scratch of the candidate / bitmask pipeline (see engine.cu): masks [n_tiles*128] u32 x2, candidate keys
  // entries [n_tiles*4096] x {u32 key, u32 offset}, counts [n_tiles*16] u32
  void set_scratch(int64_t pos_mask, int64_t dec_mask, int64_t cand, int64_t cand_cnt) {
    P.pos_mask = reinterpret_cast<uint32_t*>(pos_mask); P.dec_mask = reinterpret_cast<uint32_t*>(dec_mask);
    P.cand = reinterpret_cast<uint2*>(cand); P.cand_cnt = reinterpret_cast<uint32_t*>(cand_cnt);
  }
  void set_peer_timeout_ms(int64_t ms) { P.peer_timeout_ms = (uint32_t)ms; }
  void set_fault(int f) { P.fault = f; }
  void set_deterministic(int d) { P.deterministic = d; }
  void set_cost_prefix(int64_t p) { P.cost_prefix = reinterpret_cast<const uint32_t*>(p); }
  void set_debug_times(int64_t p) { P.debug_times = reinterpret_cast<unsigned long long*>(p); }
  void set_cuts(int64_t p, int64_t grid) { P.cuts = reinterpret_cast<const uint32_t*>(p); P.cuts_grid = (uint32_t)grid; }
  void set_grid_cap(int cap) { grid_cap = cap; }
  void set_multicast(int64_t p) { P.mc_arena = reinterpret_cast<uint32_t*>(p); }

  void set_shard(int shard, int64_t s2_words, int64_t s2_cap) {
    P.shard = shard; P.s2_words = (uint32_t)s2_words; P.s2_cap = (uint32_t)s2_cap;
  }

  void set_buffers(int64_t grad, int64_t resid) {
    P.grad = reinterpret_cast<float*>(grad); P.resid = reinterpret_cast<float*>(resid);
  }

  int get_grid() {
    if (grid == 0) grid = dr::engine_max_grid(blocks_per_sm, dyn_smem);
    return grid;
  }

  void run_on(uint32_t epoch, int phase_begin, int phase_end, cudaStream_t st) {
    EngineParams Q = P;
    Q.epoch = epoch; Q.phase_begin = phase_begin; Q.phase_end = phase_end;
    TORCH_CHECK(P.pos_mask && P.cand, "Engine: set_scratch() was not called");
    int g = get_grid();
    if (grid_cap > 0 && grid_cap < g) g = grid_cap;
    cudaError_t e = dr::engine_launch(Q, g, blocks_per_sm, dyn_smem, st);
    TORCH_CHECK(e == cudaSuccess, "engine launch failed: ", cudaGetErrorString(e));
  }

  void run(int64_t epoch, int phase_begin, int phase_end) { run_on((uint32_t)epoch, phase_begin, phase_end, cur_stream()); }
};

// ---------------------------------------------------------------------------
// background launch thread: buckets are handed over as soon as their gradients
// are ready; the thread issues wait(ready) -> engine kernel -> record(done) on
// a high-priority side stream so the exchange overlaps the rest of backward.
// ---------------------------------------------------------------------------
struct Scheduler {
  struct Item { Engine* eng; uint32_t epoch; cudaEvent_t ready; cudaEvent_t done; };
  std::thread worker;
  std::mutex mu;
  std::condition_variable cv, cv_done;
  std::deque<Item> q;
  bool stop = false;
  int64_t submitted = 0, completed = 0;
  cudaStream_t side = nullptr;
  int device = 0;
  std::vector<cudaEvent_t> ready_ev, done_ev;
  std::string error;

  explicit Scheduler(int n_buckets) {
    cudaGetDevice(&device);
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);
    cudaStreamCreateWithPriority(&side, cudaStreamNonBlocking, hi);
    ready_ev.resize(n_buckets); done_ev.resize(n_buckets);
    for (int i = 0; i < n_buckets; ++i) {
      cudaEventCreateWithFlags(&ready_ev[i], cudaEventDisableTiming);
      cudaEventCreateWithFlags(&done_ev[i], cudaEventDisableTiming);
    }
    worker = std::thread([this] { loop(); });
  }

  ~Scheduler() { shutdown(); }

  void shutdown() {
    {
      std::lock_guard<std::mutex> l(mu);
      if (stop) return;
      stop = true;
    }
    cv.notify_all();
    if (worker.joinable()) worker.join();
    for (auto e : ready_ev) cudaEventDestroy(e);
    for (auto e : done_ev) cudaEventDestroy(e);
    if (side) cudaStreamDestroy(side);
    side = nullptr;
  }

  void loop() {
    cudaSetDevice(device);
    while (true) {
      Item it;
      {
        std::unique_lock<std::mutex> l(mu);
        cv.wait(l, [this] { return stop || !q.empty(); });
        if (q.empty()) return;
        it = q.front(); q.pop_front();
      }
      cudaStreamWaitEvent(side, it.ready, 0);
      try {
        it.eng->run_on(it.epoch, dr::kPhAccum, dr::kPhEnd, side);
      } catch (const std::exception& ex) {
        std::lock_guard<std::mutex> l(mu);
        error = ex.what();
      }
      cudaEventRecord(it.done, side);
      {
        std::lock_guard<std::mutex> l(mu);
        ++completed;
      }
      cv_done.notify_all();
    }
  }

  // main thread: gradients of `bucket` are final on the current stream
  void submit(int bucket, Engine* eng, int64_t epoch) {
    cudaEventRecord(ready_ev[bucket], cur_stream());
    {
      std::lock_guard<std::mutex> l(mu);
      q.push_back(Item{eng, (uint32_t)epoch, ready_ev[bucket], done_ev[bucket]});
      ++submitted;
    }
    cv.notify_one();
  }

  // main thread: make the current stream wait for every submitted bucket
  void wait_all() {
    py::gil_scoped_release rel;
    {
      std::unique_lock<std::mutex> l(mu);
      cv_done.wait(l, [this] { return completed == submitted; });
      TORCH_CHECK(error.empty(), "background engine launch failed: ", error);
    }
    for (auto e : done_ev) cudaStreamWaitEvent(cur_stream(), e, 0);
  }
};

// ---------------------------------------------------------------------------
// arena
// ---------------------------------------------------------------------------
static int64_t arena_alloc(int64_t bytes) {
  void* p = dr::arena_alloc((size_t)bytes);
  TORCH_CHECK(p != nullptr, "arena cudaMalloc failed");
  return (int64_t)p;
}
static py::bytes arena_export(int64_t p) {
  dr::ArenaHandle h = dr::arena_export((void*)p);
  return py::bytes((const char*)h.bytes, sizeof(h.bytes));
}
static int64_t arena_import(const std::string& b) {
  TORCH_CHECK(b.size() == sizeof(dr::ArenaHandle), "bad handle");
  dr::ArenaHandle h;
  memcpy(h.bytes, b.data(), sizeof(h.bytes));
  void* p = dr::arena_import(h);
  TORCH_CHECK(p != nullptr, "cudaIpcOpenMemHandle failed (peer access / IPC unavailable)");
  return (int64_t)p;
}
static torch::Tensor arena_as_tensor(int64_t p, int64_t n_words, int64_t device) {
  auto opts = torch::TensorOptions().dtype(torch::kInt32).device(torch::kCUDA, (int)device);
  return torch::from_blob((void*)p, {n_words}, opts);
}

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("launch_count", [] { return (int64_t)dr::launch_count(); });
  m.def("bloom_insert", &bloom_insert);
  m.def("bloom_select", &bloom_select);
  m.def("qsgd_encode", &qsgd_encode);
  m.def("qsgd_decode", &qsgd_decode);
  m.def("pack_bits", &pack_bits);
  m.def("unpack_bits", &unpack_bits);
  m.def("polyfit_fit", &polyfit_fit);
  m.def("polyfit_eval", &polyfit_eval);
  m.def("dexp_fit", &dexp_fit);
  m.def("conflict_sets_pick", &conflict_sets_pick);
  m.def("delta_bp128_encode", &delta_bp128_encode);
  m.def("delta_bp128_decode", &delta_bp128_decode);
  m.def("u8_to_nhwc_norm", &u8_to_nhwc_norm);
  m.def("bn_stats", &bn_stats, py::arg("x"), py::arg("running_mean"), py::arg("running_var"), py::arg("momentum"),
        py::arg("eps"), py::arg("torch_kernel") = false);
  m.def("bn_apply", &bn_apply, py::arg("mode"), py::arg("x"), py::arg("p"), py::arg("z") = py::none(),
        py::arg("pz") = std::vector<torch::Tensor>{});
  m.def("bn_apply_pool", &bn_apply_pool, py::arg("x"), py::arg("p"), py::arg("kernel_size") = 3, py::arg("stride") = 2,
        py::arg("padding") = 1, py::arg("dilation") = 1, py::arg("ceil_mode") = false);
  m.def("bn_backward", &bn_backward, py::arg("mode"), py::arg("go"), py::arg("mask"), py::arg("x"), py::arg("p"),
        py::arg("z") = py::none(), py::arg("pz") = std::vector<torch::Tensor>{}, py::arg("go2") = py::none());
  m.def("rle_runs", &rle_runs);
  m.def("rle_indices", &rle_indices);
  m.def("arena_alloc", &arena_alloc);
  m.def("arena_free", [](int64_t p) { dr::arena_free((void*)p); });
  m.def("arena_export", &arena_export);
  m.def("arena_import", &arena_import);
  m.def("arena_close", [](int64_t p) { dr::arena_close((void*)p); });
  m.def("arena_as_tensor", &arena_as_tensor);
  m.def("enable_peer_access", [](std::vector<int> devices) { return dr::arena_enable_peer_access(devices.data(), (int)devices.size()); });
  m.attr("TILE") = dr::kTile;
  m.attr("ARENA_HDR_WORDS") = dr::kArenaHdrWords;
  m.attr("SLOT_HEADER_WORDS") = dr::kSlotHeaderWords;
  m.attr("HIST_BINS") = dr::kHistBins;
  m.attr("NUM_HIST") = dr::kNumHist;
  m.attr("PH_END") = (int)dr::kPhEnd;

  py::class_<Engine>(m, "Engine")
      .def(py::init<int64_t, int64_t, int64_t, int64_t, int64_t, int64_t, int64_t, int64_t, int64_t, int64_t, int64_t,
                    int64_t, int64_t, int64_t, std::vector<int64_t>, int, int>())
      .def("configure", &Engine::configure)
      .def("set_buffers", &Engine::set_buffers)
      .def("set_poly", &Engine::set_poly)
      .def("set_shard", &Engine::set_shard)
      .def("set_has_rle", &Engine::set_has_rle)
      .def("set_scratch", &Engine::set_scratch)
      .def("set_peer_timeout_ms", &Engine::set_peer_timeout_ms)
      .def("set_fault", &Engine::set_fault)
      .def("set_deterministic", &Engine::set_deterministic)
      .def("set_cost_prefix", &Engine::set_cost_prefix)
      .def("set_debug_times", &Engine::set_debug_times)
      .def("set_cuts", &Engine::set_cuts)
      .def("set_grid_cap", &Engine::set_grid_cap)
      .def("set_multicast", &Engine::set_multicast)
      .def("grid", &Engine::get_grid)
      .def("run", &Engine::run);

  py::class_<Scheduler>(m, "Scheduler")
      .def(py::init<int>())
      .def("submit", &Scheduler::submit)
      .def("wait_all", &Scheduler::wait_all)
      .def("shutdown", &Scheduler::shutdown);
}
