// pybind11 bindings: at::Tensor <-> plain-C launch API (include/b200_ops.h). The only TU that includes torch headers.
#include <ATen/cuda/CUDAContext.h>
#include <ATen/cuda/CUDAGeneratorImpl.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <algorithm>
#include <atomic>
#include <optional>
#include <vector>

#include "include/b200_ops.h"
#include "runtime/runtime.h"
#include "runtime/tracer.h"

namespace {

std::atomic<int64_t> g_launches{0};

using torch::Tensor;
using OptT = std::optional<Tensor>;

int dt_code(const Tensor& t) {
  switch (t.scalar_type()) {
    case at::kFloat: return 0;
    case at::kHalf: return 1;
    case at::kBFloat16: return 2;
    default: TORCH_CHECK(false, "paddle_b200: unsupported dtype ", t.scalar_type());
  }
}
int dt_code(at::ScalarType st) {
  switch (st) {
    case at::kFloat: return 0;
    case at::kHalf: return 1;
    case at::kBFloat16: return 2;
    default: TORCH_CHECK(false, "paddle_b200: unsupported dtype ", st);
  }
}
cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }
void check_err() {
  const char* e = b200::take_last_error();
  TORCH_CHECK(e[0] == 0, "paddle_b200 kernel error: ", e);
}
const void* optp(const OptT& t) { return t.has_value() && t->defined() ? t->data_ptr() : nullptr; }
void check_cuda_contig(const Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor");
  TORCH_CHECK(t.is_contiguous(), name, " must be contiguous");
}

// ------------------------------------------------------------------------------------------------ norm
std::vector<Tensor> rms_norm_fwd(const Tensor& x, const OptT& residual, const OptT& w, const OptT& b, double eps) {
  check_cuda_contig(x, "x");
  c10::cuda::CUDAGuard guard(x.device());
  const int cols = (int)x.size(-1);
  const int64_t rows = x.numel() / cols;
  Tensor y = torch::empty_like(x);
  Tensor rstd = torch::empty({rows}, x.options().dtype(at::kFloat));
  Tensor res_out;
  if (residual.has_value() && residual->defined()) res_out = torch::empty_like(x);
  b200::rms_norm_fwd(x.data_ptr(), optp(residual), optp(w), optp(b), y.data_ptr(), res_out.defined() ? res_out.data_ptr() : nullptr,
                     rstd.data_ptr<float>(), rows, cols, (float)eps, dt_code(x), cur_stream());
  g_launches += 1;
  check_err();
  return {y, rstd, res_out.defined() ? res_out : Tensor()};
}

std::vector<Tensor> rms_norm_bwd(const Tensor& dy, const Tensor& x, const OptT& w, const Tensor& rstd) {
  check_cuda_contig(dy, "dy");
  check_cuda_contig(x, "x");
  c10::cuda::CUDAGuard guard(x.device());
  const int cols = (int)x.size(-1);
  const int64_t rows = x.numel() / cols;
  Tensor dx = torch::empty_like(x);
  const bool has_w = w.has_value() && w->defined();
  const int np = b200::norm_bwd_num_partials(rows);
  Tensor dwp, dw;
  if (has_w) dwp = torch::empty({np, cols}, x.options().dtype(at::kFloat));
  b200::rms_norm_bwd(dy.data_ptr(), x.data_ptr(), optp(w), rstd.data_ptr<float>(), dx.data_ptr(),
                     has_w ? dwp.data_ptr<float>() : nullptr, nullptr, rows, cols, dt_code(x), np, cur_stream());
  g_launches += 1;
  if (has_w) {
    dw = torch::empty_like(*w);
    b200::reduce_partials(dwp.data_ptr<float>(), dw.data_ptr(), np, cols, dt_code(*w), cur_stream());
    g_launches += 1;
  }
  check_err();
  return {dx, dw};
}

std::vector<Tensor> layer_norm_fwd(const Tensor& x, const OptT& w, const OptT& b, double eps) {
  check_cuda_contig(x, "x");
  c10::cuda::CUDAGuard guard(x.device());
  const int cols = (int)x.size(-1);
  const int64_t rows = x.numel() / cols;
  Tensor y = torch::empty_like(x);
  Tensor mean = torch::empty({rows}, x.options().dtype(at::kFloat));
  Tensor rstd = torch::empty({rows}, x.options().dtype(at::kFloat));
  b200::layer_norm_fwd(x.data_ptr(), optp(w), optp(b), y.data_ptr(), mean.data_ptr<float>(), rstd.data_ptr<float>(), rows, cols,
                       (float)eps, dt_code(x), cur_stream());
  g_launches += 1;
  check_err();
  return {y, mean, rstd};
}

std::vector<Tensor> layer_norm_bwd(const Tensor& dy, const Tensor& x, const OptT& w, const Tensor& mean, const Tensor& rstd, bool need_db) {
  check_cuda_contig(dy, "dy");
  check_cuda_contig(x, "x");
  c10::cuda::CUDAGuard guard(x.device());
  const int cols = (int)x.size(-1);
  const int64_t rows = x.numel() / cols;
  Tensor dx = torch::empty_like(x);
  const int np = b200::norm_bwd_num_partials(rows);
  Tensor dwp = torch::empty({np, cols}, x.options().dtype(at::kFloat));
  Tensor dbp = torch::empty({np, cols}, x.options().dtype(at::kFloat));
  b200::layer_norm_bwd(dy.data_ptr(), x.data_ptr(), optp(w), mean.data_ptr<float>(), rstd.data_ptr<float>(), dx.data_ptr(),
                       dwp.data_ptr<float>(), dbp.data_ptr<float>(), rows, cols, dt_code(x), np, cur_stream());
  auto pdt = (w.has_value() && w->defined()) ? w->scalar_type() : x.scalar_type();
  Tensor dw = torch::empty({cols}, x.options().dtype(pdt));
  Tensor db = torch::empty({cols}, x.options().dtype(pdt));
  b200::reduce_partials(dwp.data_ptr<float>(), dw.data_ptr(), np, cols, dt_code(pdt), cur_stream());
  b200::reduce_partials(dbp.data_ptr<float>(), db.data_ptr(), np, cols, dt_code(pdt), cur_stream());
  g_launches += 3;
  check_err();
  return {dx, dw, db};
}

// ------------------------------------------------------------------------------------------------ elementwise
// out = dropout(x + bias) (upscale_in_train) + y; returns (out, mask uint8).  seed / offset: Philox counter of this call
std::vector<Tensor> bias_dropout_add(const Tensor& x, const OptT& bias, const OptT& y, double p, bool upscale, int64_t seed, int64_t offset) {
  TORCH_CHECK(x.is_cuda() && x.is_contiguous() && x.dim() >= 1, "bias_dropout_add: contiguous CUDA tensor required");
  const int64_t cols = x.size(-1);
  if (bias.has_value() && bias->defined()) TORCH_CHECK(bias->is_contiguous() && bias->numel() == cols && bias->scalar_type() == x.scalar_type(), "bias_dropout_add: bias [cols] in x dtype");
  if (y.has_value() && y->defined()) TORCH_CHECK(y->is_contiguous() && y->numel() == x.numel() && y->scalar_type() == x.scalar_type(), "bias_dropout_add: y must match x");
  c10::cuda::CUDAGuard guard(x.device());
  Tensor out = torch::empty_like(x);
  Tensor mask = torch::empty(x.sizes(), x.options().dtype(at::kByte));
  b200::bias_dropout_add_fwd(x.data_ptr(), optp(bias), optp(y), out.data_ptr(), mask.data_ptr<uint8_t>(), x.numel(), (int)cols, (float)p, upscale ? 1 : 0, (uint64_t)seed,
                             (uint64_t)offset, dt_code(x), cur_stream());
  g_launches += 1;
  check_err();
  return {out, mask};
}

Tensor dropout_bwd(const Tensor& dout, const Tensor& mask, double p, bool upscale) {
  TORCH_CHECK(dout.is_cuda() && dout.is_contiguous() && mask.is_contiguous() && mask.scalar_type() == at::kByte && mask.numel() == dout.numel(), "dropout_bwd: dout + uint8 mask of the same size");
  c10::cuda::CUDAGuard guard(dout.device());
  Tensor dx = torch::empty_like(dout);
  b200::dropout_bwd(dout.data_ptr(), mask.data_ptr<uint8_t>(), dx.data_ptr(), dout.numel(), (float)p, upscale ? 1 : 0, dt_code(dout), cur_stream());
  g_launches += 1;
  check_err();
  return dx;
}

// act(x + bias): act 0 gelu / 1 relu / 2 silu; gated (swiglu / geglu): the second half of the row multiplies the activated first half
Tensor bias_act(const Tensor& x, const OptT& bias, int64_t act, bool gated) {
  TORCH_CHECK(x.is_cuda() && x.is_contiguous() && x.dim() >= 1, "bias_act: contiguous CUDA tensor required");
  const int64_t cols = x.size(-1), rows = x.numel() / cols;
  if (bias.has_value() && bias->defined()) TORCH_CHECK(bias->is_contiguous() && bias->numel() == cols && bias->scalar_type() == x.scalar_type(), "bias_act: bias [cols] in x dtype");
  c10::cuda::CUDAGuard guard(x.device());
  auto shape = x.sizes().vec();
  if (gated) shape.back() = cols / 2;
  Tensor out = torch::empty(shape, x.options());
  b200::bias_act_fwd(x.data_ptr(), optp(bias), out.data_ptr(), rows, (int)cols, (int)act, gated ? 1 : 0, dt_code(x), cur_stream());
  g_launches += 1;
  check_err();
  return out;
}

Tensor swiglu_fwd(const Tensor& gate, const OptT& up) {
  check_cuda_contig(gate, "gate");
  c10::cuda::CUDAGuard guard(gate.device());
  const bool packed = !(up.has_value() && up->defined());
  const int cols = packed ? (int)gate.size(-1) / 2 : (int)gate.size(-1);
  const int64_t rows = gate.numel() / gate.size(-1);
  auto sizes = gate.sizes().vec();
  sizes.back() = cols;
  Tensor out = torch::empty(sizes, gate.options());
  b200::swiglu_fwd(gate.data_ptr(), optp(up), out.data_ptr(), rows, cols, dt_code(gate), cur_stream());
  g_launches += 1;
  check_err();
  return out;
}

std::vector<Tensor> swiglu_bwd(const Tensor& dout, const Tensor& gate, const OptT& up) {
  check_cuda_contig(dout, "dout");
  c10::cuda::CUDAGuard guard(gate.device());
  const bool packed = !(up.has_value() && up->defined());
  const int cols = packed ? (int)gate.size(-1) / 2 : (int)gate.size(-1);
  const int64_t rows = gate.numel() / gate.size(-1);
  Tensor dgate = torch::empty_like(gate);
  Tensor dup;
  if (!packed) dup = torch::empty_like(*up);
  b200::swiglu_bwd(dout.data_ptr(), gate.data_ptr(), optp(up), dgate.data_ptr(), packed ? nullptr : dup.data_ptr(), rows, cols,
                   dt_code(gate), cur_stream());
  g_launches += 1;
  check_err();
  return {dgate, dup};
}

Tensor rope(const Tensor& x, const Tensor& cos_t, const Tensor& sin_t, const OptT& pos_ids, int64_t seq, bool neox, bool backward) {
  check_cuda_contig(x, "x");
  TORCH_CHECK(x.dim() >= 3, "rope expects [..., seq, heads, dim]");
  c10::cuda::CUDAGuard guard(x.device());
  const int dim = (int)x.size(-1), heads = (int)x.size(-2);
  const int64_t tokens = x.numel() / ((int64_t)dim * heads);
  Tensor y = torch::empty_like(x);
  const int64_t* pid = nullptr;
  Tensor pos;
  if (pos_ids.has_value() && pos_ids->defined()) {
    pos = pos_ids->to(at::kLong).contiguous();
    pid = pos.data_ptr<int64_t>();
  }
  b200::rope_apply(x.data_ptr(), y.data_ptr(), cos_t.data_ptr<float>(), sin_t.data_ptr<float>(), pid, tokens, (int)seq, heads, dim,
                   neox ? 1 : 0, backward ? 1 : 0, dt_code(x), 0, cur_stream());
  g_launches += 1;
  check_err();
  return y;
}

// In-place rotary on the first `rope_heads` heads of a packed [tokens, total_heads, dim] tensor (fused QKV: q and k heads
// rotate, v heads are left untouched) -> no split/concat copies around the attention.
void rope_packed_(Tensor x, const Tensor& cos_t, const Tensor& sin_t, const OptT& pos_ids, int64_t seq, int64_t rope_heads,
                  int64_t total_heads, int64_t dim, bool neox, bool backward) {
  check_cuda_contig(x, "x");
  c10::cuda::CUDAGuard guard(x.device());
  const int64_t tokens = x.numel() / (total_heads * dim);
  const int64_t* pid = nullptr;
  Tensor pos;
  if (pos_ids.has_value() && pos_ids->defined()) {
    pos = pos_ids->to(at::kLong).contiguous();
    pid = pos.data_ptr<int64_t>();
  }
  b200::rope_apply(x.data_ptr(), x.data_ptr(), cos_t.data_ptr<float>(), sin_t.data_ptr<float>(), pid, tokens, (int)seq, (int)rope_heads,
                   (int)dim, neox ? 1 : 0, backward ? 1 : 0, dt_code(x), total_heads * dim, cur_stream());
  g_launches += 1;
  check_err();
}

// ------------------------------------------------------------------------------------------------ loss
std::vector<Tensor> softmax_ce_fwd(const Tensor& logits, const Tensor& labels, int64_t ignore_index) {
  check_cuda_contig(logits, "logits");
  c10::cuda::CUDAGuard guard(logits.device());
  const int vocab = (int)logits.size(-1);
  const int64_t rows = logits.numel() / vocab;
  Tensor lab = labels.to(at::kLong).contiguous();
  Tensor loss = torch::empty({rows}, logits.options().dtype(at::kFloat));
  Tensor lse = torch::empty({rows}, logits.options().dtype(at::kFloat));
  b200::softmax_ce_fwd(logits.data_ptr(), lab.data_ptr<int64_t>(), loss.data_ptr<float>(), lse.data_ptr<float>(), rows, vocab,
                       ignore_index, dt_code(logits), cur_stream());
  g_launches += 1;
  check_err();
  return {loss, lse};
}

Tensor softmax_ce_bwd(const Tensor& logits, const Tensor& labels, const Tensor& lse, const Tensor& dloss, int64_t ignore_index, bool inplace) {
  check_cuda_contig(logits, "logits");
  c10::cuda::CUDAGuard guard(logits.device());
  const int vocab = (int)logits.size(-1);
  const int64_t rows = logits.numel() / vocab;
  Tensor lab = labels.to(at::kLong).contiguous();
  Tensor dl = dloss.to(at::kFloat).contiguous();
  Tensor out = inplace ? logits : torch::empty_like(logits);
  b200::softmax_ce_bwd(logits.data_ptr(), lab.data_ptr<int64_t>(), lse.data_ptr<float>(), dl.data_ptr<float>(), out.data_ptr(), rows,
                       vocab, ignore_index, dt_code(logits), cur_stream());
  g_launches += 1;
  check_err();
  return out;
}

Tensor vp_ce_max(const Tensor& logits) {
  check_cuda_contig(logits, "logits");
  c10::cuda::CUDAGuard guard(logits.device());
  const int vocab = (int)logits.size(-1);
  const int64_t rows = logits.numel() / vocab;
  Tensor mx = torch::empty({rows}, logits.options().dtype(at::kFloat));
  b200::vocab_parallel_ce_stats(logits.data_ptr(), nullptr, mx.data_ptr<float>(), rows, vocab, dt_code(logits), cur_stream());
  g_launches += 1;
  check_err();
  return mx;
}

std::vector<Tensor> vp_ce_sumexp(const Tensor& logits, const Tensor& labels, const Tensor& row_max, int64_t vocab_start) {
  c10::cuda::CUDAGuard guard(logits.device());
  const int vocab = (int)logits.size(-1);
  const int64_t rows = logits.numel() / vocab;
  Tensor lab = labels.to(at::kLong).contiguous();
  Tensor se = torch::empty({rows}, logits.options().dtype(at::kFloat));
  Tensor tl = torch::empty({rows}, logits.options().dtype(at::kFloat));
  b200::vocab_parallel_ce_sumexp(logits.data_ptr(), lab.data_ptr<int64_t>(), row_max.data_ptr<float>(), se.data_ptr<float>(),
                                 tl.data_ptr<float>(), rows, vocab, vocab_start, dt_code(logits), cur_stream());
  g_launches += 1;
  check_err();
  return {se, tl};
}

Tensor vp_ce_bwd(const Tensor& logits, const Tensor& labels, const Tensor& row_max, const Tensor& sumexp, const Tensor& dloss,
                 int64_t vocab_start, int64_t ignore_index, bool inplace) {
  c10::cuda::CUDAGuard guard(logits.device());
  const int vocab = (int)logits.size(-1);
  const int64_t rows = logits.numel() / vocab;
  Tensor lab = labels.to(at::kLong).contiguous();
  Tensor dl = dloss.to(at::kFloat).contiguous();
  Tensor out = inplace ? logits : torch::empty_like(logits);
  b200::vocab_parallel_ce_bwd(logits.data_ptr(), lab.data_ptr<int64_t>(), row_max.data_ptr<float>(), sumexp.data_ptr<float>(),
                              dl.data_ptr<float>(), out.data_ptr(), rows, vocab, vocab_start, ignore_index, dt_code(logits), cur_stream());
  g_launches += 1;
  check_err();
  return out;
}

// ------------------------------------------------------------------------------------------------ optimizer
static void adamw_step_impl(Tensor p, const Tensor& g, const OptT& master, Tensor m, Tensor v, double lr, double beta1, double beta2, double eps,
                            double weight_decay, int64_t step, const OptT& grad_sq_norm, double max_norm, const OptT& found_inf, const OptT& inv_scale,
                            const OptT& dyn) {
  check_cuda_contig(p, "param");
  check_cuda_contig(g, "grad");
  c10::cuda::CUDAGuard guard(p.device());
  b200::AdamWArgs a;
  a.lr = (float)lr; a.beta1 = (float)beta1; a.beta2 = (float)beta2; a.eps = (float)eps; a.weight_decay = (float)weight_decay;
  a.bias_c1 = (float)(1.0 - std::pow(beta1, (double)step));
  a.bias_c2 = (float)(1.0 - std::pow(beta2, (double)step));
  a.grad_sq_norm = (const float*)optp(grad_sq_norm);
  a.max_norm = (float)max_norm;
  a.found_inf = (const float*)optp(found_inf);
  a.inv_scale = (const float*)optp(inv_scale);
  a.dyn = (const float*)optp(dyn);
  if (a.dyn) TORCH_CHECK(dyn->scalar_type() == at::kFloat && dyn->numel() >= 3 && dyn->is_cuda(), "adamw dyn hparams: float32 CUDA tensor of 3");
  float* mp = nullptr;
  int16_t* lo = nullptr;
  if (master.has_value() && master->defined()) {
    TORCH_CHECK(master->numel() == p.numel() && master->is_cuda() && master->is_contiguous(), "adamw: master weights must match the parameter slab");
    if (master->scalar_type() == at::kShort) lo = master->data_ptr<int16_t>();      // split master: bf16 parameter + int16 residual
    else mp = master->data_ptr<float>();
  }
  b200::adamw_step(p.data_ptr(), g.data_ptr(), mp, m.data_ptr(), v.data_ptr(), p.numel(), dt_code(p), dt_code(g), dt_code(m), a, cur_stream(), lo);
  g_launches += 1;
  check_err();
}

void adamw_step(Tensor p, const Tensor& g, const OptT& master, Tensor m, Tensor v, double lr, double beta1, double beta2, double eps,
                double weight_decay, int64_t step, const OptT& grad_sq_norm, double max_norm, const OptT& found_inf, const OptT& inv_scale) {
  adamw_step_impl(p, g, master, m, v, lr, beta1, beta2, eps, weight_decay, step, grad_sq_norm, max_norm, found_inf, inv_scale, std::nullopt);
}

// Graph-capturable form: lr and the bias corrections come from the device tensor `dyn` = {lr, 1-b1^t, 1-b2^t}; `lr_mult` scales dyn[0].
void adamw_step_dyn(Tensor p, const Tensor& g, const OptT& master, Tensor m, Tensor v, double lr_mult, double beta1, double beta2, double eps,
                    double weight_decay, const OptT& grad_sq_norm, double max_norm, const OptT& found_inf, const OptT& inv_scale, const Tensor& dyn) {
  adamw_step_impl(p, g, master, m, v, lr_mult, beta1, beta2, eps, weight_decay, 1, grad_sq_norm, max_norm, found_inf, inv_scale, dyn);
}

void grad_sq_norm(const Tensor& g, Tensor out, const OptT& found_inf) {
  check_cuda_contig(g, "grad");
  c10::cuda::CUDAGuard guard(g.device());
  float* fi = found_inf.has_value() && found_inf->defined() ? found_inf->data_ptr<float>() : nullptr;
  b200::grad_sq_norm(g.data_ptr(), g.numel(), dt_code(g), out.data_ptr<float>(), fi, cur_stream());
  g_launches += 1;
  check_err();
}

void scale_inplace(Tensor g, const OptT& scale_dev, double scale_host) {
  check_cuda_contig(g, "tensor");
  c10::cuda::CUDAGuard guard(g.device());
  b200::scale_inplace(g.data_ptr(), g.numel(), dt_code(g), (const float*)optp(scale_dev), (float)scale_host, cur_stream());
  g_launches += 1;
  check_err();
}

void sgd_step(Tensor p, const Tensor& g, const OptT& master, const OptT& mom, double lr, double momentum, double wd, bool nesterov) {
  check_cuda_contig(p, "param");
  c10::cuda::CUDAGuard guard(p.device());
  float* mp = master.has_value() && master->defined() ? master->data_ptr<float>() : nullptr;
  void* mo = mom.has_value() && mom->defined() ? mom->data_ptr() : nullptr;
  b200::sgd_momentum_step(p.data_ptr(), g.data_ptr(), mp, mo, p.numel(), dt_code(p), dt_code(g), (float)lr, (float)momentum, (float)wd,
                          nesterov ? 1 : 0, cur_stream());
  g_launches += 1;
  check_err();
}

void lamb_step(Tensor p, const Tensor& g, const OptT& master, Tensor m, Tensor v, double lr, double beta1, double beta2, double eps,
               double wd, int64_t step) {
  check_cuda_contig(p, "param");
  c10::cuda::CUDAGuard guard(p.device());
  Tensor upd = torch::empty({p.numel()}, p.options().dtype(at::kFloat));
  Tensor sq = torch::zeros({2}, p.options().dtype(at::kFloat));
  const float* mp = master.has_value() && master->defined() ? master->data_ptr<float>() : nullptr;
  b200::lamb_stage1(p.data_ptr(), g.data_ptr(), mp, m.data_ptr(), v.data_ptr(), upd.data_ptr<float>(), p.numel(), dt_code(p), dt_code(g),
                    (float)beta1, (float)beta2, (float)eps, (float)wd, (float)(1.0 - std::pow(beta1, (double)step)),
                    (float)(1.0 - std::pow(beta2, (double)step)), sq.data_ptr<float>(), sq.data_ptr<float>() + 1, cur_stream());
  b200::lamb_stage2(p.data_ptr(), const_cast<float*>(mp), upd.data_ptr<float>(), p.numel(), dt_code(p), (float)lr, sq.data_ptr<float>(),
                    sq.data_ptr<float>() + 1, cur_stream());
  g_launches += 2;
  check_err();
}

// ------------------------------------------------------------------------------------------------ gemm
// a: [.., M, K] (or [.., K, M] when a_is_km); b: [.., N, K] when b_is_nk else [.., K, N]. Last-dim stride must be 1.
bool gemm_supported(const Tensor& a, const Tensor& b, bool a_is_km, bool b_is_nk) {
  if (!a.is_cuda() || a.scalar_type() != b.scalar_type()) return false;
  if (a.scalar_type() != at::kBFloat16 && a.scalar_type() != at::kHalf) return false;
  if (a.dim() < 2 || b.dim() < 2 || a.dim() > 3 || b.dim() != a.dim()) return false;
  if (a.stride(-1) != 1 || b.stride(-1) != 1) return false;
  const int64_t m = a_is_km ? a.size(-1) : a.size(-2), k = a_is_km ? a.size(-2) : a.size(-1);
  const int64_t n = b_is_nk ? b.size(-2) : b.size(-1), kb = b_is_nk ? b.size(-1) : b.size(-2);
  if (k != kb) return false;
  if (a.dim() == 3 && (a.size(0) != b.size(0) || a.stride(0) % 8 || b.stride(0) % 8)) return false;
  if ((reinterpret_cast<uintptr_t>(a.data_ptr()) & 15) || (reinterpret_cast<uintptr_t>(b.data_ptr()) & 15)) return false;
  return b200::gemm_tcgen05_supported((int)m, (int)n, (int)k, a.stride(-2), b.stride(-2), n, a_is_km, b_is_nk) != 0;
}

Tensor gemm(const Tensor& a, const Tensor& b, const OptT& bias, bool a_is_km, bool b_is_nk, int64_t epilogue, const OptT& out,
            const std::optional<at::ScalarType>& out_dtype, const std::vector<int64_t>& rs_dst, int64_t rs_rows,
            const std::vector<int64_t>& ag_src, const std::vector<int64_t>& ag_pad, const OptT& ag_flags, int64_t ag_rank, int64_t ag_rows,
            int64_t ag_epoch) {
  TORCH_CHECK(gemm_supported(a, b, a_is_km, b_is_nk), "paddle_b200.gemm: unsupported operands for the tcgen05 path");
  c10::cuda::CUDAGuard guard(a.device());
  b200::GemmArgs g;
  g.m = (int)(a_is_km ? a.size(-1) : a.size(-2));
  g.k = (int)(a_is_km ? a.size(-2) : a.size(-1));
  g.n = (int)(b_is_nk ? b.size(-2) : b.size(-1));
  g.batch = a.dim() == 3 ? (int)a.size(0) : 1;
  Tensor d;
  if (out.has_value() && out->defined()) {
    d = *out;
    TORCH_CHECK(d.stride(-1) == 1, "gemm: out must have unit inner stride");
  } else {
    auto od = out_dtype.has_value() ? *out_dtype : a.scalar_type();
    d = g.batch > 1 ? torch::empty({g.batch, g.m, g.n}, a.options().dtype(od)) : torch::empty({g.m, g.n}, a.options().dtype(od));
  }
  g.a = a.data_ptr(); g.b = b.data_ptr(); g.d = d.data_ptr();
  g.bias = optp(bias);
  g.lda = a.stride(-2); g.ldb = b.stride(-2); g.ldd = d.stride(-2);
  g.a_is_km = a_is_km; g.b_is_nk = b_is_nk;
  g.epilogue = (int)epilogue;
  g.dtype = dt_code(a);
  g.out_dtype = dt_code(d);
  g.stride_a = a.dim() == 3 ? a.stride(0) : 0;
  g.stride_b = b.dim() == 3 ? b.stride(0) : 0;
  g.stride_d = d.dim() == 3 ? d.stride(0) : 0;
  if (!rs_dst.empty()) {   // fused reduce-scatter: rows are pushed into the owners' staging slots, `d` is not written
    TORCH_CHECK(g.batch == 1 && rs_dst.size() <= 8 && rs_rows > 0 && (int64_t)g.m == rs_rows * (int64_t)rs_dst.size() && g.n % 8 == 0,
                "gemm: bad reduce-scatter push arguments");
    g.rs_world = (int)rs_dst.size();
    g.rs_rows = (int)rs_rows;
    for (size_t i = 0; i < rs_dst.size(); ++i) g.rs_dst[i] = reinterpret_cast<void*>(rs_dst[i]);
  }
  if (!ag_src.empty()) {   // fused all-gather of the A rows (see GemmArgs)
    TORCH_CHECK(ag_src.size() <= 8 && ag_pad.size() == ag_src.size() && ag_flags.has_value() && ag_flags->defined() && !a_is_km &&
                a.is_contiguous() && ag_rows > 0, "gemm: bad fused all-gather arguments");
    g.ag_world = (int)ag_src.size(); g.ag_rank = (int)ag_rank; g.ag_rows = (int)ag_rows; g.ag_epoch = (uint32_t)ag_epoch;
    for (size_t i = 0; i < ag_src.size(); ++i) { g.ag_src[i] = reinterpret_cast<const void*>(ag_src[i]); g.ag_pad[i] = reinterpret_cast<void*>(ag_pad[i]); }
    g.ag_flags = ag_flags->data_ptr();
  }
  if (g.bias) TORCH_CHECK(bias->scalar_type() == a.scalar_type() || bias->scalar_type() == at::kFloat, "gemm: bias dtype");
  if (g.bias && bias->scalar_type() == at::kFloat && a.scalar_type() != at::kFloat) {
    // epilogue reads bias in the input dtype
    Tensor bb = bias->to(a.scalar_type());
    g.bias = bb.data_ptr();
    int rc = b200::gemm_tcgen05(g, cur_stream());
    g_launches += 1;
    check_err();
    TORCH_CHECK(rc == 0, "paddle_b200.gemm launch failed rc=", rc);
    return d;
  }
  int rc = b200::gemm_tcgen05(g, cur_stream());
  g_launches += 1;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.gemm launch failed rc=", rc);
  return d;
}

// Grouped GEMM over stacked expert weights (see GemmArgs::grouped == 1): a [Mpad, K] rows grouped by expert in 256-row aligned
// segments, b [E, K, N] (or [E, N, K] with b_is_nk), tile_expert int32 [Mpad / 256] -> out [Mpad, N].
Tensor gemm_grouped(const Tensor& a, const Tensor& b, const Tensor& tile_expert, bool b_is_nk, const OptT& out) {
  TORCH_CHECK(a.is_cuda() && a.dim() == 2 && b.dim() == 3 && a.is_contiguous() && b.is_contiguous() && a.scalar_type() == b.scalar_type(),
              "gemm_grouped: a [M,K] and stacked b [E,*,*] contiguous, same dtype");
  TORCH_CHECK(a.scalar_type() == at::kBFloat16 || a.scalar_type() == at::kHalf, "gemm_grouped: bf16 / fp16 only");
  const int64_t m = a.size(0), k = a.size(1), n = b_is_nk ? b.size(1) : b.size(2), kb = b_is_nk ? b.size(2) : b.size(1);
  TORCH_CHECK(k == kb && m % 256 == 0 && m >= 256 && n >= 256 && k % 8 == 0 && n % 8 == 0, "gemm_grouped: M multiple of 256, N >= 256, K/N multiples of 8");
  TORCH_CHECK(tile_expert.is_cuda() && tile_expert.scalar_type() == at::kInt && tile_expert.numel() == m / 256 && tile_expert.is_contiguous(),
              "gemm_grouped: tile_expert must be int32 [M / 256] on the device");
  c10::cuda::CUDAGuard guard(a.device());
  Tensor d = out.has_value() && out->defined() ? *out : torch::empty({m, n}, a.options());
  TORCH_CHECK(d.is_contiguous() && d.size(0) == m && d.size(1) == n, "gemm_grouped: out must be [M, N] contiguous");
  b200::GemmArgs g;
  g.m = (int)m; g.n = (int)n; g.k = (int)k; g.batch = 1;
  g.a = a.data_ptr(); g.b = b.data_ptr(); g.d = d.data_ptr(); g.bias = nullptr;
  g.lda = k; g.ldb = b.stride(1); g.ldd = n;
  g.a_is_km = 0; g.b_is_nk = b_is_nk; g.epilogue = 0; g.dtype = dt_code(a); g.out_dtype = dt_code(d);
  g.stride_a = 0; g.stride_b = b.stride(0); g.stride_d = 0;
  g.grouped = 1; g.groups = (int)b.size(0); g.tile_expert = tile_expert.data_ptr<int>();
  int rc = b200::gemm_tcgen05(g, cur_stream());
  g_launches += 1;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.gemm_grouped launch failed rc=", rc);
  return d;
}

// Per-expert weight gradients (GemmArgs::grouped == 2): out[e] += x[rows_e]^T @ dy[rows_e]; x [R, K_in], dy [R, N], out [E, K_in, N];
// expert_k0 / expert_kb int32 [E] = first row and number of 64-row blocks of every expert's (padded) segment.
void gemm_grouped_wgrad(const Tensor& x, const Tensor& dy, const Tensor& expert_k0, const Tensor& expert_kb, Tensor out) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && dy.dim() == 2 && x.is_contiguous() && dy.is_contiguous() && x.size(0) == dy.size(0) &&
              x.scalar_type() == dy.scalar_type(), "gemm_grouped_wgrad: x [R,K] and dy [R,N] contiguous, same dtype");
  TORCH_CHECK(out.dim() == 3 && out.is_contiguous() && out.size(1) == x.size(1) && out.size(2) == dy.size(1), "gemm_grouped_wgrad: out must be [E, K, N]");
  TORCH_CHECK(expert_k0.scalar_type() == at::kInt && expert_kb.scalar_type() == at::kInt && expert_k0.numel() == out.size(0) && expert_kb.numel() == out.size(0) &&
              expert_k0.is_cuda() && expert_kb.is_cuda(), "gemm_grouped_wgrad: expert_k0 / expert_kb int32 [E] on the device");
  TORCH_CHECK(x.size(1) >= 256 && dy.size(1) >= 256 && x.size(1) % 8 == 0 && dy.size(1) % 8 == 0 && x.size(0) % 64 == 0, "gemm_grouped_wgrad: shapes");
  c10::cuda::CUDAGuard guard(x.device());
  b200::GemmArgs g;
  g.m = (int)x.size(1); g.n = (int)dy.size(1); g.k = (int)x.size(0); g.batch = 1;
  g.a = x.data_ptr(); g.b = dy.data_ptr(); g.d = out.data_ptr(); g.bias = nullptr;
  g.lda = x.size(1); g.ldb = dy.size(1); g.ldd = out.size(2);
  g.a_is_km = 1; g.b_is_nk = 0; g.epilogue = 4; g.dtype = dt_code(x); g.out_dtype = dt_code(out);
  g.stride_a = 0; g.stride_b = 0; g.stride_d = out.stride(0);
  g.grouped = 2; g.groups = (int)out.size(0); g.expert_k0 = expert_k0.data_ptr<int>(); g.expert_kb = expert_kb.data_ptr<int>();
  int rc = b200::gemm_tcgen05(g, cur_stream());
  g_launches += 1;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.gemm_grouped_wgrad launch failed rc=", rc);
}

// ------------------------------------------------------------------------------------------------ MoE routing (csrc/moe.cu)
static void check_i64(const Tensor& t, const char* what) {
  TORCH_CHECK(t.is_cuda() && t.is_contiguous() && t.scalar_type() == at::kLong, what, ": int64 CUDA contiguous tensor expected");
}
Tensor moe_number_count(const Tensor& idx, int64_t upper) {
  check_i64(idx, "number_count");
  c10::cuda::CUDAGuard guard(idx.device());
  Tensor counts = torch::zeros({upper}, idx.options());
  b200::moe_number_count(idx.data_ptr<int64_t>(), idx.numel(), counts.data_ptr<int64_t>(), (int)upper, cur_stream());
  g_launches += 1; check_err();
  return counts;
}
Tensor moe_assign_pos(const Tensor& idx, const Tensor& cum_count, int64_t n_valid) {
  check_i64(idx, "assign_pos"); check_i64(cum_count, "assign_pos");
  c10::cuda::CUDAGuard guard(idx.device());
  Tensor cursor = cum_count.clone();
  Tensor pos = torch::empty({n_valid}, idx.options());
  b200::moe_assign_pos(idx.data_ptr<int64_t>(), idx.numel(), cursor.data_ptr<int64_t>(), pos.data_ptr<int64_t>(), cur_stream());
  g_launches += 1; check_err();
  return pos;
}
Tensor moe_limit_by_capacity(const Tensor& expert_count, const Tensor& capacity, int64_t n_worker) {
  check_i64(expert_count, "limit_by_capacity"); check_i64(capacity, "limit_by_capacity");
  c10::cuda::CUDAGuard guard(expert_count.device());
  const int n_expert = (int)capacity.numel();
  TORCH_CHECK(expert_count.numel() == n_expert * n_worker, "limit_by_capacity: expert_count must hold n_worker * n_expert entries");
  Tensor out = torch::empty_like(expert_count);
  b200::moe_limit_by_capacity(expert_count.data_ptr<int64_t>(), capacity.data_ptr<int64_t>(), out.data_ptr<int64_t>(), n_expert, (int)n_worker, cur_stream());
  g_launches += 1; check_err();
  return out;
}
Tensor moe_prune_gate_by_capacity(const Tensor& gate_idx, const Tensor& expert_count) {
  check_i64(gate_idx, "prune_gate_by_capacity"); check_i64(expert_count, "prune_gate_by_capacity");
  c10::cuda::CUDAGuard guard(gate_idx.device());
  Tensor remaining = expert_count.clone();
  Tensor out = torch::empty_like(gate_idx);
  b200::moe_prune_gate(gate_idx.data_ptr<int64_t>(), gate_idx.numel(), remaining.data_ptr<int64_t>(), out.data_ptr<int64_t>(), cur_stream());
  g_launches += 1; check_err();
  return out;
}
// expert ids of the token slots ([S] int64, -1 = dropped) -> (dest int32 [S], tile_expert int32 [MT], expert_k0 int32 [E], expert_kb int32 [E],
// seg_start int32 [E+1], counts int64 [E]); rows_cap = static upper bound of the padded row count (multiple of 256)
std::vector<Tensor> moe_route(const Tensor& idx, int64_t n_expert, int64_t rows_cap) {
  check_i64(idx, "moe_route");
  TORCH_CHECK(rows_cap % 256 == 0 && rows_cap > 0, "moe_route: rows_cap must be a positive multiple of 256");
  c10::cuda::CUDAGuard guard(idx.device());
  auto i32 = idx.options().dtype(at::kInt);
  Tensor counts = torch::zeros({n_expert}, idx.options());
  Tensor dest = torch::empty({idx.numel()}, i32), tile_expert = torch::empty({rows_cap / 256}, i32);
  Tensor k0 = torch::empty({n_expert}, i32), kb = torch::empty({n_expert}, i32), seg = torch::empty({n_expert + 1}, i32), cursor = torch::empty({n_expert}, i32);
  auto st = cur_stream();
  b200::moe_number_count(idx.data_ptr<int64_t>(), idx.numel(), counts.data_ptr<int64_t>(), (int)n_expert, st);
  b200::moe_plan(counts.data_ptr<int64_t>(), (int)n_expert, (int)(rows_cap / 256), seg.data_ptr<int>(), cursor.data_ptr<int>(), tile_expert.data_ptr<int>(),
                 k0.data_ptr<int>(), kb.data_ptr<int>(), st);
  b200::moe_dest(idx.data_ptr<int64_t>(), idx.numel(), cursor.data_ptr<int>(), dest.data_ptr<int>(), st);
  g_launches += 3; check_err();
  return {dest, tile_expert, k0, kb, seg, counts};
}
Tensor moe_rows_scatter(const Tensor& src, const Tensor& dest, const OptT& scale, int64_t topk, int64_t rows_out) {
  TORCH_CHECK(src.is_cuda() && src.dim() == 2 && src.is_contiguous() && dest.scalar_type() == at::kInt && dest.is_contiguous(), "moe_rows_scatter: bad operands");
  c10::cuda::CUDAGuard guard(src.device());
  Tensor dst = torch::zeros({rows_out, src.size(1)}, src.options());
  const float* sc = scale.has_value() && scale->defined() ? scale->data_ptr<float>() : nullptr;
  b200::moe_rows_scatter(src.data_ptr(), dest.data_ptr<int>(), sc, dest.numel(), (int)topk, (int)src.size(1), dst.data_ptr(), dt_code(src), cur_stream());
  g_launches += 1; check_err();
  return dst;
}
Tensor moe_rows_combine(const Tensor& src, const Tensor& dest, const OptT& w, int64_t topk) {
  TORCH_CHECK(src.is_cuda() && src.dim() == 2 && src.is_contiguous() && dest.scalar_type() == at::kInt && dest.is_contiguous() && dest.numel() % topk == 0,
              "moe_rows_combine: bad operands");
  c10::cuda::CUDAGuard guard(src.device());
  const int64_t n_tok = dest.numel() / topk;
  Tensor out = torch::empty({n_tok, src.size(1)}, src.options());
  const float* wp = w.has_value() && w->defined() ? w->data_ptr<float>() : nullptr;
  b200::moe_rows_combine(src.data_ptr(), dest.data_ptr<int>(), wp, n_tok, (int)topk, (int)src.size(1), out.data_ptr(), dt_code(src), cur_stream());
  g_launches += 1; check_err();
  return out;
}
Tensor moe_rows_dot(const Tensor& src, const Tensor& dest, const Tensor& g, int64_t topk) {
  TORCH_CHECK(src.is_cuda() && src.is_contiguous() && g.is_contiguous() && src.scalar_type() == g.scalar_type() && src.size(1) == g.size(1), "moe_rows_dot: bad operands");
  c10::cuda::CUDAGuard guard(src.device());
  Tensor dw = torch::empty({dest.numel()}, src.options().dtype(at::kFloat));
  b200::moe_rows_dot(src.data_ptr(), dest.data_ptr<int>(), g.data_ptr(), dest.numel(), (int)topk, (int)src.size(1), dw.data_ptr<float>(), dt_code(src), cur_stream());
  g_launches += 1; check_err();
  return dw;
}

// ---- weight-only GEMM and dequantisation.  Failing checks use literal messages only: with this extension's host toolchain a failing
// TORCH_CHECK that formats an integer aborts instead of raising.  experts: every weight operand carries a leading [E].

// w int8 [N, K] (int4 packed [N, K/2]) contiguous and non-empty on a CUDA device, and its scales fp32 [N] per channel (group_size <= 0)
// or [K / group_size, N], contiguous on w's device.  Messages name `op`.  Returns K.
int64_t check_wo_weight(const char* op, const Tensor& w, const Tensor& scale, bool int4, int64_t group_size, bool experts) {
  const char* lead = experts ? "E, " : "";
  TORCH_CHECK(w.is_cuda() && w.dim() == (experts ? 3 : 2) && w.is_contiguous() && w.scalar_type() == at::kChar && w.numel() > 0,
              op, ": w int8 [", lead, "N, K] (int4: [", lead, "N, K/2]) contiguous");
  const int64_t n = w.size(-2), k = int4 ? 2 * w.size(-1) : w.size(-1);
  const bool scale_ok = scale.scalar_type() == at::kFloat && scale.is_contiguous();
  if (group_size <= 0) {
    TORCH_CHECK(scale_ok && (experts ? scale.dim() == 2 && scale.size(0) == w.size(0) && scale.size(1) == n : scale.numel() == n),
                op, ": scale float32 [", lead, "N] contiguous");
  } else {
    TORCH_CHECK(k % group_size == 0, op, ": K is not a multiple of group_size");
    TORCH_CHECK(scale_ok && scale.dim() == (experts ? 3 : 2) && (!experts || scale.size(0) == w.size(0)) && scale.size(-2) == k / group_size &&
                scale.size(-1) == n, op, ": scale float32 [", lead, "K / group_size, N] contiguous");
  }
  TORCH_CHECK(scale.device() == w.device(), op, ": w and scale on one device");
  return k;
}

// The operands of weight_only_gemm and weight_only_gemm_experts: x [M, K] bf16 / fp16 contiguous on a CUDA device, w and scale as in
// check_wo_weight with group_size -1, 64 or 128, bias [N] in x's dtype or None, every operand on x's device, and E, N, K, M in range.
void check_wo_operands(const char* op, const Tensor& x, const Tensor& w, const Tensor& scale, const OptT& bias, bool int4, int64_t group_size,
                       bool experts) {
  const char* lead = experts ? "E, " : "";
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.is_contiguous() && (x.scalar_type() == at::kBFloat16 || x.scalar_type() == at::kHalf),
              op, ": x [M, K] bf16 / fp16 contiguous");
  TORCH_CHECK(group_size <= 0 || group_size == 64 || group_size == 128, op, ": group_size must be -1, 64 or 128");
  const int64_t K = check_wo_weight(op, w, scale, int4, group_size, experts), N = w.size(-2), E = experts ? w.size(0) : 1;
  TORCH_CHECK(x.size(1) == K, op, ": x [M, K] and w [", lead, "N, K] (int4: [", lead, "N, K/2]) disagree on K");
  TORCH_CHECK(E <= 1024 && K < (int64_t)1 << 30 && N < (int64_t)1 << 30 && x.size(0) > 0 && x.size(0) < (int64_t)1 << 30, op, ": dimensions out of range");
  if (bias.has_value() && bias->defined())
    TORCH_CHECK(bias->is_cuda() && bias->scalar_type() == x.scalar_type() && bias->numel() == E * N && bias->is_contiguous(),
                op, ": bias [", lead, "N] contiguous CUDA tensor in x dtype");
  TORCH_CHECK(w.device() == x.device() && (!bias.has_value() || !bias->defined() || bias->device() == x.device()), op, ": all operands on one device");
}

// the arguments of gemm_weight_only for checked operands; the expert binding adds its plan
b200::WoGemmArgs wo_gemm_args(const Tensor& x, const Tensor& w, const Tensor& scale, const OptT& bias, const Tensor& out, bool int4, int64_t group_size) {
  b200::WoGemmArgs g;
  g.m = (int)x.size(0); g.k = (int)x.size(1); g.n = (int)w.size(-2);
  g.x = x.data_ptr(); g.w = w.data_ptr(); g.scale = scale.data_ptr<float>(); g.out = out.data_ptr();
  g.bias = bias.has_value() && bias->defined() ? bias->data_ptr() : nullptr;
  g.int4 = int4 ? 1 : 0; g.bf16 = x.scalar_type() == at::kBFloat16 ? 1 : 0;
  g.group_size = group_size > 0 ? (int)group_size : 0;
  return g;
}

// x [M, K] bf16 / fp16, w int8 [N, K] (or int4 packed [N, K/2]), scale float [N] (group_size <= 0) or [K / group_size, N] (64 / 128),
// bias [N] or None -> [M, N]
Tensor weight_only_gemm(const Tensor& x, const Tensor& w, const Tensor& scale, const OptT& bias, bool int4, int64_t group_size) {
  check_wo_operands("weight_only_gemm", x, w, scale, bias, int4, group_size, false);
  c10::cuda::CUDAGuard guard(x.device());
  Tensor out = torch::empty({x.size(0), w.size(0)}, x.options());
  int rc = b200::gemm_weight_only(wo_gemm_args(x, w, scale, bias, out, int4, group_size), cur_stream());
  g_launches += 1;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.weight_only_gemm: unsupported shape (K multiple of 64, N multiple of 8, M <= 64, 16-byte aligned)");
  return out;
}

// w int8 [(E,) N, K] (int4 packed [(E,) N, K/2]), scale float [(E,) N] or [(E,) K / group_size, N] -> [(E,) K, N] in out_dtype (bf16 / fp16 /
// fp32); one launch for all experts, every expert bit-equal to weight_dequantize of its slice
Tensor dequantize_wo(const char* op, const Tensor& w, const Tensor& scale, bool int4, int64_t group_size, at::ScalarType out_dtype, bool experts) {
  TORCH_CHECK(out_dtype == at::kBFloat16 || out_dtype == at::kHalf || out_dtype == at::kFloat, op, ": out_dtype bf16 / fp16 / fp32");
  const int64_t k = check_wo_weight(op, w, scale, int4, group_size, experts), n = w.size(-2), E = experts ? w.size(0) : 1;
  TORCH_CHECK(E <= 65535 && n < (int64_t)1 << 31 && k < (int64_t)1 << 31, op, ": dimensions too large");
  c10::cuda::CUDAGuard guard(w.device());
  Tensor out = experts ? torch::empty({E, k, n}, w.options().dtype(out_dtype)) : torch::empty({k, n}, w.options().dtype(out_dtype));
  int rc = b200::weight_dequantize(w.data_ptr(), scale.data_ptr<float>(), out.data_ptr(), (int)n, (int)k, int4 ? 1 : 0, group_size > 0 ? (int)group_size : 0,
                                   dt_code(out_dtype), cur_stream(), (int)E);
  g_launches += 1;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.", op, ": unsupported shape");
  return out;
}
Tensor weight_dequantize(const Tensor& w, const Tensor& scale, bool int4, int64_t group_size, at::ScalarType out_dtype) {
  return dequantize_wo("weight_dequantize", w, scale, int4, group_size, out_dtype, false);
}

// ---- weight-only MoE experts.  Failing checks use literal messages only, as above.
// expert ids of the token slots ([S] int64, -1 = dropped) -> (dest int32 [S], offsets int32 [E + 1], work int32 [1 + 2 * items]): the
// compact plan of weight_only_gemm_experts for S rows.  Three launches (count, plan, dest), no host read.
std::vector<Tensor> moe_wo_plan(const Tensor& idx, int64_t n_expert) {
  check_i64(idx, "moe_wo_plan");
  TORCH_CHECK(n_expert > 0 && n_expert <= 1024, "moe_wo_plan: 1 to 1024 experts");
  TORCH_CHECK(idx.numel() > 0 && idx.numel() < (int64_t)1 << 30, "moe_wo_plan: bad slot count");
  c10::cuda::CUDAGuard guard(idx.device());
  const int m = (int)idx.numel(), ntok = b200::wo_expert_ntok(m);
  auto i32 = idx.options().dtype(at::kInt);
  Tensor counts = torch::zeros({n_expert}, idx.options());
  Tensor dest = torch::empty({m}, i32), offsets = torch::empty({n_expert + 1}, i32), cursor = torch::empty({n_expert}, i32);
  Tensor work = torch::empty({1 + 2 * (int64_t)b200::wo_expert_items(m, (int)n_expert, ntok)}, i32);
  auto st = cur_stream();
  b200::moe_number_count(idx.data_ptr<int64_t>(), m, counts.data_ptr<int64_t>(), (int)n_expert, st);
  b200::moe_wo_plan(counts.data_ptr<int64_t>(), (int)n_expert, ntok, offsets.data_ptr<int>(), cursor.data_ptr<int>(), work.data_ptr<int>(), st);
  b200::moe_dest(idx.data_ptr<int64_t>(), m, cursor.data_ptr<int>(), dest.data_ptr<int>(), st);
  g_launches += 3; check_err();
  return {dest, offsets, work};
}

// xp [R, K] bf16 / fp16 (routed rows grouped by expert), w int8 [E, N, K] (int4 [E, N, K/2]), scale fp32 [E, N] or [E, K / group_size, N],
// bias [E, N] in xp's dtype or None, offsets / work from moe_wo_plan over R slots -> out [R, N]; rows past offsets[E] are left unwritten
Tensor weight_only_gemm_experts(const Tensor& xp, const Tensor& w, const Tensor& scale, const OptT& bias, const Tensor& offsets, const Tensor& work,
                                bool int4, int64_t group_size) {
  const char* op = "weight_only_gemm_experts";
  check_wo_operands(op, xp, w, scale, bias, int4, group_size, true);
  const int64_t E = w.size(0);
  const int m = (int)xp.size(0);
  TORCH_CHECK(offsets.is_cuda() && offsets.scalar_type() == at::kInt && offsets.is_contiguous() && offsets.numel() == E + 1,
              op, ": offsets int32 [E + 1] from moe_wo_plan");
  TORCH_CHECK(work.is_cuda() && work.scalar_type() == at::kInt && work.is_contiguous() &&
              work.numel() == 1 + 2 * (int64_t)b200::wo_expert_items(m, (int)E, b200::wo_expert_ntok(m)),
              op, ": work must come from moe_wo_plan over the rows of xp");
  TORCH_CHECK(offsets.device() == xp.device() && work.device() == xp.device(), op, ": all operands on one device");
  c10::cuda::CUDAGuard guard(xp.device());
  Tensor out = torch::empty({m, w.size(1)}, xp.options());
  b200::WoGemmArgs g = wo_gemm_args(xp, w, scale, bias, out, int4, group_size);
  g.experts = (int)E; g.offsets = offsets.data_ptr<int>(); g.work = work.data_ptr<int>();
  int rc = b200::gemm_weight_only(g, cur_stream());
  g_launches += 1;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.weight_only_gemm_experts: unsupported shape (K multiple of 64, N multiple of 8, 16-byte aligned)");
  return out;
}

Tensor weight_dequantize_experts(const Tensor& w, const Tensor& scale, bool int4, int64_t group_size, at::ScalarType out_dtype) {
  return dequantize_wo("weight_dequantize_experts", w, scale, int4, group_size, out_dtype, true);
}

// D = act(scale * A[M,K] @ B[N,K]^T + bias), A/B fp8 (e4m3 / e5m2), D half / bf16 / fp32
// (q [M,K] fp8, qT [K,M] fp8 or undefined, inv_scale float[1]) of a 2-D bf16 / fp16 / fp32 tensor; two launches, no host sync
std::vector<Tensor> quantize_fp8(const Tensor& x, bool e5m2, bool want_transpose) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.is_contiguous() && x.size(0) % 64 == 0 && x.size(1) % 64 == 0, "quantize_fp8: contiguous [M, K] with M, K multiples of 64");
  c10::cuda::CUDAGuard guard(x.device());
  const auto f8 = e5m2 ? at::kFloat8_e5m2 : at::kFloat8_e4m3fn;
  Tensor q = torch::empty({x.size(0), x.size(1)}, x.options().dtype(f8));
  Tensor qT = want_transpose ? torch::empty({x.size(1), x.size(0)}, x.options().dtype(f8)) : Tensor();
  Tensor st = torch::zeros({2}, x.options().dtype(at::kFloat));      // [amax, inv_scale]
  auto s = cur_stream();
  b200::fp8_amax(x.data_ptr(), x.numel(), dt_code(x), st.data_ptr<float>(), s);
  b200::fp8_cast_transpose(x.data_ptr(), x.size(0), x.size(1), dt_code(x), st.data_ptr<float>(), e5m2 ? 1 : 0, q.data_ptr(),
                           want_transpose ? qT.data_ptr() : nullptr, st.data_ptr<float>() + 1, s);
  g_launches += 2;
  check_err();
  return {q, qT, st.slice(0, 1, 2)};
}

Tensor gemm_fp8(const Tensor& a, const Tensor& b, const OptT& bias, double scale, int64_t act, at::ScalarType out_dtype, const OptT& scale_a,
                const OptT& scale_b) {
  TORCH_CHECK(a.is_cuda() && b.is_cuda() && a.dim() == 2 && b.dim() == 2 && a.is_contiguous() && b.is_contiguous() && a.size(1) == b.size(1),
              "gemm_fp8: operands must be contiguous [M,K] and [N,K]");
  auto is8 = [](const Tensor& t) { return t.scalar_type() == at::kFloat8_e4m3fn || t.scalar_type() == at::kFloat8_e5m2; };
  TORCH_CHECK(is8(a) && is8(b), "gemm_fp8: fp8 operands required");
  c10::cuda::CUDAGuard guard(a.device());
  b200::GemmFp8Args g;
  g.m = (int)a.size(0); g.k = (int)a.size(1); g.n = (int)b.size(0);
  Tensor d = torch::empty({g.m, g.n}, a.options().dtype(out_dtype));
  g.a = a.data_ptr(); g.b = b.data_ptr(); g.d = d.data_ptr();
  g.bias = nullptr;
  if (bias.has_value() && bias->defined()) {
    TORCH_CHECK(bias->scalar_type() == out_dtype && bias->numel() == g.n, "gemm_fp8: bias must be [N] in the output dtype");
    g.bias = bias->data_ptr();
  }
  g.lda = a.stride(0); g.ldb = b.stride(0); g.ldd = d.stride(0);
  g.a_e5m2 = a.scalar_type() == at::kFloat8_e5m2; g.b_e5m2 = b.scalar_type() == at::kFloat8_e5m2;
  g.scale = (float)scale; g.act = (int)act; g.out_dtype = dt_code(d); g.batch = 1;
  if (scale_a.has_value() && scale_a->defined()) { TORCH_CHECK(scale_a->is_cuda() && scale_a->scalar_type() == at::kFloat, "gemm_fp8: scale_a must be a CUDA float tensor"); g.scale_a_dev = scale_a->data_ptr<float>(); }
  if (scale_b.has_value() && scale_b->defined()) { TORCH_CHECK(scale_b->is_cuda() && scale_b->scalar_type() == at::kFloat, "gemm_fp8: scale_b must be a CUDA float tensor"); g.scale_b_dev = scale_b->data_ptr<float>(); }
  g.stride_a = g.stride_b = g.stride_d = 0;
  int rc = b200::gemm_fp8_tcgen05(g, cur_stream());
  g_launches += 1;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.gemm_fp8 launch failed rc=", rc);
  return d;
}

// int8 x int8 GEMM (csrc/gemm_fp8_sm100.cu, gemm_s8_kernel): a [M,K] / [B,M,K], b [N,K] / [B,N,K] int8 contiguous, K % 16 == 0
b200::GemmS8Args s8_args(const Tensor& a, const Tensor& b, const char* name) {
  TORCH_CHECK(a.is_cuda() && b.is_cuda() && a.scalar_type() == at::kChar && b.scalar_type() == at::kChar, name, ": int8 CUDA operands required");
  TORCH_CHECK(a.dim() == b.dim() && (a.dim() == 2 || a.dim() == 3) && a.is_contiguous() && b.is_contiguous() && a.size(-1) == b.size(-1)
              && (a.dim() == 2 || a.size(0) == b.size(0)), name, ": operands must be contiguous [M,K] and [N,K] (or [B,M,K] and [B,N,K])");
  TORCH_CHECK(a.device() == b.device(), name, ": operands on one device");
  TORCH_CHECK(a.size(-1) % 16 == 0, name, ": K must be a multiple of 16");
  b200::GemmS8Args g;
  g.a = a.data_ptr(); g.b = b.data_ptr();
  g.m = (int)a.size(-2); g.n = (int)b.size(-2); g.k = (int)a.size(-1);
  g.lda = a.stride(-2); g.ldb = b.stride(-2);
  g.batch = a.dim() == 3 ? (int)a.size(0) : 1;
  g.stride_a = a.dim() == 3 ? a.stride(0) : 0;
  g.stride_b = b.dim() == 3 ? b.stride(0) : 0;
  return g;
}

Tensor gemm_int8(const Tensor& a, const Tensor& b) {
  b200::GemmS8Args g = s8_args(a, b, "gemm_int8");
  c10::cuda::CUDAGuard guard(a.device());
  Tensor d = a.dim() == 3 ? torch::empty({a.size(0), g.m, g.n}, a.options().dtype(at::kInt)) : torch::empty({g.m, g.n}, a.options().dtype(at::kInt));
  if (g.batch == 0 || g.m == 0 || g.n == 0) return d;
  g.d = d.data_ptr(); g.ldd = d.stride(-2); g.stride_d = a.dim() == 3 ? d.stride(0) : 0;
  g.out_i32 = 1; g.out_dtype = 0;
  int rc = b200::gemm_s8(g, cur_stream());
  g_launches += 1;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.gemm_int8 launch failed rc=", rc);
  return d;
}

// (float(a @ b^T) * row_scale[m]) * col_scale[n] (+ bias[n]) in out_dtype; row_scale fp32 [M], col_scale fp32 [N], bias fp32 [N]
Tensor gemm_int8_dequant(const Tensor& a, const Tensor& b, const Tensor& row_scale, const Tensor& col_scale, const OptT& bias, at::ScalarType out_dtype) {
  TORCH_CHECK(a.dim() == 2, "gemm_int8_dequant: 2-D operands");
  b200::GemmS8Args g = s8_args(a, b, "gemm_int8_dequant");
  auto vec = [&](const Tensor& t, int64_t n) {
    return t.is_cuda() && t.device() == a.device() && t.scalar_type() == at::kFloat && t.dim() == 1 && t.numel() == n && t.is_contiguous();
  };
  TORCH_CHECK(vec(row_scale, g.m) && vec(col_scale, g.n), "gemm_int8_dequant: row_scale / col_scale must be contiguous float32 [M] / [N]");
  const bool has_bias = bias.has_value() && bias->defined();
  TORCH_CHECK(!has_bias || vec(*bias, g.n), "gemm_int8_dequant: bias must be contiguous float32 [N]");
  c10::cuda::CUDAGuard guard(a.device());
  Tensor d = torch::empty({g.m, g.n}, a.options().dtype(out_dtype));
  if (g.m == 0 || g.n == 0) return d;
  g.d = d.data_ptr(); g.ldd = d.stride(0); g.stride_d = 0;
  g.out_i32 = 0; g.out_dtype = dt_code(out_dtype);
  g.row_scale = row_scale.data_ptr<float>(); g.col_scale = col_scale.data_ptr<float>();
  g.bias = has_bias ? bias->data_ptr<float>() : nullptr;
  int rc = b200::gemm_s8(g, cur_stream());
  g_launches += 1;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.gemm_int8_dequant launch failed rc=", rc);
  return d;
}

// per-token int8 quantisation of a contiguous [M, K] bf16 / fp16 / fp32 tensor (K % 16 == 0): (q int8 [M, K], row_scale fp32 [M]);
// columns where mask (bool [K]) is set are left out of the scale and written as 0.  One launch.
std::vector<Tensor> quantize_int8_rows(const Tensor& x, const OptT& mask) {
  check_cuda_contig(x, "quantize_int8_rows: x");
  TORCH_CHECK(x.dim() == 2 && x.size(1) % 16 == 0 && reinterpret_cast<uintptr_t>(x.data_ptr()) % 16 == 0,
              "quantize_int8_rows: x must be a 16-byte aligned [M, K] with K a multiple of 16");
  const bool has_mask = mask.has_value() && mask->defined();
  TORCH_CHECK(!has_mask || (mask->is_cuda() && mask->device() == x.device() && mask->scalar_type() == at::kBool && mask->dim() == 1
                            && mask->numel() == x.size(1) && mask->is_contiguous()), "quantize_int8_rows: mask must be a contiguous bool [K] on x's device");
  c10::cuda::CUDAGuard guard(x.device());
  Tensor q = torch::empty({x.size(0), x.size(1)}, x.options().dtype(at::kChar));
  Tensor sc = torch::empty({x.size(0)}, x.options().dtype(at::kFloat));
  b200::quantize_rows_s8(x.data_ptr(), has_mask ? reinterpret_cast<const uint8_t*>(mask->data_ptr<bool>()) : nullptr, x.size(0), x.size(1), dt_code(x),
                         q.data_ptr<int8_t>(), sc.data_ptr<float>(), cur_stream());
  g_launches += 1;
  check_err();
  return {q, sc};
}

// OCP MX quantisation of a contiguous [rows, K] tensor (rows, K multiples of 128) along K: (q e4m3 [rows, K], sf uint8 [rows / 128 * K / 128 * 512])
std::vector<Tensor> quantize_mx(const Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.is_contiguous() && x.size(0) % 128 == 0 && x.size(1) % 128 == 0, "quantize_mx: contiguous [rows, K] with rows, K multiples of 128");
  c10::cuda::CUDAGuard guard(x.device());
  Tensor q = torch::empty({x.size(0), x.size(1)}, x.options().dtype(at::kFloat8_e4m3fn));
  Tensor sf = torch::empty({x.size(0) / 128 * (x.size(1) / 128) * 512}, x.options().dtype(at::kByte));
  int rc = b200::mx_quantize(x.data_ptr(), x.size(0), x.size(1), dt_code(x), q.data_ptr(), sf.data_ptr<uint8_t>(), cur_stream());
  g_launches += 1;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.quantize_mx failed rc=", rc);
  return {q, sf};
}

Tensor dequantize_mx(const Tensor& q, const Tensor& sf) {
  TORCH_CHECK(q.is_cuda() && q.dim() == 2 && q.is_contiguous() && q.scalar_type() == at::kFloat8_e4m3fn && sf.scalar_type() == at::kByte && sf.is_contiguous()
              && sf.numel() == q.size(0) / 128 * (q.size(1) / 128) * 512, "dequantize_mx: (q e4m3 [rows, K], sf) as produced by quantize_mx");
  c10::cuda::CUDAGuard guard(q.device());
  Tensor out = torch::empty({q.size(0), q.size(1)}, q.options().dtype(at::kFloat));
  int rc = b200::mx_dequantize(q.data_ptr(), sf.data_ptr<uint8_t>(), q.size(0), q.size(1), out.data_ptr<float>(), cur_stream());
  g_launches += 1;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.dequantize_mx failed rc=", rc);
  return out;
}

// D[M,N] = (A * 2^sfa) (B * 2^sfb)^T: both operands e4m3 K-major with one E8M0 scale per 32 k (quantize_mx); M, N, K multiples of 128
Tensor gemm_fp8_mx(const Tensor& a, const Tensor& sfa, const Tensor& b, const Tensor& sfb, const OptT& bias, at::ScalarType out_dtype) {
  TORCH_CHECK(a.is_cuda() && b.is_cuda() && a.dim() == 2 && b.dim() == 2 && a.is_contiguous() && b.is_contiguous() && a.size(1) == b.size(1),
              "gemm_fp8_mx: operands must be contiguous [M,K] and [N,K]");
  TORCH_CHECK(a.scalar_type() == at::kFloat8_e4m3fn && b.scalar_type() == at::kFloat8_e4m3fn, "gemm_fp8_mx: e4m3 operands required");
  TORCH_CHECK(a.size(0) % 128 == 0 && b.size(0) % 128 == 0 && a.size(1) % 128 == 0, "gemm_fp8_mx: M, N, K must be multiples of 128");
  TORCH_CHECK(sfa.scalar_type() == at::kByte && sfb.scalar_type() == at::kByte && sfa.is_contiguous() && sfb.is_contiguous()
              && sfa.numel() == a.size(0) / 128 * (a.size(1) / 128) * 512 && sfb.numel() == b.size(0) / 128 * (b.size(1) / 128) * 512, "gemm_fp8_mx: scale blocks do not match the operands");
  c10::cuda::CUDAGuard guard(a.device());
  b200::GemmFp8Args g;
  g.m = (int)a.size(0); g.k = (int)a.size(1); g.n = (int)b.size(0);
  Tensor d = torch::empty({g.m, g.n}, a.options().dtype(out_dtype));
  g.a = a.data_ptr(); g.b = b.data_ptr(); g.d = d.data_ptr();
  g.bias = nullptr;
  if (bias.has_value() && bias->defined()) {
    TORCH_CHECK(bias->scalar_type() == out_dtype && bias->numel() == g.n, "gemm_fp8_mx: bias must be [N] in the output dtype");
    g.bias = bias->data_ptr();
  }
  g.lda = a.stride(0); g.ldb = b.stride(0); g.ldd = d.stride(0);
  g.a_e5m2 = 0; g.b_e5m2 = 0;
  g.scale = 1.f; g.act = 0; g.out_dtype = dt_code(d); g.batch = 1;
  g.sfa = sfa.data_ptr<uint8_t>(); g.sfb = sfb.data_ptr<uint8_t>();
  g.stride_a = g.stride_b = g.stride_d = 0;
  int rc = b200::gemm_fp8_tcgen05(g, cur_stream());
  g_launches += 1;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.gemm_fp8_mx launch failed rc=", rc);
  return d;
}

// q [B,H,D], k_cache / v_cache [B,Hkv,S_max,D] contiguous, lens int32 [B] -> out [B,H,D]; window > 0: the last `window` positions only
Tensor decode_attention(const Tensor& q, const Tensor& k_cache, const Tensor& v_cache, const Tensor& lens, double scale, int64_t window) {
  TORCH_CHECK(q.is_cuda() && q.dim() == 3 && k_cache.dim() == 4 && v_cache.dim() == 4 && q.is_contiguous() && k_cache.is_contiguous() && v_cache.is_contiguous(),
              "decode_attention: q [B,H,D], caches [B,Hkv,S,D] contiguous");
  TORCH_CHECK(lens.scalar_type() == at::kInt && lens.is_contiguous() && lens.numel() == q.size(0), "decode_attention: lens must be int32 [B]");
  c10::cuda::CUDAGuard guard(q.device());
  const int b = (int)q.size(0), h = (int)q.size(1), d = (int)q.size(2), hkv = (int)k_cache.size(1), smax = (int)k_cache.size(2);
  const int w = window > 0 ? (int)std::min<int64_t>(window, smax) : 0;
  const int splits = b200::decode_attention_splits(b, h, w > 0 ? w : smax);
  Tensor out = torch::empty_like(q);
  Tensor pacc = torch::empty({b, h, splits, d}, q.options().dtype(at::kFloat));
  Tensor pml = torch::empty({b, h, splits, 2}, q.options().dtype(at::kFloat));
  int rc = b200::decode_attention(q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), lens.data_ptr<int>(), out.data_ptr(), pacc.data_ptr<float>(),
                                  pml.data_ptr<float>(), b, h, hkv, smax, d, splits, (float)scale, dt_code(q), cur_stream(), nullptr, 0, 0, w);
  g_launches += 2;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.decode_attention: unsupported shape (head_dim 128 or 64, fp16/bf16 only) rc=", rc);
  return out;
}

// 8-bit KV caches (int8 / fp8 e4m3): the cache dtype code, after checking that k and v caches share it and that the dequant scales are
// fp32 [Hkv] on q's device; -1 when no scales are given (the caches must then be of q's dtype, checked by the caller).
constexpr int kKvI8 = 3, kKvE4M3 = 4;   // b200::DType codes of the 8-bit cache formats
int kv8_code(const char* op, const Tensor& q, const Tensor& k_cache, const Tensor& v_cache, const OptT& k_dq, const OptT& v_dq) {
  const bool has_k = k_dq.has_value() && k_dq->defined(), has_v = v_dq.has_value() && v_dq->defined();
  TORCH_CHECK(has_k == has_v, op, ": k_dequant_scales and v_dequant_scales go together");
  if (!has_k) return -1;
  const auto st = k_cache.scalar_type();
  TORCH_CHECK(v_cache.scalar_type() == st && (st == at::kChar || st == at::kFloat8_e4m3fn),
              op, ": dequant scales need int8 or float8_e4m3fn caches of one dtype, got ", st, " and ", v_cache.scalar_type());
  TORCH_CHECK(q.scalar_type() == at::kHalf || q.scalar_type() == at::kBFloat16, op, ": q must be fp16 or bf16 with 8-bit caches");
  const int64_t hkv = k_cache.size(1);
  for (const Tensor* t : {&*k_dq, &*v_dq})
    TORCH_CHECK(t->scalar_type() == at::kFloat && t->device() == q.device() && t->is_contiguous() && t->dim() == 1 && t->size(0) == hkv,
                op, ": dequant scales must be fp32 [Hkv] = [", hkv, "] on the device of q");
  return st == at::kChar ? kKvI8 : kKvE4M3;
}

// The operands the paged attention bindings share, checked with messages that name `op`: q a CUDA [T,H,D] view with unit head_dim
// stride, caches contiguous [num_blocks,Hkv,block_size,D] of one shape on q's device (8-bit with their dequant scales, or of q's dtype),
// block_tables int32 [B, max_blocks > 0] on the device, the per-sequence vectors `seq` (named `seq_names` in messages) int32 [B] on the
// device, and out (when given) [T, H*D] of q's dtype with unit inner stride.  Returns the 8-bit cache code (kv8_code).
int check_paged_operands(const char* op, const Tensor& q, const Tensor& k_cache, const Tensor& v_cache, const Tensor& block_tables,
                         const OptT& k_dq, const OptT& v_dq, std::initializer_list<const Tensor*> seq, const char* seq_names, const Tensor* out) {
  TORCH_CHECK(q.is_cuda() && q.dim() == 3 && q.stride(2) == 1, op, ": q must be a CUDA [T,H,D] view with unit head_dim stride");
  TORCH_CHECK(k_cache.dim() == 4 && v_cache.dim() == 4 && k_cache.is_contiguous() && v_cache.is_contiguous() && k_cache.sizes() == v_cache.sizes(),
              op, ": caches must be contiguous [num_blocks,Hkv,block_size,D] of one shape");
  TORCH_CHECK(k_cache.device() == q.device() && v_cache.device() == q.device(), op, ": q and caches must be on one device");
  const int kv = kv8_code(op, q, k_cache, v_cache, k_dq, v_dq);
  if (kv == -1)
    TORCH_CHECK(k_cache.scalar_type() == q.scalar_type() && v_cache.scalar_type() == q.scalar_type(), op, ": q and caches must share a dtype");
  TORCH_CHECK(block_tables.device() == q.device() && block_tables.scalar_type() == at::kInt && block_tables.is_contiguous() && block_tables.dim() == 2
              && block_tables.size(1) > 0, op, ": block_tables must be int32 [B, max_blocks] on the device");
  for (const Tensor* t : seq)
    TORCH_CHECK(t->device() == q.device() && t->scalar_type() == at::kInt && t->is_contiguous() && t->numel() == block_tables.size(0), op, ": ",
                seq_names, " must be int32 [B] on the device");
  if (out)
    TORCH_CHECK(out->device() == q.device() && out->scalar_type() == q.scalar_type() && out->dim() == 2 && out->size(0) == q.size(0) &&
                out->size(1) == q.size(1) * q.size(2) && out->stride(1) == 1, op, ": out must be [T, H*D] with unit inner stride");
  return kv;
}

// paged KV cache: q [B,H,D], caches [num_blocks,Hkv,block_size,D], lens int32 [B] (positions valid per sequence), block_tables int32 [B,max_blocks];
// int8 / fp8 e4m3 caches take fp32 [Hkv] k_dequant_scales / v_dequant_scales; window > 0: the last `window` positions only
Tensor decode_attention_paged(const Tensor& q, const Tensor& k_cache, const Tensor& v_cache, const Tensor& lens, const Tensor& block_tables, double scale,
                              const OptT& k_dequant_scales, const OptT& v_dequant_scales, int64_t window) {
  const char* op = "decode_attention_paged";
  const int kv = check_paged_operands(op, q, k_cache, v_cache, block_tables, k_dequant_scales, v_dequant_scales, {&lens}, "lens", nullptr);
  TORCH_CHECK(q.is_contiguous() && block_tables.size(0) == q.size(0), op, ": q must be contiguous [B,H,D] with one block table row per sequence");
  c10::cuda::CUDAGuard guard(q.device());
  const int b = (int)q.size(0), h = (int)q.size(1), d = (int)q.size(2), hkv = (int)k_cache.size(1), bs = (int)k_cache.size(2), mb = (int)block_tables.size(1);
  const int w = window > 0 ? (int)std::min<int64_t>(window, (int64_t)mb * bs) : 0;
  const int splits = b200::decode_attention_splits(b, h, w > 0 ? w : mb * bs);
  Tensor out = torch::empty_like(q);
  Tensor pacc = torch::empty({b, h, splits, d}, q.options().dtype(at::kFloat));
  Tensor pml = torch::empty({b, h, splits, 2}, q.options().dtype(at::kFloat));
  if (kv != -1) {
    int rc = b200::decode_attention_paged_q8(q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), lens.data_ptr<int>(), out.data_ptr(),
                                             pacc.data_ptr<float>(), pml.data_ptr<float>(), b, h, hkv, d, splits, (float)scale, dt_code(q), kv,
                                             k_dequant_scales->data_ptr<float>(), v_dequant_scales->data_ptr<float>(), block_tables.data_ptr<int>(),
                                             mb, bs, cur_stream(), w);
    g_launches += 2;
    check_err();
    TORCH_CHECK(rc == 0, "paddle_b200.decode_attention_paged: unsupported shape (head_dim 128, H % Hkv == 0) rc=", rc);
    return out;
  }
  int rc = b200::decode_attention(q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), lens.data_ptr<int>(), out.data_ptr(), pacc.data_ptr<float>(),
                                  pml.data_ptr<float>(), b, h, hkv, mb * bs, d, splits, (float)scale, dt_code(q), cur_stream(), block_tables.data_ptr<int>(), mb, bs, w);
  g_launches += 2;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.decode_attention_paged: unsupported shape (head_dim 128 or 64, fp16/bf16 only) rc=", rc);
  return out;
}

static bool fill_attn(b200::AttnArgs& a, const Tensor& q, const Tensor& k, const Tensor& v, double scale, bool causal) {
  if (q.dim() != 4 || k.dim() != 4 || v.dim() != 4) return false;
  if (q.stride(3) != 1 || k.stride(3) != 1 || v.stride(3) != 1) return false;
  if (q.scalar_type() != k.scalar_type() || q.scalar_type() != v.scalar_type()) return false;
  if (q.scalar_type() != at::kBFloat16 && q.scalar_type() != at::kHalf) return false;
  a.q = q.data_ptr(); a.k = k.data_ptr(); a.v = v.data_ptr();
  a.b = (int)q.size(0); a.sq = (int)q.size(1); a.h = (int)q.size(2); a.d = (int)q.size(3);
  a.sk = (int)k.size(1); a.hk = (int)k.size(2);
  if (k.size(0) != q.size(0) || v.size(0) != q.size(0) || v.size(1) != k.size(1) || v.size(2) != k.size(2) || k.size(3) != q.size(3) || v.size(3) != q.size(3)) return false;
  for (int i = 0; i < 3; ++i) { a.q_strides[i] = q.stride(i); a.k_strides[i] = k.stride(i); a.v_strides[i] = v.stride(i); }
  a.scale = (float)scale; a.causal = causal ? 1 : 0; a.dtype = dt_code(q);
  a.o = nullptr; a.lse = nullptr;
  a.o_strides[0] = (int64_t)a.sq * a.h * a.d; a.o_strides[1] = (int64_t)a.h * a.d; a.o_strides[2] = a.d;
  return true;
}

bool attention_supported(const Tensor& q, const Tensor& k, const Tensor& v) {
  b200::AttnArgs a;
  if (!q.is_cuda() || !fill_attn(a, q, k, v, 1.0, false)) return false;
  a.o = const_cast<void*>(a.q);   // alignment probe only
  return b200::attention_fwd_supported(a) != 0;
}

// q [B,Sq,H,D], k/v [B,Sk,Hk,D] (strided views allowed) -> (out [B,Sq,H,D] contiguous, lse fp32 [B,H,Sq])
// mask_skip: the call takes the kernels that skip the tiles the mask hides (csrc/attention_flashmask_sm100.cu); the returned scratch holds
// their tile summary, built on the device by a small kernel the call launches first.  That kernel is not counted in the launch count,
// which counts attention kernels alike for both kinds of masked call.  Otherwise the masked kernels test every element.
static Tensor set_colmask(b200::AttnArgs& a, const OptT& colmask, bool mask_skip) {
  if (!(colmask.has_value() && colmask->defined())) return Tensor();
  const Tensor& m = *colmask;
  TORCH_CHECK(m.is_cuda() && m.scalar_type() == at::kInt && m.is_contiguous() && m.dim() == 4 && m.size(0) == a.b && m.size(2) == a.sk && m.size(3) == 4 &&
              (m.size(1) == 1 || m.size(1) == a.h), "attention: colmask must be int32 [B, 1|H, Sk, 4] (lt_start, lt_end, ut_start, ut_end)");
  a.colmask = m.data_ptr<int>();
  a.mask_heads = (int)m.size(1);
  if (!mask_skip) return Tensor();
  Tensor scratch = torch::empty({b200::attention_mask_tiles_ints(a.b, a.mask_heads, a.sq, a.sk)}, m.options());
  a.mask_tiles = scratch.data_ptr<int>();
  return scratch;
}

// Attention dropout's generator state.  fixed_seed_offset (int64 [2] = (seed, offset), on the host or the device) is used as given;
// otherwise the call takes B*H offsets of torch's default CUDA generator as a PhiloxCudaState, which the kernel resolves on the device,
// so a call captured in a CUDA graph reads the graph's seed and offset slots at every replay and draws a fresh mask each time.
static b200::AttnDropoutArgs dropout_args(double p, const OptT& fixed_seed_offset, const Tensor& seed_offset, int64_t planes, c10::Device dev) {
  b200::AttnDropoutArgs d;
  d.p = p;
  d.seed_offset = seed_offset.data_ptr<int64_t>();
  if (fixed_seed_offset.has_value() && fixed_seed_offset->defined()) {
    const Tensor& f = *fixed_seed_offset;
    TORCH_CHECK(f.scalar_type() == at::kLong && f.numel() == 2 && f.is_contiguous(), "attention: fixed_seed_offset must be int64 [2] (seed, offset)");
    if (f.is_cuda()) {
      TORCH_CHECK(f.device() == dev, "attention: fixed_seed_offset is on another device");
      d.seed_ptr = f.data_ptr<int64_t>(); d.offset_ptr = d.seed_ptr + 1;
    } else {
      d.seed = (uint64_t)f.data_ptr<int64_t>()[0]; d.offset = (uint64_t)f.data_ptr<int64_t>()[1];
    }
    return d;
  }
  auto* gen = at::get_generator_or_default<at::CUDAGeneratorImpl>(std::nullopt, at::cuda::detail::getDefaultCUDAGenerator(dev.index()));
  at::PhiloxCudaState st;
  {
    std::lock_guard<std::mutex> lock(gen->mutex_);
    st = gen->philox_cuda_state((uint64_t)planes);
  }
  if (st.captured_) {
    d.seed_ptr = st.seed_.ptr; d.offset_ptr = st.offset_.ptr; d.offset_add = (int64_t)st.offset_intragraph_;
  } else {
    d.seed = st.seed_.val; d.offset = st.offset_.val;
  }
  return d;
}

static void check_dropout(double p, const char* what) {
  TORCH_CHECK(p >= 0.0 && p < 1.0, what, ": dropout_p must be in [0, 1)");
}

// dropout_p > 0: attention dropout (csrc/attention_dropout_sm100.cu); also returns the int64 [2] (seed, offset) the mask was drawn with
std::vector<Tensor> attention_fwd(const Tensor& q, const Tensor& k, const Tensor& v, double scale, bool causal, bool out_seq_major, const OptT& colmask,
                                  double dropout_p, const OptT& fixed_seed_offset, bool mask_skip) {
  c10::cuda::CUDAGuard guard(q.device());
  check_dropout(dropout_p, "attention_fwd");
  b200::AttnArgs a;
  TORCH_CHECK(fill_attn(a, q, k, v, scale, causal), "paddle_b200.attention_fwd: unsupported operands");
  const Tensor tiles = set_colmask(a, colmask, mask_skip);
  // out_seq_major: the output is laid out [Sq,B,H,D] (sequence-parallel layers consume it without a transpose copy)
  Tensor out = out_seq_major ? torch::empty({a.sq, a.b, a.h, a.d}, q.options()) : torch::empty({a.b, a.sq, a.h, a.d}, q.options());
  if (out_seq_major) { a.o_strides[0] = (int64_t)a.h * a.d; a.o_strides[1] = (int64_t)a.b * a.h * a.d; a.o_strides[2] = a.d; }
  Tensor lse = torch::empty({a.b, a.h, a.sq}, q.options().dtype(at::kFloat));
  a.o = out.data_ptr(); a.lse = lse.data_ptr<float>();
  if (dropout_p > 0.0) {
    Tensor seed_offset = torch::empty({2}, q.options().dtype(at::kLong));
    const b200::AttnDropoutArgs d = dropout_args(dropout_p, fixed_seed_offset, seed_offset, (int64_t)a.b * a.h, q.device());
    int rc = b200::attention_fwd_dropout(a, d, cur_stream());
    g_launches += 1;
    check_err();
    TORCH_CHECK(rc == 0, "paddle_b200.attention_fwd (dropout) launch failed rc=", rc);
    return {out, lse, seed_offset};
  }
  int rc = b200::attention_fwd(a, cur_stream());
  g_launches += 1;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.attention_fwd launch failed rc=", rc);
  return {out, lse};
}

// Causal prefill over the paged KV cache (new K / V already written to the caches): q [T,H,D] view of the packed qkv rows, caches
// [num_blocks,Hkv,block_size,D], block_tables int32 [B,max_blocks], cu_q / n_q / past int32 [B] (n_q = 0: sequence skipped); writes
// out [T,H*D] at the new tokens' rows only, and lse fp32 [H,T] at the same rows when given.  No host read of the lengths.
// int8 / fp8 e4m3 caches take fp32 [Hkv] k_dequant_scales / v_dequant_scales.  window > 0: sliding window, new row r sees keys
// (past + r - window, past + r].
void attention_fwd_paged(const Tensor& q, const Tensor& k_cache, const Tensor& v_cache, const Tensor& block_tables, const Tensor& cu_q,
                         const Tensor& n_q, const Tensor& past, double scale, const Tensor& out, const OptT& lse, const OptT& k_dequant_scales,
                         const OptT& v_dequant_scales, int64_t window) {
  const int kv = check_paged_operands("attention_fwd_paged", q, k_cache, v_cache, block_tables, k_dequant_scales, v_dequant_scales,
                                      {&cu_q, &n_q, &past}, "cu_q / n_q / past", &out);
  const int64_t b = block_tables.size(0);
  b200::PagedAttnArgs a;
  a.q = q.data_ptr(); a.k_cache = k_cache.data_ptr(); a.v_cache = v_cache.data_ptr(); a.o = out.data_ptr(); a.lse = nullptr;
  a.t = (int)q.size(0); a.h = (int)q.size(1); a.d = (int)q.size(2);
  a.num_blocks = (int)k_cache.size(0); a.hk = (int)k_cache.size(1); a.block_size = (int)k_cache.size(2);
  TORCH_CHECK(k_cache.size(3) == q.size(2), "attention_fwd_paged: head_dim of q and caches differ");
  a.b = (int)b; a.max_blocks = (int)block_tables.size(1);
  a.q_strides[0] = q.stride(0); a.q_strides[1] = q.stride(1);
  a.o_strides[0] = out.stride(0); a.o_strides[1] = a.d;
  a.block_tables = block_tables.data_ptr<int>(); a.cu_q = cu_q.data_ptr<int>(); a.n_q = n_q.data_ptr<int>(); a.past = past.data_ptr<int>();
  a.scale = (float)scale; a.dtype = dt_code(q);
  a.window = window > 0 ? (int)std::min<int64_t>(window, INT32_MAX) : 0;
  if (kv != -1) { a.kv_dtype = kv; a.k_dq = k_dequant_scales->data_ptr<float>(); a.v_dq = v_dequant_scales->data_ptr<float>(); }
  if (lse.has_value() && lse->defined()) {
    TORCH_CHECK(lse->device() == q.device() && lse->scalar_type() == at::kFloat && lse->is_contiguous() && lse->dim() == 2 && lse->size(0) == a.h &&
                lse->size(1) == a.t, "attention_fwd_paged: lse must be fp32 [H, T]");
    a.lse = lse->data_ptr<float>();
  }
  TORCH_CHECK(b200::attention_paged_prefill_supported(a), "attention_fwd_paged: unsupported operands (head_dim 128, or 64 on 16-bit caches, "
              "fp16/bf16, H % Hkv == 0, block_size in {16, 32, 64, 128, 256}, 16-byte aligned rows)");
  c10::cuda::CUDAGuard guard(q.device());
  Tensor scratch = torch::empty({b200::attention_paged_prefill_scratch_ints(a.t, a.b)}, q.options().dtype(at::kInt));
  a.scratch = scratch.data_ptr<int>();
  int rc = b200::attention_paged_prefill(a, cur_stream());
  g_launches += 2;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.attention_fwd_paged launch failed rc=", rc);
}

// Multi-token decode over the paged KV cache (the verify rows of speculative decoding; new K / V already written): q [T,H,D] view of the
// packed qkv rows, caches [num_blocks,Hkv,block_size,D], block_tables int32 [B,max_blocks], cu_q / n_q / past int32 [B] (n_q = 0: sequence
// skipped); writes out [T, H*D] at the new tokens' rows only.  n_q * (H / Hkv) may not exceed 64 (a sequence beyond it gets NaN rows: the
// lengths are not read on the host).  int8 / fp8 e4m3 caches take fp32 [Hkv] k_dequant_scales / v_dequant_scales.  window > 0: sliding
// window, new token r sees keys (past + r - window, past + r].
void decode_attention_paged_multi(const Tensor& q, const Tensor& k_cache, const Tensor& v_cache, const Tensor& block_tables, const Tensor& cu_q,
                                  const Tensor& n_q, const Tensor& past, double scale, const Tensor& out, const OptT& k_dequant_scales,
                                  const OptT& v_dequant_scales, int64_t window) {
  TORCH_CHECK(q.scalar_type() == at::kHalf || q.scalar_type() == at::kBFloat16, "decode_attention_paged_multi: q must be fp16 or bf16");
  const int kv = check_paged_operands("decode_attention_paged_multi", q, k_cache, v_cache, block_tables, k_dequant_scales, v_dequant_scales,
                                      {&cu_q, &n_q, &past}, "cu_q / n_q / past", &out);
  const int64_t b = block_tables.size(0);
  TORCH_CHECK(q.size(2) == k_cache.size(3) && (q.size(2) == 128 || (q.size(2) == 64 && kv == -1)),
              "decode_attention_paged_multi: head_dim must be 128, or 64 on 16-bit caches");
  const int64_t hkv = k_cache.size(1);
  TORCH_CHECK(hkv > 0 && q.size(1) % hkv == 0 && q.size(1) / hkv <= 64, "decode_attention_paged_multi: H must be a multiple of Hkv with H / Hkv <= 64, "
              "and n_q * (H / Hkv) <= 64 per sequence");
  b200::PagedMultiArgs a;
  a.q = q.data_ptr(); a.k_cache = k_cache.data_ptr(); a.v_cache = v_cache.data_ptr(); a.out = out.data_ptr();
  a.block_tables = block_tables.data_ptr<int>(); a.cu_q = cu_q.data_ptr<int>(); a.n_q = n_q.data_ptr<int>(); a.past = past.data_ptr<int>();
  a.q_st = q.stride(0); a.q_sh = q.stride(1); a.o_st = out.stride(0);
  a.b = (int)b; a.h = (int)q.size(1); a.hkv = (int)hkv; a.d = (int)q.size(2);
  a.max_blocks = (int)block_tables.size(1); a.block_size = (int)k_cache.size(2);
  a.window = window > 0 ? (int)std::min<int64_t>(window, (int64_t)a.max_blocks * a.block_size) : 0;
  a.splits = b200::decode_attention_splits(a.b, a.hkv, a.window > 0 ? a.window : a.max_blocks * a.block_size);
  a.scale = (float)scale; a.dtype = dt_code(q);
  if (kv != -1) { a.kv_dtype = kv; a.k_dq = k_dequant_scales->data_ptr<float>(); a.v_dq = v_dequant_scales->data_ptr<float>(); }
  c10::cuda::CUDAGuard guard(q.device());
  Tensor pacc = torch::empty({b, hkv, a.splits, 64, a.d}, q.options().dtype(at::kFloat));
  Tensor pml = torch::empty({b, hkv, a.splits, 64, 2}, q.options().dtype(at::kFloat));
  a.part_acc = pacc.data_ptr<float>(); a.part_ml = pml.data_ptr<float>();
  int rc = b200::decode_attention_paged_multi(a, cur_stream());
  g_launches += 2;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.decode_attention_paged_multi: unsupported operands (16-byte aligned rows and caches) rc=", rc);
}

// Shared-prefix decode over the paged KV cache (new K / V already written): q [T,H,D] view of the packed qkv rows, caches
// [num_blocks,Hkv,block_size,D], block_tables int32 [B,max_blocks], cu_q / lens int32 [B] on the device (lens: keys including the new
// token).  Groups on the host: cu_groups int32 [G+1], group_seqs int32 [n] (distinct batch indices), prefix_len int32 [G] (positive
// multiples of block_size); every member of group g shares its first prefix_len[g] / block_size table entries with the others.  Writes
// out [T, H*D] at the members' rows only.  The host builds the task list (prefix tiles of up to 64 / (H / Hkv) members, one suffix task
// per member, split counts) and copies it to the device; no device value is read.  A member breaking the contract gets NaN rows.
void decode_attention_paged_shared(const Tensor& q, const Tensor& k_cache, const Tensor& v_cache, const Tensor& block_tables, const Tensor& cu_q,
                                   const Tensor& lens, const Tensor& cu_groups, const Tensor& group_seqs, const Tensor& prefix_len, double scale,
                                   const Tensor& out, const OptT& k_dequant_scales, const OptT& v_dequant_scales) {
  const char* fn = "decode_attention_paged_shared";
  TORCH_CHECK(q.scalar_type() == at::kHalf || q.scalar_type() == at::kBFloat16, fn, ": q must be fp16 or bf16");
  const int kv = check_paged_operands(fn, q, k_cache, v_cache, block_tables, k_dequant_scales, v_dequant_scales, {&cu_q, &lens}, "cu_q / lens", &out);
  const int64_t b = block_tables.size(0);
  for (const Tensor* t : {&cu_groups, &group_seqs, &prefix_len})
    TORCH_CHECK(t->device().is_cpu() && t->scalar_type() == at::kInt && t->is_contiguous() && t->dim() == 1, fn,
                ": cu_groups / group_seqs / prefix_len must be int32 1-D tensors on the host");
  TORCH_CHECK(q.size(2) == 128 && k_cache.size(3) == 128, fn, ": head_dim must be 128");
  const int64_t hkv = k_cache.size(1), h = q.size(1), bs = k_cache.size(2), max_blocks = block_tables.size(1);
  TORCH_CHECK(hkv > 0 && h % hkv == 0 && h / hkv <= 64, fn, ": H must be a multiple of Hkv with H / Hkv <= 64");
  const int64_t g_size = h / hkv, ng = prefix_len.numel(), n = group_seqs.numel();
  const int* cg = cu_groups.data_ptr<int>();
  const int* gs = group_seqs.data_ptr<int>();
  const int* pl = prefix_len.data_ptr<int>();
  TORCH_CHECK(cu_groups.numel() == ng + 1 && cg[0] == 0 && cg[ng] == n, fn, ": cu_groups must be [G + 1] from 0 to len(group_seqs)");
  std::vector<char> seen(b, 0);
  for (int64_t g = 0; g < ng; ++g) {
    TORCH_CHECK(cg[g + 1] > cg[g], fn, ": every group needs at least one member (cu_groups must rise strictly)");
    // messages take std::to_string: a number streamed into TORCH_CHECK's ostringstream crashes this extension (DESIGN.md section 2)
    TORCH_CHECK(pl[g] > 0 && pl[g] % bs == 0 && pl[g] / bs <= max_blocks, fn, ": prefix_len must be a positive multiple of block_size ",
                std::to_string(bs), " within the block table, got ", std::to_string(pl[g]));
  }
  for (int64_t i = 0; i < n; ++i) {
    TORCH_CHECK(gs[i] >= 0 && gs[i] < b, fn, ": group_seqs holds batch index ", std::to_string(gs[i]), " outside [0, ", std::to_string(b), ")");
    TORCH_CHECK(!seen[gs[i]], fn, ": sequence ", std::to_string(gs[i]), " is in more than one group");
    seen[gs[i]] = 1;
  }
  if (n == 0) return;
  // task list: every group's prefix tiles (split over its prefix), then one suffix task per member (split over the longest possible suffix)
  const int sm = at::cuda::getDeviceProperties(q.device().index())->multiProcessorCount;
  const int64_t per_tile = 64 / g_size;
  int64_t n_tiles = 0;
  for (int64_t g = 0; g < ng; ++g) n_tiles += (cg[g + 1] - cg[g] + per_tile - 1) / per_tile;
  auto splits_for = [&](int64_t ctas, int64_t keys) {
    int64_t s = (2 * sm + ctas * hkv - 1) / (ctas * hkv);
    s = std::min(s, std::max<int64_t>((keys + 255) / 256, 1));
    return (int)std::max<int64_t>(1, std::min<int64_t>(s, 64));
  };
  int min_plen = pl[0];
  for (int64_t g = 1; g < ng; ++g) min_plen = std::min(min_plen, pl[g]);
  const int suf_splits = splits_for(n, max_blocks * bs - min_plen);
  std::vector<int> tasks, members(n * b200::kSharedMemberInts);
  int64_t rows = 0;
  auto add_task = [&](int tb, int m0, int cnt, int lo, int hi, int splits) {
    const int64_t t0 = (int64_t)tasks.size() / b200::kSharedTaskInts;
    for (int s = 0; s < splits; ++s) {
      tasks.insert(tasks.end(), {tb, m0, cnt, lo, hi, s, splits, (int)rows});
      rows += cnt * g_size;
    }
    return (int)t0;
  };
  for (int64_t g = 0; g < ng; ++g) {
    const int splits = splits_for(n_tiles, pl[g]);
    for (int m0 = cg[g]; m0 < cg[g + 1]; m0 += per_tile) {
      const int cnt = std::min<int>(per_tile, cg[g + 1] - m0);
      const int t0 = add_task(gs[cg[g]], m0, cnt, 0, pl[g], splits);
      for (int i = m0; i < m0 + cnt; ++i) {
        int* mi = members.data() + (int64_t)i * b200::kSharedMemberInts;
        mi[0] = t0; mi[1] = (int)((i - m0) * g_size); mi[3] = gs[cg[g]]; mi[4] = pl[g]; mi[5] = gs[i];
      }
    }
  }
  for (int64_t g = 0; g < ng; ++g)
    for (int i = cg[g]; i < cg[g + 1]; ++i) members[(int64_t)i * b200::kSharedMemberInts + 2] = add_task(gs[i], i, 1, pl[g], -1, suf_splits);
  const int64_t n_tasks = (int64_t)tasks.size() / b200::kSharedTaskInts;
  TORCH_CHECK(rows < INT32_MAX && n_tasks < INT32_MAX, fn, ": too many tasks");
  c10::cuda::CUDAGuard guard(q.device());
  // one pinned host buffer (group_seqs | tasks | members), one asynchronous copy
  Tensor host = torch::empty({n + (int64_t)tasks.size() + (int64_t)members.size()}, at::TensorOptions().dtype(at::kInt).pinned_memory(true));
  int* hp = host.data_ptr<int>();
  std::copy(gs, gs + n, hp);
  std::copy(tasks.begin(), tasks.end(), hp + n);
  std::copy(members.begin(), members.end(), hp + n + tasks.size());
  Tensor dev = host.to(q.device(), /*non_blocking=*/true);
  b200::PagedSharedArgs a;
  a.q = q.data_ptr(); a.k_cache = k_cache.data_ptr(); a.v_cache = v_cache.data_ptr(); a.out = out.data_ptr();
  a.block_tables = block_tables.data_ptr<int>(); a.cu_q = cu_q.data_ptr<int>(); a.lens = lens.data_ptr<int>();
  a.group_seqs = dev.data_ptr<int>(); a.tasks = a.group_seqs + n; a.members = a.tasks + tasks.size();
  a.q_st = q.stride(0); a.q_sh = q.stride(1); a.o_st = out.stride(0);
  a.n_tasks = (int)n_tasks; a.n_members = (int)n; a.rows = (int)rows;
  a.h = (int)h; a.hkv = (int)hkv; a.d = (int)q.size(2); a.max_blocks = (int)max_blocks; a.block_size = (int)bs;
  a.scale = (float)scale; a.dtype = dt_code(q);
  if (kv != -1) { a.kv_dtype = kv; a.k_dq = k_dequant_scales->data_ptr<float>(); a.v_dq = v_dequant_scales->data_ptr<float>(); }
  Tensor pacc = torch::empty({hkv, rows, 128}, q.options().dtype(at::kFloat));
  Tensor pml = torch::empty({hkv, rows, 2}, q.options().dtype(at::kFloat));
  a.part_acc = pacc.data_ptr<float>(); a.part_ml = pml.data_ptr<float>();
  int rc = b200::decode_attention_paged_shared(a, cur_stream());
  g_launches += 2;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.decode_attention_paged_shared: unsupported operands (16-byte aligned rows and caches) rc=", std::to_string(rc));
}

// Write of every sequence's new K / V rows into the paged caches: qkv [T, (H + 2 Hkv) * D] packed rows (unit inner stride), caches
// [num_blocks, Hkv, block_size, D], cu_q int32 [B + 1], seq_lens_encoder / seq_lens_decoder int32 [B], block_tables int32 [B, max_blocks].
// int8 / fp8 e4m3 caches take quant scales fp32 [Hkv]: y = (max_bound * scale) * x rounded (round_type 0: rint, 1: roundf) and clamped to
// the bounds; 16-bit caches (the compute type) take a copy.  The optional rest is block_multihead_attention's qkv prologue, applied to
// each row first (csrc/kv_cache_quant.cu): int32 qkv with qkv_out_scale fp32 [W]; qkv_bias [W] of the compute type; rope_cos / rope_sin
// fp32 [S, 64] (interleaved pairs) or [S, 128] (neox halves, neox = true), every new token's position < S; qkv_out [T, W] of the
// compute type receives the processed rows (it may be qkv itself).  The compute type is qkv's dtype, or qkv_out's for int32 qkv.
void paged_kv_cache_write(const Tensor& qkv, const Tensor& k_cache, const Tensor& v_cache, const Tensor& cu_q, const Tensor& seq_lens_encoder,
                          const Tensor& seq_lens_decoder, const Tensor& block_tables, const OptT& k_quant_scales, const OptT& v_quant_scales,
                          int64_t round_type, double max_bound, double min_bound, const OptT& qkv_out, const OptT& qkv_out_scale,
                          const OptT& qkv_bias, const OptT& rope_cos, const OptT& rope_sin, bool neox) {
  const bool i32 = qkv.scalar_type() == at::kInt;
  TORCH_CHECK(qkv.is_cuda() && qkv.dim() == 2 && qkv.stride(1) == 1 && (qkv.scalar_type() == at::kHalf || qkv.scalar_type() == at::kBFloat16 || i32),
              "paged_kv_cache_write: qkv must be a CUDA fp16 / bf16 / int32 [T, (H + 2 Hkv) * D] tensor with unit inner stride");
  const bool has_out = qkv_out.has_value() && qkv_out->defined();
  TORCH_CHECK(!i32 || has_out, "paged_kv_cache_write: int32 qkv needs qkv_out, whose dtype is the compute type");
  const auto ct = i32 ? qkv_out->scalar_type() : qkv.scalar_type();
  TORCH_CHECK(ct == at::kHalf || ct == at::kBFloat16, "paged_kv_cache_write: the compute type must be fp16 or bf16");
  TORCH_CHECK(k_cache.dim() == 4 && k_cache.is_contiguous() && v_cache.is_contiguous() && k_cache.sizes() == v_cache.sizes() &&
              k_cache.device() == qkv.device() && v_cache.device() == qkv.device(),
              "paged_kv_cache_write: caches must be contiguous [num_blocks, Hkv, block_size, D] of one shape on the device of qkv");
  const auto st = k_cache.scalar_type();
  const bool kv16 = st == ct;
  TORCH_CHECK(v_cache.scalar_type() == st && (st == at::kChar || st == at::kFloat8_e4m3fn || kv16),
              "paged_kv_cache_write: caches must both be int8, float8_e4m3fn or of the compute type");
  const int64_t hkv = k_cache.size(1), d = k_cache.size(3);
  if (!kv16) {
    TORCH_CHECK(round_type == 0 || round_type == 1, "paged_kv_cache_write: round_type must be 0 (rint) or 1 (round half away from zero)");
    TORCH_CHECK(min_bound <= max_bound, "paged_kv_cache_write: min_bound must not exceed max_bound");
    if (st == at::kFloat8_e4m3fn) {
      TORCH_CHECK(max_bound <= 448.0 && min_bound >= -448.0, "paged_kv_cache_write: fp8 e4m3 bounds must lie within [-448, 448]");
    } else {
      TORCH_CHECK(max_bound <= 127.0 && min_bound >= -128.0, "paged_kv_cache_write: int8 bounds must lie within [-128, 127]");
    }
    for (const OptT* t : {&k_quant_scales, &v_quant_scales})
      TORCH_CHECK(t->has_value() && (*t)->device() == qkv.device() && (*t)->scalar_type() == at::kFloat && (*t)->is_contiguous() && (*t)->dim() == 1 &&
                  (*t)->size(0) == hkv, "paged_kv_cache_write: quant scales must be fp32 [Hkv] on the device");
  }
  const int64_t w = qkv.size(1);
  TORCH_CHECK(w % d == 0 && w / d > 2 * hkv, "paged_kv_cache_write: qkv row width must be (H + 2 Hkv) * D");
  TORCH_CHECK(qkv.stride(0) % 4 == 0 && reinterpret_cast<uintptr_t>(qkv.data_ptr()) % 8 == 0, "paged_kv_cache_write: qkv rows must be 8-byte aligned");
  TORCH_CHECK(block_tables.device() == qkv.device() && block_tables.scalar_type() == at::kInt && block_tables.is_contiguous() && block_tables.dim() == 2,
              "paged_kv_cache_write: block_tables must be int32 [B, max_blocks] on the device");
  const int64_t b = block_tables.size(0);
  TORCH_CHECK(cu_q.device() == qkv.device() && cu_q.scalar_type() == at::kInt && cu_q.is_contiguous() && cu_q.numel() == b + 1,
              "paged_kv_cache_write: cu_q must be int32 [B + 1] on the device");
  for (const Tensor* t : {&seq_lens_encoder, &seq_lens_decoder})
    TORCH_CHECK(t->device() == qkv.device() && t->scalar_type() == at::kInt && t->is_contiguous() && t->numel() == b,
                "paged_kv_cache_write: seq_lens_encoder / seq_lens_decoder must be int32 [B] on the device");
  auto aligned16 = [](const Tensor& t) { return reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0; };
  const bool has_scale = qkv_out_scale.has_value() && qkv_out_scale->defined(), has_bias = qkv_bias.has_value() && qkv_bias->defined();
  const bool has_cos = rope_cos.has_value() && rope_cos->defined(), has_sin = rope_sin.has_value() && rope_sin->defined();
  const bool prologue = i32 || has_out || has_scale || has_bias || has_cos || has_sin || kv16;
  if (prologue) {
    TORCH_CHECK((qkv.stride(0) * qkv.element_size()) % 16 == 0 && aligned16(qkv), "paged_kv_cache_write: qkv rows must be 16-byte aligned");
    TORCH_CHECK(i32 == has_scale, "paged_kv_cache_write: qkv_out_scale goes with int32 qkv, and only with it");
    if (has_scale)
      TORCH_CHECK(qkv_out_scale->device() == qkv.device() && qkv_out_scale->scalar_type() == at::kFloat && qkv_out_scale->is_contiguous() &&
                  qkv_out_scale->numel() == w && aligned16(*qkv_out_scale), "paged_kv_cache_write: qkv_out_scale must be fp32 [W] on the device");
    if (has_bias)
      TORCH_CHECK(qkv_bias->device() == qkv.device() && qkv_bias->scalar_type() == ct && qkv_bias->is_contiguous() && qkv_bias->numel() == w &&
                  aligned16(*qkv_bias), "paged_kv_cache_write: qkv_bias must be [W] of the compute type on the device");
    TORCH_CHECK(has_cos == has_sin, "paged_kv_cache_write: rope_cos and rope_sin go together");
    if (has_cos)
      for (const OptT* t : {&rope_cos, &rope_sin})
        TORCH_CHECK((*t)->device() == qkv.device() && (*t)->scalar_type() == at::kFloat && (*t)->is_contiguous() && (*t)->dim() == 2 &&
                    (*t)->sizes() == rope_cos->sizes() && (*t)->size(1) == (neox ? d : d / 2) && aligned16(**t),
                    "paged_kv_cache_write: rope_cos / rope_sin must be fp32 [S, D / 2] (neox: [S, D]) on the device");
    if (has_out)
      TORCH_CHECK(qkv_out->device() == qkv.device() && qkv_out->scalar_type() == ct && qkv_out->dim() == 2 && qkv_out->size(0) == qkv.size(0) && qkv_out->size(1) == w &&
                  qkv_out->stride(1) == 1 && (qkv_out->stride(0) * qkv_out->element_size()) % 16 == 0 && aligned16(*qkv_out),
                  "paged_kv_cache_write: qkv_out must be [T, W] of the compute type with 16-byte aligned rows");
  }
  b200::PagedKvWriteArgs a;
  a.qkv = qkv.data_ptr(); a.k_cache = k_cache.data_ptr(); a.v_cache = v_cache.data_ptr(); a.row_stride = qkv.stride(0);
  a.t = (int)qkv.size(0); a.hkv = (int)hkv; a.d = (int)d; a.h = (int)(w / d - 2 * hkv); a.b = (int)b;
  a.block_size = (int)k_cache.size(2); a.max_blocks = (int)block_tables.size(1);
  a.cu_q = cu_q.data_ptr<int>(); a.enc = seq_lens_encoder.data_ptr<int>(); a.dec = seq_lens_decoder.data_ptr<int>(); a.block_tables = block_tables.data_ptr<int>();
  a.k_quant_scales = kv16 ? nullptr : k_quant_scales->data_ptr<float>(); a.v_quant_scales = kv16 ? nullptr : v_quant_scales->data_ptr<float>();
  a.round_type = (int)round_type; a.max_bound = (float)max_bound; a.min_bound = (float)min_bound;
  a.dtype = dt_code(ct); a.kv_dtype = kv16 ? a.dtype : st == at::kChar ? kKvI8 : kKvE4M3;
  if (prologue) {
    a.qkv_int32 = i32 ? 1 : 0;
    a.col_scale = has_scale ? qkv_out_scale->data_ptr<float>() : nullptr;
    a.bias = has_bias ? qkv_bias->data_ptr() : nullptr;
    a.rope = has_cos ? (neox ? 2 : 1) : 0;
    a.rope_cos = has_cos ? rope_cos->data_ptr<float>() : nullptr; a.rope_sin = has_cos ? rope_sin->data_ptr<float>() : nullptr;
    a.rope_stride = has_cos ? (int)rope_cos->size(1) : 0;
    a.out = has_out ? qkv_out->data_ptr() : nullptr; a.out_stride = has_out ? qkv_out->stride(0) : 0;
  }
  c10::cuda::CUDAGuard guard(qkv.device());
  int rc = b200::paged_kv_cache_write(a, cur_stream());
  g_launches += 1;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.paged_kv_cache_write: unsupported operands (head_dim 128) rc=", rc);
}

// Output quantization of block_multihead_attention (out_scale > 0): x [rows, cols] fp16 / bf16 contiguous -> y int8 / float8_e4m3fn of the
// same shape, y = quantize(max_bound * out_scale * x) under the cache rounding rules; shift / smooth [cols] of x's dtype, both or neither:
// x is first replaced by ((x + shift) * smooth), each step rounded to x's dtype.
void attention_out_quant(const Tensor& x, const Tensor& y, double out_scale, const OptT& shift, const OptT& smooth, int64_t round_type,
                         double max_bound, double min_bound) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.is_contiguous() && (x.scalar_type() == at::kHalf || x.scalar_type() == at::kBFloat16) &&
              reinterpret_cast<uintptr_t>(x.data_ptr()) % 16 == 0 && x.size(1) % 8 == 0,
              "attention_out_quant: x must be a contiguous CUDA fp16 / bf16 [rows, cols] tensor, cols a multiple of 8, 16-byte aligned");
  TORCH_CHECK(y.device() == x.device() && y.is_contiguous() && y.sizes() == x.sizes() && (y.scalar_type() == at::kChar || y.scalar_type() == at::kFloat8_e4m3fn) &&
              reinterpret_cast<uintptr_t>(y.data_ptr()) % 8 == 0, "attention_out_quant: y must be a contiguous int8 / float8_e4m3fn tensor shaped like x");
  TORCH_CHECK(round_type == 0 || round_type == 1, "attention_out_quant: round_type must be 0 (rint) or 1 (round half away from zero)");
  TORCH_CHECK(min_bound <= max_bound, "attention_out_quant: min_bound must not exceed max_bound");
  if (y.scalar_type() == at::kFloat8_e4m3fn) {
    TORCH_CHECK(max_bound <= 448.0 && min_bound >= -448.0, "attention_out_quant: fp8 e4m3 bounds must lie within [-448, 448]");
  } else {
    TORCH_CHECK(max_bound <= 127.0 && min_bound >= -128.0, "attention_out_quant: int8 bounds must lie within [-128, 127]");
  }
  const bool has_shift = shift.has_value() && shift->defined(), has_smooth = smooth.has_value() && smooth->defined();
  TORCH_CHECK(has_shift == has_smooth, "attention_out_quant: shift and smooth go together");
  if (has_shift)
    for (const OptT* t : {&shift, &smooth})
      TORCH_CHECK((*t)->device() == x.device() && (*t)->scalar_type() == x.scalar_type() && (*t)->is_contiguous() && (*t)->numel() == x.size(1) &&
                  reinterpret_cast<uintptr_t>((*t)->data_ptr()) % 16 == 0, "attention_out_quant: shift / smooth must be [cols] of x's dtype on the device");
  b200::OutQuantArgs a;
  a.x = x.data_ptr(); a.y = y.data_ptr(); a.rows = x.size(0); a.cols = (int)x.size(1);
  a.shift = optp(shift); a.smooth = optp(smooth);
  a.scale = (float)max_bound * (float)out_scale;
  a.round_type = (int)round_type; a.max_bound = (float)max_bound; a.min_bound = (float)min_bound;
  a.dtype = dt_code(x); a.out_dtype = y.scalar_type() == at::kChar ? kKvI8 : kKvE4M3;
  c10::cuda::CUDAGuard guard(x.device());
  int rc = b200::attention_out_quant(a, cur_stream());
  g_launches += 1;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.attention_out_quant: unsupported operands rc=", rc);
}

static bool g_deterministic = false;     // FLAGS_cudnn_deterministic: the attention backward takes its bitwise-reproducible two-kernel path

// The backward's launch: dropout_p > 0 takes the mask of seed_offset, the (seed, offset) pair the forward returned.
static int launch_bwd(const b200::AttnBwdArgs& a, double dropout_p, const OptT& seed_offset, const char* what) {
  if (dropout_p == 0.0) return b200::attention_bwd(a, cur_stream());
  TORCH_CHECK(seed_offset.has_value() && seed_offset->defined() && seed_offset->is_cuda() && seed_offset->scalar_type() == at::kLong &&
              seed_offset->numel() == 2, what, ": dropout needs the forward's seed_offset (int64 [2] on the device)");
  b200::AttnDropoutArgs d;
  d.p = dropout_p;
  d.seed_offset = seed_offset->data_ptr<int64_t>();
  return b200::attention_bwd_dropout(a, d, cur_stream());
}

// backward of attention_fwd: returns (dq [B,Sq,H,D], dk, dv [B,Sk,Hk,D]) in the input dtype
std::vector<Tensor> attention_bwd(const Tensor& q, const Tensor& k, const Tensor& v, const Tensor& out, const Tensor& lse, const Tensor& d_out,
                                  double scale, bool causal, const OptT& colmask, double dropout_p, const OptT& seed_offset, bool mask_skip) {
  c10::cuda::CUDAGuard guard(q.device());
  check_dropout(dropout_p, "attention_bwd");
  b200::AttnBwdArgs a;
  TORCH_CHECK(fill_attn(a.fwd, q, k, v, scale, causal), "paddle_b200.attention_bwd: unsupported operands");
  const Tensor tiles = set_colmask(a.fwd, colmask, mask_skip);
  TORCH_CHECK(out.is_contiguous() && d_out.is_contiguous() && lse.is_contiguous() && lse.scalar_type() == at::kFloat, "attention_bwd: out / d_out / lse layout");
  a.fwd.o = out.data_ptr(); a.fwd.lse = lse.data_ptr<float>();
  Tensor dq32 = torch::empty({a.fwd.b, a.fwd.sq, a.fwd.h, a.fwd.d}, q.options().dtype(at::kFloat));
  Tensor dk = torch::empty({a.fwd.b, a.fwd.sk, a.fwd.hk, a.fwd.d}, q.options());
  Tensor dv = torch::empty_like(dk);
  Tensor stats = torch::empty({a.fwd.b, a.fwd.h, 2, b200::attention_bwd_stats_pad(a.fwd.sq)}, q.options().dtype(at::kFloat));
  a.d_o = d_out.data_ptr(); a.stats = stats.data_ptr<float>(); a.dq = dq32.data_ptr<float>(); a.dk = dk.data_ptr(); a.dv = dv.data_ptr();
  a.deterministic = g_deterministic;
  for (int i = 0; i < 3; ++i) { a.dkv_strides[i] = dk.stride(i); a.o_strides[i] = out.stride(i); a.dq_strides[i] = dq32.stride(i); }
  int rc = launch_bwd(a, dropout_p, seed_offset, "attention_bwd");
  g_launches += a.deterministic ? 3 : 2;     // prep + dK/dV + dQ, or prep + single pass
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.attention_bwd launch failed rc=", rc);
  return {dq32.to(q.scalar_type()), dk, dv};
}

// packed variant: qkv [B,S,nh+2*nkv,D] (q heads | k heads | v heads); returns d(qkv) of the same shape, written in place by
// the kernel (dk/dv slices) plus one cast-copy of the fp32 dq accumulator - no slice-backward zero fills / adds.  colmask: as attention_bwd,
// over the [B,S] view
Tensor attention_bwd_packed(const Tensor& qkv, int64_t nh, int64_t nkv, const Tensor& out, const Tensor& lse, const Tensor& d_out, double scale,
                            bool causal, bool seq_major, double dropout_p, const OptT& seed_offset, const OptT& colmask, bool mask_skip) {
  c10::cuda::CUDAGuard guard(qkv.device());
  check_dropout(dropout_p, "attention_bwd_packed");
  TORCH_CHECK(qkv.dim() == 4 && qkv.is_contiguous() && qkv.size(2) == nh + 2 * nkv, "attention_bwd_packed: qkv layout");
  // seq_major: qkv / out / d_out memory is [S,B,*,D]; the kernels see [B,S,*,D] views of it (strides only, no copies)
  auto bs = [&](const Tensor& t) { return seq_major ? t.transpose(0, 1) : t; };
  Tensor q = bs(qkv.narrow(2, 0, nh)), k = bs(qkv.narrow(2, nh, nkv)), v = bs(qkv.narrow(2, nh + nkv, nkv));
  b200::AttnBwdArgs a;
  TORCH_CHECK(fill_attn(a.fwd, q, k, v, scale, causal), "paddle_b200.attention_bwd_packed: unsupported operands");
  const Tensor tiles = set_colmask(a.fwd, colmask, mask_skip);
  TORCH_CHECK(out.is_contiguous() && d_out.is_contiguous() && lse.is_contiguous() && out.sizes() == d_out.sizes(), "attention_bwd_packed: out / d_out / lse layout");
  Tensor ov = bs(out);
  a.fwd.o = out.data_ptr(); a.fwd.lse = lse.data_ptr<float>();
  Tensor dqkv = torch::empty_like(qkv);
  Tensor dk = bs(dqkv.narrow(2, nh, nkv)), dv = bs(dqkv.narrow(2, nh + nkv, nkv));
  Tensor dq32_mem = torch::empty(out.sizes(), qkv.options().dtype(at::kFloat));     // same memory order as `out`
  Tensor dq32 = bs(dq32_mem);
  Tensor stats = torch::empty({a.fwd.b, a.fwd.h, 2, b200::attention_bwd_stats_pad(a.fwd.sq)}, qkv.options().dtype(at::kFloat));
  a.d_o = d_out.data_ptr(); a.stats = stats.data_ptr<float>(); a.dq = dq32_mem.data_ptr<float>(); a.dk = dk.data_ptr(); a.dv = dv.data_ptr();
  a.deterministic = g_deterministic;
  for (int i = 0; i < 3; ++i) { a.dkv_strides[i] = dk.stride(i); a.o_strides[i] = ov.stride(i); a.dq_strides[i] = dq32.stride(i); }
  int rc = launch_bwd(a, dropout_p, seed_offset, "attention_bwd_packed");
  g_launches += a.deterministic ? 3 : 2;     // prep + dK/dV + dQ, or prep + single pass
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.attention_bwd_packed launch failed rc=", rc);
  dqkv.narrow(2, 0, nh).copy_(dq32_mem);
  return dqkv;
}

// ------------------------------------------------------------------------------------------------ token sampling (csrc/sampling.cu)
// x [rows, vocab] fp32 / fp16 / bf16 with unit column stride (any row stride); per-row parameters are contiguous CUDA vectors on x's
// device.  Returns (ids int64 [rows], vals [rows] in x's dtype, top_vals [rows, k_out], top_ids int64 [rows, k_out]).  One launch,
// no host read.  Failing checks use literal messages only.
std::vector<Tensor> sample_tokens(const Tensor& x, const Tensor& temperature, const Tensor& top_k, const Tensor& top_p, const OptT& threshold,
                                  const Tensor& seed, const Tensor& offset, bool is_prob, bool truncated, int64_t k_out) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.stride(1) == 1 && x.size(1) > 0, "sample_tokens: x must be a CUDA [rows, vocab] matrix with unit column stride");
  TORCH_CHECK(x.size(1) < ((int64_t)1 << 30) && x.size(0) < ((int64_t)1 << 31), "sample_tokens: too many rows or tokens");
  TORCH_CHECK(k_out >= 0 && k_out <= b200::sample_max_top() && k_out <= x.size(1), "sample_tokens: k_out must be in [0, min(1024, vocab)]");
  const int64_t rows = x.size(0);
  auto vec = [&](const Tensor& t, at::ScalarType st, const char* msg) {
    TORCH_CHECK(t.device() == x.device() && t.scalar_type() == st && t.dim() == 1 && t.size(0) == rows && t.is_contiguous(), msg);
  };
  vec(temperature, at::kFloat, "sample_tokens: temperature must be float32 [rows] on x's device");
  vec(top_k, at::kInt, "sample_tokens: top_k must be int32 [rows] on x's device");
  vec(top_p, at::kFloat, "sample_tokens: top_p must be float32 [rows] on x's device");
  vec(seed, at::kLong, "sample_tokens: seed must be int64 [rows] on x's device");
  vec(offset, at::kLong, "sample_tokens: offset must be int64 [rows] on x's device");
  const bool has_thr = threshold.has_value() && threshold->defined();
  if (has_thr) vec(*threshold, at::kFloat, "sample_tokens: threshold must be float32 [rows] on x's device");
  c10::cuda::CUDAGuard guard(x.device());
  Tensor ids = torch::empty({rows}, x.options().dtype(at::kLong));
  Tensor vals = torch::empty({rows}, x.options());
  Tensor top_vals = torch::empty({rows, k_out}, x.options());
  Tensor top_ids = torch::empty({rows, k_out}, x.options().dtype(at::kLong));
  b200::SampleArgs a{};
  a.x = x.data_ptr(); a.rows = rows; a.stride = rows > 1 ? x.stride(0) : x.size(1); a.vocab = (int)x.size(1);
  a.temperature = temperature.data_ptr<float>(); a.top_k = top_k.data_ptr<int>(); a.top_p = top_p.data_ptr<float>();
  a.threshold = has_thr ? threshold->data_ptr<float>() : nullptr;
  a.seed = seed.data_ptr<int64_t>(); a.offset = offset.data_ptr<int64_t>();
  a.ids = ids.data_ptr<int64_t>(); a.vals = vals.data_ptr(); a.top_vals = top_vals.data_ptr(); a.top_ids = top_ids.data_ptr<int64_t>();
  a.k_out = (int)k_out; a.is_prob = is_prob ? 1 : 0; a.truncated = truncated ? 1 : 0; a.dtype = dt_code(x);
  const int rc = b200::sample_tokens(a, cur_stream());
  g_launches += 1;
  check_err();
  TORCH_CHECK(rc == 0, "paddle_b200.sample_tokens: unsupported shape");
  return {ids, vals, top_vals, top_ids};
}

// the uniforms the sampling race draws for (seed, offset), tokens 0 .. n-1 (float32 [n] on `device`)
Tensor sampling_uniforms(int64_t seed, int64_t offset, int64_t n, const Tensor& like) {
  TORCH_CHECK(like.is_cuda() && n >= 0 && n < ((int64_t)1 << 30), "sampling_uniforms: n in [0, 2^30) on a CUDA device");
  c10::cuda::CUDAGuard guard(like.device());
  Tensor out = torch::empty({n}, like.options().dtype(at::kFloat));
  b200::sampling_uniforms(seed, offset, (int)n, out.data_ptr<float>(), cur_stream());
  g_launches += 1;
  check_err();
  return out;
}

// Every kernel entry point is bound through traced(): when the tracer is on (profiler.Profiler) the call becomes a host range
// plus a cudaEvent pair on the launching stream; when it is off the cost is one relaxed atomic load.
template <typename R, typename... A>
auto traced(const char* name, R (*f)(A...)) {
  return [name, f](A... a) -> R {
    b200::runtime::TraceScope scope(name);
    return f(std::forward<A>(a)...);
  };
}

int64_t launch_count() { return g_launches.load(); }
void reset_launch_count() { g_launches.store(0); }
void add_launches(int64_t n) { g_launches += n; }

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("rms_norm_fwd", traced("rms_norm_fwd", &rms_norm_fwd));
  m.def("rms_norm_bwd", traced("rms_norm_bwd", &rms_norm_bwd));
  m.def("layer_norm_fwd", traced("layer_norm_fwd", &layer_norm_fwd));
  m.def("layer_norm_bwd", traced("layer_norm_bwd", &layer_norm_bwd));
  m.def("bias_dropout_add", traced("bias_dropout_add", &bias_dropout_add));
  m.def("dropout_bwd", traced("dropout_bwd", &dropout_bwd));
  m.def("bias_act", traced("bias_act", &bias_act));
  m.def("swiglu_fwd", traced("swiglu_fwd", &swiglu_fwd));
  m.def("swiglu_bwd", traced("swiglu_bwd", &swiglu_bwd));
  m.def("rope", traced("rope", &rope));
  m.def("rope_packed_", traced("rope_packed_", &rope_packed_));
  m.def("softmax_ce_fwd", traced("softmax_ce_fwd", &softmax_ce_fwd));
  m.def("softmax_ce_bwd", traced("softmax_ce_bwd", &softmax_ce_bwd));
  m.def("vp_ce_max", traced("vp_ce_max", &vp_ce_max));
  m.def("vp_ce_sumexp", traced("vp_ce_sumexp", &vp_ce_sumexp));
  m.def("vp_ce_bwd", traced("vp_ce_bwd", &vp_ce_bwd));
  m.def("adamw_step", traced("adamw_step", &adamw_step));
  m.def("adamw_step_dyn", traced("adamw_step", &adamw_step_dyn));
  m.def("grad_sq_norm", traced("grad_sq_norm", &grad_sq_norm));
  m.def("scale_inplace", traced("scale_inplace", &scale_inplace));
  m.def("sgd_step", traced("sgd_step", &sgd_step));
  m.def("lamb_step", traced("lamb_step", &lamb_step));
  m.def("gemm_supported", &gemm_supported);
  m.def("gemm", traced("gemm", &gemm), pybind11::arg("a"), pybind11::arg("b"), pybind11::arg("bias") = pybind11::none(), pybind11::arg("a_is_km") = false,
        pybind11::arg("b_is_nk") = false, pybind11::arg("epilogue") = 0, pybind11::arg("out") = pybind11::none(),
        pybind11::arg("out_dtype") = pybind11::none(), pybind11::arg("rs_dst") = std::vector<int64_t>(), pybind11::arg("rs_rows") = 0,
        pybind11::arg("ag_src") = std::vector<int64_t>(), pybind11::arg("ag_pad") = std::vector<int64_t>(), pybind11::arg("ag_flags") = pybind11::none(),
        pybind11::arg("ag_rank") = 0, pybind11::arg("ag_rows") = 0, pybind11::arg("ag_epoch") = 0);
  m.def("moe_number_count", traced("moe_number_count", &moe_number_count));
  m.def("moe_assign_pos", traced("moe_assign_pos", &moe_assign_pos));
  m.def("moe_limit_by_capacity", traced("moe_limit_by_capacity", &moe_limit_by_capacity));
  m.def("moe_prune_gate_by_capacity", traced("moe_prune_gate_by_capacity", &moe_prune_gate_by_capacity));
  m.def("moe_route", traced("moe_route", &moe_route));
  m.def("moe_rows_scatter", traced("moe_rows_scatter", &moe_rows_scatter), pybind11::arg("src"), pybind11::arg("dest"), pybind11::arg("scale") = pybind11::none(),
        pybind11::arg("topk") = 1, pybind11::arg("rows_out") = 0);
  m.def("moe_rows_combine", traced("moe_rows_combine", &moe_rows_combine), pybind11::arg("src"), pybind11::arg("dest"), pybind11::arg("w") = pybind11::none(),
        pybind11::arg("topk") = 1);
  m.def("moe_rows_dot", traced("moe_rows_dot", &moe_rows_dot));
  m.def("weight_only_gemm", traced("weight_only_gemm", &weight_only_gemm), pybind11::arg("x"), pybind11::arg("w"), pybind11::arg("scale"), pybind11::arg("bias") = pybind11::none(),
        pybind11::arg("int4") = false, pybind11::arg("group_size") = -1);
  m.def("weight_dequantize", traced("weight_dequantize", &weight_dequantize), pybind11::arg("w"), pybind11::arg("scale"), pybind11::arg("int4") = false,
        pybind11::arg("group_size") = -1, pybind11::arg("out_dtype") = at::kBFloat16);
  m.def("moe_wo_plan", traced("moe_wo_plan", &moe_wo_plan));
  m.def("weight_only_gemm_experts", traced("weight_only_gemm_experts", &weight_only_gemm_experts), pybind11::arg("xp"), pybind11::arg("w"),
        pybind11::arg("scale"), pybind11::arg("bias"), pybind11::arg("offsets"), pybind11::arg("work"), pybind11::arg("int4") = false,
        pybind11::arg("group_size") = -1);
  m.def("weight_dequantize_experts", traced("weight_dequantize_experts", &weight_dequantize_experts), pybind11::arg("w"), pybind11::arg("scale"),
        pybind11::arg("int4") = false, pybind11::arg("group_size") = -1, pybind11::arg("out_dtype") = at::kBFloat16);
  m.def("gemm_grouped", traced("gemm_grouped", &gemm_grouped), pybind11::arg("a"), pybind11::arg("b"), pybind11::arg("tile_expert"), pybind11::arg("b_is_nk") = false,
        pybind11::arg("out") = pybind11::none());
  m.def("gemm_grouped_wgrad", traced("gemm_grouped_wgrad", &gemm_grouped_wgrad));
  m.def("gemm_fp8", traced("gemm_fp8", &gemm_fp8), pybind11::arg("a"), pybind11::arg("b"), pybind11::arg("bias") = pybind11::none(), pybind11::arg("scale") = 1.0,
        pybind11::arg("act") = 0, pybind11::arg("out_dtype") = at::kBFloat16, pybind11::arg("scale_a") = pybind11::none(), pybind11::arg("scale_b") = pybind11::none());
  m.def("quantize_mx", traced("quantize_mx", &quantize_mx));
  m.def("dequantize_mx", traced("dequantize_mx", &dequantize_mx));
  m.def("gemm_fp8_mx", traced("gemm_fp8_mx", &gemm_fp8_mx), pybind11::arg("a"), pybind11::arg("sfa"), pybind11::arg("b"), pybind11::arg("sfb"), pybind11::arg("bias") = pybind11::none(),
        pybind11::arg("out_dtype") = at::kBFloat16);
  m.def("gemm_int8", traced("gemm_int8", &gemm_int8), pybind11::arg("a"), pybind11::arg("b"));
  m.def("gemm_int8_dequant", traced("gemm_int8_dequant", &gemm_int8_dequant), pybind11::arg("a"), pybind11::arg("b"), pybind11::arg("row_scale"),
        pybind11::arg("col_scale"), pybind11::arg("bias") = pybind11::none(), pybind11::arg("out_dtype") = at::kFloat);
  m.def("quantize_int8_rows", traced("quantize_int8_rows", &quantize_int8_rows), pybind11::arg("x"), pybind11::arg("mask") = pybind11::none());
  m.def("quantize_fp8", traced("quantize_fp8", &quantize_fp8), pybind11::arg("x"), pybind11::arg("e5m2") = false, pybind11::arg("want_transpose") = false);
  m.def("set_deterministic", [](bool on) { g_deterministic = on; });
  m.def("deterministic", []() { return g_deterministic; });
  m.def("decode_attention", traced("decode_attention", &decode_attention), pybind11::arg("q"), pybind11::arg("k_cache"), pybind11::arg("v_cache"),
        pybind11::arg("lens"), pybind11::arg("scale"), pybind11::arg("window") = 0);
  m.def("decode_attention_paged", traced("decode_attention_paged", &decode_attention_paged), pybind11::arg("q"), pybind11::arg("k_cache"),
        pybind11::arg("v_cache"), pybind11::arg("lens"), pybind11::arg("block_tables"), pybind11::arg("scale"),
        pybind11::arg("k_dequant_scales") = pybind11::none(), pybind11::arg("v_dequant_scales") = pybind11::none(), pybind11::arg("window") = 0);
  m.def("paged_kv_cache_write", traced("paged_kv_cache_write", &paged_kv_cache_write), pybind11::arg("qkv"), pybind11::arg("k_cache"),
        pybind11::arg("v_cache"), pybind11::arg("cu_q"), pybind11::arg("seq_lens_encoder"), pybind11::arg("seq_lens_decoder"),
        pybind11::arg("block_tables"), pybind11::arg("k_quant_scales"), pybind11::arg("v_quant_scales"), pybind11::arg("round_type") = 1,
        pybind11::arg("max_bound") = 127.0, pybind11::arg("min_bound") = -127.0, pybind11::arg("qkv_out") = pybind11::none(),
        pybind11::arg("qkv_out_scale") = pybind11::none(), pybind11::arg("qkv_bias") = pybind11::none(), pybind11::arg("rope_cos") = pybind11::none(),
        pybind11::arg("rope_sin") = pybind11::none(), pybind11::arg("neox") = false);
  m.def("attention_out_quant", traced("attention_out_quant", &attention_out_quant), pybind11::arg("x"), pybind11::arg("y"), pybind11::arg("out_scale"),
        pybind11::arg("shift") = pybind11::none(), pybind11::arg("smooth") = pybind11::none(), pybind11::arg("round_type") = 1,
        pybind11::arg("max_bound") = 127.0, pybind11::arg("min_bound") = -127.0);
  m.def("attention_supported", &attention_supported);
  m.def("attention_fwd", traced("attention_fwd", &attention_fwd), pybind11::arg("q"), pybind11::arg("k"), pybind11::arg("v"), pybind11::arg("scale"), pybind11::arg("causal"),
        pybind11::arg("out_seq_major") = false, pybind11::arg("colmask") = pybind11::none(), pybind11::arg("dropout_p") = 0.0,
        pybind11::arg("seed_offset") = pybind11::none(), pybind11::arg("mask_skip") = true);
  m.def("attention_fwd_paged", traced("attention_fwd_paged", &attention_fwd_paged), pybind11::arg("q"), pybind11::arg("k_cache"),
        pybind11::arg("v_cache"), pybind11::arg("block_tables"), pybind11::arg("cu_q"), pybind11::arg("n_q"), pybind11::arg("past"), pybind11::arg("scale"),
        pybind11::arg("out"), pybind11::arg("lse") = pybind11::none(), pybind11::arg("k_dequant_scales") = pybind11::none(),
        pybind11::arg("v_dequant_scales") = pybind11::none(), pybind11::arg("window") = 0);
  m.def("decode_attention_paged_multi", traced("decode_attention_paged_multi", &decode_attention_paged_multi), pybind11::arg("q"),
        pybind11::arg("k_cache"), pybind11::arg("v_cache"), pybind11::arg("block_tables"), pybind11::arg("cu_q"), pybind11::arg("n_q"),
        pybind11::arg("past"), pybind11::arg("scale"), pybind11::arg("out"), pybind11::arg("k_dequant_scales") = pybind11::none(),
        pybind11::arg("v_dequant_scales") = pybind11::none(), pybind11::arg("window") = 0);
  m.def("decode_attention_paged_shared", traced("decode_attention_paged_shared", &decode_attention_paged_shared), pybind11::arg("q"),
        pybind11::arg("k_cache"), pybind11::arg("v_cache"), pybind11::arg("block_tables"), pybind11::arg("cu_q"), pybind11::arg("lens"),
        pybind11::arg("cu_groups"), pybind11::arg("group_seqs"), pybind11::arg("prefix_len"), pybind11::arg("scale"), pybind11::arg("out"),
        pybind11::arg("k_dequant_scales") = pybind11::none(), pybind11::arg("v_dequant_scales") = pybind11::none());
  m.def("attention_bwd", traced("attention_bwd", &attention_bwd), pybind11::arg("q"), pybind11::arg("k"), pybind11::arg("v"), pybind11::arg("out"), pybind11::arg("lse"),
        pybind11::arg("d_out"), pybind11::arg("scale"), pybind11::arg("causal"), pybind11::arg("colmask") = pybind11::none(),
        pybind11::arg("dropout_p") = 0.0, pybind11::arg("seed_offset") = pybind11::none(), pybind11::arg("mask_skip") = true);
  m.def("attention_bwd_packed", traced("attention_bwd_packed", &attention_bwd_packed), pybind11::arg("qkv"), pybind11::arg("nh"), pybind11::arg("nkv"), pybind11::arg("out"),
        pybind11::arg("lse"), pybind11::arg("d_out"), pybind11::arg("scale"), pybind11::arg("causal"), pybind11::arg("seq_major") = false,
        pybind11::arg("dropout_p") = 0.0, pybind11::arg("seed_offset") = pybind11::none(), pybind11::arg("colmask") = pybind11::none(),
        pybind11::arg("mask_skip") = true);
  m.def("sample_tokens", traced("sample_tokens", &sample_tokens), pybind11::arg("x"), pybind11::arg("temperature"), pybind11::arg("top_k"),
        pybind11::arg("top_p"), pybind11::arg("threshold"), pybind11::arg("seed"), pybind11::arg("offset"), pybind11::arg("is_prob") = false,
        pybind11::arg("truncated") = true, pybind11::arg("k_out") = 0);
  m.def("sampling_uniforms", traced("sampling_uniforms", &sampling_uniforms));
  m.def("launch_count", &launch_count);
  m.def("reset_launch_count", &reset_launch_count);
  m.def("add_launches", &add_launches);
  b200::runtime::bind(m);
}
