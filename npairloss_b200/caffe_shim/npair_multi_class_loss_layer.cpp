// NPairMultiClassLossLayer host side: Caffe plugin surface over the C ABI (include/npair_b200.h).
// Replaces reference npair_multi_class_loss.cpp:19-191 and the host parts of npair_multi_class_loss.cu:207-499.
#include "npair_multi_class_loss_layer.hpp"

#include <cuda_runtime.h>

#include <cstdlib>

#include "caffe/layer_factory.hpp"
#include "npair_b200.h"

namespace caffe {

template <typename Dtype>
NPairMultiClassLossLayer<Dtype>::~NPairMultiClassLossLayer() {
  if (ctx_) npair_destroy(ctx_);
  if (f32_feat_) cudaFree(f32_feat_);
  if (f32_label_) cudaFree(f32_label_);
  if (f32_diff_) cudaFree(f32_diff_);
  if (f32_weight_) cudaFree(f32_weight_);
}

template <typename Dtype>
void NPairMultiClassLossLayer<Dtype>::LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  CHECK(bottom[0]->num() == bottom[1]->num());                                  // reference .cpp:23
  num_ = bottom[0]->num();
  dim_ = bottom[0]->channels() * bottom[0]->height() * bottom[0]->width();      // reference .cu:215
  CHECK_GE(bottom[1]->count(), num_) << "label blob holds fewer than num labels";
  if (bottom.size() > 2) CHECK_EQ(bottom[2]->count(), num_) << "the anchor weight blob holds one weight per sample";

  npair_config cfg;
  npair_config_default(&cfg, num_, dim_);
  const NPairLossParameter& p = this->layer_param().npair_loss_param();         // reference .cpp:32-42
  cfg.margin_ident = p.margin_ident();
  cfg.margin_diff = p.margin_diff();
  cfg.identsn = p.identsn();
  cfg.diffsn = p.diffsn();
  cfg.ap_region = static_cast<int32_t>(p.ap_mining_region());                   // re-read every forward upstream (.cu:277-348)
  cfg.ap_method = static_cast<int32_t>(p.ap_mining_method());
  cfg.an_region = static_cast<int32_t>(p.an_mining_region());
  cfg.an_method = static_cast<int32_t>(p.an_mining_method());
  cfg.world = Caffe::NUM_GPU;                                                   // reference .cu:214
  cfg.rank = Caffe::RANK;                                                       // reference .cu:220
  cfg.num_tops = static_cast<int32_t>(top.size());
  if (sim_precision_ >= 0) cfg.sim_precision = sim_precision_;
  if (const char* e = getenv("NPAIR_SIM_PRECISION")) cfg.sim_precision = atoi(e);
  if (cfg.world > 1) CHECK(Caffe::nccl_unique_id() != nullptr) << "NUM_GPU > 1 needs Caffe::set_nccl_unique_id()";
  npair_ctx* old = ctx_;                   // destroyed AFTER the new context exists: the shared communicator stays referenced
  ctx_ = nullptr;
  // every layer instance of this process passes the same id: the library keeps ONE communicator per (process, id), so a second
  // instance (TRAIN + TEST nets) or a repeated LayerSetUp does not consume the ncclUniqueId again
  const int rc = npair_create(&cfg, Caffe::NUM_GPU > 1 ? Caffe::nccl_unique_id() : nullptr, &ctx_);
  if (old) npair_destroy(old);
  CHECK_EQ(rc, NPAIR_OK) << "npair_create: " << npair_last_error(nullptr);
  if (sizeof(Dtype) == 8) {
    CUDA_CHECK(cudaMalloc(&f32_feat_, sizeof(float) * static_cast<size_t>(num_) * dim_));
    CUDA_CHECK(cudaMalloc(&f32_label_, sizeof(float) * num_));
    CUDA_CHECK(cudaMalloc(&f32_diff_, sizeof(float) * static_cast<size_t>(num_) * dim_));
    if (bottom.size() > 2) CUDA_CHECK(cudaMalloc(&f32_weight_, sizeof(float) * num_));
  }
}

template <typename Dtype>
void NPairMultiClassLossLayer<Dtype>::Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  // batch size is frozen at setup upstream as well (reference .cpp:24-30, SURVEY Q13)
  CHECK_EQ(bottom[0]->num(), num_) << "NPairMultiClassLoss: batch size changed after LayerSetUp";
  if (bottom.size() > 2) CHECK_EQ(bottom[2]->count(), num_) << "the anchor weight blob holds one weight per sample";
  vector<int> shape(0);                                                         // 0-axis scalars (reference .cpp:160-163)
  for (size_t i = 0; i < top.size(); ++i) top[i]->Reshape(shape);
}

template <typename Dtype>
void NPairMultiClassLossLayer<Dtype>::Forward_cpu(const vector<Blob<Dtype>*>&, const vector<Blob<Dtype>*>&) {
  // The reference body is empty (npair_multi_class_loss.cpp:172-176), i.e. it silently produces nothing.
  // This build refuses instead: there is no CPU fallback for the product path.
  LOG(FATAL) << "NPairMultiClassLossLayer has no CPU path (reference Forward_cpu is empty); use Caffe::GPU on an H100";
}

template <typename Dtype>
void NPairMultiClassLossLayer<Dtype>::Backward_cpu(const vector<Blob<Dtype>*>&, const vector<bool>&, const vector<Blob<Dtype>*>&) {
  LOG(FATAL) << "NPairMultiClassLossLayer has no CPU path (reference Backward_cpu is empty); use Caffe::GPU on an H100";
}

template <typename Dtype>
void NPairMultiClassLossLayer<Dtype>::Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  float tops[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
  const bool weighted = bottom.size() > 2;
  int rc;
  if (sizeof(Dtype) == 4) {
    if (weighted) npair_set_anchor_io(ctx_, reinterpret_cast<const float*>(bottom[2]->gpu_data()), nullptr);
    rc = npair_forward(ctx_, reinterpret_cast<const float*>(bottom[0]->gpu_data()), reinterpret_cast<const float*>(bottom[1]->gpu_data()), tops, nullptr);
  } else {
    rc = npair_util_f64_to_f32(reinterpret_cast<const double*>(bottom[0]->gpu_data()), f32_feat_, static_cast<size_t>(num_) * dim_, nullptr);
    if (rc == NPAIR_OK) rc = npair_util_f64_to_f32(reinterpret_cast<const double*>(bottom[1]->gpu_data()), f32_label_, num_, nullptr);
    if (rc == NPAIR_OK && weighted) rc = npair_util_f64_to_f32(reinterpret_cast<const double*>(bottom[2]->gpu_data()), f32_weight_, num_, nullptr);
    if (rc == NPAIR_OK && weighted) npair_set_anchor_io(ctx_, f32_weight_, nullptr);
    if (rc == NPAIR_OK) rc = npair_forward(ctx_, f32_feat_, f32_label_, tops, nullptr);
  }
  // the weights are in the row records now (the backward reads those): the context's next forward is unweighted unless set again
  if (weighted) npair_set_anchor_io(ctx_, nullptr, nullptr);
  CHECK_EQ(rc, NPAIR_OK) << "npair_forward: " << npair_last_error(ctx_);
  // [loss, retrieve top-1, top-5, top-10, feature asum]; the last top is always the asum (reference .cu:388-401)
  for (size_t i = 0; i < top.size(); ++i) top[i]->mutable_cpu_data()[0] = static_cast<Dtype>(tops[i]);
}

template <typename Dtype>
void NPairMultiClassLossLayer<Dtype>::Backward_gpu(const vector<Blob<Dtype>*>& top, const vector<bool>& /*propagate_down: ignored upstream too (.cu:421-422)*/,
                                                  const vector<Blob<Dtype>*>& bottom) {
  const float loss_weight = static_cast<float>(top[0]->cpu_diff()[0]);          // reference .cu:435
  int rc;
  if (sizeof(Dtype) == 4) {
    rc = npair_backward(ctx_, loss_weight, reinterpret_cast<float*>(bottom[0]->mutable_gpu_diff()), nullptr);
  } else {
    rc = npair_backward(ctx_, loss_weight, f32_diff_, nullptr);
    if (rc == NPAIR_OK) rc = npair_util_f32_to_f64(f32_diff_, reinterpret_cast<double*>(bottom[0]->mutable_gpu_diff()), static_cast<size_t>(num_) * dim_, nullptr);
  }
  CHECK_EQ(rc, NPAIR_OK) << "npair_backward: " << npair_last_error(ctx_);
}

INSTANTIATE_CLASS(NPairMultiClassLossLayer);
REGISTER_LAYER_CLASS(NPairMultiClassLoss);

}  // namespace caffe
