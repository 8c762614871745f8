// NPairMultiClassLossLayer -- H100-native drop-in for the reference layer (quziyan/NPairLoss
// npair_multi_class_loss.hpp:17-79).  Same class name, registry type string, virtuals, blob-count contract and top
// layout; the implementation is new: every device computation sits behind the C ABI of include/npair_b200.h, so this
// class is ~100 lines of plain C++ (no .cu file, no cuBLAS, no MPI, no host loops over the similarity matrix).
#ifndef CAFFE_NPAIR_MULTI_CLASS_LOSS_LAYER_HPP_
#define CAFFE_NPAIR_MULTI_CLASS_LOSS_LAYER_HPP_

#include <string>
#include <vector>

#include "caffe/blob.hpp"
#include "caffe/common.hpp"
#include "caffe/layer.hpp"
#include "caffe/loss_layers.hpp"
#include "caffe/proto/caffe.pb.h"

struct npair_ctx;   // include/npair_b200.h

namespace caffe {

template <typename Dtype>
class NPairMultiClassLossLayer : public LossLayer<Dtype> {
 public:
  explicit NPairMultiClassLossLayer(const LayerParameter& param) : LossLayer<Dtype>(param) {}
  virtual ~NPairMultiClassLossLayer();
  virtual void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);

  virtual inline const char* type() const { return "NPairMultiClassLoss"; }   // reference .hpp:30
  // features, labels (.hpp:31), and, as an extension, an optional third bottom of num anchor weights in [0, 1] (npair_set_anchor_io,
  // DESIGN 4.5): the loss becomes -(1/num) sum_i w_i log(A_i / T_i) and the gradient that of it.  The weights get no gradient.
  virtual inline int ExactNumBottomBlobs() const { return -1; }
  virtual inline int MinBottomBlobs() const { return 2; }
  virtual inline int MaxBottomBlobs() const { return 3; }
  virtual inline int ExactNumTopBlobs() const { return -1; }                  // .hpp:32
  virtual inline int MinTopBlobs() const { return 1; }                        // .hpp:33
  virtual inline int MaxTopBlobs() const { return 5; }                        // .hpp:34

  // Extension (not in the reference): operand precision of the tensor-core contractions, NPAIR_PREC_* of
  // include/npair_b200.h.  Default NPAIR_PREC_FP32_FP16X2; environment NPAIR_SIM_PRECISION overrides at LayerSetUp.
  void set_sim_precision(int p) { sim_precision_ = p; }

 protected:
  virtual void Forward_cpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual void Backward_cpu(const vector<Blob<Dtype>*>& top, const vector<bool>& propagate_down, const vector<Blob<Dtype>*>& bottom);
  virtual void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual void Backward_gpu(const vector<Blob<Dtype>*>& top, const vector<bool>& propagate_down, const vector<Blob<Dtype>*>& bottom);

 private:
  npair_ctx* ctx_ = nullptr;
  int num_ = 0, dim_ = 0;
  int sim_precision_ = -1;
  // Dtype == double: the device path is fp32 (as is the reference's expf/logf/FLT_MAX arithmetic, SURVEY Q14);
  // features/labels/gradients are converted on the device through these staging buffers.
  float *f32_feat_ = nullptr, *f32_label_ = nullptr, *f32_diff_ = nullptr, *f32_weight_ = nullptr;
};

}  // namespace caffe
#endif
