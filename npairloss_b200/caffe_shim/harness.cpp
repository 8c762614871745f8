// C-callable test/bench harness around the Caffe-style layer (libnpair_caffe.so).  It plays the role of Caffe's Net for
// exactly one layer: parses a prototxt, builds bottoms/tops, calls Layer::SetUp / Forward / Backward.  Used by the
// Python tests and by bench.py's end-to-end leg (host bottoms -> H2D inside Blob::gpu_data(), D2H inside cpu_diff()).
#include <cstring>
#include <string>

#include "caffe/blob.hpp"
#include "caffe/common.hpp"
#include "caffe/layer_factory.hpp"
#include "caffe/proto/caffe.pb.h"

using namespace caffe;

namespace {
struct Net {
  shared_ptr<Layer<float> > layer;
  Blob<float> feat, label, weight;      // weight: the optional third bottom (anchor weights), when the layer block names one
  std::vector<Blob<float>*> bottom, top;
  std::vector<Blob<float> > top_store;
  LayerParameter param;
  std::string err;
  // optional second bottom set + copy stream: the role of Caffe's BasePrefetchingDataLayer (next batch goes to the device on
  // its own stream while the net computes on the current one)
  Blob<float> feat2, label2;
  std::vector<Blob<float>*> bottom2;
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ready[2] = {nullptr, nullptr}, done[2] = {nullptr, nullptr};
  std::vector<Blob<float>*>& set(int s) { return s ? bottom2 : bottom; }
};
thread_local std::string g_err;
void set_err(char* buf, int len, const std::string& m) {
  g_err = m;
  if (buf && len > 0) { strncpy(buf, m.c_str(), len - 1); buf[len - 1] = 0; }
}
}  // namespace

extern "C" {

// Parses `prototxt` (a whole net or a single layer block), instantiates the first layer of type NPairMultiClassLoss
// through the registry with bottoms shaped (num, channels, height, width) and (num) -- plus a third (num) bottom of anchor weights,
// all 1, when the layer block lists three bottoms -- and runs Layer::SetUp.
// world/rank set the fork statics Caffe::NUM_GPU / Caffe::RANK; nccl_id (128 B) is required when world > 1.
void* npc_net_create(const char* prototxt, int num, int channels, int height, int width, int world, int rank,
                     const void* nccl_id, int sim_precision, char* errbuf, int errlen) {
  try {
    std::vector<LayerParameter> layers;
    std::string perr;
    if (!ReadLayersFromText(prototxt ? prototxt : "", &layers, &perr)) { set_err(errbuf, errlen, "prototxt: " + perr); return nullptr; }
    const LayerParameter* lp = nullptr;
    for (size_t i = 0; i < layers.size(); ++i) if (layers[i].type() == "NPairMultiClassLoss") { lp = &layers[i]; break; }
    if (!lp) { set_err(errbuf, errlen, "no layer of type NPairMultiClassLoss in the prototxt"); return nullptr; }
    Caffe::set_mode(Caffe::GPU);
    Caffe::NUM_GPU = world; Caffe::RANK = rank; Caffe::MULTI_GPU = world > 1;
    Caffe::set_nccl_unique_id(nccl_id);
    if (sim_precision >= 0) setenv("NPAIR_SIM_PRECISION", std::to_string(sim_precision).c_str(), 1); else unsetenv("NPAIR_SIM_PRECISION");
    Net* n = new Net();
    n->param = *lp;
    n->feat.Reshape(num, channels, height, width);
    std::vector<int> ls(1, num);
    n->label.Reshape(ls);
    n->bottom.push_back(&n->feat); n->bottom.push_back(&n->label);
    if (lp->bottom_size() > 2) {
      n->weight.Reshape(ls);
      float* w = n->weight.mutable_cpu_data();
      for (int i = 0; i < num; ++i) w[i] = 1.f;
      n->bottom.push_back(&n->weight);
    }
    n->top_store.resize(lp->top_size());
    for (int t = 0; t < lp->top_size(); ++t) n->top.push_back(&n->top_store[t]);
    n->layer = LayerRegistry<float>::CreateLayer(n->param);
    n->layer->SetUp(n->bottom, n->top);
    return n;
  } catch (const std::exception& e) { set_err(errbuf, errlen, e.what()); return nullptr; }
}

void npc_net_destroy(void* h) {
  Net* n = static_cast<Net*>(h);
  if (n && n->copy_stream) {
    cudaStreamSynchronize(n->copy_stream);
    for (int s = 0; s < 2; ++s) { cudaEventDestroy(n->ready[s]); cudaEventDestroy(n->done[s]); }
    cudaStreamDestroy(n->copy_stream);
  }
  delete n;
}
const char* npc_last_error(void) { return g_err.c_str(); }

int npc_num_tops(void* h) { return static_cast<int>(static_cast<Net*>(h)->top.size()); }
const char* npc_layer_type(void* h) { return static_cast<Net*>(h)->layer->type(); }
// returns 8 floats: margin_ident, margin_diff, identsn, diffsn, ap_region, ap_method, an_region, an_method
void npc_layer_params(void* h, float* out8) {
  const NPairLossParameter& p = static_cast<Net*>(h)->param.npair_loss_param();
  out8[0] = p.margin_ident(); out8[1] = p.margin_diff(); out8[2] = p.identsn(); out8[3] = p.diffsn();
  out8[4] = static_cast<float>(p.ap_mining_region()); out8[5] = static_cast<float>(p.ap_mining_method());
  out8[6] = static_cast<float>(p.an_mining_region()); out8[7] = static_cast<float>(p.an_mining_method());
}
float npc_loss_weight(void* h, int top) { return static_cast<Net*>(h)->layer->loss(top); }

// Host (pinned) storage of bottom i's data; calling this marks the blob CPU-dirty exactly like a data layer writing a
// new batch through mutable_cpu_data(), so the next Forward pays the H2D copy.
float* npc_bottom_mutable_cpu_data(void* h, int i) {
  try { return static_cast<Net*>(h)->bottom[i]->mutable_cpu_data(); } catch (const std::exception& e) { g_err = e.what(); return nullptr; }
}
// Layer::Forward: returns 0 on success; tops5 receives top[i]->cpu_data()[0]; *loss the weighted loss
int npc_forward(void* h, float* tops5, float* loss) {
  Net* n = static_cast<Net*>(h);
  try {
    const float l = n->layer->Forward(n->bottom, n->top);
    for (size_t t = 0; t < n->top.size() && t < 5; ++t) tops5[t] = n->top[t]->cpu_data()[0];
    if (loss) *loss = l;
    return 0;
  } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
// Layer::Backward with propagate_down = {true, false}
int npc_backward(void* h) {
  Net* n = static_cast<Net*>(h);
  try {
    std::vector<bool> pd(2, false); pd[0] = true;
    n->layer->Backward(n->top, pd, n->bottom);
    return 0;
  } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
// bottom[0]->cpu_diff(): blocking D2H of the gradient into the blob's pinned host mirror
const float* npc_bottom_cpu_diff(void* h) {
  try { return static_cast<Net*>(h)->bottom[0]->cpu_diff(); } catch (const std::exception& e) { g_err = e.what(); return nullptr; }
}
// ---- prefetching (double-buffered bottoms) ----
int npc_prefetch_enable(void* h) {
  Net* n = static_cast<Net*>(h);
  try {
    if (n->copy_stream) return 0;
    n->feat2.Reshape(n->feat.shape()); n->label2.Reshape(n->label.shape());
    n->bottom2.clear(); n->bottom2.push_back(&n->feat2); n->bottom2.push_back(&n->label2);
    CUDA_CHECK(cudaStreamCreateWithFlags(&n->copy_stream, cudaStreamNonBlocking));     // must not serialise with the legacy stream
    for (int s = 0; s < 2; ++s) {
      CUDA_CHECK(cudaEventCreateWithFlags(&n->ready[s], cudaEventDisableTiming));
      CUDA_CHECK(cudaEventCreateWithFlags(&n->done[s], cudaEventDisableTiming));
      CUDA_CHECK(cudaEventRecord(n->done[s], 0));
    }
    return 0;
  } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
// host storage of bottom i of set s (marks it CPU-dirty)
float* npc_set_mutable_cpu_data(void* h, int s, int i) {
  try { return static_cast<Net*>(h)->set(s)[i]->mutable_cpu_data(); } catch (const std::exception& e) { g_err = e.what(); return nullptr; }
}
// start the H2D copy of set s on the copy stream, after the last step that used this set has finished on the device
int npc_prefetch(void* h, int s) {
  Net* n = static_cast<Net*>(h);
  try {
    CUDA_CHECK(cudaStreamWaitEvent(n->copy_stream, n->done[s], 0));
    n->set(s)[0]->data()->async_gpu_push(n->copy_stream);
    n->set(s)[1]->data()->async_gpu_push(n->copy_stream);
    CUDA_CHECK(cudaEventRecord(n->ready[s], n->copy_stream));
    return 0;
  } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
// Forward + Backward on set s: the layer's stream (legacy default) waits for the set's copy
int npc_step_set(void* h, int s, float* tops5) {
  Net* n = static_cast<Net*>(h);
  try {
    CUDA_CHECK(cudaStreamWaitEvent(0, n->ready[s], 0));
    n->layer->Forward(n->set(s), n->top);
    for (size_t t = 0; t < n->top.size() && t < 5; ++t) tops5[t] = n->top[t]->cpu_data()[0];
    std::vector<bool> pd(2, false); pd[0] = true;
    n->layer->Backward(n->top, pd, n->set(s));
    CUDA_CHECK(cudaEventRecord(n->done[s], 0));
    return 0;
  } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
const float* npc_set_cpu_diff(void* h, int s) {
  try { return static_cast<Net*>(h)->set(s)[0]->cpu_diff(); } catch (const std::exception& e) { g_err = e.what(); return nullptr; }
}

// Forward through the CPU entry point (fails loudly: no CPU path)
int npc_forward_cpu_mode(void* h) {
  Net* n = static_cast<Net*>(h);
  Caffe::set_mode(Caffe::CPU);
  int rc = 0;
  try { n->layer->Forward(n->bottom, n->top); } catch (const std::exception& e) { g_err = e.what(); rc = -1; }
  Caffe::set_mode(Caffe::GPU);
  return rc;
}
// prototxt reader only (no GPU): returns the number of layers or -1; fills out8 from the first NPairMultiClassLoss layer
int npc_parse_only(const char* prototxt, float* out8, int* ntops, int* nloss_weights, char* errbuf, int errlen) {
  std::vector<LayerParameter> layers;
  std::string perr;
  if (!ReadLayersFromText(prototxt ? prototxt : "", &layers, &perr)) { set_err(errbuf, errlen, perr); return -1; }
  for (size_t i = 0; i < layers.size(); ++i)
    if (layers[i].type() == "NPairMultiClassLoss") {
      const NPairLossParameter& p = layers[i].npair_loss_param();
      out8[0] = p.margin_ident(); out8[1] = p.margin_diff(); out8[2] = p.identsn(); out8[3] = p.diffsn();
      out8[4] = static_cast<float>(p.ap_mining_region()); out8[5] = static_cast<float>(p.ap_mining_method());
      out8[6] = static_cast<float>(p.an_mining_region()); out8[7] = static_cast<float>(p.an_mining_method());
      if (ntops) *ntops = layers[i].top_size();
      if (nloss_weights) *nloss_weights = layers[i].loss_weight_size();
      return static_cast<int>(layers.size());
    }
  set_err(errbuf, errlen, "no NPairMultiClassLoss layer");
  return -1;
}
// prototxt reader only: the number of bottoms of the first NPairMultiClassLoss layer, or -1
int npc_parse_num_bottoms(const char* prototxt) {
  std::vector<LayerParameter> layers;
  std::string perr;
  if (!ReadLayersFromText(prototxt ? prototxt : "", &layers, &perr)) return -1;
  for (size_t i = 0; i < layers.size(); ++i)
    if (layers[i].type() == "NPairMultiClassLoss") return layers[i].bottom_size();
  return -1;
}

}  // extern "C"
