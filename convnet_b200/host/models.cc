// models.cc — ModelConfig builders for the BASELINE configs (the reference reads these from pbtxt).
#include <cstdio>
#include <cstdlib>
#include <stdexcept>

#include "convnet.h"

namespace cnbhost {

namespace {
LayerConfig L(const char* name, int ch, Activation act = LINEAR, float dropprob = 0.f) {
  LayerConfig l; l.name = name; l.num_channels = ch; l.activation = act; l.dropprob = dropprob; return l;
}
EdgeConfig E(EdgeType t, int k = 1, int s = 1, int p = 0) {
  EdgeConfig e; e.edge_type = t; e.kernel_size = k; e.stride = s; e.padding = p;
  e.weight_optimizer.epsilon = 0.01f; e.weight_optimizer.final_momentum = 0.9f;
  e.bias_optimizer.epsilon = 0.01f; e.bias_optimizer.final_momentum = 0.9f;
  return e;
}
EdgeConfig Conv(int k, int s, int p, float l2 = 0.f) { EdgeConfig e = E(CONVOLUTIONAL, k, s, p); e.weight_optimizer.l2_decay = l2; return e; }
EdgeConfig Pool(int k, int s, int p) { return E(MAXPOOL, k, s, p); }
EdgeConfig RNorm(float add = 0.0005f, float pow = 0.75f, float frac = 0.25f) {
  EdgeConfig e = E(RESPONSE_NORM); e.add_scale = add; e.pow_scale = pow; e.frac_of_filters_response_norm = frac; return e;
}
void finish(ModelConfig& m) {
  for (size_t i = 0; i < m.edge.size(); i++) {
    m.edge[i].source = m.layer[i].name; m.edge[i].dest = m.layer[i + 1].name;
    m.edge[i].name = m.layer[i].name + ":" + m.layer[i + 1].name;
  }
}
}  // namespace

// examples/imagenet/CLS_net_20140801232522.pbtxt (SURVEY.md Appendix B, net A)
ModelConfig BuildAlexNet() {
  ModelConfig m; m.name = "CLS_net_20140801232522";
  LayerConfig in = L("input", 3); in.is_input = true; in.image_size_y = in.image_size_x = 224; in.image_size_t = 1;
  m.layer = {in,
             L("hidden1_conv", 96, RECTIFIED_LINEAR), L("hidden1_maxpool", 96), L("hidden1_rnorm", 96, RECTIFIED_LINEAR),
             L("hidden2_conv", 256, RECTIFIED_LINEAR), L("hidden2_conv_nin1", 256, RECTIFIED_LINEAR),
             L("hidden2_maxpool", 256), L("hidden2_rnorm", 256, RECTIFIED_LINEAR),
             L("hidden3_conv", 384, RECTIFIED_LINEAR), L("hidden3_conv_nin1", 768, RECTIFIED_LINEAR),
             L("hidden4_conv", 384, RECTIFIED_LINEAR), L("hidden4_conv_nin1", 768, RECTIFIED_LINEAR, 0.1f),
             L("hidden4_conv_nin2", 384, RECTIFIED_LINEAR),
             L("hidden5_conv", 512, RECTIFIED_LINEAR), L("hidden5_conv_nin1", 1024, RECTIFIED_LINEAR, 0.3f),
             L("hidden5_conv_nin2", 512, RECTIFIED_LINEAR), L("hidden5_maxpool", 512),
             L("hidden6", 4096, RECTIFIED_LINEAR, 0.5f), L("hidden7", 4096, RECTIFIED_LINEAR, 0.5f),
             L("output", 1000, SOFTMAX)};
  m.layer.back().is_output = true;
  m.edge = {Conv(7, 2, 1), Pool(3, 2, 1), RNorm(),
            Conv(5, 2, 1), E(CONV_ONETOONE), Pool(3, 2, 1), RNorm(),
            Conv(3, 1, 1, 0.0005f), E(CONV_ONETOONE),
            Conv(3, 1, 1, 0.0005f), E(CONV_ONETOONE), E(CONV_ONETOONE),
            Conv(3, 1, 0, 0.0005f), E(CONV_ONETOONE), E(CONV_ONETOONE), Pool(3, 2, 1),
            E(FC), E(FC), E(FC)};
  finish(m);
  return m;
}

// examples/mnist-conv/net.pbtxt (net M): 28x28x1 -conv4x4-> 25x25x48 -pool4/2-> 11x11x48 -conv4x4-> 8x8x128 -pool4/2-> 3x3x128 -fc-> 10
ModelConfig BuildLeNet() {
  ModelConfig m; m.name = "mnist-conv";
  LayerConfig in = L("input", 1); in.is_input = true; in.image_size_y = in.image_size_x = 28;
  m.layer = {in, L("hidden1_conv", 48, RECTIFIED_LINEAR), L("hidden1_maxpool", 48),
             L("hidden2_conv", 128, RECTIFIED_LINEAR), L("hidden2_maxpool", 128), L("output", 10, SOFTMAX)};
  m.layer.back().is_output = true;
  m.edge = {Conv(4, 1, 0, 0.0005f), Pool(4, 2, 0), Conv(4, 1, 0, 0.0005f), Pool(4, 2, 0), E(FC)};
  for (EdgeConfig& e : m.edge) { e.weight_optimizer.final_momentum = 0.95f; e.bias_optimizer.final_momentum = 0.95f; }
  finish(m);
  return m;
}

// C3D-style video net (SURVEY.md §8(d) cfg4): 16 x 112 x 112 x 3 clips, 3x3x3 kernels, pad y/x 1, pad t 0
ModelConfig BuildC3D() {
  ModelConfig m; m.name = "c3d";
  LayerConfig in = L("input", 3); in.is_input = true; in.image_size_y = in.image_size_x = 112; in.image_size_t = 16;
  m.layer = {in, L("conv1a", 64, RECTIFIED_LINEAR), L("pool1", 64), L("conv2a", 128, RECTIFIED_LINEAR), L("pool2", 128),
             L("conv3a", 256, RECTIFIED_LINEAR), L("pool3", 256), L("output", 101, SOFTMAX)};
  m.layer.back().is_output = true;
  auto c3 = []() { EdgeConfig e = Conv(3, 1, 1); e.kernel_size_t = 3; e.stride_t = 1; e.padding_t = 0; return e; };
  auto p3 = [](int kt) { EdgeConfig e = Pool(2, 2, 0); e.kernel_size_t = kt; e.stride_t = kt; e.padding_t = 0; return e; };
  EdgeConfig gp = Pool(0, 1, 0); gp.kernel_size_t = 0; gp.stride_t = 1;     // global pooling before the classifier
  m.edge = {c3(), p3(1), c3(), p3(2), c3(), gp, E(FC)};
  finish(m);
  return m;
}

// small net touching every edge type, used by tests and the grad check
ModelConfig BuildTinyNet() {
  ModelConfig m; m.name = "tiny";
  LayerConfig in = L("input", 8); in.is_input = true; in.image_size_y = in.image_size_x = 12;
  m.layer = {in, L("conv1", 16, RECTIFIED_LINEAR), L("pool1", 16), L("rnorm1", 16, RECTIFIED_LINEAR),
             L("nin1", 24, RECTIFIED_LINEAR), L("conv2", 16, RECTIFIED_LINEAR), L("avgpool", 16), L("output", 10, SOFTMAX)};
  m.layer.back().is_output = true;
  EdgeConfig ap = E(AVGPOOL, 2, 2, 0);
  m.edge = {Conv(3, 1, 1), Pool(3, 2, 1), RNorm(0.01f, 0.75f, 0.5f), E(CONV_ONETOONE), Conv(3, 2, 1), ap, E(FC)};
  for (EdgeConfig& e : m.edge) { e.grad_check = true; e.grad_check_num_params = 8; e.grad_check_epsilon = {1e-2f, 3e-3f, 1e-3f}; }
  finish(m);
  return m;
}

// net for run_grad_check: one edge of every weighted type around pooling and response-norm, with SMOOTH
// activations (linear units, average pooling).  Finite differences are only meaningful away from kinks: with
// ReLU / max-pool a unit that sits within epsilon of its kink makes the central difference the AVERAGE of two
// one-sided slopes at every epsilon (observed: float64 finite differences show the same), so the reference's 1 %
// criterion (grad_check.cc:61) is a data lottery there.  The ReLU / max-pool backward ops are verified against
// float64 autograd instead (tests/test_gpu_net.py::test_backprop_matches_float64_autograd).
ModelConfig BuildGradCheckNet() {
  ModelConfig m; m.name = "gradcheck";
  LayerConfig in = L("input", 4); in.is_input = true; in.image_size_y = in.image_size_x = 8;
  m.layer = {in, L("conv1", 8), L("pool1", 8), L("rnorm1", 8), L("nin1", 12), L("output", 5, SOFTMAX)};
  m.layer.back().is_output = true;
  m.edge = {Conv(3, 1, 1), E(AVGPOOL, 3, 2, 1), RNorm(0.01f, 0.75f, 0.5f), E(CONV_ONETOONE), E(FC)};
  for (EdgeConfig& e : m.edge) { e.grad_check = true; e.grad_check_num_params = 10; e.grad_check_epsilon = {1e-2f, 3e-3f, 1e-3f}; }
  finish(m);
  return m;
}

// the gradcheck net with logistic units in every hidden layer: the grad check of a smooth nonlinearity through the conv,
// average-pooling, response-norm, 1x1 and FC edges (sigma after the pooling and sigma' into its undo run as passes).
// init_wt 3: each sigma' scales the derivative by at most 1/4, and at the default scale the derivative reaching conv1
// through four logistic layers sits at the float32 noise floor of the finite differences
ModelConfig BuildLogCheckNet() {
  ModelConfig m = BuildGradCheckNet();
  m.name = "logcheck";
  for (LayerConfig& l : m.layer)
    if (!l.is_input && !l.is_output) l.activation = LOGISTIC;
  for (EdgeConfig& e : m.edge)
    if (e.edge_type == CONVOLUTIONAL || e.edge_type == CONV_ONETOONE || e.edge_type == FC) e.init_wt = 3.f;
  return m;
}

// conv + locally connected classifier (cuda-convnet's conv+local nets, scaled to 96 x 96 inputs): the two LOCAL edges
// carry a filter bank per output position (42 and 29 MB in bf16) and sit near the HBM / tensor-core balance point at
// batch 128.  init_wt = sqrt(modules): the reference scales a local edge's initial weights by 1/sqrt(K*modules/3)
// (weights_.GetCols(), edge_with_weight.cc:126); this undoes the modules factor, giving a conv-like initial scale.
ModelConfig BuildLcNet() {
  ModelConfig m; m.name = "lcnet";
  LayerConfig in = L("input", 3); in.is_input = true; in.image_size_y = in.image_size_x = 96;
  m.layer = {in, L("conv1", 64, RECTIFIED_LINEAR), L("pool1", 64), L("conv2", 128, RECTIFIED_LINEAR), L("pool2", 128),
             L("local3", 128, RECTIFIED_LINEAR), L("local4", 128, RECTIFIED_LINEAR), L("fc5", 1024, RECTIFIED_LINEAR, 0.5f),
             L("output", 1000, SOFTMAX)};
  m.layer.back().is_output = true;
  EdgeConfig l3 = E(LOCAL, 3, 1, 1), l4 = E(LOCAL, 3, 1, 0);
  l3.init_wt = 12.f;                                        // sqrt(12 x 12 modules)
  l4.init_wt = 10.f;                                        // sqrt(10 x 10 modules)
  m.edge = {Conv(5, 2, 2), Pool(3, 2, 1), Conv(3, 1, 1), Pool(3, 2, 1), l3, l4, E(FC), E(FC)};
  finish(m);
  return m;
}

// run_grad_check net for the LOCAL edge, smooth like BuildGradCheckNet (linear units, average pooling): one local edge
// with padding, one with stride 2 and no padding, then an FC.  init_wt = sqrt(modules) as in lcnet: with the reference's
// 1/sqrt(K*modules/3) scale the derivative reaching local1 is so small that its per-feature bias gradients sit at the
// float32 noise floor of the finite differences.  The check reads the FIRST parameters of a tensor, which for a local edge
// are the taps of module 0 (the top-left corner).  With padding 1, 5 of local1's 9 taps there only ever read padding, so
// local1 checks 72 parameters: all 8 outputs x 9 taps of input channel 0 of module 0, 32 of them live (the pairs whose
// analytic and numeric gradients are both exactly 0 do not enter the mean).
ModelConfig BuildLocalCheckNet() {
  ModelConfig m; m.name = "localcheck";
  LayerConfig in = L("input", 4); in.is_input = true; in.image_size_y = in.image_size_x = 8;
  m.layer = {in, L("local1", 8), L("pool1", 8), L("local2", 8), L("output", 5, SOFTMAX)};
  m.layer.back().is_output = true;
  EdgeConfig l1 = E(LOCAL, 3, 1, 1), l2 = E(LOCAL, 3, 2, 0);
  l1.init_wt = 8.f;                                         // sqrt(8 x 8 modules)
  l2.init_wt = 3.f;                                         // sqrt(3 x 3 modules)
  m.edge = {l1, E(AVGPOOL, 2, 1, 0), l2, E(FC)};
  for (EdgeConfig& e : m.edge) { e.grad_check = true; e.grad_check_num_params = 10; e.grad_check_epsilon = {1e-2f, 3e-3f, 1e-3f}; }
  m.edge[0].grad_check_num_params = 8 * 9;
  finish(m);
  return m;
}

EdgeConfig Sample(EdgeType t, int f) { EdgeConfig e = E(t); e.sample_factor = f; return e; }

// encoder-decoder at bench size: a YUV front end, two 2x down-samplings and two 2x up-samplings between 3x3 convs, and a
// LINEAR 3-channel output trained on a float target per pixel (SQUARED_ERROR).  128 x 128 inputs; the up-sampled 128-channel
// layer is the largest tensor (8 MB per image)
ModelConfig BuildUpDownNet() {
  ModelConfig m; m.name = "updown";
  LayerConfig in = L("input", 3); in.is_input = true; in.image_size_y = in.image_size_x = 128;
  m.layer = {in, L("yuv", 3), L("conv1", 64, RECTIFIED_LINEAR), L("down1", 64), L("conv2", 128, RECTIFIED_LINEAR),
             L("down2", 128), L("conv3", 256, RECTIFIED_LINEAR), L("up3", 256), L("conv4", 128, RECTIFIED_LINEAR),
             L("up4", 128), L("conv5", 64, RECTIFIED_LINEAR), L("output", 3)};
  LayerConfig& out = m.layer.back();
  out.is_output = true; out.loss_function = SQUARED_ERROR; out.performance_metric = SQUARED_ERROR;
  m.edge = {E(RGBTOYUV), Conv(3, 1, 1), Sample(DOWNSAMPLE, 2), Conv(3, 1, 1), Sample(DOWNSAMPLE, 2), Conv(3, 1, 1),
            Sample(UPSAMPLE, 2), Conv(3, 1, 1), Sample(UPSAMPLE, 2), Conv(3, 1, 1), Conv(3, 1, 1)};
  finish(m);
  return m;
}

// run_grad_check net for the sampling edges, smooth like BuildGradCheckNet: down- and up-sampling by 3 and by 2, a conv
// under every sampling edge, a logistic layer written by an UPSAMPLE (sigma after the up-sampling, sigma' into its block
// sum as passes) and LINEAR units elsewhere, then an FC into a softmax as in gradcheck: the loss of a per-pixel regression
// output (SQUARED_ERROR on random targets) is so large that its float32 rounding drowns the finite differences
ModelConfig BuildUpDownCheckNet() {
  ModelConfig m; m.name = "updowncheck";
  LayerConfig in = L("input", 4); in.is_input = true; in.image_size_y = in.image_size_x = 6;
  m.layer = {in, L("conv1", 8), L("down1", 8), L("conv2", 8), L("up2", 8, LOGISTIC), L("conv3", 6), L("down3", 6),
             L("conv4", 6), L("up4", 6), L("output", 5, SOFTMAX)};
  m.layer.back().is_output = true;
  m.edge = {Conv(3, 1, 1), Sample(DOWNSAMPLE, 3), Conv(3, 1, 1), Sample(UPSAMPLE, 3), Conv(3, 1, 1), Sample(DOWNSAMPLE, 2),
            Conv(3, 1, 1), Sample(UPSAMPLE, 2), E(FC)};
  for (EdgeConfig& e : m.edge) { e.grad_check = true; e.grad_check_num_params = 10; e.grad_check_epsilon = {1e-2f, 3e-3f, 1e-3f}; }
  finish(m);
  return m;
}

// weight sharing (EdgeConfig::tied_to) on the training path: one 64 -> 64 3x3 conv runs at three geometries — 32 x 32
// with padding 1, 16 x 16 after a max-pool, and with stride 2 — so one filter tensor keeps three sets of dgrad banks; and
// two 256 -> 256 FC edges share weights with the LOWER edge naming the higher one, so the shared slice sits at the tied
// edge rather than at its owner.  Dropout on the owner's output layer, a softmax classifier
ModelConfig BuildTiedNet() {
  ModelConfig m; m.name = "tiednet";
  LayerConfig in = L("input", 3); in.is_input = true; in.image_size_y = in.image_size_x = 32;
  m.layer = {in, L("conv1", 64, RECTIFIED_LINEAR), L("conv2", 64, RECTIFIED_LINEAR), L("pool2", 64),
             L("conv3", 64, RECTIFIED_LINEAR), L("conv4", 64, RECTIFIED_LINEAR), L("fc5", 256, RECTIFIED_LINEAR),
             L("fc6", 256, RECTIFIED_LINEAR), L("fc7", 256, RECTIFIED_LINEAR, 0.5f), L("output", 10, SOFTMAX)};
  m.layer.back().is_output = true;
  m.edge = {Conv(3, 1, 1), Conv(3, 1, 1), Pool(2, 2, 0), Conv(3, 1, 1), Conv(3, 2, 1), E(FC), E(FC), E(FC), E(FC)};
  finish(m);
  m.edge[3].tied_to = m.edge[4].tied_to = m.edge[1].name;          // pool2:conv3 and conv3:conv4 run conv1:conv2's filters
  m.edge[6].tied_to = m.edge[7].name;                                // fc5:fc6 runs with fc6:fc7's weights
  return m;
}

// run_grad_check net for ties, smooth like BuildGradCheckNet (linear units, average pooling): a conv used at padding 1
// and padding 0, a CONV_ONETOONE, a LOCAL and an FC tie (the FC one named by the lower edge).  grad_check is set on every
// edge with parameters of its own; an owner's check perturbs the shared tensors, so it checks the summed gradient
ModelConfig BuildTiedCheckNet() {
  ModelConfig m; m.name = "tiedcheck";
  LayerConfig in = L("input", 4); in.is_input = true; in.image_size_y = in.image_size_x = 8;
  m.layer = {in, L("c0", 8), L("c1", 8), L("c2", 8), L("pool", 8), L("o1", 8), L("o2", 8), L("l1", 8), L("l2", 8),
             L("f1", 16), L("f2", 16), L("f3", 16), L("output", 5, SOFTMAX)};
  m.layer.back().is_output = true;
  EdgeConfig l1 = E(LOCAL, 3, 1, 1);
  l1.init_wt = 3.f;                                         // sqrt(3 x 3 modules), as in localcheck
  m.edge = {Conv(3, 1, 1), Conv(3, 1, 1), Conv(3, 1, 0), E(AVGPOOL, 2, 2, 0), E(CONV_ONETOONE), E(CONV_ONETOONE), l1, l1,
            E(FC), E(FC), E(FC), E(FC)};
  finish(m);
  m.edge[2].tied_to = m.edge[1].name;                                // 8 x 8 at padding 1, then at padding 0
  m.edge[5].tied_to = m.edge[4].name;
  m.edge[7].tied_to = m.edge[6].name;
  m.edge[9].tied_to = m.edge[10].name;
  for (EdgeConfig& e : m.edge) {
    e.grad_check = e.tied_to.empty(); e.grad_check_num_params = 10; e.grad_check_epsilon = {1e-2f, 3e-3f, 1e-3f};
  }
  m.edge[6].grad_check_num_params = 8 * 9;                 // module 0's taps of input channel 0 (see localcheck)
  return m;
}

// "<model>+ref-optimizer": the optimizer blocks of the model's pbtxt exactly (BuildAlexNet / BuildLeNet keep the constant
// momentum and leave out the norm rules and the FC l2_decay)
static void UseReferenceOptimizers(const std::string& base, ModelConfig& m) {
  OptimizerConfig o;                                        // every weight and bias optimizer of both files
  o.epsilon = 0.01f;
  if (base == "alexnet") {        // examples/imagenet/CLS_net_20140801232522.pbtxt:148-505
    o.initial_momentum = 0.5f; o.final_momentum = 0.9f; o.momentum_transition_timescale = 2000;
    for (EdgeConfig& e : m.edge) {
      const float l2 = e.weight_optimizer.l2_decay;        // conv3-5: 0.0005, as BuildAlexNet has it
      e.weight_optimizer = o; e.bias_optimizer = o;
      e.weight_optimizer.l2_decay = l2;
      if (e.edge_type == CONV_ONETOONE) e.weight_optimizer.weight_norm_constraint = 1.f;
      if (e.edge_type == FC) { e.weight_optimizer.weight_norm_limit = 4.f; e.weight_optimizer.l2_decay = 0.0005f; }
    }
  } else {                        // examples/mnist-conv/net.pbtxt:60-127
    OptimizerConfig w = o, b = o;
    w.initial_momentum = 0.5f; w.final_momentum = 0.95f; w.l2_decay = 0.0005f;    // no transition timescale: 0.95 throughout
    b.final_momentum = 0.95f;
    for (EdgeConfig& e : m.edge) {
      e.weight_optimizer = w; e.bias_optimizer = b;
      if (e.edge_type == FC) e.weight_optimizer.weight_norm_limit = 4.f;
    }
  }
}

// "<model>+bn": batch_normalize on every hidden layer written by a conv, 1x1 or FC edge.  gamma trains with the writing
// edge's weight optimizer and beta with its bias optimizer, both without L2 decay and norm rules (a per-channel scale and
// shift are not weights of a unit; the reference's norm rules would not apply to a [1 x channels] row anyway)
static void UseBatchNorm(const std::string& name, ModelConfig& m) {
  if (m.layer.front().image_size_t > 1)
    throw std::invalid_argument("model '" + name + "': batch normalisation is not supported on 3-D layers (image_size_t > 1)");
  for (size_t i = 0; i < m.edge.size(); i++) {
    const EdgeConfig& e = m.edge[i];
    LayerConfig& l = m.layer[i + 1];
    if (l.is_output || (e.edge_type != CONVOLUTIONAL && e.edge_type != CONV_ONETOONE && e.edge_type != FC && e.edge_type != LOCAL))
      continue;
    if (l.batch_normalize) throw std::invalid_argument("model '" + name + "': +bn is given twice");
    l.batch_normalize = true;
    l.gamma_optimizer = e.weight_optimizer;
    l.beta_optimizer = e.bias_optimizer;
    for (OptimizerConfig* o : {&l.gamma_optimizer, &l.beta_optimizer}) {
      o->l2_decay = 0.f; o->weight_norm_limit = 0.f; o->weight_norm_constraint = 0.f;
    }
  }
}

// "<model>+adagrad" / "<model>+rmsprop": every weight, bias, gamma and beta optimizer of the model switched to that rule,
// the other fields kept except epsilon, which is scaled so that the step stays near the plain model's:
//   +adagrad  adagrad_delta 1 (the proto's default), epsilon x 0.1.  While sqrt(sum g^2) is small against delta the rule is
//             SGD with its gradient scaled by sqrt(step + 1) (5.6 at step 30, 10 at step 100); the 0.1 keeps the first
//             ~100 steps at or below the plain model's step size.
//   +rmsprop  rms_prop_factor 0.9, epsilon x 0.01.  Once s tracks the root mean square of the gradient, the step of every
//             element is about epsilon / (1 - momentum) = 10 epsilon: 1e-3 at the models' epsilon 0.01, the usual step of
//             a normalised-gradient method.
static void UseAdaptiveOptimizers(int type, ModelConfig& m) {
  auto use = [type](OptimizerConfig& o) {
    o.optimizer_type = type;
    if (type == ADAGRAD_SGD) { o.adagrad_delta = 1.f; o.epsilon *= 0.1f; o.minimum_epsilon *= 0.1f; }
    else { o.rms_prop_factor = 0.9f; o.epsilon *= 0.01f; o.minimum_epsilon *= 0.01f; }
  };
  for (EdgeConfig& e : m.edge) { use(e.weight_optimizer); use(e.bias_optimizer); }
  for (LayerConfig& l : m.layer)
    if (l.batch_normalize) { use(l.gamma_optimizer); use(l.beta_optimizer); }
}

// "<model>+logistic": every hidden RECTIFIED_LINEAR layer becomes LOGISTIC (the parameter layout does not change)
static void UseLogisticUnits(const std::string& name, ModelConfig& m) {
  bool any = false;
  for (LayerConfig& l : m.layer)
    if (!l.is_output && l.activation == RECTIFIED_LINEAR) { l.activation = LOGISTIC; any = true; }
  if (!any) throw std::invalid_argument("model '" + name + "': +logistic finds no RECTIFIED_LINEAR hidden layer");
}

// the output suffixes: the output layer's activation, loss function and performance metric (at most one per model)
//   +squared-error  LINEAR, SQUARED_ERROR, metric SQUARED_ERROR (regression on a float target per output unit)
//   +binary-ce      LOGISTIC, CROSS_ENTROPY_BINARY, metric CLASSIFICATION_BINARY (independent binary labels; t < 0: don't care)
//   +soft-targets   SOFTMAX_DIST, CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED, metric the same (a distribution over the classes)
struct OutputSuffix { const char* suffix; Activation act; int loss, metric; };
static const OutputSuffix kOutputSuffixes[] = {
    {"+squared-error", LINEAR, SQUARED_ERROR, SQUARED_ERROR},
    {"+binary-ce", LOGISTIC, CROSS_ENTROPY_BINARY, CLASSIFICATION_BINARY},
    {"+soft-targets", SOFTMAX_DIST, CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED, CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED}};

static bool EndsWith(const std::string& s, const std::string& suffix) {
  return s.size() > suffix.size() && s.compare(s.size() - suffix.size(), suffix.size(), suffix) == 0;
}

ModelConfig BuildModel(const std::string& name) {
  if (EndsWith(name, ".pbtxt")) return ReadModelFile(name);          // no suffix ends in ".pbtxt"
  for (const OutputSuffix& o : kOutputSuffixes) {
    if (!EndsWith(name, o.suffix)) continue;
    ModelConfig m = BuildModel(name.substr(0, name.size() - std::string(o.suffix).size()));
    LayerConfig& out = m.layer.back();
    if (out.activation != SOFTMAX || out.loss_function != CROSS_ENTROPY_MULTINOMIAL)
      throw std::invalid_argument("model '" + name + "': one output suffix only (+squared-error, +binary-ce, +soft-targets)");
    out.activation = o.act; out.loss_function = o.loss; out.performance_metric = o.metric;
    return m;
  }
  if (EndsWith(name, "+logistic")) {
    ModelConfig m = BuildModel(name.substr(0, name.size() - 9));
    UseLogisticUnits(name, m);
    return m;
  }
  for (const auto& [suffix, type] : {std::make_pair(std::string("+adagrad"), (int)ADAGRAD_SGD),
                                     std::make_pair(std::string("+rmsprop"), (int)RMSPROP_SGD)}) {
    if (name.size() > suffix.size() && name.compare(name.size() - suffix.size(), suffix.size(), suffix) == 0) {
      ModelConfig m = BuildModel(name.substr(0, name.size() - suffix.size()));
      for (const EdgeConfig& e : m.edge)
        if (IsAdaptive(e.weight_optimizer)) throw std::invalid_argument("model '" + name + "': one adaptive rule only");
      UseAdaptiveOptimizers(type, m);
      return m;
    }
  }
  const std::string bn = "+bn";
  if (name.size() > bn.size() && name.compare(name.size() - bn.size(), bn.size(), bn) == 0) {
    ModelConfig m = BuildModel(name.substr(0, name.size() - bn.size()));
    UseBatchNorm(name, m);
    return m;
  }
  const std::string ref = "+ref-optimizer";
  if (name.size() > ref.size() && name.compare(name.size() - ref.size(), ref.size(), ref) == 0) {
    const std::string base = name.substr(0, name.size() - ref.size());
    if (base != "alexnet" && base != "lenet")
      throw std::invalid_argument("model '" + name + "': +ref-optimizer is defined for alexnet and lenet only");
    ModelConfig m = BuildModel(base);
    UseReferenceOptimizers(base, m);
    return m;
  }
  // "<model>+gradcheck": the model with run_grad_check's edge flags as BASELINE config 1 states them
  // (grad_check_num_params: 10, grad_check_epsilon: [1e-2, 1e-3, 1e-4]; src/grad_check.cc:20-61)
  const std::string suffix = "+gradcheck";
  if (name.size() > suffix.size() && name.compare(name.size() - suffix.size(), suffix.size(), suffix) == 0) {
    ModelConfig m = BuildModel(name.substr(0, name.size() - suffix.size()));
    const int frozen = FrozenEdges(m.edge);
    for (int i = 0; i < (int)m.edge.size(); i++) {        // (a tied edge is checked through its owner, a frozen one not at all)
      EdgeConfig& e = m.edge[i];
      e.grad_check = e.tied_to.empty() && i >= frozen; e.grad_check_num_params = 10; e.grad_check_epsilon = {1e-2f, 1e-3f, 1e-4f};
    }
    return m;
  }
  // "<model>+finetune": block_backprop on every edge below the lowest FC edge, whose grad_check flags go (a frozen edge has
  // no gradient to check): the trunk keeps its weights and the FC classifier trains on its features
  if (EndsWith(name, "+finetune")) {
    ModelConfig m = BuildModel(name.substr(0, name.size() - 9));
    size_t fc = 0;
    while (fc < m.edge.size() && m.edge[fc].edge_type != FC) fc++;
    if (fc == m.edge.size()) throw std::invalid_argument("model '" + name + "': +finetune trains the FC edges, and it has none");
    for (size_t i = 0; i < fc; i++) { m.edge[i].block_backprop = true; m.edge[i].grad_check = false; }
    return m;
  }
  if (name == "gradcheck") return BuildGradCheckNet();
  if (name == "tiednet") return BuildTiedNet();
  if (name == "tiedcheck") return BuildTiedCheckNet();
  if (name == "logcheck") return BuildLogCheckNet();
  if (name == "alexnet") return BuildAlexNet();
  if (name == "lenet") return BuildLeNet();
  if (name == "c3d") return BuildC3D();
  if (name == "tiny") return BuildTinyNet();
  if (name == "lcnet") return BuildLcNet();
  if (name == "localcheck") return BuildLocalCheckNet();
  if (name == "updown") return BuildUpDownNet();
  if (name == "updowncheck") return BuildUpDownCheckNet();
  throw std::invalid_argument("unknown model '" + name + "'");
}

}  // namespace cnbhost
