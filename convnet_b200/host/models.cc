// models.cc — the built-in models, each a config::Model text that ReadModelText (model_file.cc) reads as it reads a model
// file, and the name suffixes that derive a variant of any model ("+bn", "+rmsprop", ...).
#include <stdexcept>

#include "convnet.h"

namespace cnbhost {

namespace {
// The reader applies the proto's defaults, so each text states where a model departs from them: the seed, the optimizers'
// epsilon and momentum, shared_bias on every convolution, DENSE_UNIFORM_SQRT_FAN_IN on every edge with weights of its
// own, the response-norm constants, the sampling factors and the grad_check settings.  A block too long for one line
// continues on the next
struct BuiltIn { const char* name; const char* text; };
const BuiltIn kBuiltIns[] = {
{"alexnet", R"pb(
# examples/imagenet/CLS_net_20140801232522.pbtxt (SURVEY.md Appendix B, net A), with constant momentum and without the
# norm rules and the FC l2_decay ("alexnet+ref-optimizer" has the file's optimizer blocks exactly)
name: "CLS_net_20140801232522"
seed: 42
default_weight_optimizer { epsilon: 0.01 final_momentum: 0.9 }
default_bias_optimizer { epsilon: 0.01 final_momentum: 0.9 }
layer { name: "input" num_channels: 3 image_size_y: 224 image_size_x: 224 }
layer { name: "hidden1_conv" num_channels: 96 activation: RECTIFIED_LINEAR }
layer { name: "hidden1_maxpool" num_channels: 96 }
layer { name: "hidden1_rnorm" num_channels: 96 activation: RECTIFIED_LINEAR }
layer { name: "hidden2_conv" num_channels: 256 activation: RECTIFIED_LINEAR }
layer { name: "hidden2_conv_nin1" num_channels: 256 activation: RECTIFIED_LINEAR }
layer { name: "hidden2_maxpool" num_channels: 256 }
layer { name: "hidden2_rnorm" num_channels: 256 activation: RECTIFIED_LINEAR }
layer { name: "hidden3_conv" num_channels: 384 activation: RECTIFIED_LINEAR }
layer { name: "hidden3_conv_nin1" num_channels: 768 activation: RECTIFIED_LINEAR }
layer { name: "hidden4_conv" num_channels: 384 activation: RECTIFIED_LINEAR }
layer { name: "hidden4_conv_nin1" num_channels: 768 activation: RECTIFIED_LINEAR dropprob: 0.1 }
layer { name: "hidden4_conv_nin2" num_channels: 384 activation: RECTIFIED_LINEAR }
layer { name: "hidden5_conv" num_channels: 512 activation: RECTIFIED_LINEAR }
layer { name: "hidden5_conv_nin1" num_channels: 1024 activation: RECTIFIED_LINEAR dropprob: 0.3 }
layer { name: "hidden5_conv_nin2" num_channels: 512 activation: RECTIFIED_LINEAR }
layer { name: "hidden5_maxpool" num_channels: 512 }
layer { name: "hidden6" num_channels: 4096 activation: RECTIFIED_LINEAR dropprob: 0.5 }
layer { name: "hidden7" num_channels: 4096 activation: RECTIFIED_LINEAR dropprob: 0.5 }
layer { name: "output" num_channels: 1000 activation: SOFTMAX }
edge { source: "input" dest: "hidden1_conv" edge_type: CONVOLUTIONAL kernel_size: 7 stride: 2 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "hidden1_conv" dest: "hidden1_maxpool" edge_type: MAXPOOL kernel_size: 3 stride: 2 padding: 1 }
edge { source: "hidden1_maxpool" dest: "hidden1_rnorm" edge_type: RESPONSE_NORM
       add_scale: 0.0005 pow_scale: 0.75 frac_of_filters_response_norm: 0.25 }
edge { source: "hidden1_rnorm" dest: "hidden2_conv" edge_type: CONVOLUTIONAL kernel_size: 5 stride: 2 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "hidden2_conv" dest: "hidden2_conv_nin1" edge_type: CONV_ONETOONE
       initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "hidden2_conv_nin1" dest: "hidden2_maxpool" edge_type: MAXPOOL kernel_size: 3 stride: 2 padding: 1 }
edge { source: "hidden2_maxpool" dest: "hidden2_rnorm" edge_type: RESPONSE_NORM
       add_scale: 0.0005 pow_scale: 0.75 frac_of_filters_response_norm: 0.25 }
edge { source: "hidden2_rnorm" dest: "hidden3_conv" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN weight_optimizer { l2_decay: 0.0005 } }
edge { source: "hidden3_conv" dest: "hidden3_conv_nin1" edge_type: CONV_ONETOONE
       initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "hidden3_conv_nin1" dest: "hidden4_conv" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN weight_optimizer { l2_decay: 0.0005 } }
edge { source: "hidden4_conv" dest: "hidden4_conv_nin1" edge_type: CONV_ONETOONE
       initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "hidden4_conv_nin1" dest: "hidden4_conv_nin2" edge_type: CONV_ONETOONE
       initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "hidden4_conv_nin2" dest: "hidden5_conv" edge_type: CONVOLUTIONAL kernel_size: 3
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN weight_optimizer { l2_decay: 0.0005 } }
edge { source: "hidden5_conv" dest: "hidden5_conv_nin1" edge_type: CONV_ONETOONE
       initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "hidden5_conv_nin1" dest: "hidden5_conv_nin2" edge_type: CONV_ONETOONE
       initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "hidden5_conv_nin2" dest: "hidden5_maxpool" edge_type: MAXPOOL kernel_size: 3 stride: 2 padding: 1 }
edge { source: "hidden5_maxpool" dest: "hidden6" edge_type: FC initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "hidden6" dest: "hidden7" edge_type: FC initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "hidden7" dest: "output" edge_type: FC initialization: DENSE_UNIFORM_SQRT_FAN_IN }
)pb"},

{"lenet", R"pb(
# examples/mnist-conv/net.pbtxt (net M), with constant momentum and without the norm rule and the FC l2_decay
# ("lenet+ref-optimizer" has the file's optimizer blocks exactly):
# 28x28x1 -conv4x4-> 25x25x48 -pool4/2-> 11x11x48 -conv4x4-> 8x8x128 -pool4/2-> 3x3x128 -fc-> 10
name: "mnist-conv"
seed: 42
default_weight_optimizer { epsilon: 0.01 final_momentum: 0.95 }
default_bias_optimizer { epsilon: 0.01 final_momentum: 0.95 }
layer { name: "input" num_channels: 1 image_size_y: 28 image_size_x: 28 }
layer { name: "hidden1_conv" num_channels: 48 activation: RECTIFIED_LINEAR }
layer { name: "hidden1_maxpool" num_channels: 48 }
layer { name: "hidden2_conv" num_channels: 128 activation: RECTIFIED_LINEAR }
layer { name: "hidden2_maxpool" num_channels: 128 }
layer { name: "output" num_channels: 10 activation: SOFTMAX }
edge { source: "input" dest: "hidden1_conv" edge_type: CONVOLUTIONAL kernel_size: 4
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN weight_optimizer { l2_decay: 0.0005 } }
edge { source: "hidden1_conv" dest: "hidden1_maxpool" edge_type: MAXPOOL kernel_size: 4 stride: 2 }
edge { source: "hidden1_maxpool" dest: "hidden2_conv" edge_type: CONVOLUTIONAL kernel_size: 4
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN weight_optimizer { l2_decay: 0.0005 } }
edge { source: "hidden2_conv" dest: "hidden2_maxpool" edge_type: MAXPOOL kernel_size: 4 stride: 2 }
edge { source: "hidden2_maxpool" dest: "output" edge_type: FC initialization: DENSE_UNIFORM_SQRT_FAN_IN }
)pb"},

{"c3d", R"pb(
# C3D-style video net (SURVEY.md §8(d) cfg4): 16 x 112 x 112 x 3 clips, 3x3x3 kernels, padding 1 in y and x and none in t
name: "c3d"
seed: 42
default_weight_optimizer { epsilon: 0.01 final_momentum: 0.9 }
default_bias_optimizer { epsilon: 0.01 final_momentum: 0.9 }
layer { name: "input" num_channels: 3 image_size_y: 112 image_size_x: 112 image_size_t: 16 }
layer { name: "conv1a" num_channels: 64 activation: RECTIFIED_LINEAR }
layer { name: "pool1" num_channels: 64 }
layer { name: "conv2a" num_channels: 128 activation: RECTIFIED_LINEAR }
layer { name: "pool2" num_channels: 128 }
layer { name: "conv3a" num_channels: 256 activation: RECTIFIED_LINEAR }
layer { name: "pool3" num_channels: 256 }
layer { name: "output" num_channels: 101 activation: SOFTMAX }
edge { source: "input" dest: "conv1a" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1 kernel_size_t: 3
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "conv1a" dest: "pool1" edge_type: MAXPOOL kernel_size: 2 stride: 2 }
edge { source: "pool1" dest: "conv2a" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1 kernel_size_t: 3
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "conv2a" dest: "pool2" edge_type: MAXPOOL kernel_size: 2 stride: 2 kernel_size_t: 2 stride_t: 2 }
edge { source: "pool2" dest: "conv3a" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1 kernel_size_t: 3
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN }
# global pooling before the classifier (a window of 0 covers the whole image)
edge { source: "conv3a" dest: "pool3" edge_type: MAXPOOL kernel_size: 0 kernel_size_t: 0 }
edge { source: "pool3" dest: "output" edge_type: FC initialization: DENSE_UNIFORM_SQRT_FAN_IN }
)pb"},

{"tiny", R"pb(
# small net touching every edge type, used by tests and the grad check
name: "tiny"
seed: 42
default_weight_optimizer { epsilon: 0.01 final_momentum: 0.9 }
default_bias_optimizer { epsilon: 0.01 final_momentum: 0.9 }
layer { name: "input" num_channels: 8 image_size_y: 12 image_size_x: 12 }
layer { name: "conv1" num_channels: 16 activation: RECTIFIED_LINEAR }
layer { name: "pool1" num_channels: 16 }
layer { name: "rnorm1" num_channels: 16 activation: RECTIFIED_LINEAR }
layer { name: "nin1" num_channels: 24 activation: RECTIFIED_LINEAR }
layer { name: "conv2" num_channels: 16 activation: RECTIFIED_LINEAR }
layer { name: "avgpool" num_channels: 16 }
layer { name: "output" num_channels: 10 activation: SOFTMAX }
edge { source: "input" dest: "conv1" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN
       grad_check: true grad_check_num_params: 8 grad_check_epsilon: [0.01, 0.003, 0.001] }
edge { source: "conv1" dest: "pool1" edge_type: MAXPOOL kernel_size: 3 stride: 2 padding: 1 }
edge { source: "pool1" dest: "rnorm1" edge_type: RESPONSE_NORM
       add_scale: 0.01 pow_scale: 0.75 frac_of_filters_response_norm: 0.5 }
edge { source: "rnorm1" dest: "nin1" edge_type: CONV_ONETOONE initialization: DENSE_UNIFORM_SQRT_FAN_IN
       grad_check: true grad_check_num_params: 8 grad_check_epsilon: [0.01, 0.003, 0.001] }
edge { source: "nin1" dest: "conv2" edge_type: CONVOLUTIONAL kernel_size: 3 stride: 2 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN
       grad_check: true grad_check_num_params: 8 grad_check_epsilon: [0.01, 0.003, 0.001] }
edge { source: "conv2" dest: "avgpool" edge_type: AVERAGE_POOL kernel_size: 2 stride: 2 }
edge { source: "avgpool" dest: "output" edge_type: FC initialization: DENSE_UNIFORM_SQRT_FAN_IN
       grad_check: true grad_check_num_params: 8 grad_check_epsilon: [0.01, 0.003, 0.001] }
)pb"},

{"gradcheck", R"pb(
# net for run_grad_check: one edge of every weighted type around pooling and response-norm, with SMOOTH activations
# (linear units, average pooling).  Finite differences are only meaningful away from kinks: with ReLU / max-pool a unit
# that sits within epsilon of its kink makes the central difference the AVERAGE of two one-sided slopes at every epsilon
# (observed: float64 finite differences show the same), so the reference's 1 % criterion (grad_check.cc:61) is a data
# lottery there.  The ReLU / max-pool backward ops are verified against float64 autograd instead
# (tests/test_gpu_net.py::test_backprop_matches_float64_autograd).
name: "gradcheck"
seed: 42
default_weight_optimizer { epsilon: 0.01 final_momentum: 0.9 }
default_bias_optimizer { epsilon: 0.01 final_momentum: 0.9 }
layer { name: "input" num_channels: 4 image_size_y: 8 image_size_x: 8 }
layer { name: "conv1" num_channels: 8 }
layer { name: "pool1" num_channels: 8 }
layer { name: "rnorm1" num_channels: 8 }
layer { name: "nin1" num_channels: 12 }
layer { name: "output" num_channels: 5 activation: SOFTMAX }
edge { source: "input" dest: "conv1" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN
       grad_check: true grad_check_num_params: 10 grad_check_epsilon: [0.01, 0.003, 0.001] }
edge { source: "conv1" dest: "pool1" edge_type: AVERAGE_POOL kernel_size: 3 stride: 2 padding: 1 }
edge { source: "pool1" dest: "rnorm1" edge_type: RESPONSE_NORM
       add_scale: 0.01 pow_scale: 0.75 frac_of_filters_response_norm: 0.5 }
edge { source: "rnorm1" dest: "nin1" edge_type: CONV_ONETOONE initialization: DENSE_UNIFORM_SQRT_FAN_IN
       grad_check: true grad_check_num_params: 10 grad_check_epsilon: [0.01, 0.003, 0.001] }
edge { source: "nin1" dest: "output" edge_type: FC initialization: DENSE_UNIFORM_SQRT_FAN_IN
       grad_check: true grad_check_num_params: 10 grad_check_epsilon: [0.01, 0.003, 0.001] }
)pb"},

{"logcheck", R"pb(
# the gradcheck net with logistic units in every hidden layer: the grad check of a smooth nonlinearity through the conv,
# average-pooling, response-norm, 1x1 and FC edges (sigma after the pooling and sigma' into its undo run as passes).
# init_wt 3: each sigma' scales the derivative by at most 1/4, and at the default scale the derivative reaching conv1
# through four logistic layers sits at the float32 noise floor of the finite differences
name: "logcheck"
seed: 42
default_weight_optimizer { epsilon: 0.01 final_momentum: 0.9 }
default_bias_optimizer { epsilon: 0.01 final_momentum: 0.9 }
layer { name: "input" num_channels: 4 image_size_y: 8 image_size_x: 8 }
layer { name: "conv1" num_channels: 8 activation: LOGISTIC }
layer { name: "pool1" num_channels: 8 activation: LOGISTIC }
layer { name: "rnorm1" num_channels: 8 activation: LOGISTIC }
layer { name: "nin1" num_channels: 12 activation: LOGISTIC }
layer { name: "output" num_channels: 5 activation: SOFTMAX }
edge { source: "input" dest: "conv1" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN init_wt: 3
       grad_check: true grad_check_num_params: 10 grad_check_epsilon: [0.01, 0.003, 0.001] }
edge { source: "conv1" dest: "pool1" edge_type: AVERAGE_POOL kernel_size: 3 stride: 2 padding: 1 }
edge { source: "pool1" dest: "rnorm1" edge_type: RESPONSE_NORM
       add_scale: 0.01 pow_scale: 0.75 frac_of_filters_response_norm: 0.5 }
edge { source: "rnorm1" dest: "nin1" edge_type: CONV_ONETOONE initialization: DENSE_UNIFORM_SQRT_FAN_IN init_wt: 3
       grad_check: true grad_check_num_params: 10 grad_check_epsilon: [0.01, 0.003, 0.001] }
edge { source: "nin1" dest: "output" edge_type: FC initialization: DENSE_UNIFORM_SQRT_FAN_IN init_wt: 3
       grad_check: true grad_check_num_params: 10 grad_check_epsilon: [0.01, 0.003, 0.001] }
)pb"},

{"lcnet", R"pb(
# conv + locally connected classifier (cuda-convnet's conv+local nets, scaled to 96 x 96 inputs): the two LOCAL edges
# carry a filter bank per output position (42 and 29 MB in bf16) and sit near the HBM / tensor-core balance point at
# batch 128.  init_wt = sqrt(modules): the reference scales a local edge's initial weights by 1/sqrt(K*modules/3)
# (weights_.GetCols(), edge_with_weight.cc:126); this undoes the modules factor, giving a conv-like initial scale.
name: "lcnet"
seed: 42
default_weight_optimizer { epsilon: 0.01 final_momentum: 0.9 }
default_bias_optimizer { epsilon: 0.01 final_momentum: 0.9 }
layer { name: "input" num_channels: 3 image_size_y: 96 image_size_x: 96 }
layer { name: "conv1" num_channels: 64 activation: RECTIFIED_LINEAR }
layer { name: "pool1" num_channels: 64 }
layer { name: "conv2" num_channels: 128 activation: RECTIFIED_LINEAR }
layer { name: "pool2" num_channels: 128 }
layer { name: "local3" num_channels: 128 activation: RECTIFIED_LINEAR }
layer { name: "local4" num_channels: 128 activation: RECTIFIED_LINEAR }
layer { name: "fc5" num_channels: 1024 activation: RECTIFIED_LINEAR dropprob: 0.5 }
layer { name: "output" num_channels: 1000 activation: SOFTMAX }
edge { source: "input" dest: "conv1" edge_type: CONVOLUTIONAL kernel_size: 5 stride: 2 padding: 2
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "conv1" dest: "pool1" edge_type: MAXPOOL kernel_size: 3 stride: 2 padding: 1 }
edge { source: "pool1" dest: "conv2" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "conv2" dest: "pool2" edge_type: MAXPOOL kernel_size: 3 stride: 2 padding: 1 }
edge { source: "pool2" dest: "local3" edge_type: LOCAL kernel_size: 3 padding: 1
       initialization: DENSE_UNIFORM_SQRT_FAN_IN init_wt: 12 }                # sqrt(12 x 12 modules)
edge { source: "local3" dest: "local4" edge_type: LOCAL kernel_size: 3
       initialization: DENSE_UNIFORM_SQRT_FAN_IN init_wt: 10 }                # sqrt(10 x 10 modules)
edge { source: "local4" dest: "fc5" edge_type: FC initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "fc5" dest: "output" edge_type: FC initialization: DENSE_UNIFORM_SQRT_FAN_IN }
)pb"},

{"localcheck", R"pb(
# run_grad_check net for the LOCAL edge, smooth like gradcheck (linear units, average pooling): one local edge with
# padding, one with stride 2 and no padding, then an FC.  init_wt = sqrt(modules) as in lcnet: with the reference's
# 1/sqrt(K*modules/3) scale the derivative reaching local1 is so small that its per-feature bias gradients sit at the
# float32 noise floor of the finite differences.  The check reads the FIRST parameters of a tensor, which for a local
# edge are the taps of module 0 (the top-left corner).  With padding 1, 5 of local1's 9 taps there only ever read
# padding, so local1 checks 72 parameters: all 8 outputs x 9 taps of input channel 0 of module 0, 32 of them live (the
# pairs whose analytic and numeric gradients are both exactly 0 do not enter the mean).
name: "localcheck"
seed: 42
default_weight_optimizer { epsilon: 0.01 final_momentum: 0.9 }
default_bias_optimizer { epsilon: 0.01 final_momentum: 0.9 }
layer { name: "input" num_channels: 4 image_size_y: 8 image_size_x: 8 }
layer { name: "local1" num_channels: 8 }
layer { name: "pool1" num_channels: 8 }
layer { name: "local2" num_channels: 8 }
layer { name: "output" num_channels: 5 activation: SOFTMAX }
edge { source: "input" dest: "local1" edge_type: LOCAL kernel_size: 3 padding: 1
       initialization: DENSE_UNIFORM_SQRT_FAN_IN init_wt: 8                   # sqrt(8 x 8 modules)
       grad_check: true grad_check_num_params: 72 grad_check_epsilon: [0.01, 0.003, 0.001] }
edge { source: "local1" dest: "pool1" edge_type: AVERAGE_POOL kernel_size: 2 }
edge { source: "pool1" dest: "local2" edge_type: LOCAL kernel_size: 3 stride: 2
       initialization: DENSE_UNIFORM_SQRT_FAN_IN init_wt: 3                   # sqrt(3 x 3 modules)
       grad_check: true grad_check_num_params: 10 grad_check_epsilon: [0.01, 0.003, 0.001] }
edge { source: "local2" dest: "output" edge_type: FC initialization: DENSE_UNIFORM_SQRT_FAN_IN
       grad_check: true grad_check_num_params: 10 grad_check_epsilon: [0.01, 0.003, 0.001] }
)pb"},

{"updown", R"pb(
# encoder-decoder at bench size: a YUV front end, two 2x down-samplings and two 2x up-samplings between 3x3 convs, and a
# LINEAR 3-channel output trained on a float target per pixel (SQUARED_ERROR).  128 x 128 inputs; the up-sampled
# 128-channel layer is the largest tensor (8 MB per image)
name: "updown"
seed: 42
default_weight_optimizer { epsilon: 0.01 final_momentum: 0.9 }
default_bias_optimizer { epsilon: 0.01 final_momentum: 0.9 }
layer { name: "input" num_channels: 3 image_size_y: 128 image_size_x: 128 }
layer { name: "yuv" num_channels: 3 }
layer { name: "conv1" num_channels: 64 activation: RECTIFIED_LINEAR }
layer { name: "down1" num_channels: 64 }
layer { name: "conv2" num_channels: 128 activation: RECTIFIED_LINEAR }
layer { name: "down2" num_channels: 128 }
layer { name: "conv3" num_channels: 256 activation: RECTIFIED_LINEAR }
layer { name: "up3" num_channels: 256 }
layer { name: "conv4" num_channels: 128 activation: RECTIFIED_LINEAR }
layer { name: "up4" num_channels: 128 }
layer { name: "conv5" num_channels: 64 activation: RECTIFIED_LINEAR }
layer { name: "output" num_channels: 3 loss_function: SQUARED_ERROR performance_metric: SQUARED_ERROR }
edge { source: "input" dest: "yuv" edge_type: RGBTOYUV }
edge { source: "yuv" dest: "conv1" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "conv1" dest: "down1" edge_type: DOWNSAMPLE sample_factor: 2 }
edge { source: "down1" dest: "conv2" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "conv2" dest: "down2" edge_type: DOWNSAMPLE sample_factor: 2 }
edge { source: "down2" dest: "conv3" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "conv3" dest: "up3" edge_type: UPSAMPLE sample_factor: 2 }
edge { source: "up3" dest: "conv4" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "conv4" dest: "up4" edge_type: UPSAMPLE sample_factor: 2 }
edge { source: "up4" dest: "conv5" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "conv5" dest: "output" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN }
)pb"},

{"updowncheck", R"pb(
# run_grad_check net for the sampling edges, smooth like gradcheck: down- and up-sampling by 3 and by 2, a conv under
# every sampling edge, a logistic layer written by an UPSAMPLE (sigma after the up-sampling, sigma' into its block sum
# as passes) and LINEAR units elsewhere, then an FC into a softmax as in gradcheck: the loss of a per-pixel regression
# output (SQUARED_ERROR on random targets) is so large that its float32 rounding drowns the finite differences
name: "updowncheck"
seed: 42
default_weight_optimizer { epsilon: 0.01 final_momentum: 0.9 }
default_bias_optimizer { epsilon: 0.01 final_momentum: 0.9 }
layer { name: "input" num_channels: 4 image_size_y: 6 image_size_x: 6 }
layer { name: "conv1" num_channels: 8 }
layer { name: "down1" num_channels: 8 }
layer { name: "conv2" num_channels: 8 }
layer { name: "up2" num_channels: 8 activation: LOGISTIC }
layer { name: "conv3" num_channels: 6 }
layer { name: "down3" num_channels: 6 }
layer { name: "conv4" num_channels: 6 }
layer { name: "up4" num_channels: 6 }
layer { name: "output" num_channels: 5 activation: SOFTMAX }
edge { source: "input" dest: "conv1" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN
       grad_check: true grad_check_num_params: 10 grad_check_epsilon: [0.01, 0.003, 0.001] }
edge { source: "conv1" dest: "down1" edge_type: DOWNSAMPLE sample_factor: 3 }
edge { source: "down1" dest: "conv2" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN
       grad_check: true grad_check_num_params: 10 grad_check_epsilon: [0.01, 0.003, 0.001] }
edge { source: "conv2" dest: "up2" edge_type: UPSAMPLE sample_factor: 3 }
edge { source: "up2" dest: "conv3" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN
       grad_check: true grad_check_num_params: 10 grad_check_epsilon: [0.01, 0.003, 0.001] }
edge { source: "conv3" dest: "down3" edge_type: DOWNSAMPLE sample_factor: 2 }
edge { source: "down3" dest: "conv4" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN
       grad_check: true grad_check_num_params: 10 grad_check_epsilon: [0.01, 0.003, 0.001] }
edge { source: "conv4" dest: "up4" edge_type: UPSAMPLE sample_factor: 2 }
edge { source: "up4" dest: "output" edge_type: FC initialization: DENSE_UNIFORM_SQRT_FAN_IN
       grad_check: true grad_check_num_params: 10 grad_check_epsilon: [0.01, 0.003, 0.001] }
)pb"},

{"tiednet", R"pb(
# weight sharing (tied_to) on the training path: one 64 -> 64 3x3 conv runs at three geometries — 32 x 32 with padding
# 1, 16 x 16 after a max-pool, and with stride 2 — so one filter tensor keeps three sets of dgrad banks; and two
# 256 -> 256 FC edges share weights with the LOWER edge naming the higher one, so the shared slice sits at the tied edge
# rather than at its owner.  Dropout on the owner's output layer, a softmax classifier
name: "tiednet"
seed: 42
default_weight_optimizer { epsilon: 0.01 final_momentum: 0.9 }
default_bias_optimizer { epsilon: 0.01 final_momentum: 0.9 }
layer { name: "input" num_channels: 3 image_size_y: 32 image_size_x: 32 }
layer { name: "conv1" num_channels: 64 activation: RECTIFIED_LINEAR }
layer { name: "conv2" num_channels: 64 activation: RECTIFIED_LINEAR }
layer { name: "pool2" num_channels: 64 }
layer { name: "conv3" num_channels: 64 activation: RECTIFIED_LINEAR }
layer { name: "conv4" num_channels: 64 activation: RECTIFIED_LINEAR }
layer { name: "fc5" num_channels: 256 activation: RECTIFIED_LINEAR }
layer { name: "fc6" num_channels: 256 activation: RECTIFIED_LINEAR }
layer { name: "fc7" num_channels: 256 activation: RECTIFIED_LINEAR dropprob: 0.5 }
layer { name: "output" num_channels: 10 activation: SOFTMAX }
edge { source: "input" dest: "conv1" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "conv1" dest: "conv2" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "conv2" dest: "pool2" edge_type: MAXPOOL kernel_size: 2 stride: 2 }
# pool2:conv3 and conv3:conv4 run conv1:conv2's filters
edge { source: "pool2" dest: "conv3" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1 shared_bias: true
       tied_to: "conv1:conv2" }
edge { source: "conv3" dest: "conv4" edge_type: CONVOLUTIONAL kernel_size: 3 stride: 2 padding: 1 shared_bias: true
       tied_to: "conv1:conv2" }
edge { source: "conv4" dest: "fc5" edge_type: FC initialization: DENSE_UNIFORM_SQRT_FAN_IN }
# fc5:fc6 runs with fc6:fc7's weights
edge { source: "fc5" dest: "fc6" edge_type: FC tied_to: "fc6:fc7" }
edge { source: "fc6" dest: "fc7" edge_type: FC initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "fc7" dest: "output" edge_type: FC initialization: DENSE_UNIFORM_SQRT_FAN_IN }
)pb"},

{"tiedcheck", R"pb(
# run_grad_check net for ties, smooth like gradcheck (linear units, average pooling): a conv used at padding 1 and
# padding 0, a CONV_ONETOONE, a LOCAL and an FC tie (the FC one named by the lower edge).  grad_check is set on every
# edge with parameters of its own; an owner's check perturbs the shared tensors, so it checks the summed gradient
name: "tiedcheck"
seed: 42
default_weight_optimizer { epsilon: 0.01 final_momentum: 0.9 }
default_bias_optimizer { epsilon: 0.01 final_momentum: 0.9 }
layer { name: "input" num_channels: 4 image_size_y: 8 image_size_x: 8 }
layer { name: "c0" num_channels: 8 }
layer { name: "c1" num_channels: 8 }
layer { name: "c2" num_channels: 8 }
layer { name: "pool" num_channels: 8 }
layer { name: "o1" num_channels: 8 }
layer { name: "o2" num_channels: 8 }
layer { name: "l1" num_channels: 8 }
layer { name: "l2" num_channels: 8 }
layer { name: "f1" num_channels: 16 }
layer { name: "f2" num_channels: 16 }
layer { name: "f3" num_channels: 16 }
layer { name: "output" num_channels: 5 activation: SOFTMAX }
edge { source: "input" dest: "c0" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN
       grad_check: true grad_check_num_params: 10 grad_check_epsilon: [0.01, 0.003, 0.001] }
edge { source: "c0" dest: "c1" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN
       grad_check: true grad_check_num_params: 10 grad_check_epsilon: [0.01, 0.003, 0.001] }
# 8 x 8 at padding 1, then at padding 0
edge { source: "c1" dest: "c2" edge_type: CONVOLUTIONAL kernel_size: 3 shared_bias: true tied_to: "c0:c1" }
edge { source: "c2" dest: "pool" edge_type: AVERAGE_POOL kernel_size: 2 stride: 2 }
edge { source: "pool" dest: "o1" edge_type: CONV_ONETOONE initialization: DENSE_UNIFORM_SQRT_FAN_IN
       grad_check: true grad_check_num_params: 10 grad_check_epsilon: [0.01, 0.003, 0.001] }
edge { source: "o1" dest: "o2" edge_type: CONV_ONETOONE tied_to: "pool:o1" }
edge { source: "o2" dest: "l1" edge_type: LOCAL kernel_size: 3 padding: 1
       initialization: DENSE_UNIFORM_SQRT_FAN_IN init_wt: 3                   # sqrt(3 x 3 modules), as in localcheck
       # module 0's taps of input channel 0 (see localcheck)
       grad_check: true grad_check_num_params: 72 grad_check_epsilon: [0.01, 0.003, 0.001] }
edge { source: "l1" dest: "l2" edge_type: LOCAL kernel_size: 3 padding: 1 tied_to: "o2:l1" }
edge { source: "l2" dest: "f1" edge_type: FC initialization: DENSE_UNIFORM_SQRT_FAN_IN
       grad_check: true grad_check_num_params: 10 grad_check_epsilon: [0.01, 0.003, 0.001] }
edge { source: "f1" dest: "f2" edge_type: FC tied_to: "f2:f3" }
edge { source: "f2" dest: "f3" edge_type: FC initialization: DENSE_UNIFORM_SQRT_FAN_IN
       grad_check: true grad_check_num_params: 10 grad_check_epsilon: [0.01, 0.003, 0.001] }
edge { source: "f3" dest: "output" edge_type: FC initialization: DENSE_UNIFORM_SQRT_FAN_IN
       grad_check: true grad_check_num_params: 10 grad_check_epsilon: [0.01, 0.003, 0.001] }
)pb"},
};
}  // namespace

// "<model>+ref-optimizer": the optimizer blocks of the model's pbtxt exactly (the alexnet and lenet texts keep the constant
// momentum and leave out the norm rules and the FC l2_decay)
static void UseReferenceOptimizers(const std::string& base, ModelConfig& m) {
  OptimizerConfig o;                                        // every weight and bias optimizer of both files
  o.epsilon = 0.01f;
  if (base == "alexnet") {        // examples/imagenet/CLS_net_20140801232522.pbtxt:148-505
    o.initial_momentum = 0.5f; o.final_momentum = 0.9f; o.momentum_transition_timescale = 2000;
    for (EdgeConfig& e : m.edge) {
      const float l2 = e.weight_optimizer.l2_decay;        // conv3-5: 0.0005, as the alexnet text has it
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
  for (const BuiltIn& b : kBuiltIns)
    if (name == b.name) return ReadModelText(b.text, name, true);
  throw std::invalid_argument("unknown model '" + name + "'");
}

}  // namespace cnbhost
