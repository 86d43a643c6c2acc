"""ctypes door onto the native host code (convnet_b200/host: Matrix / Edge / ConvNet / GradChecker /
DataParallelSync -> lib/libconvnet_b200_host.so).  Python only launches; sequencing, memory and the
NCCL gradient sync live in C++ like the reference's src/convnet.cc."""
import ctypes as ct
import os

from . import lib as _lib


class OptimizerConfig(ct.Structure):
    """host/edge.h OptimizerConfig: the SGD, Adagrad and RMSProp fields of the reference's proto Optimizer
    (proto/convnet_config.proto:64-113), same names, same defaults, same order as the C struct."""
    _fields_ = [("epsilon", ct.c_float), ("epsilon_decay", ct.c_int), ("epsilon_decay_timescale", ct.c_int),
                ("minimum_epsilon", ct.c_float), ("decay_factor", ct.c_float), ("initial_momentum", ct.c_float),
                ("final_momentum", ct.c_float), ("momentum_transition_timescale", ct.c_int), ("l2_decay", ct.c_float),
                ("gradient_clip", ct.c_float), ("start_optimization_after", ct.c_int), ("weight_norm_limit", ct.c_float),
                ("weight_norm_constraint", ct.c_float), ("optimizer_type", ct.c_int), ("adagrad_delta", ct.c_float),
                ("rms_prop_factor", ct.c_float)]
    DEFAULTS = {"decay_factor": 1.0, "gradient_clip": -1.0, "adagrad_delta": 1.0}
    DECAY = {"NONE": 0, "INVERSE_T": 1, "EXPONENTIAL": 2, "LINEAR": 3, "EXPONENTIAL_STEP": 4}
    TYPE = {"STOCHASTIC_GRADIENT_DESCENT": 0, "LBFGS": 1, "ADAGRAD_SGD": 2, "RMSPROP_SGD": 3}

    @classmethod
    def from_dict(cls, d):
        """an optimizer block as a dict of proto field names (epsilon_decay and optimizer_type also by name); unset fields
        take the proto's defaults.  Fields outside these paths (Nesterov, LBFGS's memory, shared prior) are not supported,
        and the host refuses optimizer_type LBFGS."""
        c = cls(**cls.DEFAULTS)
        names = [f[0] for f in cls._fields_]
        for k, v in d.items():
            if k not in names:
                raise KeyError("unsupported optimizer field %r (known: %s)" % (k, ", ".join(names)))
            if k == "epsilon_decay" and isinstance(v, str):
                v = cls.DECAY[v]
            if k == "optimizer_type" and isinstance(v, str):
                v = cls.TYPE[v]
            setattr(c, k, v)
        return c

    def to_dict(self):
        return {f[0]: getattr(self, f[0]) for f in self._fields_}


class DatasetOrder(ct.Structure):
    """host/data.h DatasetOrder: the batch-order fields of the reference's DatasetConfig (proto/convnet_config.proto:371-382),
    same names, same defaults."""
    _fields_ = [("batch_size", ct.c_int), ("chunk_size", ct.c_int), ("max_reuse_count", ct.c_int),
                ("pipeline_loads", ct.c_int), ("randomize_cpu", ct.c_int), ("randomize_gpu", ct.c_int),
                ("random_access_chunk_size", ct.c_int), ("multiplicity", ct.c_int)]
    DEFAULTS = {"batch_size": 1, "random_access_chunk_size": 1, "multiplicity": 1}

    @classmethod
    def from_dict(cls, d):
        c = cls(**cls.DEFAULTS)
        names = [f[0] for f in cls._fields_]
        for k, v in d.items():
            if k not in names:
                raise KeyError("unsupported dataset field %r (known: %s)" % (k, ", ".join(names)))
            setattr(c, k, int(v))
        return c

    def to_dict(self):
        return {f[0]: getattr(self, f[0]) for f in self._fields_}


HOST_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libconvnet_b200_host.so")
_host = None


def load_host():
    global _host
    if _host is None:
        _lib.load()                    # the kernel library first (RTLD_GLOBAL not needed: host lib has an rpath)
        if not os.path.exists(HOST_LIB_PATH):
            raise RuntimeError("convnet_b200: %s is missing - run __graft_entry__.build()" % HOST_LIB_PATH)
        H = ct.CDLL(HOST_LIB_PATH)
        vp, i, ll, d, f = ct.c_void_p, ct.c_int, ct.c_longlong, ct.c_double, ct.c_float
        sig = {
            "cnb_model_open": ([ct.c_char_p, i], vp),
            "cnb_net_create": ([ct.c_char_p, i, ct.c_uint, i], vp), "cnb_net_destroy": ([vp], None),
            "cnb_net_num_params": ([vp], ll), "cnb_net_num_edges": ([vp], i), "cnb_net_edge_name": ([vp, i], ct.c_char_p),
            "cnb_net_edge_flops": ([vp, i], d), "cnb_net_edge_offset": ([vp, i], ll), "cnb_net_edge_size": ([vp, i], ll),
            "cnb_net_edge_slice": ([vp, i], ll), "cnb_net_edge_fusion": ([vp, i, ct.POINTER(i), ct.POINTER(i)], i),
            "cnb_net_layer_passes": ([vp, i], i),
            "cnb_net_flops_fprop": ([vp], d), "cnb_net_flops_train": ([vp], d),
            "cnb_net_input": ([vp], vp), "cnb_net_input_floats": ([vp], ll), "cnb_net_labels": ([vp], vp),
            "cnb_net_output": ([vp], vp), "cnb_net_num_classes": ([vp], i), "cnb_net_params": ([vp], vp),
            "cnb_net_grads": ([vp], vp), "cnb_net_layer_state": ([vp, i], vp), "cnb_net_layer_floats": ([vp, i], ll),
            "cnb_net_num_layers": ([vp], i), "cnb_net_device_loss": ([vp], vp),
            "cnb_net_fprop": ([vp, i], i), "cnb_net_bprop": ([vp], i), "cnb_net_update": ([vp], i),
            "cnb_net_loss": ([vp, ct.POINTER(f)], i), "cnb_net_train_step": ([vp, ct.POINTER(f)], i),
            "cnb_net_trace_step": ([vp, ct.POINTER(f), i], i),
            "cnb_data_create": ([i, i, i, i, i, i, i, i, ct.c_ulonglong], vp), "cnb_data_destroy": ([vp], None),
            "cnb_data_upload": ([vp, vp, i, i], i), "cnb_data_get_batch": ([vp, vp, i, i], i),
            "cnb_data_last_noise": ([vp, ct.POINTER(f), i], i),
            "cnb_data_view_offset": ([i, i, i, ct.POINTER(i), ct.POINTER(i)], None),
            "cnb_dp_unique_id": ([ct.c_char_p], i), "cnb_net_dp_init": ([vp, i, i, ct.c_char_p, ll], i),
            "cnb_plan_buckets": ([i, ct.POINTER(ll), ct.POINTER(ll), ll, i, ct.POINTER(ll), ct.POINTER(ll), ct.POINTER(i)], i),
            "cnb_net_reduce_learning_rate": ([vp, f], None),
            "cnb_net_set_optimizer": ([vp, ct.c_char_p, ct.POINTER(OptimizerConfig)], i),
            "cnb_net_adaptive_state": ([vp], vp),
            "cnb_net_get_optimizer_state": ([vp, ct.c_char_p, ct.POINTER(ll), ct.POINTER(f), ct.POINTER(f),
                                             ct.POINTER(OptimizerConfig)], ll),
            "cnb_optimizer_schedule": ([ct.POINTER(OptimizerConfig), ll, ct.POINTER(f), ct.POINTER(f)], i),
            "cnb_net_grad_check": ([vp, ct.c_uint, i, ct.c_char_p, ct.POINTER(f), ct.POINTER(f), ct.POINTER(f)], i),
            "cnb_net_layer_name": ([vp, i], ct.c_char_p), "cnb_net_layer_channels": ([vp, i], i),
            "cnb_net_layer_bn": ([vp, i, ct.POINTER(f), ct.POINTER(f)], None),
            "cnb_net_bn_offset": ([vp, i], ll), "cnb_net_bn_stat": ([vp, i, i], vp),
            "cnb_bn_optimizer_check": ([ct.POINTER(OptimizerConfig)], i),
            "cnb_net_targets": ([vp], vp), "cnb_net_targets_floats": ([vp], ll), "cnb_net_metric": ([vp, ct.POINTER(f)], i),
            "cnb_net_output_layer": ([vp, ct.POINTER(i), ct.POINTER(i), ct.POINTER(i), ct.POINTER(f), ct.POINTER(i)], None),
            "cnb_net_model_text": ([vp, ct.c_char_p, ll], ll),
            "cnb_net_initial_weights": ([vp, i, ct.c_uint, ct.POINTER(f), ll], ll),
            "cnb_net_history": ([vp], vp), "cnb_last_error": ([], ct.c_char_p), "cnb_last_status": ([], i),
            "cnb_net_save": ([vp, ct.c_char_p], i),
            "cnb_net_load": ([vp, ct.c_char_p], i), "cnb_net_iteration": ([vp], ll),
            "cnb_net_polyak_insert": ([vp], i), "cnb_net_load_polyak_weights": ([vp], i),
            "cnb_net_load_current_weights": ([vp], i), "cnb_net_polyak_count": ([vp], i),
            "cnb_net_polyak": ([vp, ct.POINTER(i), ct.POINTER(i), ct.POINTER(i), ct.POINTER(i)], i),
            "cnb_net_polyak_due": ([vp, ll], i),
            "cnb_net_edge_tied_to": ([vp, i], ct.c_char_p),
            "cnb_net_layer_deriv": ([vp, i], vp),
            "cnb_net_dropout_seed": ([vp, i], ct.c_ulonglong),
            "cnb_net_frozen_edges": ([vp, ct.POINTER(ll)], i),
            "cnb_schedule_create": ([ct.POINTER(DatasetOrder), i, ct.c_ulonglong], vp), "cnb_schedule_destroy": ([vp], None),
            "cnb_schedule_chunk_size": ([vp], i),
            "cnb_schedule_next": ([vp, ct.POINTER(i), ct.POINTER(i), ct.POINTER(i), ct.POINTER(i)], i),
            "cnb_schedule_seek": ([vp, i], i),
            "cnb_handler_create": ([ct.POINTER(DatasetOrder), i, i, i, i, i, i, i, i, vp, vp, vp, i, ct.c_ulonglong], vp),
            "cnb_handler_destroy": ([vp], None), "cnb_handler_get_batch": ([vp, vp], i), "cnb_handler_seek": ([vp, i], i),
            "cnb_handler_last": ([vp, ct.POINTER(i), ct.POINTER(i), ct.POINTER(i), ct.POINTER(f)], i),
            "cnb_net_dataset": ([vp, i, ct.POINTER(DatasetOrder), ct.POINTER(i), ct.POINTER(i), ct.POINTER(i),
                                 ct.POINTER(i)], i),
            "cnb_net_schedule": ([vp, ct.POINTER(i), ct.POINTER(f), ct.POINTER(ct.c_char_p), ct.POINTER(ct.c_char_p)], None),
            "cnb_reduce_lr_due": ([ct.POINTER(f), i, i, f, i], i),
            "cnb_net_train_dry_run": ([vp, ll, i, i, ct.POINTER(f), i, ll, ct.POINTER(ll), ct.POINTER(i)], ll),
            "cnb_net_validate": ([vp, vp, ct.POINTER(f)], i),
            "cnb_net_train": ([vp, vp, vp, ct.c_char_p, ct.c_char_p], i),
            "cnb_net_train_event": ([vp, i, ct.POINTER(ll), ct.POINTER(i), ct.POINTER(f), ct.POINTER(i), ct.POINTER(i)], i),
            "cnb_net_lr_reduce_counter": ([vp], i),
        }
        for name, (args, res) in sig.items():
            fn = getattr(H, name)
            fn.argtypes, fn.restype = args, res
        _host = H
    return _host


def _check(rc):
    """the result of a host call that can fail: a status, count or handle passes through; a failure raises, with the host's
    reason (cnb_last_error) as its message: ValueError for a refusal (-1), RuntimeError for a failed CUDA or NCCL call
    (-2), and for a NULL handle whichever of the two cnb_last_status() names.  After a RuntimeError in the middle of a
    step the net's state is undefined, and close() is the only safe call left on it."""
    H = load_host()
    if rc is None:
        rc = H.cnb_last_status()
    if rc >= 0:
        return rc
    raise (RuntimeError if rc == -2 else ValueError)(H.cnb_last_error().decode())


class Model:
    """A model's chain built on the host only, for describing it: its edges, layers, parameter layout, fusion plan and
    FLOPs at `batch`, without device memory.  `model` is a built-in name or a model file, with suffixes, as for Net.  A
    model that cannot be read or run raises ValueError with the reason (for a file: its line and field)."""

    def __init__(self, model, batch=1):
        self._open(model, batch, load_host().cnb_model_open(model.encode(), batch))

    def _open(self, model, batch, h):
        self.H, self.h, self.model, self.batch_size = load_host(), None, model, batch
        self.h = _check(h)

    def close(self):
        if self.h:
            self.H.cnb_net_destroy(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    num_params = property(lambda s: s.H.cnb_net_num_params(s.h))
    flops_fprop = property(lambda s: s.H.cnb_net_flops_fprop(s.h))
    flops_train = property(lambda s: s.H.cnb_net_flops_train(s.h))

    def _frozen(self):
        off = ct.c_longlong(0)
        return self.H.cnb_net_frozen_edges(self.h, ct.byref(off)), off.value

    trained_offset = property(lambda s: s._frozen()[1],
                              doc="floats at the start of params_tensor() held by frozen edges and layers, which nothing trains")

    def edges(self):
        return [(self.H.cnb_net_edge_name(self.h, i).decode(), self.H.cnb_net_edge_flops(self.h, i),
                 self.H.cnb_net_edge_offset(self.h, i), self.H.cnb_net_edge_size(self.h, i))
                for i in range(self.H.cnb_net_num_edges(self.h))]

    def _edge_name(self, edge):
        """the name of `edge` (index or name); "" for an index out of range, whose tensors the host then does not find.
        ValueError for a tied edge, whose optimizers are its owner's"""
        names = [e[0] for e in self.edges()]
        if isinstance(edge, str):
            if edge not in names:
                raise KeyError("no edge %r (edges: %s)" % (edge, ", ".join(names)))
            i = names.index(edge)
        elif 0 <= int(edge) < len(names):
            i = int(edge)
        else:
            return ""
        owner = self.H.cnb_net_edge_tied_to(self.h, i).decode()
        if owner:
            raise ValueError("edge %r is tied to %r: its weights, bias and optimizers are those of %r" % (edge, owner, owner))
        return names[i]

    def bn_layers(self):
        """[(layer index, name, channels, offset of [gamma | beta] in params_tensor())] of the batch-normalised layers"""
        out = []
        for i in range(self.H.cnb_net_num_layers(self.h)):
            off = self.H.cnb_net_bn_offset(self.h, i)
            if off >= 0:
                out.append((i, self.H.cnb_net_layer_name(self.h, i).decode(), self.H.cnb_net_layer_channels(self.h, i), off))
        return out

    def _optimizer_config(self, tensor):
        """the optimizer settings (a dict) of trained tensor `tensor`; None when there is none or it holds no floats"""
        c, step, v = OptimizerConfig(), ct.c_longlong(0), ct.c_float(0)
        n = self.H.cnb_net_get_optimizer_state(self.h, tensor.encode(), ct.byref(step), ct.byref(v), ct.byref(v), ct.byref(c))
        return c.to_dict() if n > 0 else None


class Net(Model):
    """A chain ConvNet built natively, from a built-in name ("alexnet" | "lenet" | "c3d" | "tiny" | "lcnet" | "gradcheck" |
    "logcheck" | "localcheck" | "tiednet" | "tiedcheck" | "updown" | "updowncheck") or from a model file: any name ending in ".pbtxt" is the path of a config::Model text proto
    as the reference writes them (examples/*/net.pbtxt), read with the proto's defaults (model_text() prints any model
    as one).  The file's seed is printed but not used: `seed` decides, for files as for built-ins.  Suffixes compose with
    both ("net.pbtxt+rmsprop"):
    "+ref-optimizer" (alexnet and lenet): train with the optimizer blocks of the reference's pbtxt files.
    "+bn": batch normalisation on every hidden layer written by a conv, 1x1 or FC edge; gamma / beta train with that
    edge's weight / bias optimizer, without L2 decay and norm rules ("tiny+bn", "lenet+bn", "alexnet+bn", "gradcheck+bn",
    "alexnet+ref-optimizer+bn"; not "c3d+bn": 3-D layers are not supported).
    "+adagrad" / "+rmsprop": every weight, bias, gamma and beta optimizer on ADAGRAD_SGD (adagrad_delta 1, epsilon x 0.1) /
    RMSPROP_SGD (rms_prop_factor 0.9, epsilon x 0.01); they compose with the others ("alexnet+ref-optimizer+rmsprop",
    "tiny+bn+adagrad").
    "+gradcheck": run_grad_check's edge flags on the trained edges (e.g. "tiny+bn+gradcheck").
    "+finetune": block_backprop on every edge below the lowest FC edge: the trunk keeps its weights and the FC classifier
    trains ("alexnet+finetune", "alexnet+ref-optimizer+finetune", "tiny+bn+finetune"; refused without an FC edge).
    "+logistic": every hidden RECTIFIED_LINEAR layer becomes LOGISTIC (same parameters; "alexnet+logistic", "tiny+bn+logistic").
    One output suffix at most: "+squared-error" (LINEAR output, SQUARED_ERROR), "+binary-ce" (LOGISTIC output,
    CROSS_ENTROPY_BINARY, metric CLASSIFICATION_BINARY), "+soft-targets" (SOFTMAX_DIST, CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED);
    such outputs train on targets_tensor() instead of labels_tensor().  "logcheck": the gradcheck net with logistic units.
    A model that cannot be read or run raises ValueError with the reason (for a file: its line and field), as Model does;
    a device that cannot hold it (or no device) RuntimeError with the CUDA error.

    Tied edges (the reference's Edge.tied_to, see model_ties()) run with their owner's weights and bias and add their
    gradients to the owner's: they own no parameters (edges() reports size 0 and the owner's offset), and the owner's
    optimizers, tensors ("<owner>:weight", "<owner>:bias") and checkpoint records serve the whole group.

    Checkpoints (the reference's ConvNet::Save / Load): save(path) writes the parameters, the optimizers' histories, step
    counts and adaptive state, the batch-norm running statistics, the iteration, the seed and the optimizer settings in
    force; load(path) into a net of the same model resumes training bit for bit, whatever seed the Net was built with.
    A model file with polyak_after and polyak_queue_size averages the parameters over a queue on the device, as the
    reference's Save() does beside each checkpoint:
        if polyak_due(model, net.iteration): net.polyak_insert()          # after each train_step
        net.save(p)
        net.load_polyak_weights(); net.save(p + "polyak"); net.load_current_weights()

    Fine-tuning (the reference's Edge.block_backprop, see model_frozen()): a blocked edge and every edge below it are frozen.
    They run their forward pass only (dropout and batch statistics as in training, running statistics updated); they get
    no gradient and no optimizer step, and the hidden layers they write no derivative (layer_deriv() is None).  Their
    parameters stay in the buffers, as the prefix [0, trained_offset) of params_tensor(), which no update, all-reduce or
    Polyak average touches; checkpoints save them.  A model file's subnet blocks (the reference's Model.subnet) pull
    another model file in, optionally PRETRAINED from a checkpoint and blocked: the usual way to train a new head on a
    trained trunk."""

    def __init__(self, model, batch_size, seed=42, grad_checker=False):
        self._open(model, batch_size, load_host().cnb_net_create(model.encode(), batch_size, seed, int(grad_checker)))

    num_classes = property(lambda s: s.H.cnb_net_num_classes(s.h))
    input_floats = property(lambda s: s.H.cnb_net_input_floats(s.h))

    # --- device buffers as torch tensors (zero-copy views)
    def _view(self, ptr, n, dtype):
        import torch
        # torch has no from_address; go through the CUDA array interface

        class _W:
            pass
        w = _W()
        w.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4" if dtype == "f" else "<i4",
                                      "data": (ptr, False), "version": 2}
        return torch.as_tensor(w, device="cuda")

    def input_tensor(self):
        return self._view(self.H.cnb_net_input(self.h), self.input_floats, "f")

    def labels_tensor(self):
        return self._view(self.H.cnb_net_labels(self.h), self.batch_size, "i")

    def output_tensor(self):
        return self._view(self.H.cnb_net_output(self.h), self.batch_size * self.num_classes, "f")

    def targets_tensor(self):
        """the output layer's float targets, column-major (element n + batch * j is feature j of image n), written by the
        caller; None for an output layer trained on labels (labels_tensor())"""
        n = self.H.cnb_net_targets_floats(self.h)
        return self._view(self.H.cnb_net_targets(self.h), n, "f") if n else None

    def params_tensor(self):
        return self._view(self.H.cnb_net_params(self.h), self.num_params, "f")

    def grads_tensor(self):
        return self._view(self.H.cnb_net_grads(self.h), self.num_params, "f")

    def history_tensor(self):
        """the optimizers' momentum history (gradient_history), laid out like params_tensor()"""
        return self._view(self.H.cnb_net_history(self.h), self.num_params, "f")

    def adaptive_state_tensor(self):
        """the per-parameter state of the ADAGRAD_SGD / RMSPROP_SGD optimizers, laid out like params_tensor(); None while
        no optimizer of the net is adaptive (the buffer is allocated by the first one)"""
        ptr = self.H.cnb_net_adaptive_state(self.h)
        return self._view(ptr, self.num_params, "f") if ptr else None

    def layer_state(self, i):
        return self._view(self.H.cnb_net_layer_state(self.h, i), self.H.cnb_net_layer_floats(self.h, i), "f")

    def layer_deriv(self, i):
        """the derivative of the loss with respect to layer i's state after bprop, laid out like layer_state(i); None for
        a layer that receives no derivative: the input layer, the layer an RGBTOYUV edge writes and every hidden layer a
        frozen edge writes (block_backprop)"""
        ptr = self.H.cnb_net_layer_deriv(self.h, i)
        return self._view(ptr, self.H.cnb_net_layer_floats(self.h, i), "f") if ptr else None

    def dropout_seed(self, i):
        """the seed of the keep mask the next training step draws for layer i (element k of the state is kept when
        float32(hash(seed + k)) * 2^-32 >= dropprob, csrc/common.cuh); 0 for a layer without dropout"""
        return self.H.cnb_net_dropout_seed(self.h, i)

    # --- compute
    def fprop(self, train=False):
        _check(self.H.cnb_net_fprop(self.h, int(train)))

    def bprop(self):
        _check(self.H.cnb_net_bprop(self.h))

    def update(self):
        _check(self.H.cnb_net_update(self.h))

    def loss(self):
        """loss_function_weight times the batch's loss under the output layer's loss function (after fprop)"""
        v = ct.c_float(0)
        _check(self.H.cnb_net_loss(self.h, ct.byref(v)))
        return v.value

    def metric(self):
        """the output layer's performance metric summed over the batch (after fprop): correct images for
        CLASSIFICATION_MULTINOMIAL, the per-image share of correct features for CLASSIFICATION_BINARY, or a loss"""
        v = ct.c_float(0)
        _check(self.H.cnb_net_metric(self.h, ct.byref(v)))
        return v.value

    # --- optimizer (SGDOptimizer, src/optimizer.cc): one per trained tensor, named "<edge>:weight", "<edge>:bias",
    # "<layer>:gamma", "<layer>:beta" as in checkpoints
    def _set_optimizer(self, tensor, d):
        _check(self.H.cnb_net_set_optimizer(self.h, tensor.encode(), ct.byref(OptimizerConfig.from_dict(d))))

    def _optimizer_state(self, tensor):
        step, eps, mom = ct.c_longlong(0), ct.c_float(0), ct.c_float(0)
        n = self.H.cnb_net_get_optimizer_state(self.h, tensor.encode(), ct.byref(step), ct.byref(eps), ct.byref(mom), None)
        return {"step": step.value, "epsilon": eps.value, "momentum": mom.value} if n >= 0 else None

    def set_optimizer(self, edge, weights=None, bias=None):
        """replace the settings of the weight and / or bias optimizer of `edge` (index or name) with the optimizer block
        `weights` / `bias` (dicts of proto field names, unset fields at the proto's defaults).  Step counts and momentum
        histories are kept.  ValueError for a frozen edge (block_backprop), which nothing trains."""
        name = self._edge_name(edge)
        if name and [e[0] for e in self.edges()].index(name) < self._frozen()[0]:
            raise ValueError("edge %r is blocked (block_backprop): it is frozen, and no optimizer trains it" % (name,))
        for kind, d in ((":weight", weights), (":bias", bias)):
            if d is not None:
                self._set_optimizer(name + kind, d)

    def optimizer_state(self, edge):
        """{"weights": {...}, "bias": {...}}: updates counted so far ("step") and the epsilon / momentum of the next one"""
        name = self._edge_name(edge)
        out = {"weights": self._optimizer_state(name + ":weight"), "bias": self._optimizer_state(name + ":bias")}
        if out["weights"] is None:
            raise ValueError("edge %r has no parameters" % (edge,))
        return out

    def reduce_learning_rate(self, factor):
        """multiply the base epsilon of every optimizer by `factor` (ConvNet::ReduceLearningRate)"""
        self.H.cnb_net_reduce_learning_rate(self.h, factor)

    # --- batch normalisation (Layer::ApplyBatchNormalization, src/layer.cc:452-510)
    def _bn_layer(self, layer):
        for entry in self.bn_layers():
            if layer in (entry[0], entry[1]):
                return entry
        raise KeyError("layer %r is not batch-normalised (those that are: %s)" % (layer, [e[1] for e in self.bn_layers()]))

    def bn_state(self, layer):
        """the tensors of a batch-normalised layer (index or name), as zero-copy views: gamma / beta (into params_tensor()),
        grad_gamma / grad_beta (into grads_tensor(): mean over the layer's N * pixels values, the reference's scaling),
        running_mean / running_sigma, and batch_mean / batch_sigma of the last training-mode fprop"""
        i, _, c, off = self._bn_layer(layer)
        p, g = self.params_tensor(), self.grads_tensor()
        stat = [self._view(self.H.cnb_net_bn_stat(self.h, i, k), c, "f") for k in range(4)]
        return {"gamma": p[off:off + c], "beta": p[off + c:off + 2 * c], "grad_gamma": g[off:off + c],
                "grad_beta": g[off + c:off + 2 * c], "running_mean": stat[0], "running_sigma": stat[1],
                "batch_mean": stat[2], "batch_sigma": stat[3]}

    def set_bn_optimizer(self, layer, gamma=None, beta=None):
        """replace the settings of the gamma and / or beta optimizer of a batch-normalised layer (optimizer blocks as for
        set_optimizer; norm rules are refused).  Step counts and momentum histories are kept."""
        name = self._bn_layer(layer)[1]
        for key, d in (("gamma", gamma), ("beta", beta)):
            if d is not None:
                self._set_optimizer(name + ":" + key, d)

    def bn_optimizer_state(self, layer):
        """{"gamma": {...}, "beta": {...}}: updates counted so far ("step") and the epsilon / momentum of the next one"""
        name = self._bn_layer(layer)[1]
        return {key: self._optimizer_state(name + ":" + key) for key in ("gamma", "beta")}

    # --- checkpoints and Polyak averaging (ConvNet::Save / Load / InsertPolyak / LoadPolyakWeights / LoadCurrentWeights)
    def save(self, path):
        """write the net's state to `path` (through path + "temp", fsynced and renamed), after every pending step"""
        _check(self.H.cnb_net_save(self.h, os.fsencode(path)))

    def load(self, path):
        """restore the state `save` wrote from a net of the same model: ValueError (naming the record) if the file does not
        fit this net, which is then unchanged"""
        _check(self.H.cnb_net_load(self.h, os.fsencode(path)))

    iteration = property(lambda s: s.H.cnb_net_iteration(s.h), doc="train_step calls so far (restored by load)")
    polyak_count = property(lambda s: s.H.cnb_net_polyak_count(s.h), doc="filled slots of the Polyak queue")

    def polyak_insert(self):
        """copy the parameters into the next slot of the Polyak queue (a ring of polyak_queue_size slots)"""
        _check(self.H.cnb_net_polyak_insert(self.h))

    def load_polyak_weights(self):
        """keep the parameters aside and replace them with the average of the filled queue slots"""
        _check(self.H.cnb_net_load_polyak_weights(self.h))

    def load_current_weights(self):
        """restore the parameters load_polyak_weights kept aside"""
        _check(self.H.cnb_net_load_current_weights(self.h))

    lr_reduce_counter = property(lambda s: s.H.cnb_net_lr_reduce_counter(s.h),
                                 doc="learning-rate reductions train() has applied (kept by save, restored by load)")

    # --- the reference's Validate and Train loop (host/train.cc)
    def validate(self, handler):
        """the output layer's performance metric per image over the DataHandler `handler` (ConvNet::Validate): seek(0),
        then dataset_size // batch_size test-mode batches (the rest is dropped), averaged as the reference's float running
        mean.  ValueError for a handler of another batch size."""
        v = ct.c_float(0)
        _check(self.H.cnb_net_validate(self.h, handler.h, ct.byref(v)))
        return v.value

    def train(self, train, valid=None, *, checkpoint_dir=None, run_name=None):
        """train to the model's schedule (ConvNet::Train, the reference's Train loop) from DataHandler `train`, validating
        on DataHandler `valid` if given, from `iteration` to max_iter.  The schedule is the model's: model_schedule(model)
        for the fields; the periods act where the iteration modulo the period is 0, so an unset print_after or save_after
        (-1) prints or checkpoints after every step.  Files go under checkpoint_dir (default: the model's, else "."), named
        after run_name (default "<model name>_<timestamp>"): <run>.pbtxt, <run>_train.log ("iteration seconds value"
        per print), <run>_valid.log ("iteration value" per validation), <run>.ckpt and with Polyak <run>.ckptpolyak.
        Validation with Polyak on loads the average and training continues from it, as in the reference; with the queue
        still empty it runs on the current weights.  Returns the events, in order: {"iteration", "kind": "train" (the
        metric per image since the last print) | "valid", "value", "lr_reduced", "polyak" (validated on the average)}.
        ValueError for a schedule the loop refuses, a handler of another batch size or a data-parallel net."""
        n = _check(self.H.cnb_net_train(self.h, train.h, valid.h if valid is not None else None,
                                        None if checkpoint_dir is None else os.fsencode(checkpoint_dir),
                                        None if run_name is None else run_name.encode()))
        out = []
        for k in range(n):
            it, kind, v, red, pol = ct.c_longlong(0), ct.c_int(0), ct.c_float(0), ct.c_int(0), ct.c_int(0)
            self.H.cnb_net_train_event(self.h, k, ct.byref(it), ct.byref(kind), ct.byref(v), ct.byref(red), ct.byref(pol))
            out.append({"iteration": it.value, "kind": ("train", "valid")[kind.value], "value": v.value,
                        "lr_reduced": bool(red.value), "polyak": bool(pol.value)})
        return out

    def train_step(self, want_loss=True):
        if want_loss:
            v = ct.c_float(0)
            _check(self.H.cnb_net_train_step(self.h, ct.byref(v)))
            return v.value
        _check(self.H.cnb_net_train_step(self.h, None))
        return None

    def trace_step(self):
        """One extra training step with timing events on the three streams (ConvNet::TraceStep): device milliseconds since
        the step began of the pipeline's milestones, and per gradient bucket its size, exchange window and SGD end."""
        buf = (ct.c_float * 512)()
        n = min(512, _check(self.H.cnb_net_trace_step(self.h, buf, 512)))
        v = [buf[k] for k in range(n)]
        out = {"fprop_end_ms": v[0], "bprop_compute_end_ms": v[1], "step_end_ms": v[2], "buckets": []}
        for b in range(int(v[3])):
            mb, c0, c1, s1 = v[4 + 4 * b:8 + 4 * b]
            out["buckets"].append({"MB": round(mb, 3), "exchange_begin_ms": c0, "exchange_end_ms": c1, "sgd_end_ms": s1})
        return out

    def dp_init(self, rank, world, id_bytes, bucket_floats=32 << 20):
        """join the data-parallel group: RuntimeError when NCCL cannot be loaded or initialised"""
        assert len(id_bytes) == 128
        _check(self.H.cnb_net_dp_init(self.h, rank, world, bytes(id_bytes), bucket_floats))

    def grad_check(self, seed=1, cap=64):
        names = ct.create_string_buffer(64 * cap)
        eps, dw, db = (ct.c_float * cap)(), (ct.c_float * cap)(), (ct.c_float * cap)()
        n = _check(self.H.cnb_net_grad_check(self.h, seed, cap, names, eps, dw, db))
        out = []
        for k in range(n):
            out.append((names.raw[64 * k:64 * (k + 1)].split(b"\0")[0].decode(), eps[k], dw[k], db[k]))
        return out


def model_edge_params(model, batch=1):
    """parameter count of every edge of a model (host-only: no device memory is touched)."""
    with Model(model, batch) as m:
        return [e[3] for e in m.edges()]


def model_edge_optimizer(model, edge, which="weights"):
    """the optimizer config (dict of proto field names) a model gives edge `edge` (host-only); None for an edge without
    parameters"""
    kind = {"weights": ":weight", "bias": ":bias"}[which]
    with Model(model) as m:
        names = [e[0] for e in m.edges()]
        return m._optimizer_config(names[edge] + kind) if 0 <= edge < len(names) else None


def model_bn_layers(model):
    """the batch-normalised layers of a model (host-only): [{"layer", "name", "channels", "bn_f", "bn_epsilon",
    "gamma_optimizer", "beta_optimizer"}] in chain order"""
    out = []
    with Model(model) as m:
        for i, name, channels, _ in m.bn_layers():
            f_, eps = ct.c_float(0), ct.c_float(0)
            m.H.cnb_net_layer_bn(m.h, i, ct.byref(f_), ct.byref(eps))
            out.append({"layer": i, "name": name, "channels": channels, "bn_f": f_.value, "bn_epsilon": eps.value,
                        "gamma_optimizer": m._optimizer_config(name + ":gamma"),
                        "beta_optimizer": m._optimizer_config(name + ":beta")})
    return out


ACTIVATIONS = ("LINEAR", "RECTIFIED_LINEAR", "SOFTMAX", "LOGISTIC", "SOFTMAX_DIST")
LOSS_FUNCTIONS = ("SQUARED_ERROR", "LINEAR_ERROR", "CROSS_ENTROPY_MULTINOMIAL", "CROSS_ENTROPY_BINARY",
                  "CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED", "CLASSIFICATION_MULTINOMIAL", "CLASSIFICATION_BINARY",
                  "HINGE_LINEAR", "HINGE_QUADRATIC")


def model_output_layer(model):
    """the output layer a model configures (host-only): {"activation", "loss_function", "performance_metric" (names),
    "loss_function_weight", "labels" (True: trained on integer labels, False: on float targets)}"""
    a, lf, pm, lab, w = ct.c_int(0), ct.c_int(0), ct.c_int(0), ct.c_int(0), ct.c_float(0)
    with Model(model) as m:
        m.H.cnb_net_output_layer(m.h, ct.byref(a), ct.byref(lf), ct.byref(pm), ct.byref(w), ct.byref(lab))
    return {"activation": ACTIVATIONS[a.value], "loss_function": LOSS_FUNCTIONS[lf.value],
            "performance_metric": LOSS_FUNCTIONS[pm.value], "loss_function_weight": w.value, "labels": bool(lab.value)}


def model_text(model):
    """the resolved configuration of a model (built-in, suffixed or file) as a config::Model text proto: every field the
    host reads for each layer and edge explicit, floats printed so that they read back bit-exactly.  Written to a file
    ending in ".pbtxt", it builds the same model."""
    with Model(model) as m:
        n = m.H.cnb_net_model_text(m.h, None, 0)
        buf = ct.create_string_buffer(n + 1)
        m.H.cnb_net_model_text(m.h, buf, n + 1)
    return buf.value.decode()


def model_initial_weights(model, edge, seed=42):
    """the initial weights (a list of floats, without the bias) of edge `edge` of a model under RNG seed `seed`
    (host-only; the net seeds edge i with its seed + 17 i), or a PRETRAINED edge's weights from its checkpoint; None for
    an edge without parameters of its own (a tied edge starts from its owner's)"""
    with Model(model) as m:
        n = _check(m.H.cnb_net_initial_weights(m.h, edge, seed, None, 0))
        if n == 0:
            return None
        buf = (ct.c_float * n)()
        m.H.cnb_net_initial_weights(m.h, edge, seed, buf, n)
    return list(buf)


def model_ties(model):
    """the tied edges of a model (host-only): {tied edge name: the name of the edge whose parameters it uses}"""
    with Model(model) as m:
        owners = [(e[0], m.H.cnb_net_edge_tied_to(m.h, i).decode()) for i, e in enumerate(m.edges())]
    return {name: owner for name, owner in owners if owner}


def model_flops(model, batch):
    """{"fprop", "train"}: the FLOPs of one forward pass and of one training step of a model at `batch` (host-only; the
    flops_fprop / flops_train of a Net)"""
    with Model(model, batch) as m:
        return {"fprop": m.flops_fprop, "train": m.flops_train}


def model_frozen(model):
    """the frozen part of a model (host-only): {"edges": the blocked edges and those below them, "layers": the hidden layers
    they write}, in chain order"""
    with Model(model) as m:
        n, layers = m._frozen()[0], m.H.cnb_net_num_layers(m.h)
        return {"edges": [e[0] for e in m.edges()[:n]],
                "layers": [m.H.cnb_net_layer_name(m.h, i).decode() for i in range(1, n + 1) if i < layers - 1]}


def model_polyak(model):
    """a model's Polyak averaging (host-only): None when it is off, else {"polyak_after", "polyak_queue_size",
    "validate_after", "save_after"}"""
    v = [ct.c_int(0) for _ in range(4)]
    with Model(model) as m:
        on = m.H.cnb_net_polyak(m.h, *[ct.byref(x) for x in v])
    return dict(zip(("polyak_after", "polyak_queue_size", "validate_after", "save_after"), (x.value for x in v))) if on else None


def polyak_due(model, iteration):
    """whether the reference's training loop inserts into the Polyak queue after train_step number `iteration`"""
    with Model(model) as m:
        return bool(m.H.cnb_net_polyak_due(m.h, iteration))


def model_param_layout(model, batch=1):
    """the flat parameter buffer of a model (host-only): {"edge_offsets": [...], "bn_offsets": per layer (None: not
    batch-normalised), "total": floats with padding}"""
    with Model(model, batch) as m:
        bn = [m.H.cnb_net_bn_offset(m.h, i) for i in range(m.H.cnb_net_num_layers(m.h))]
        return {"edge_offsets": [m.H.cnb_net_edge_slice(m.h, i) for i in range(m.H.cnb_net_num_edges(m.h))],
                "bn_offsets": [off if off >= 0 else None for off in bn], "total": m.num_params}


FUSION_FLAGS = ("dropout_up", "scale_down", "sums_bias_below", "offers_bias_grad")


def model_fusion(model, batch=1):
    """the epilogue fusion plan of a model (host-only): {"edges": per edge {"up_act", "down_act" (CNB_ACT_* codes: 0 none,
    1 ReLU, 2 logistic), "dropout_up", "scale_down", "sums_bias_below", "offers_bias_grad"}, "layers": per layer
    {"activation_pass", "deriv_pass"} (True: a separate pass remains)}"""
    edges = []
    with Model(model, batch) as m:
        for i in range(m.H.cnb_net_num_edges(m.h)):
            up, down = ct.c_int(0), ct.c_int(0)
            flags = m.H.cnb_net_edge_fusion(m.h, i, ct.byref(up), ct.byref(down))
            edges.append(dict(up_act=up.value, down_act=down.value,
                              **{f: bool(flags >> b & 1) for b, f in enumerate(FUSION_FLAGS)}))
        passes = [m.H.cnb_net_layer_passes(m.h, i) for i in range(m.H.cnb_net_num_layers(m.h))]
    return {"edges": edges, "layers": [{"activation_pass": bool(p & 1), "deriv_pass": bool(p & 2)} for p in passes]}


def check_bn_optimizer(config):
    """raise ValueError if the optimizer block `config` (a dict) cannot train gamma / beta"""
    _check(load_host().cnb_bn_optimizer_check(ct.byref(OptimizerConfig.from_dict(config))))


def optimizer_schedule(config, step):
    """(epsilon, momentum) of the update after `step` earlier ones under the optimizer block `config` (a dict)"""
    eps, mom = ct.c_float(0), ct.c_float(0)
    c = OptimizerConfig.from_dict(config)
    _check(load_host().cnb_optimizer_schedule(ct.byref(c), step, ct.byref(eps), ct.byref(mom)))
    return eps.value, mom.value


def plan_buckets(edge_sizes, bucket_floats):
    """(lo, hi, trigger_edge) gradient buckets over the flat 128-float-padded parameter buffer (convnet.cc PlanBuckets)."""
    H = load_host()
    n = len(edge_sizes)
    offs, total = [], 0
    for sz in edge_sizes:
        offs.append(total)
        total += (sz + 127) // 128 * 128
    A = ct.c_longlong * n
    cap = n + 1
    lo, hi, trig = (ct.c_longlong * cap)(), (ct.c_longlong * cap)(), (ct.c_int * cap)()
    k = H.cnb_plan_buckets(n, A(*offs), A(*edge_sizes), bucket_floats, cap, lo, hi, trig)
    return [(lo[j], hi[j], trig[j]) for j in range(k)], total


def dp_unique_id():
    buf = ct.create_string_buffer(128)
    _check(load_host().cnb_dp_unique_id(buf))
    return buf.raw


class DataIterator:
    """Device side of the reference's input pipeline (host/data.h; src/datahandler.cc:146-200, 520-568): a chunk of images
    resident on the GPU, and per minibatch a random (or centre / corner) crop + mirror into the net's input layer.
    ValueError for a crop larger than the image, or a chunk_size or channels below 1."""

    def __init__(self, chunk_size, channels, image_size, gpu_image_size, translate=True, flip=True, seed=1):
        self.H, self.h = load_host(), None
        isy, isx = (image_size, image_size) if isinstance(image_size, int) else image_size
        gy, gx = (gpu_image_size, gpu_image_size) if isinstance(gpu_image_size, int) else gpu_image_size
        self.chunk_size, self.dims = chunk_size, channels * isy * isx
        self.h = _check(self.H.cnb_data_create(chunk_size, channels, isy, isx, gy, gx, int(translate), int(flip), seed))

    def close(self):
        if self.h:
            self.H.cnb_data_destroy(self.h)
            self.h = None

    def upload(self, host_tensor, first=0):
        """host_tensor: float32 CPU tensor [count, channels, rows, cols] (pinned for an asynchronous copy)"""
        import torch
        t = host_tensor.contiguous()
        assert t.dtype == torch.float32 and t.device.type == "cpu" and t[0].numel() == self.dims
        _check(self.H.cnb_data_upload(self.h, t.data_ptr(), first, t.shape[0]))
        self._keep = t                                   # the copy is asynchronous

    def get_batch(self, net, start=0, multiplicity_id=0):
        _check(self.H.cnb_data_get_batch(self.h, net.h, start, multiplicity_id))

    def last_noise(self, batch):
        buf = (ct.c_float * (3 * batch))()
        n = self.H.cnb_data_last_noise(self.h, buf, 3 * batch)
        assert n == batch
        v = [buf[k] for k in range(3 * batch)]
        return v[:batch], v[batch:2 * batch], v[2 * batch:]


def view_offset(multiplicity_id, max_offset_x, max_offset_y):
    """(w, h) of the deterministic crop number multiplicity_id (host logic only, no GPU)"""
    H = load_host()
    w, h = ct.c_int(0), ct.c_int(0)
    H.cnb_data_view_offset(multiplicity_id, max_offset_x, max_offset_y, ct.byref(w), ct.byref(h))
    return w.value, h.value


class DataHandler:
    """The reference's DataHandler (src/datahandler.cc; host/data.h) over a data set already in host memory: float pixels
    `images` [N, channels, rows, cols] (a CPU float32 tensor, pinned for copies that overlap the step), integer `labels`
    [N] and / or float `targets` [N, features].  It keeps a chunk of chunk_size images on the GPU (the whole data set when
    chunk_size is 0 or larger), and get_batch(net) writes the next minibatch into the net's input layer, randomly cropped
    to gpu_image_size (when `translate`; else the centre / corner view of multiplicity_id) and mirrored (when `flip`; else
    views 5..9), together with the labels or the targets the net's output layer trains on, in one kernel launch.

    The order follows the reference's rules: a chunk is reused max_reuse_count times before the next one is loaded,
    randomize_gpu reshuffles the chunk's order for every pass, randomize_cpu loads chunks of random_access_chunk_size-row
    blocks from random places (else consecutive rows, wrapping around), every batch is served `multiplicity` times with
    multiplicity_id 0, 1, ..., and pipeline_loads copies the next chunk while the net trains.  dataset_schedule() gives
    the same order without a GPU.  The tensors must outlive the handler (it keeps references)."""

    def __init__(self, images, labels=None, targets=None, *, batch_size, chunk_size=0, gpu_image_size=None, translate=False,
                 flip=False, randomize_gpu=False, randomize_cpu=False, random_access_chunk_size=1, max_reuse_count=0,
                 multiplicity=1, pipeline_loads=False, seed=1):
        import torch
        self.H = load_host()
        self.h = None
        assert images.dtype == torch.float32 and images.device.type == "cpu" and images.dim() == 4
        n, c, isy, isx = images.shape
        gy, gx = ((isy, isx) if gpu_image_size is None else
                  (gpu_image_size, gpu_image_size) if isinstance(gpu_image_size, int) else gpu_image_size)
        self._images = images.contiguous()
        self._labels = None if labels is None else labels.to(torch.int32).contiguous()
        self._targets = None if targets is None else targets.to(torch.float32).reshape(n, -1).contiguous()
        for t in (self._labels, self._targets):
            assert t is None or (t.device.type == "cpu" and t.shape[0] == n), "labels / targets: one row per image, on the host"
        self.order = DatasetOrder.from_dict(dict(
            batch_size=batch_size, chunk_size=chunk_size, max_reuse_count=max_reuse_count, pipeline_loads=pipeline_loads,
            randomize_cpu=randomize_cpu, randomize_gpu=randomize_gpu, random_access_chunk_size=random_access_chunk_size,
            multiplicity=multiplicity))
        self.batch_size = batch_size
        ptr = lambda t: None if t is None else t.data_ptr()
        self.h = _check(self.H.cnb_handler_create(
            ct.byref(self.order), n, c, isy, isx, gy, gx, int(translate), int(flip), ptr(self._images), ptr(self._labels),
            ptr(self._targets), 0 if self._targets is None else self._targets.shape[1], seed))

    @classmethod
    def from_model(cls, model, images, labels=None, which="train_dataset", *, targets=None, net=None, seed=1):
        """a handler configured by a model file's train_dataset or valid_dataset: its batch order, and the crop
        (gpu_image_size_y / _x), can_translate and can_flip of the data stream whose layer_name is the input layer.
        ValueError when the model has no such block, or when its batch_size differs from `net`'s."""
        cfg = model_dataset(model, which)
        if cfg is None:
            raise ValueError("model %r has no %s" % (model, which))
        if net is not None and cfg["batch_size"] != net.batch_size:
            raise ValueError("%s of %r has batch_size %d and the net %d" % (which, model, cfg["batch_size"], net.batch_size))
        gy, gx = cfg.pop("gpu_image_size_y"), cfg.pop("gpu_image_size_x")
        gy, gx = gy or images.shape[2], gx or images.shape[3]
        return cls(images, labels, targets, gpu_image_size=(gy, gx), seed=seed, **cfg)

    def close(self):
        if self.h:
            self.H.cnb_handler_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def get_batch(self, net):
        """the next minibatch into net's input layer, and its labels or targets into labels_tensor() / targets_tensor()"""
        if net.batch_size != self.batch_size:
            raise ValueError("the net's batch size is %d and the handler's %d" % (net.batch_size, self.batch_size))
        _check(self.H.cnb_handler_get_batch(self.h, net.h))

    def seek(self, row):
        """restart the schedule at data set row `row` (DataHandler::Seek): the next batch loads a chunk from there"""
        _check(self.H.cnb_handler_seek(self.h, row))

    def last_indices(self):
        """{"start", "multiplicity_id", "rows": the data set row of each image of the last batch, "width_offset",
        "height_offset", "flip": its jitter}"""
        b = self.batch_size
        start, mid, rows, noise = ct.c_int(0), ct.c_int(0), (ct.c_int * b)(), (ct.c_float * (3 * b))()
        self.H.cnb_handler_last(self.h, ct.byref(start), ct.byref(mid), rows, noise)
        v = list(noise)
        return {"start": start.value, "multiplicity_id": mid.value, "rows": list(rows), "width_offset": v[:b],
                "height_offset": v[b:2 * b], "flip": v[2 * b:]}


def dataset_schedule(config, dataset_size, steps, seed=1, seeks=None):
    """the order a DataHandler with batch-order fields `config` (a dict of DatasetConfig names) and seed `seed` serves a
    data set of dataset_size images in (host logic only, no GPU): for each of `steps` minibatches a tuple (rows, start,
    multiplicity_id, permutation): rows is the list of data set rows of the chunk loaded for that batch (None when the
    resident chunk is kept), and batch image n is chunk column permutation[start + n].  seeks: {step: row} calls seek(row)
    before that step.  ValueError for a configuration the handler refuses."""
    H = load_host()
    order = DatasetOrder.from_dict(config)
    s = _check(H.cnb_schedule_create(ct.byref(order), dataset_size, seed))
    try:
        chunk = H.cnb_schedule_chunk_size(s)
        rows, perm, start, mid, out = (ct.c_int * chunk)(), (ct.c_int * chunk)(), ct.c_int(0), ct.c_int(0), []
        for k in range(steps):
            if seeks and k in seeks:
                _check(H.cnb_schedule_seek(s, seeks[k]))
            loaded = H.cnb_schedule_next(s, ct.byref(start), ct.byref(mid), rows, perm)
            out.append((list(rows) if loaded else None, start.value, mid.value, list(perm)))
        return out
    finally:
        H.cnb_schedule_destroy(s)


def model_dataset(model, which="train_dataset"):
    """a model's train_dataset or valid_dataset block (host-only): None when it has none, else its batch-order fields
    (DatasetOrder names) with translate, flip, gpu_image_size_y and gpu_image_size_x (0: not set) of the data stream that
    feeds the input layer"""
    o, v = DatasetOrder(), [ct.c_int(0) for _ in range(4)]
    with Model(model) as m:
        present = m.H.cnb_net_dataset(m.h, {"train_dataset": 0, "valid_dataset": 1}[which], ct.byref(o),
                                      *[ct.byref(x) for x in v])
    if not present:
        return None
    d = {k: (bool(x) if k in ("pipeline_loads", "randomize_cpu", "randomize_gpu") else x) for k, x in o.to_dict().items()}
    d.update(zip(("translate", "flip", "gpu_image_size_y", "gpu_image_size_x"), (bool(v[0].value), bool(v[1].value),
                                                                                   v[2].value, v[3].value)))
    return d


SCHEDULE_INTS = ("max_iter", "print_after", "validate_after", "save_after", "reduce_lr_num_steps", "reduce_lr_max",
                 "smaller_is_better")


def model_schedule(model):
    """a model's training schedule (host-only), the fields Net.train reads, at the proto's defaults where unset:
    {"max_iter", "print_after", "validate_after", "save_after", "reduce_lr_factor", "reduce_lr_threshold",
    "reduce_lr_num_steps", "reduce_lr_max", "smaller_is_better", "reduce_lr_layer_name", "checkpoint_dir"}"""
    ints, floats, layer, cdir = (ct.c_int * 7)(), (ct.c_float * 2)(), ct.c_char_p(), ct.c_char_p()
    with Model(model) as m:
        m.H.cnb_net_schedule(m.h, ints, floats, ct.byref(layer), ct.byref(cdir))
        layer, cdir = layer.value, cdir.value
    out = dict(zip(SCHEDULE_INTS, ints))
    out["smaller_is_better"] = bool(out["smaller_is_better"])
    out.update(reduce_lr_factor=floats[0], reduce_lr_threshold=floats[1], reduce_lr_layer_name=layer.decode(),
               checkpoint_dir=os.fsdecode(cdir))
    return out


def reduce_lr_due(history, num_steps, threshold, smaller_is_better):
    """the reference's CheckReduceLearningRate, the test Net.train applies after each validation: False while `history`
    (validation values, oldest first) holds fewer than num_steps values; else whether the float running mean of the
    second half of its last num_steps values (the larger half when num_steps is odd) improves on the first half's by less
    than `threshold` (improves: is smaller when smaller_is_better, else larger)"""
    h = (ct.c_float * max(1, len(history)))(*history)
    return bool(load_host().cnb_reduce_lr_due(h, len(history), num_steps, threshold, int(smaller_is_better)))


TRAIN_ACTIONS = ("print", "insert", "validate", "save", "lr_reduced", "polyak", "final")


def train_dry_run(model, valid_values=None, *, iteration=0, lr_reduce_counter=0):
    """what Net.train does with `model`'s schedule from train_step number `iteration` + 1 to max_iter, without a GPU
    (host/train.cc TrainSchedule, the code Net.train decides with): a list of (iteration, set of actions) for every
    iteration with an action, in order; actions are "print", "insert" (into the Polyak queue), "validate", "save",
    "lr_reduced" (after this validation), "polyak" (this validation runs on the Polyak average).  The checkpoint after
    the loop is a last record (max_iter, {"save", "final"}).  valid_values: the validation values, in order (None: no
    validation set).  ValueError for a schedule Net.train refuses, or fewer values than validations."""
    vals = list(valid_values or [])
    fv = (ct.c_float * max(1, len(vals)))(*vals)
    cap = 1024
    with Model(model) as m:
        while True:
            its, acts = (ct.c_longlong * cap)(), (ct.c_int * cap)()
            n = _check(m.H.cnb_net_train_dry_run(m.h, iteration, lr_reduce_counter, int(valid_values is not None), fv,
                                                 len(vals), cap, its, acts))
            if n <= cap:
                return [(its[k], {a for b, a in enumerate(TRAIN_ACTIONS) if acts[k] >> b & 1}) for k in range(n)]
            cap = n


Net.model_output_layer = staticmethod(model_output_layer)
