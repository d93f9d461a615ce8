"""Flag system: a small absl/`tf.app.flags` work-alike.

The reference scatters `tf.app.flags.DEFINE_*` calls over three modules and
merges them into one global ``FLAGS`` by import side-effect
(reference: src/distributed_train.py:36-99, src/nn_eval.py:36-45,
src/sync_replicas_optimizer_modified/sync_replicas_optimizer_modified.py:38).
Here every flag lives in one registry with the *same names and defaults*, so
command lines written for the reference keep working, plus a small set of new
flags (model choice, synthetic data, straggler injection, backend selection)
that the single-box H100 design needs.

Accepted syntaxes (same as absl): ``--name=value``, ``--name value``,
``--flag`` / ``--noflag`` for booleans, and ``true/false/1/0/yes/no/t/f`` as
boolean values in any case.
"""
from __future__ import annotations

import sys
from dataclasses import dataclass
from typing import Any, Callable, Dict, List, Optional, Sequence

_TRUE = {"true", "t", "1", "yes", "y"}
_FALSE = {"false", "f", "0", "no", "n"}


class FlagError(ValueError):
    pass


@dataclass
class _Flag:
    name: str
    default: Any
    help: str
    kind: str  # 'boolean' | 'integer' | 'float' | 'string'
    value: Any = None
    present: bool = False  # set on the command line

    def parse(self, text: str) -> Any:
        if self.kind == "boolean":
            low = text.strip().lower()
            if low in _TRUE:
                return True
            if low in _FALSE:
                return False
            raise FlagError("flag --%s: %r is not a boolean" % (self.name, text))
        if self.kind == "integer":
            try:
                return int(text, 0) if isinstance(text, str) else int(text)
            except ValueError:
                raise FlagError("flag --%s: %r is not an integer" % (self.name, text))
        if self.kind == "float":
            try:
                return float(text)
            except ValueError:
                raise FlagError("flag --%s: %r is not a float" % (self.name, text))
        return str(text)


class FlagValues:
    """Registry + attribute access (``FLAGS.batch_size``)."""

    def __init__(self) -> None:
        object.__setattr__(self, "_flags", {})
        object.__setattr__(self, "_parsed", False)

    # ---- definition -----------------------------------------------------
    def _define(self, kind: str, name: str, default: Any, help: str) -> None:
        flags: Dict[str, _Flag] = self._flags
        if name in flags:
            # Re-definition with identical spec is a no-op (modules may be
            # re-imported by the compat shims); anything else is a bug.
            old = flags[name]
            if old.kind != kind or old.default != default:
                raise FlagError("flag --%s defined twice with different specs" % name)
            return
        flags[name] = _Flag(name=name, default=default, help=help, kind=kind, value=default)

    def DEFINE_boolean(self, name: str, default: bool, help: str = "") -> None:
        self._define("boolean", name, default, help)

    DEFINE_bool = DEFINE_boolean

    def DEFINE_integer(self, name: str, default: int, help: str = "") -> None:
        self._define("integer", name, default, help)

    def DEFINE_float(self, name: str, default: float, help: str = "") -> None:
        self._define("float", name, default, help)

    def DEFINE_string(self, name: str, default: str, help: str = "") -> None:
        self._define("string", name, default, help)

    # ---- access ---------------------------------------------------------
    def __getattr__(self, name: str) -> Any:
        flags = object.__getattribute__(self, "_flags")
        if name in flags:
            return flags[name].value
        raise AttributeError("unknown flag %r" % name)

    def __setattr__(self, name: str, value: Any) -> None:
        flags = self._flags
        if name not in flags:
            raise AttributeError("unknown flag %r" % name)
        f = flags[name]
        f.value = f.parse(value) if isinstance(value, str) and f.kind != "string" else value

    def __contains__(self, name: str) -> bool:
        return name in self._flags

    def is_present(self, name: str) -> bool:
        return self._flags[name].present

    def flag_values_dict(self) -> Dict[str, Any]:
        return {k: f.value for k, f in self._flags.items()}

    def defaults_dict(self) -> Dict[str, Any]:
        return {k: f.default for k, f in self._flags.items()}

    def reset(self) -> None:
        for f in self._flags.values():
            f.value = f.default
            f.present = False
        object.__setattr__(self, "_parsed", False)

    # ---- parsing --------------------------------------------------------
    def parse(self, argv: Optional[Sequence[str]] = None, known_only: bool = False) -> List[str]:
        """Parse ``argv`` (without the program name). Returns leftover positionals.

        Unknown ``--flags`` raise unless ``known_only`` (then they are returned).
        """
        flags: Dict[str, _Flag] = self._flags
        args = list(sys.argv[1:] if argv is None else argv)
        rest: List[str] = []
        i = 0
        while i < len(args):
            a = args[i]
            i += 1
            if a == "--":
                rest.extend(args[i:])
                break
            if not a.startswith("-") or a == "-":
                rest.append(a)
                continue
            body = a.lstrip("-")
            if "=" in body:
                name, text = body.split("=", 1)
                has_value = True
            else:
                name, text, has_value = body, "", False
            name = name.replace("-", "_")
            if name not in flags:
                if name.startswith("no") and name[2:] in flags and flags[name[2:]].kind == "boolean" and not has_value:
                    f = flags[name[2:]]
                    f.value, f.present = False, True
                    continue
                if known_only:
                    rest.append(a)
                    continue
                raise FlagError("unknown flag --%s" % name)
            f = flags[name]
            if not has_value:
                if f.kind == "boolean":
                    # `--flag` alone means true; `--flag false` is also accepted.
                    if i < len(args) and args[i].strip().lower() in (_TRUE | _FALSE):
                        text = args[i]
                        i += 1
                    else:
                        text = "true"
                else:
                    if i >= len(args):
                        raise FlagError("flag --%s needs a value" % name)
                    text = args[i]
                    i += 1
            # Strip one level of shell-style quotes that survive cfg templating
            # (the reference wraps host lists in single quotes, cfg/*:79-80).
            if len(text) >= 2 and text[0] == text[-1] and text[0] in "'\"":
                text = text[1:-1]
            f.value = f.parse(text)
            f.present = True
        object.__setattr__(self, "_parsed", True)
        return rest

    def usage(self) -> str:
        lines = []
        for name in sorted(self._flags):
            f = self._flags[name]
            lines.append("  --%s (%s, default %r)\n      %s" % (name, f.kind, f.default, f.help))
        return "\n".join(lines)


FLAGS = FlagValues()


def define_reference_flags(F: FlagValues = FLAGS) -> FlagValues:
    """Every flag of the reference, same name and default (SURVEY §2.2)."""
    # reference: src/distributed_train.py:36-39
    F.DEFINE_boolean("worker_times_cdf_method", False, "Track worker times cdf (full-barrier mode with timing capture)")
    F.DEFINE_boolean("interval_method", False, "Use the fixed wall-clock interval aggregation method")
    F.DEFINE_boolean("async_method", False, "Asynchronous SGD: every replica applies its own gradient to the shared "
                                            "weights at once, without waiting for or averaging with any other; reports "
                                            "the staleness of its updates (workerN_staleness.json)")
    F.DEFINE_integer("ssp_staleness", -1, "Stale synchronous parallel, with --async_method: no replica starts an "
                                          "iteration more than s of its own updates ahead of the slowest replica that "
                                          "is still running (s = this value, 0 <= s < 2^31; -1 = off, plain "
                                          "asynchronous SGD); reports its waits (workerN_ssp.json)")
    F.DEFINE_integer("local_sgd_steps", 0, "Local SGD (periodic model averaging): every replica applies its own "
                                           "gradients to its own weights, and every H-th global step the replicas' "
                                           "weights are replaced by their mean (H = this value; 0 = off); reports the "
                                           "averaging rounds and their barrier waits (workerN_local_sgd.json)")
    F.DEFINE_boolean("gossip_method", False, "Gossip (decentralized) SGD on a ring: every step each replica averages its "
                                             "half step w - lr * g with those of its two ring neighbours, waiting for "
                                             "those two only; the run ends with one average of every replica; reports "
                                             "the barrier waits (workerN_gossip.json)")
    F.DEFINE_boolean("should_summarize", False, "Whether the chief should write summaries")
    F.DEFINE_boolean("timeline_logging", False, "Dump a chrome-trace timeline json per step")
    # reference: src/distributed_train.py:40-48
    F.DEFINE_string("job_name", "", 'One of "ps", "worker"')
    F.DEFINE_string("ps_hosts", "", "Comma-separated hostname:port list of parameter servers (accepted for "
                    "compatibility; the H100 engine has no parameter server)")
    F.DEFINE_string("worker_hosts", "", "Comma-separated hostname:port list of workers; its length is the "
                    "number of replicas when WORLD_SIZE is not set")
    # reference: src/distributed_train.py:50-63
    F.DEFINE_string("train_dir", "/tmp/imagenet_train", "Directory for checkpoints, timelines and .npy results")
    F.DEFINE_integer("rpc_port", 1235, "Port of the timing/ready control plane (rendezvous store port here)")
    F.DEFINE_integer("save_results_period", 1000, "Period (global steps) of saving worker<id>_time_acc.npy")
    F.DEFINE_integer("max_steps", 1000000, "Number of batches to run")
    F.DEFINE_boolean("drop_connect", False, "Multiply gradients by a Bernoulli mask before aggregation")
    F.DEFINE_integer("batch_size", 128, "Batch size per replica")
    F.DEFINE_string("subset", "train", 'Either "train" or "validation" (unused, kept for compatibility)')
    F.DEFINE_boolean("log_device_placement", False, "Log which device every kernel runs on")
    # reference: src/distributed_train.py:68-78
    F.DEFINE_integer("task_id", 0, "Replica index; replica 0 is the chief")
    F.DEFINE_integer("num_replicas_to_aggregate", -1, "Gradients to collect before updating (K of N); -1 = all")
    F.DEFINE_float("save_interval_secs", 20, "Checkpoint interval in seconds (chief); fractions allowed: an H100 step takes ~0.15 ms")
    F.DEFINE_integer("save_summaries_secs", 300, "Summary interval in seconds (chief)")
    # reference: src/distributed_train.py:92-98
    F.DEFINE_float("initial_learning_rate", 0.1, "Initial learning rate")
    F.DEFINE_float("num_epochs_per_decay", 2.0, "Epochs after which the learning rate decays")
    F.DEFINE_float("learning_rate_decay_factor", 0.999, "Learning rate decay factor")
    F.DEFINE_float("drop_connect_probability", 0.9, "Keep probability of gradient drop-connect")
    # reference: sync_replicas_optimizer_modified.py:38
    F.DEFINE_integer("interval_ms", 1000, "Aggregation period of the interval method, milliseconds")
    # reference: src/nn_eval.py:36-45
    F.DEFINE_string("eval_dir", "/tmp/imagenet_eval", "Directory where the evaluator writes its event log")
    F.DEFINE_string("checkpoint_dir", "/tmp/imagenet_train", "Directory the evaluator polls for checkpoints")
    F.DEFINE_float("eval_interval_secs", 1, "How often the evaluator polls (seconds, fractions allowed)")
    F.DEFINE_boolean("run_once", False, "Evaluate once and exit")
    return F


def define_engine_flags(F: FlagValues = FLAGS) -> FlagValues:
    """New flags of the H100 engine (no analogue in the reference)."""
    F.DEFINE_string("model", "lenet", "lenet | mlp2 | mlp3")
    F.DEFINE_integer("mlp_hidden", 1024, "Hidden width of the MLP models")
    F.DEFINE_string("data_dir", "MNIST-data", "Directory with the four MNIST IDX .gz files (never downloaded)")
    F.DEFINE_boolean("synthetic_data", True, "Generate MNIST-shaped synthetic data when the IDX files are absent")
    F.DEFINE_boolean("fake_data", False, "Constant all-ones images / label 0 (reference mnist_data.py fake_data)")
    F.DEFINE_integer("seed", 66478, "Base RNG seed (per-replica streams are derived from it)")
    F.DEFINE_string("compute_dtype", "bf16", "bf16 | fp32 (activations / tensor-core operand type)")
    F.DEFINE_string("backend", "auto", "auto | fused (sm_90a kernels + symmetric memory) | nccl | gloo")
    F.DEFINE_string("inject_straggler", "", "Comma-separated device-side delay injection: rank:prob:usec (fixed delay with "
                    "probability prob), or a delay drawn every iteration from rank:exp:MEAN_US, "
                    "rank:lognormal:MEDIAN_US:SIGMA or rank:profile:PATH (.npy / text file of delays in us); "
                    "rank may be * for the drawn forms (every replica, each with its own stream)")
    F.DEFINE_integer("sync_timeout_ms", 30000, "Watchdog for device-side arrival polling")
    F.DEFINE_boolean("use_cuda_graph", True, "Capture the training step in a CUDA graph")
    F.DEFINE_boolean("use_nvls", True, "Use NVLS multimem reductions when the multicast object binds")
    F.DEFINE_boolean("debug_sync", False, "Dump the aggregation control block (arrival / done words, bitmap, commit ring) "
                                          "when a device-side watchdog fires (reference: the optimizer's debug Print ops)")
    F.DEFINE_boolean("pipeline_steps", True, "GPU path: enqueue step i+1 before reading step i's loss / status words "
                                             "(page-locked result buffers, background batch packer)")
    F.DEFINE_boolean("device_data", False, "GPU path: keep each replica's training set in GPU memory and feed every step "
                                           "B int32 row indices, gathered into the input slot on the device, instead of a "
                                           "batch packed on the host (not with --fake_data; sm_90a engine only)")
    F.DEFINE_integer("log_every", 1, "Log every n-th local iteration (1 = reference behaviour)")
    F.DEFINE_float("dropout_keep_prob", 0.5, "Keep probability of the fc1 dropout (reference mnist.py:139)")
    F.DEFINE_integer("eval_every_steps", 0, "Chief: score the validation set after every E-th global step and after the last "
                                            "one (test_acc, worker0_eval.npy); 0 = off.  GPU path: lenet; K < N or interval need --eval_snapshot")
    F.DEFINE_boolean("eval_snapshot", False, "GPU path, with --eval_every_steps: score a validated snapshot of the newest "
                                             "committed weights, so K < N and --interval_method runs can be evaluated too")
    F.DEFINE_float("target_accuracy", 0.0, "With --eval_every_steps: stop the run after the first in-training evaluation "
                                           "whose validation accuracy is >= this value, and report the training time it "
                                           "took (worker0_time_to_accuracy.json); 0 = off, else 0 < A <= 1")
    F.DEFINE_float("moving_average_decay", 0.0, "Chief: keep an exponential moving average of the weights with this decay "
                                                "(TF's ExponentialMovingAverage, num_updates = global step), saved in every "
                                                "checkpoint as <variable>/ExponentialMovingAverage; 0 = off, else 0 < D < 1.  "
                                                "K = N or --worker_times_cdf_method only")
    F.DEFINE_boolean("eval_moving_average", False, "Score the moving average instead of the live weights: in training, the "
                                                   "in-training evaluation and --target_accuracy (needs --moving_average_decay "
                                                   "and --eval_every_steps); in the evaluator, the checkpoint's "
                                                   "<variable>/ExponentialMovingAverage tensors")
    F.DEFINE_boolean("keep_best_checkpoint", False, "With --eval_every_steps: keep the weights of the best-scoring "
                                                    "in-training evaluation and save them at the end of the run as "
                                                    "train_dir/best/model.ckpt-<step> plus worker0_best.json")
    F.DEFINE_integer("early_stopping_patience", 0, "With --eval_every_steps: stop the run once this many in-training "
                                                   "evaluations in a row have not beaten the best so far (by more than "
                                                   "--early_stopping_min_delta), at the scored step + 2; report in "
                                                   "worker0_early_stopping.json; 0 = off, else P >= 1")
    F.DEFINE_float("early_stopping_min_delta", 0.0, "With --early_stopping_patience: the accuracy an evaluation must beat "
                                                    "the best by to reset the patience, rounded down to whole validation "
                                                    "rows; 0 <= D < 1")
    F.DEFINE_integer("lr_plateau_patience", 0, "With --eval_every_steps: multiply the learning rate by "
                                               "--lr_plateau_factor once this many in-training evaluations in a row "
                                               "have not beaten the best so far (by more than --lr_plateau_min_delta), "
                                               "from the scored step + 2; at most 32 cuts; report in "
                                               "worker0_lr_plateau.json; 0 = off, else P >= 1")
    F.DEFINE_float("lr_plateau_factor", 0.1, "With --lr_plateau_patience: the factor each cut multiplies the learning "
                                             "rate by; 0 < F < 1")
    F.DEFINE_float("lr_plateau_min_delta", 0.0, "With --lr_plateau_patience: the accuracy an evaluation must beat the "
                                                "best by to reset the patience, rounded down to whole validation rows; "
                                                "0 <= D < 1")
    F.DEFINE_integer("lr_warmup_steps", 0, "Linear learning-rate warmup (Goyal et al. 2017): the update of global step s < W "
                                           "is made at the rate times f0 + (1 - f0) * s / W, f0 = "
                                           "--lr_warmup_start_factor; counts global steps (interval mode: ticks; K > N: "
                                           "committed steps) from 0, on top of the decay; 0 = off, else W < 2^32 - 1")
    F.DEFINE_float("lr_warmup_start_factor", 1.0 / 3, "With --lr_warmup_steps: the factor f0 of the rate at global step 0 "
                                                      "(torch's LinearLR start_factor); 0 <= f0 < 1")
    F.DEFINE_integer("lr_cosine_decay_steps", 0, "Replace the staircase decay by TF's cosine_decay over T global steps: "
                                                 "the rate is lr0 * ((1 - alpha) * (1 + cos(pi * min(s, T) / T)) / 2 + "
                                                 "alpha), from step 0 (a warmup multiplies its first steps); from step T on "
                                                 "it is lr0 * alpha, so alpha = 0 stops the weights there.  Not with "
                                                 "--learning_rate_decay_factor or --num_epochs_per_decay; 0 = off, else "
                                                 "T < 2^32 - 1")
    F.DEFINE_float("lr_cosine_alpha", 0.0, "With --lr_cosine_decay_steps: the floor alpha of the cosine decay as a fraction "
                                           "of the initial learning rate (TF's alpha); 0 <= alpha < 1")
    F.DEFINE_float("weight_decay", 0.0, "L2 weight decay of the fully connected layers (the reference model's regulariser, "
                                        "src/mnist.py:142-143): every replica differentiates CE + lambda * sum(v^2) / 2 over "
                                        "lenet's fc1/fc2 weights and biases (every layer of mlp2 / mlp3), and the logged "
                                        "training loss includes the term; 0 = off, else 0 < lambda < 1.  GPU path: lenet")
    F.DEFINE_float("augment_max_shift", 0.0, "Random affine augmentation of the training images: translate each image by "
                                             "tx, ty ~ U[-T, T] pixels; 0 <= T <= 8 (0 = no shift).  Augmentation is on "
                                             "when any --augment_max_* is non-zero; evaluation is never augmented")
    F.DEFINE_float("augment_max_rotation", 0.0, "Random affine augmentation: rotate each training image by theta ~ U[-R, R] "
                                                "degrees about its centre; 0 <= R <= 180 (0 = no rotation)")
    F.DEFINE_float("augment_max_scale", 0.0, "Random affine augmentation: zoom each training image by s ~ U[1-S, 1+S]; "
                                             "0 <= S < 1 (0 = no zoom)")
    F.DEFINE_float("augment_elastic_alpha", 0.0, "Elastic distortion of the training images (Simard et al. 2003): "
                                                 "displace each pixel by alpha pixels times uniform noise in [-1, 1] "
                                                 "smoothed by a Gaussian of width --augment_elastic_sigma, before the "
                                                 "affine warp; 0 <= alpha <= 64 (0 = off).  Augmentation is on when "
                                                 "alpha or any --augment_max_* is non-zero")
    F.DEFINE_float("augment_elastic_sigma", 4.0, "With --augment_elastic_alpha: the width in pixels of the Gaussian that "
                                                 "smooths the displacement field; 0.5 <= sigma <= 8")
    return F


define_reference_flags()
define_engine_flags()


def app_run(main: Callable[[List[str]], Any], argv: Optional[Sequence[str]] = None) -> None:
    """``tf.app.run`` work-alike: parse flags, call ``main(leftover_argv)``, exit."""
    args = list(sys.argv if argv is None else argv)
    if any(a in ("--help", "-h", "--helpfull") for a in args[1:]):
        print("flags:\n" + FLAGS.usage())
        sys.exit(0)
    rest = FLAGS.parse(args[1:])
    sys.exit(main([args[0]] + rest))
