"""distributedmnist_b200 -- a H100-native synchronous-replica training engine.

Same capabilities as agnusmaximus/DistributedMNIST (K-of-N backup-worker,
full-barrier and interval gradient aggregation; straggler telemetry; periodic
checkpoints + continuous evaluator; sweep/plot tooling), re-designed for one
8xH100 box: one process per GPU, hand-written sm_90a kernels for the model and
a single fused allreduce+scale+SGD kernel over NVLink symmetric memory instead
of a TensorFlow parameter server.  See DESIGN.md.
"""
__version__ = "0.1.0"

from .flags import FLAGS, app_run  # noqa: F401
