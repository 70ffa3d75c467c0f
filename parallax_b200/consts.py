"""Environment-variable protocol between launcher ("master") and workers.

Parity: reference `parallax/parallax/core/python/common/consts.py:18-38` and
`common/partitions.py:29-31`, `common/lib.py:59-62`.  The contract is kept
(the same script is re-executed on every worker and an env var tells the
process which role it plays) but workers are one process per GPU for *every*
run option, rendezvousing through `torch.distributed` on 127.0.0.1 / the
first host instead of mpirun + gRPC.
"""
import os
import getpass

# --- role selection ---------------------------------------------------------
PARALLAX_RUN_OPTION = "PARALLAX_RUN_OPTION"
PARALLAX_RUN_MASTER = "PARALLAX_RUN_MASTER"
PARALLAX_RUN_MPI = "PARALLAX_RUN_MPI"
PARALLAX_RUN_PS = "PARALLAX_RUN_PS"
PARALLAX_RUN_HYBRID = "PARALLAX_RUN_HYBRID"

# --- worker identity --------------------------------------------------------
PARALLAX_WORKER_ID = "PARALLAX_WORKER_ID"
PARALLAX_NUM_WORKERS = "PARALLAX_NUM_WORKERS"
PARALLAX_RESOURCE_INFO = "PARALLAX_RESOURCE_INFO"
PARALLAX_MACHINE_ID = "PARALLAX_MACHINE_ID"
PARALLAX_HOSTNAME = "PARALLAX_HOSTNAME"
PARALLAX_LOCAL_RANK = "PARALLAX_LOCAL_RANK"

# --- partition search -------------------------------------------------------
PARALLAX_MIN_PARTITIONS = "PARALLAX_MIN_PARTITIONS"
PARALLAX_PARTITIONS = "PARALLAX_PARTITIONS"
PARALLAX_SEARCH = "PARALLAX_SEARCH"
PARALLAX_SEARCH_ADDR = "PARALLAX_SEARCH_ADDR"
PARALLAX_SEARCH_AUTHKEY = "PARALLAX_SEARCH_AUTHKEY"    # per-job secret of the stats queue

# --- misc -------------------------------------------------------------------
PARALLAX_LOG_LEVEL = "PARALLAX_LOG_LEVEL"
PARALLAX_FABRIC = "PARALLAX_FABRIC"            # "nvlink" | "host" (tests)
PARALLAX_TIMELINE = "PARALLAX_TIMELINE"        # chrome-trace output path
PARALLAX_STALL_CHECK_TIME_SECONDS = "PARALLAX_STALL_CHECK_TIME_SECONDS"
PARALLAX_STALL_SHUTDOWN_TIME_SECONDS = "PARALLAX_STALL_SHUTDOWN_TIME_SECONDS"
PARALLAX_FUSION_THRESHOLD = "PARALLAX_FUSION_THRESHOLD"
PARALLAX_AUTOTUNE = "PARALLAX_AUTOTUNE"
PARALLAX_AUTOTUNE_LOG = "PARALLAX_AUTOTUNE_LOG"


# Horovod's knobs (`horovod/common/operations.h:33-46`) are honoured under their own names
# too, so a job script written for horovodrun keeps working: HOROVOD_X seeds PARALLAX_X.
HOROVOD_ENV_ALIASES = {
    "HOROVOD_TIMELINE": PARALLAX_TIMELINE,
    "HOROVOD_STALL_CHECK_TIME_SECONDS": PARALLAX_STALL_CHECK_TIME_SECONDS,
    "HOROVOD_STALL_SHUTDOWN_TIME_SECONDS": PARALLAX_STALL_SHUTDOWN_TIME_SECONDS,
    "HOROVOD_FUSION_THRESHOLD": PARALLAX_FUSION_THRESHOLD,
    "HOROVOD_AUTOTUNE": PARALLAX_AUTOTUNE,
    "HOROVOD_AUTOTUNE_LOG": PARALLAX_AUTOTUNE_LOG,
    "HOROVOD_CACHE_CAPACITY": "PARALLAX_CACHE_CAPACITY",
    "HOROVOD_LOG_LEVEL": PARALLAX_LOG_LEVEL,
    "HOROVOD_TIMELINE_MARK_CYCLES": "PARALLAX_TIMELINE_MARK_CYCLES",
}

# Knobs of Horovod's background loop that have no counterpart in a design with a static
# schedule (no 5 ms negotiation tick, no MPI, one NVSwitch domain): accepted, reported once.
HOROVOD_INERT_ENV = {
    "HOROVOD_CYCLE_TIME": "there is no negotiation cycle: collectives are launched from a "
                          "static per-step schedule",
    "HOROVOD_HIERARCHICAL_ALLREDUCE": "one NVSwitch domain per node: every GPU reaches every "
                                      "peer at full bandwidth, there is no intra/inter level",
    "HOROVOD_HIERARCHICAL_ALLGATHER": "one NVSwitch domain per node (see "
                                      "HOROVOD_HIERARCHICAL_ALLREDUCE)",
    "HOROVOD_MPI_THREADS_DISABLE": "no MPI in the process",
}


def adopt_horovod_env(environ=None):
    """copy HOROVOD_* settings to their PARALLAX_* names where the latter are unset;
    returns the names adopted"""
    env = os.environ if environ is None else environ
    adopted = []
    for src, dst in HOROVOD_ENV_ALIASES.items():
        if src in env and dst not in env:
            env[dst] = env[src]
            adopted.append(dst)
    return adopted


def inert_horovod_env(environ=None):
    """{name: why it changes nothing here} for the Horovod knobs that are set but have no
    effect in this design (logged once by `collectives.init` / the engine)."""
    env = os.environ if environ is None else environ
    return {k: why for k, why in HOROVOD_INERT_ENV.items() if k in env}


def _user():
    try:
        return getpass.getuser()
    except Exception:  # pragma: no cover - containers without passwd entry
        return str(os.getuid())


REMOTE_PARALLAX_ROOT = os.path.join("/tmp", "parallax-%s" % _user())

# Step window used to time a partition candidate
# (reference `common/session_context.py:28-29`).
NUM_ITERATIONS_FOR_WARMUP = 50
NUM_ITERATIONS_FOR_TEST = 100

# streaming multiprocessors of the target GPU (H100 SXM); grid sizes of the native kernels
NUM_SMS = 132
# bound on the per-CTA top-k lists of one fused full-softmax top-k launch (NUM_SMS · rows · k
# 8-byte entries); larger batches are evaluated in row chunks, each reading the table once
TOPK_WS_BYTES = 48 << 20
# digit width of the threshold search of truncated full-softmax sampling (top_k / top_p): one
# histogram pass over the table per digit of the 32-bit key, [NUM_SMS, rows, 2^d] 8-byte bins
# (EV_RADIX_BITS in ops/csrc/kernels/softmax_eval.cu, which refuses other digit positions)
SAMPLE_RADIX_BITS = 4
# bound on the chunk scratch of the fused full-softmax backward (sess_config
# ["full_softmax_train"] = "fused"): the gathered rows and the bf16 [N, Vc] softmax gradient of
# one vocabulary chunk of Vc rows
FULL_SOFTMAX_TRAIN_WS_BYTES = 256 << 20
# bound on the chunk scratch of the fused dense linear cross-entropy (`nn.linear_cross_entropy`):
# the fp32 logits and the bf16 softmax gradient of one chunk of rows, [n, V] each; a chunk never
# has fewer than 128 rows, so a vocabulary above ~350k rows may exceed it
LINEAR_XENT_WS_BYTES = 256 << 20

RUN_OPTIONS = ("PS", "MPI", "HYBRID")
# "AR" is accepted as a modern alias of the reference's "MPI" run option.
RUN_OPTION_ALIASES = {"AR": "MPI", "ALLREDUCE": "MPI"}

RUN_OPTION_TO_ENV = {
    "MPI": PARALLAX_RUN_MPI,
    "PS": PARALLAX_RUN_PS,
    "HYBRID": PARALLAX_RUN_HYBRID,
}
ENV_TO_RUN_OPTION = {v: k for k, v in RUN_OPTION_TO_ENV.items()}
