"""Master-side process launching.

Parity: reference `common/lib.py:70-98` (`remote_copy`, `remote_exec`: ssh
with exported env), `mpi/runner.py:36-131` (mpirun, one process per GPU),
`ps/runner.py:84-193` and `hybrid/runner.py:89-139` (ssh worker/PS launch,
redirect files ``log_worker<i>_{stdout,stderr}`` — `ps/runner.py:34-46`,
SIGINT kills all process groups `:186-192`).

Design: every run option uses the same shape — one worker process per
GPU re-executing the user's script, rendezvousing through `torch.distributed`
(MASTER_ADDR = first host).  There are no separate parameter-server
processes: a variable's "server" is the GPU that owns it.  Local workers are
plain subprocesses; workers on other hosts are started over ssh.
"""
import os
import shlex
import signal
import subprocess
import sys

from . import consts
from .log import parallax_log
from .resource import (is_local_host, routable_address, serialize_resource_info,
                       worker_layout,
                       get_empty_port)


def remote_copy(remote_machine, local_path, remote_path, port=22):
    """scp a file to `remote_machine` (reference `common/lib.py:70-76`)."""
    cmd = ["scp", "-P", str(port), local_path, "%s:%s" % (remote_machine, remote_path)]
    parallax_log.warning("\033[91m%s\033[0m", " ".join(cmd))
    return subprocess.call(cmd)


def remote_command(bash_script, remote_machine, env=None, python_venv=None, port=22,
                   secret_names=()):
    """The ssh argv for `remote_exec`.  Variables named in `secret_names` are NOT put on
    the command line (visible in `ps` on both machines): the remote shell reads them from
    stdin, one line each, with terminal echo off."""
    full = ""
    for k in secret_names:
        full += "stty -echo 2>/dev/null; IFS= read -r %s; stty echo 2>/dev/null; export %s; " \
            % (k, k)
    if env:
        full += " ".join("export %s=%s;" % (k, shlex.quote(str(v)))
                         for k, v in env.items() if k not in secret_names)
    if python_venv:
        full += " source %s/bin/activate;" % python_venv
    full += " " + bash_script
    return ["ssh", "-tt", "-p", str(port), remote_machine, "bash -c %s" % shlex.quote(full)]


def remote_exec(bash_script, remote_machine, stdout=None, stderr=None,
                env=None, python_venv=None, port=22, secret_names=()):
    """Run `bash_script` on `remote_machine` over ssh with `env` exported."""
    secret_names = [k for k in secret_names if env and k in env]
    cmd = remote_command(bash_script, remote_machine, env, python_venv, port, secret_names)
    parallax_log.warning("\033[91m%s\033[0m", " ".join(cmd))
    p = subprocess.Popen(cmd, stdout=stdout, stderr=stderr, preexec_fn=os.setsid,
                         stdin=subprocess.PIPE if secret_names else None)
    if secret_names:
        p.stdin.write(("".join("%s\n" % env[k] for k in secret_names)).encode())
        p.stdin.flush()
    return p


SECRET_ENV = (consts.PARALLAX_SEARCH_AUTHKEY,)


def _redirect(redirect_path, role, idx):
    if not redirect_path:
        return None, None
    os.makedirs(redirect_path, exist_ok=True)
    out = open(os.path.join(redirect_path, "log_%s%d_stdout" % (role, idx)), "w")
    err = open(os.path.join(redirect_path, "log_%s%d_stderr" % (role, idx)), "w")
    return out, err


def launch_workers(run_option, resource_info, config, extra_env=None,
                   argv=None):
    """Start one worker process per GPU.  Returns the list of Popen objects
    (chief first)."""
    argv = list(sys.argv if argv is None else argv)
    layout = worker_layout(resource_info)
    world = len(layout)
    master_host = resource_info["master"][0]["hostname"]
    # loopback only when EVERY worker runs on this machine; a worker started over ssh on
    # another host must be told an address it can actually reach
    everything_local = all(is_local_host(h) for h, _, _, _ in layout)
    master_addr = "127.0.0.1" if (everything_local and is_local_host(master_host)) \
        else routable_address(master_host)
    master_port = resource_info["master"][0]["port"][0] \
        if resource_info["master"][0]["port"] else get_empty_port(1)[0]
    serialized = serialize_resource_info(resource_info)
    mpi_env = config.communication_config.mpi_config.exported_env()
    procs = []
    for wid, (host, mid, lrank, gpu) in enumerate(layout):
        env = {
            consts.PARALLAX_RUN_OPTION: consts.RUN_OPTION_TO_ENV[run_option],
            consts.PARALLAX_RESOURCE_INFO: serialized,
            consts.PARALLAX_WORKER_ID: wid,
            consts.PARALLAX_NUM_WORKERS: world,
            consts.PARALLAX_MACHINE_ID: mid,
            consts.PARALLAX_HOSTNAME: host,
            consts.PARALLAX_LOCAL_RANK: lrank,
            "RANK": wid, "WORLD_SIZE": world,
            "LOCAL_RANK": gpu if gpu is not None else lrank,
            "MASTER_ADDR": master_addr, "MASTER_PORT": master_port,
        }
        env.update(mpi_env)
        if extra_env:
            env.update(extra_env)
        out, err = _redirect(config.redirect_path, "worker", wid)
        if is_local_host(host):
            penv = dict(os.environ)
            penv.update({k: str(v) for k, v in env.items()})
            cmd = [sys.executable] + argv
            parallax_log.debug("launch worker %d: %s", wid, " ".join(cmd))
            p = subprocess.Popen(cmd, env=penv, stdout=out, stderr=err,
                                 preexec_fn=os.setsid)
        else:
            for k in (consts.PARALLAX_LOG_LEVEL, consts.PARALLAX_MIN_PARTITIONS):
                if k in os.environ:
                    env.setdefault(k, os.environ[k])
            script = "cd %s; %s %s" % (
                shlex.quote(os.getcwd()), shlex.quote(sys.executable),
                " ".join(shlex.quote(a) for a in argv))
            p = remote_exec(script, host, stdout=out, stderr=err, env=env,
                            python_venv=os.environ.get("VIRTUAL_ENV"),
                            secret_names=SECRET_ENV)
        procs.append(p)
    return procs


def kill_all(procs):
    for p in procs:
        if p.poll() is None:
            try:
                os.killpg(os.getpgid(p.pid), signal.SIGTERM)
            except Exception:
                try:
                    p.terminate()
                except Exception:  # pragma: no cover
                    pass
    for p in procs:
        try:
            p.wait(timeout=10)
        except Exception:
            try:
                os.killpg(os.getpgid(p.pid), signal.SIGKILL)
            except Exception:  # pragma: no cover
                pass


def wait_all(procs, poll_secs=0.2):
    """Wait for every worker; if one fails, kill the rest.  Returns the exit
    code (0 iff all succeeded)."""
    import time
    while True:
        alive = False
        for p in procs:
            rc = p.poll()
            if rc is None:
                alive = True
            elif rc != 0:
                parallax_log.error("worker pid %d exited with %d; stopping job",
                                   p.pid, rc)
                kill_all(procs)
                return rc
        if not alive:
            return 0
        time.sleep(poll_secs)
