"""``[run] gpu_list`` (reference src/run.py:40-49): which GPU this process trains on, or one worker
process per listed GPU, started and supervised from the one ``python -m unflow_b200.run`` command.

* ``resolve`` reads the setting before any CUDA work and rejects a malformed one with one message.
* ``launch`` starts the workers with the environment ``torch.distributed.run`` gives its ranks, so each
  of them runs the data-parallel path that launcher drives; the rendezvous store lives in this process
  on a port the OS picks, and rank 0 joins it as a client.  It waits on all of them: when one fails,
  or this process is asked to stop, the others are stopped and every one is reaped.
"""
import ctypes
import os
import signal
import subprocess
import sys
import time

BATCH_MESSAGE = 'batch_size must be divisible by the number of GPUs'
_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def parse_gpu_list(value):
    """The ids of ``gpu_list`` as ``config_dict`` types it: ``3`` is an int, ``0,1`` or ``0, 1`` a str.
    ValueError for anything that is not a list of distinct non-negative integers."""
    if isinstance(value, bool) or not isinstance(value, (int, str)):
        raise ValueError('expected a GPU id or a comma-separated list of GPU ids')
    ids = []
    for item in str(value).split(','):
        try:
            ids.append(int(item.strip()))
        except ValueError:
            raise ValueError('%r is not an integer GPU id' % item.strip()) from None
    if any(i < 0 for i in ids):
        raise ValueError('GPU ids cannot be negative')
    if len(set(ids)) != len(ids):
        raise ValueError('GPU ids must be distinct')
    return ids


def resolve(run_config, device_count, environ=None):
    """What ``[run] gpu_list`` asks of this process, given ``device_count`` visible devices:

    * None -- no ``gpu_list``, or the process was started by a launcher (``WORLD_SIZE`` is set): train
      where ``LOCAL_RANK`` says, as the launcher arranged.  If the launcher's world size differs from the
      number of listed ids, rank 0 says that the launcher wins;
    * ``[k]`` -- train in this process on device k;
    * ``[k0, k1, ...]`` -- one worker per listed device (``launch``), ``batch_size / n`` pairs each.

    A malformed list, an id not below ``device_count`` or a ``batch_size`` the number of ids does not
    divide ends the command (SystemExit) with one message."""
    environ = os.environ if environ is None else environ
    if 'gpu_list' not in run_config:
        return None
    value = run_config['gpu_list']
    if 'WORLD_SIZE' in environ:
        world = int(environ['WORLD_SIZE'])
        listed = len(str(value).split(','))
        if listed != world and int(environ.get('RANK', '0')) == 0:
            print('-- gpu_list names %d GPU(s), the launcher started %d processes: the launcher\'s '
                  'world size is used' % (listed, world))
        return None
    try:
        ids = parse_gpu_list(value)
    except ValueError as e:
        raise SystemExit('[run] gpu_list = %s: %s' % (value, e))
    beyond = [i for i in ids if i >= device_count]
    if beyond:
        raise SystemExit('[run] gpu_list = %s: GPU %d does not exist (%d visible)'
                         % (value, beyond[0], device_count))
    if run_config['batch_size'] % len(ids) != 0:
        raise SystemExit('%s ([run] batch_size = %s, gpu_list = %s)'
                         % (BATCH_MESSAGE, run_config['batch_size'], value))
    return ids


def worker_env(rank, gpu_ids, port, environ=None):
    """The environment of worker ``rank``: what ``torch.distributed.run`` sets for a local rank, with
    ``CUDA_VISIBLE_DEVICES`` narrowed to the listed devices in the listed order, so that worker k's
    ``cuda:k`` is the k-th listed GPU and every worker sees all of them (NCCL keeps its peer paths).
    Ids index the devices this process sees: an inherited ``CUDA_VISIBLE_DEVICES`` is mapped through."""
    env = dict(os.environ if environ is None else environ)
    visible = env.get('CUDA_VISIBLE_DEVICES')
    visible = [v.strip() for v in visible.split(',')] if visible else None
    n = len(gpu_ids)
    env.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(n), LOCAL_WORLD_SIZE=str(n),
               MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port),
               CUDA_VISIBLE_DEVICES=','.join(visible[i] if visible else str(i) for i in gpu_ids),
               # the store is this process's: every rank, rank 0 included, connects as a client
               TORCHELASTIC_USE_AGENT_STORE='True',
               PYTHONPATH=os.pathsep.join(p for p in (_ROOT, env.get('PYTHONPATH')) if p))
    return env


def _die_with_parent(parent):
    """preexec_fn of a worker: the kernel kills it when the launcher dies, however that happens (an
    orphaned rank would otherwise wait in its next NCCL collective)."""
    if not sys.platform.startswith('linux'):
        return None
    libc = ctypes.CDLL(None, use_errno=True)
    PR_SET_PDEATHSIG = 1

    def preexec():
        libc.prctl(PR_SET_PDEATHSIG, signal.SIGKILL)
        if os.getppid() != parent:      # the launcher died before the line above
            os._exit(1)
    return preexec


def _stop(procs, sig, grace):
    """Send ``sig`` to the workers still running, SIGKILL those left after ``grace`` seconds, reap all."""
    for p in procs:
        if p.poll() is None:
            try:
                p.send_signal(sig)
            except ProcessLookupError:
                pass
    deadline = time.monotonic() + grace
    for p in procs:
        try:
            p.wait(timeout=max(deadline - time.monotonic(), 0))
        except subprocess.TimeoutExpired:
            p.kill()
            p.wait()


def _exit_code(returncode):
    return returncode if returncode >= 0 else 128 - returncode     # killed by signal s: 128 + s


def launch(argv, gpu_ids, cmd=None, grace=5.0, poll=0.1):
    """Run ``python -m unflow_b200.run <argv>`` once per id of ``gpu_ids`` (``cmd`` replaces that
    command) and wait for all of them.  Returns 0 when every worker exits 0; otherwise the first failing
    worker's exit code, after stopping the others (SIGTERM, then SIGKILL after ``grace`` seconds).
    SIGINT / SIGTERM received here are passed on to the workers, with the same reaping, and the return
    value is 128 + the signal number."""
    from torch.distributed import TCPStore
    if cmd is None:
        cmd = [sys.executable] + subprocess._args_from_interpreter_flags() + ['-m', 'unflow_b200.run'] + list(argv)
    # port 0: the OS picks a free port, so concurrent runs on one machine never collide
    store = TCPStore('127.0.0.1', 0, len(gpu_ids), is_master=True, wait_for_workers=False)
    received = []
    handlers = {}
    try:
        for s in (signal.SIGINT, signal.SIGTERM):
            handlers[s] = signal.signal(s, lambda signum, frame: received.append(signum))
    except ValueError:      # not the main thread: signals stay with the caller
        pass
    procs = []
    failed = None
    try:
        for rank in range(len(gpu_ids)):
            procs.append(subprocess.Popen(cmd, env=worker_env(rank, gpu_ids, store.port),
                                          preexec_fn=_die_with_parent(os.getpid())))
        while not received:
            codes = [p.poll() for p in procs]
            failed = next((r for r, c in enumerate(codes) if c not in (None, 0)), None)
            if failed is not None or all(c == 0 for c in codes):
                break
            time.sleep(poll)
    finally:
        _stop(procs, received[0] if received else signal.SIGTERM, grace)
        for s, h in handlers.items():
            signal.signal(s, h)
        del store
    if received:
        print('unflow_b200.run: stopped the workers on signal %d' % received[0], file=sys.stderr)
        return 128 + received[0]
    if failed is not None:
        code = _exit_code(procs[failed].returncode)
        print('unflow_b200.run: rank %d (GPU %d) exited with code %d; the other workers were stopped'
              % (failed, gpu_ids[failed], code), file=sys.stderr)
        return code
    return 0
