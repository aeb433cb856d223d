"""[run] gpu_list (reference src/run.py:40-49) on the CPU: how it resolves, what the one-command launch
gives each worker, and how the workers are supervised -- with stub children, no CUDA."""
import json
import os
import signal
import subprocess
import sys
import textwrap
import time

import pytest
import torch

from unflow_b200 import launch
from unflow_b200 import run as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def _all_devices_visible(monkeypatch):
    """The stub launches list ids that no device backs; an inherited CUDA_VISIBLE_DEVICES would map them."""
    monkeypatch.delenv('CUDA_VISIBLE_DEVICES', raising=False)


def _alive(pid):
    """True while ``pid`` runs (a zombie no one has reaped yet counts as gone)."""
    try:
        with open('/proc/%d/stat' % pid) as fh:
            return fh.read().rsplit(')', 1)[1].split()[0] != 'Z'
    except FileNotFoundError:
        return False


def _wait_for(paths, timeout=60.0):
    end = time.monotonic() + timeout
    while not all(os.path.exists(p) for p in paths):
        assert time.monotonic() < end, 'stub children did not start'
        time.sleep(0.05)


def _stub(body):
    return [sys.executable, '-c', textwrap.dedent(body)]


# --------------------------------------------------------------------------------------------
# resolution
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize('value, ids', [(0, [0]), (3, [3]), ('0,1', [0, 1]), ('2, 3', [2, 3]),
                                        ('3,0,1', [3, 0, 1])])
def test_resolve(value, ids):
    assert launch.resolve(dict(batch_size=12, gpu_list=value), 4, environ={}) == ids


def test_resolve_without_key_keeps_local_rank():
    assert launch.resolve(dict(batch_size=4), 4, environ={}) is None


@pytest.mark.parametrize('value, batch, message', [
    ('0,0', 4, 'distinct'), ('1, 1', 4, 'distinct'), (-1, 4, 'negative'), ('0,-2', 4, 'negative'),
    ('0,a', 4, 'integer'), (0.5, 4, 'GPU id'), (True, 4, 'GPU id'), ('', 4, 'integer'),
    (4, 4, 'GPU 4 does not exist'), ('0,7', 4, 'GPU 7 does not exist'),
    ('0,1,2', 4, launch.BATCH_MESSAGE)])
def test_resolve_rejects(value, batch, message):
    with pytest.raises(SystemExit, match=message):
        launch.resolve(dict(batch_size=batch, gpu_list=value), 4, environ={})


def test_external_launcher_wins(capsys):
    env = dict(WORLD_SIZE='2', RANK='0', LOCAL_RANK='0')
    assert launch.resolve(dict(batch_size=4, gpu_list='0,1'), 8, environ=env) is None
    assert capsys.readouterr().out == ''
    # a count that differs is noted once, by rank 0, and nothing is rejected
    assert launch.resolve(dict(batch_size=4, gpu_list='0,1,2,3'), 8, environ=env) is None
    assert "launcher's world size is used" in capsys.readouterr().out
    env['RANK'] = '1'
    assert launch.resolve(dict(batch_size=4, gpu_list=0), 8, environ=env) is None
    assert capsys.readouterr().out == ''


CFG = """
[dirs]
log = {d}/log
[run]
batch_size = {batch}
{gpu_list}
[train]
save_interval = 2
"""


class _Stop(Exception):
    pass


@pytest.fixture
def fake_cuda(monkeypatch):
    """run.main as far as it goes without a device: four visible GPUs, ``set_device`` stops the run (it
    is where training on this process begins) and ``launch.launch`` records its arguments."""
    calls = []
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: True)
    monkeypatch.setattr(torch.cuda, 'device_count', lambda: 4)

    def set_device(d):
        raise _Stop(d)

    def fake_launch(argv, gpu_ids):
        calls.append((list(argv), list(gpu_ids)))
        return 0
    monkeypatch.setattr(torch.cuda, 'set_device', set_device)
    monkeypatch.setattr(launch, 'launch', fake_launch)
    for k in ('WORLD_SIZE', 'RANK', 'LOCAL_RANK'):
        monkeypatch.delenv(k, raising=False)
    return calls


def _main(tmp_path, gpu_list, batch=4):
    ini = tmp_path / 'config.ini'
    ini.write_text(CFG.format(d=tmp_path, batch=batch, gpu_list=gpu_list))
    argv = ['--ex', 'x', '--config', str(ini), '--synthetic']
    return argv, lambda: R.main(argv)


def test_main_launches_workers_without_touching_a_device(tmp_path, fake_cuda):
    argv, main = _main(tmp_path, 'gpu_list = 2, 3')
    main()
    assert fake_cuda == [(argv, [2, 3])]
    assert not (tmp_path / 'log').exists()      # rank 0 writes the experiment, not the launcher


@pytest.mark.parametrize('gpu_list, device', [('gpu_list = 0', 0), ('gpu_list = 3', 3), ('', 0)])
def test_main_single_gpu_trains_in_process(tmp_path, fake_cuda, gpu_list, device):
    _, main = _main(tmp_path, gpu_list)
    with pytest.raises(_Stop) as stop:
        main()
    assert stop.value.args == (device,) and fake_cuda == []


def test_main_under_external_launcher_spawns_nothing(tmp_path, fake_cuda, monkeypatch):
    monkeypatch.setenv('WORLD_SIZE', '2')
    monkeypatch.setenv('RANK', '1')
    monkeypatch.setenv('LOCAL_RANK', '1')
    _, main = _main(tmp_path, 'gpu_list = 0,1')
    with pytest.raises(_Stop) as stop:
        main()
    assert stop.value.args == (1,) and fake_cuda == []


@pytest.mark.parametrize('gpu_list, batch', [('gpu_list = 0,0', 4), ('gpu_list = 0,-1', 4),
                                             ('gpu_list = 0,4', 4), ('gpu_list = 0,1,2', 4)])
def test_main_rejects_before_anything_starts(tmp_path, fake_cuda, gpu_list, batch):
    _, main = _main(tmp_path, gpu_list, batch)
    with pytest.raises(SystemExit):
        main()
    assert fake_cuda == [] and not (tmp_path / 'log').exists()


def test_main_keeps_the_batch_message(tmp_path, fake_cuda):
    _, main = _main(tmp_path, 'gpu_list = 0,1,2', batch=4)
    with pytest.raises(SystemExit, match='batch_size must be divisible by the number of GPUs'):
        main()


# --------------------------------------------------------------------------------------------
# the workers' environment
# --------------------------------------------------------------------------------------------
def test_worker_env():
    envs = [launch.worker_env(k, [2, 3], 41234) for k in (0, 1)]
    for k, env in enumerate(envs):
        assert (env['RANK'], env['LOCAL_RANK'], env['WORLD_SIZE'], env['LOCAL_WORLD_SIZE']) == (str(k), str(k), '2', '2')
        assert (env['MASTER_ADDR'], env['MASTER_PORT'], env['CUDA_VISIBLE_DEVICES']) == ('127.0.0.1', '41234', '2,3')
        assert env['PYTHONPATH'].split(os.pathsep)[0] == ROOT
    # ids count the devices this process sees: an inherited CUDA_VISIBLE_DEVICES maps them
    env = launch.worker_env(0, [1, 3], 1, environ={'CUDA_VISIBLE_DEVICES': '4,5,6,7'})
    assert env['CUDA_VISIBLE_DEVICES'] == '5,7'


def test_launch_gives_each_worker_its_rank_and_a_free_port(tmp_path):
    cmd = _stub("""
        import json, os, sys
        keys = ('RANK', 'LOCAL_RANK', 'WORLD_SIZE', 'LOCAL_WORLD_SIZE', 'MASTER_ADDR', 'MASTER_PORT',
                'CUDA_VISIBLE_DEVICES')
        json.dump({k: os.environ[k] for k in keys}, open(os.path.join(%r, os.environ['RANK']), 'w'))
    """ % str(tmp_path))
    ports = []
    for _ in range(2):
        assert launch.launch([], [1, 0], cmd=cmd) == 0
        envs = [json.load(open(tmp_path / str(k))) for k in (0, 1)]
        assert [e['LOCAL_RANK'] for e in envs] == ['0', '1'] and {e['WORLD_SIZE'] for e in envs} == {'2'}
        assert {e['CUDA_VISIBLE_DEVICES'] for e in envs} == {'1,0'}
        assert len({e['MASTER_PORT'] for e in envs}) == 1
        ports.append(int(envs[0]['MASTER_PORT']))
    assert all(0 < p < 65536 and p != 29500 for p in ports)


def test_workers_rendezvous_on_the_launchers_store(tmp_path):
    """The env:// rendezvous every worker performs (gloo here, NCCL in training) finds the store."""
    out = tmp_path / 'sum'
    cmd = _stub("""
        import torch, torch.distributed as dist
        dist.init_process_group('gloo')
        t = torch.tensor([float(dist.get_rank() + 1)])
        dist.all_reduce(t)
        if dist.get_rank() == 0:
            open(%r, 'w').write(str(float(t)))
        dist.destroy_process_group()
    """ % str(out))
    assert launch.launch([], [0, 1, 2], cmd=cmd) == 0
    assert out.read_text() == '6.0'


# --------------------------------------------------------------------------------------------
# supervision
# --------------------------------------------------------------------------------------------
def test_all_workers_succeed():
    assert launch.launch([], [0, 1], cmd=_stub("pass")) == 0


def test_os_exit_zero_is_success():
    # --graph workers leave through os._exit(0)
    assert launch.launch([], [0, 1], cmd=_stub("import os, sys; sys.stdout.flush(); os._exit(0)")) == 0


def test_failing_worker_stops_the_others(tmp_path, capsys):
    cmd = _stub("""
        import os, sys, time
        d, r = %r, os.environ['RANK']
        open(os.path.join(d, 'pid' + r), 'w').write(str(os.getpid()))
        if r == '1':
            while not os.path.exists(os.path.join(d, 'pid0')):
                time.sleep(0.02)
            sys.exit(3)
        time.sleep(120)
    """ % str(tmp_path))
    t0 = time.monotonic()
    assert launch.launch([], [4, 5], cmd=cmd) == 3
    assert time.monotonic() - t0 < 20
    assert 'rank 1 (GPU 5) exited with code 3' in capsys.readouterr().err
    assert not _alive(int((tmp_path / 'pid0').read_text()))


def test_worker_ignoring_sigterm_is_killed(tmp_path):
    cmd = _stub("""
        import os, signal, sys, time
        d, r = %r, os.environ['RANK']
        signal.signal(signal.SIGTERM, signal.SIG_IGN)
        open(os.path.join(d, 'pid' + r), 'w').write(str(os.getpid()))
        if r == '0':
            while not os.path.exists(os.path.join(d, 'pid1')):
                time.sleep(0.02)
            sys.exit(2)
        time.sleep(120)
    """ % str(tmp_path))
    assert launch.launch([], [0, 1], cmd=cmd, grace=0.5) == 2
    assert not _alive(int((tmp_path / 'pid1').read_text()))


SLEEPERS = """
    import os, time
    open(os.path.join(%r, 'pid' + os.environ['RANK']), 'w').write(str(os.getpid()))
    time.sleep(120)
"""


def _launcher(tmp_path):
    """A launcher process running two sleeping stub workers; returns it and the workers' pids."""
    code = ("import sys; sys.path.insert(0, %r); from unflow_b200 import launch; "
            "sys.exit(launch.launch([], [0, 1], cmd=%r))" % (ROOT, _stub(SLEEPERS % str(tmp_path))))
    p = subprocess.Popen([sys.executable, '-c', code], stderr=subprocess.PIPE, text=True)
    pid_files = [str(tmp_path / ('pid%d' % k)) for k in (0, 1)]
    try:
        _wait_for(pid_files)
    except AssertionError:
        p.kill()
        p.wait()
        raise
    return p, [int(open(f).read()) for f in pid_files]


@pytest.mark.parametrize('sig', [signal.SIGTERM, signal.SIGINT])
def test_signal_to_the_launcher_reaps_every_worker(tmp_path, sig):
    p, pids = _launcher(tmp_path)
    p.send_signal(sig)
    _, err = p.communicate(timeout=30)
    assert p.returncode == 128 + sig and 'stopped the workers on signal %d' % sig in err
    assert not any(_alive(pid) for pid in pids)


@pytest.mark.skipif(not sys.platform.startswith('linux'), reason='PR_SET_PDEATHSIG is Linux only')
def test_workers_die_with_a_killed_launcher(tmp_path):
    p, pids = _launcher(tmp_path)
    p.kill()
    p.wait()
    end = time.monotonic() + 10
    while any(_alive(pid) for pid in pids) and time.monotonic() < end:
        time.sleep(0.05)
    assert not any(_alive(pid) for pid in pids)
