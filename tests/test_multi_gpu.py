"""Multi-GPU parity (SURVEY.md 4 "distributed" row, 8e): an N-rank run (crops sharded, one all-reduce of dRGB) must reproduce the
1-rank run on the same seeds -- loss, d loss / d spectrum and the spectrum after two Adam steps. Needs >= 2 GPUs
(`python -m pytest tests/test_multi_gpu.py -m gpu` on a machine with N GPUs); skipped on a one-GPU machine.

Tolerances. A rank's loss is the mean over ITS crops, so its backward runs with gradients S/S_local times larger than the 1-rank
run's and is rescaled afterwards. With EVEN shards and a power-of-two rank count that factor is a power of two: every bf16
rounding inside the ViT backward is unchanged and only the order of the fp32 atomics / of the all-reduce differs (SURVEY 7.3) ->
norm-wise 2e-5. With UNEVEN shards (BASELINE configs[3]: S=87 over 4 ranks = 22/22/22/21; configs[4]: 190 over 8) the factor is
not a power of two, the bf16 roundings of the intermediate gradients fall differently (measured 2.5e-3), and the bound is the bf16
bar of the path (1e-2; each run is within 8e-3 of the fp32 oracle)."""
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, 'tests', 'multi_gpu_worker.py')
NGPU = torch.cuda.device_count() if torch.cuda.is_available() else 0


def _port():
    s = socket.socket(); s.bind(('127.0.0.1', 0)); p = s.getsockname()[1]; s.close(); return p


def _run(world, out, args, env_add=None):
    if world == 1:
        cmd = [sys.executable, WORKER, out] + args
    else:
        cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', str(world), '--master-addr', '127.0.0.1',
               '--master-port', str(_port()), WORKER, out] + args
    env = {k: v for k, v in os.environ.items() if k not in ('RANK', 'WORLD_SIZE', 'LOCAL_RANK')}
    env.update(env_add or {})
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    return torch.load(out)


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.mark.skipif(NGPU < 2, reason='needs at least 2 GPUs')
@pytest.mark.parametrize('mode', ['sym', 'nccl'])
@pytest.mark.parametrize('world,H,W,S,patch,sim', [(2, 360, 640, 24, 32, 'mix'), (2, 360, 640, 23, 32, 'mix'), (4, 720, 1280, 88, 16, 'cossim'), (4, 720, 1280, 87, 16, 'cossim'),
                                                   (8, 720, 1280, 192, 32, 'mix'), (8, 720, 1280, 190, 32, 'mix')])
def test_n_rank_equals_one_rank(tmp_path, world, H, W, S, patch, sim, mode):
    """mode 'sym': our own NVLS / peer-memory all-reduce kernel over symmetric memory (csrc/comm.cu); 'nccl': dist.all_reduce."""
    if NGPU < world:
        pytest.skip('needs %d GPUs' % world)
    args = [str(H), str(W), str(S), str(patch), sim]
    one = _run(1, str(tmp_path / 'one.pt'), args)
    many = _run(world, str(tmp_path / 'many.pt'), args, {'APH_COLLECTIVE': mode})
    assert many['collective'] == 'nccl' if mode == 'nccl' else many['collective'] in ('nvls', 'p2p', 'nccl')
    assert many['world'] == world and one['world'] == 1
    base, rem = divmod(S, world)
    assert many['local_crops'] == base + (1 if rem > 0 else 0)                       # rank 0 holds the larger shard
    # step 0 must agree to fp32 round-off; after one Adam step (beta1 = 0: every element moves by ~lr * sign(g)) elements whose gradient
    # is at round-off level may move the other way, so the second loss is only required to stay close
    assert abs(many['loss'][0] - one['loss'][0]) < 1e-5 and abs(many['loss'][1] - one['loss'][1]) < 3e-3
    e_g, e_p = _rel(many['grad'], one['grad']), _rel(many['params'], one['params'])
    print('world %d S=%d (%s exchange): rel err grad %.3e params-after-2-steps %.3e' % (world, S, many['collective'], e_g, e_p))
    even = S % world == 0
    assert e_g < (2e-5 if even else 1e-2)
    assert e_p < (2e-2 if even else 0.5)          # Adam with beta1 = 0 moves every element by ~lr*sign(g): elements whose gradient is at round-off level may flip
