"""``python -m es_distributed.main`` -- the reference CLI (es_distributed/main.py:29-86) on the H100 engine.

  master   --algo {es,ns-es,nsr-es,ga,rs}  --exp_file / --exp_str  [--master_socket_path] [--log_dir]
  workers  --algo ... --master_host --master_port --relay_socket_path --num_workers

There is no redis: the "workers" of the reference are the GPU ranks of one torchrun job and every rank runs
``master`` (rank 0 logs).  ``workers`` is accepted for script compatibility and explains that.  Socket/host/port
options are accepted and ignored.  New optional flags: --max_iterations, --n_slots, --seed.
"""
import errno
import json
import logging
import os
import sys

import click

from dne import shard


def mkdir_p(path):
    try:
        os.makedirs(path)
    except OSError as exc:
        if exc.errno == errno.EEXIST and os.path.isdir(path):
            pass
        else:
            raise


def import_algo(name):
    """main.py:29-40."""
    if name == 'es':
        from . import es as algo
    elif name in ('ns-es', 'nsr-es'):
        from . import nses as algo
    elif name == 'ga':
        from . import ga as algo
    elif name == 'rs':
        from . import rs as algo
    else:
        raise NotImplementedError(name)
    return algo


@click.group()
def cli():
    logging.basicConfig(format='[%(asctime)s pid=%(process)d] %(message)s', level=logging.INFO, stream=sys.stderr)


@cli.command()
@click.option('--algo')
@click.option('--exp_str')
@click.option('--exp_file')
@click.option('--master_socket_path', default=None)
@click.option('--log_dir')
@click.option('--max_iterations', type=int, default=None)
@click.option('--n_slots', type=int, default=256)
@click.option('--seed', type=int, default=None)
@click.option('--allow_synthetic_env', is_flag=True, default=False,
              help='no gym/ALE/MuJoCo backend is registered in this build: run real env ids on the synthetic stand-in '
                   '(throughput only; sets exp["allow_synthetic_env"])')
def master(algo, exp_str, exp_file, master_socket_path, log_dir, max_iterations, n_slots, seed, allow_synthetic_env):
    # main.py:48-61
    assert (exp_str is None) != (exp_file is None), 'Must provide exp_str xor exp_file to the master'
    if exp_str:
        exp = json.loads(exp_str)
    else:
        with open(exp_file, 'r') as f:
            exp = json.loads(f.read())
    if allow_synthetic_env:
        exp['allow_synthetic_env'] = True
    rank, world, local = shard.init_from_env()
    log_dir = os.path.expanduser(log_dir) if log_dir else '/tmp/es_master_{}'.format(os.getpid())
    if rank == 0:
        mkdir_p(log_dir)
    algo = import_algo(algo)
    algo.run_master({'unix_socket_path': master_socket_path}, log_dir, exp, max_iterations=max_iterations,
                    n_slots=n_slots, seed=seed)


@cli.command()
@click.option('--algo')
@click.option('--master_host')
@click.option('--master_port', default=6379, type=int)
@click.option('--relay_socket_path')
@click.option('--num_workers', type=int, default=0)
def workers(algo, master_host, master_port, relay_socket_path, num_workers):
    # main.py:64-86: forks a redis relay and num_workers rollout processes sharing one noise table.
    logging.info("es_distributed (H100 engine): rollout workers are the GPU ranks of the `master` torchrun job "
                 "(population sharded over NCCL); there is no redis relay to attach to -- nothing to do.")


if __name__ == '__main__':
    cli()
