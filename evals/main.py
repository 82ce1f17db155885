"""Local multi-process launcher for the frozen evaluations, one process per device (reference: evals/main.py:19-67).

    python -m evals.main --fname configs/evals/vitl16_k400_16x8x3.yaml --devices cuda:0 cuda:1 ...
"""
import argparse
import logging
import multiprocessing as mp
import os
import pprint

import yaml

parser = argparse.ArgumentParser()
parser.add_argument('--fname', type=str, help='name of config file to load', default='configs.yaml')
parser.add_argument('--devices', type=str, nargs='+', default=['cuda:0'], help='which devices to use on local machine')


def process_main(rank, fname, world_size, devices):
    # each process sees exactly one GPU, as cuda:0
    os.environ['CUDA_VISIBLE_DEVICES'] = str(devices[rank].split(':')[-1])

    logging.basicConfig()
    logger = logging.getLogger()
    logger.setLevel(logging.INFO if rank == 0 else logging.ERROR)
    logger.info(f'called-params {fname}')

    with open(fname, 'r') as y_file:
        params = yaml.load(y_file, Loader=yaml.FullLoader)
    logger.info('loaded params...')
    pprint.PrettyPrinter(indent=4).pprint(params)

    from evals.scaffold import main as eval_main
    from src.utils.distributed import init_distributed
    world_size, rank = init_distributed(rank_and_world_size=(rank, world_size))
    logger.info(f'Running... (rank: {rank}/{world_size})')
    eval_main(params['eval_name'], args_eval=params)


if __name__ == '__main__':
    args = parser.parse_args()
    num_gpus = len(args.devices)
    mp.set_start_method('spawn')
    procs = [mp.Process(target=process_main, args=(rank, args.fname, num_gpus, args.devices)) for rank in range(num_gpus)]
    for p in procs:
        p.start()
    for p in procs:
        p.join()
