"""Python-3 twin of the reference's training driver (scripts/train_nats.py): same `main(job_id, params)` entry, same
hyper-parameter dictionary and the same fixed settings (maxlen=500, batch 20, frequencies 10, dispFreq 1); the data
location is an argument instead of a hard-coded /disk1/$USER path.

    python -m nats_b200.train_nats --data-dir DATA --model models/model.npz [--dim 600 ...]
    python -m nats_b200.train_nats ... --reload --rl-weight 0.9      # self-critical fine-tuning of an ML model
    torchrun --nproc-per-node 8 -m nats_b200.train_nats ...      # data-parallel: each rank takes its shard of a batch
"""
import argparse
import os

from .nats import train


def main(job_id, params):
    print(params)
    data = params['data-dir'][0]
    j = lambda name: os.path.join(data, name)
    validerr = train(saveto=params['model'][0],
                     reload_=params['reload'][0],
                     dim_word=params['dim_word'][0],
                     dim=params['dim'][0],
                     dim_att=params['dim_att'][0],
                     patience=params['patience'][0],
                     n_words=params['n-words'][0],
                     decay_c=params['decay-c'][0],
                     clip_c=params['clip-c'][0],
                     lrate=params['learning-rate'][0],
                     optimizer=params['optimizer'][0],
                     maxlen=500,
                     batch_size=params.get('batch-size', [20])[0],
                     valid_batch_size=params.get('batch-size', [20])[0],
                     datasets=[j(params['train'][0]), j(params['train'][1])],
                     valid_datasets=[j(params['valid'][0]), j(params['valid'][1])],
                     dictionary=j(params['dictionary'][0]),
                     validFreq=10,
                     dispFreq=1,
                     saveFreq=10,
                     sampleFreq=10,
                     use_dropout=params['use-dropout'][0],
                     rl_weight=params.get('rl-weight', [0.])[0],
                     rl_samples=params.get('rl-samples', [4])[0],
                     rl_maxlen=params.get('rl-maxlen', [100])[0],
                     rl_seed=params.get('rl-seed', [1234])[0],
                     **({'finish_after': params['finish-after'][0]} if 'finish-after' in params else {}))
    return validerr


def _args():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--data-dir', required=True)
    ap.add_argument('--model', required=True)
    ap.add_argument('--train', nargs=2, default=['toy_train_input.txt', 'toy_train_output.txt'])
    ap.add_argument('--valid', nargs=2, default=['toy_validation_input.txt', 'toy_validation_output.txt'])
    ap.add_argument('--dictionary', default='toy_train_input.txt.pkl')
    ap.add_argument('--dim-word', type=int, default=120)
    ap.add_argument('--dim', type=int, default=600)
    ap.add_argument('--dim-att', type=int, default=100)
    ap.add_argument('--n-words', type=int, default=25000)
    ap.add_argument('--patience', type=int, default=1)
    ap.add_argument('--optimizer', default='adadelta')
    ap.add_argument('--decay-c', type=float, default=0.)
    ap.add_argument('--clip-c', type=float, default=100.)
    ap.add_argument('--learning-rate', type=float, default=0.0001)
    ap.add_argument('--batch-size', type=int, default=20)
    ap.add_argument('--finish-after', type=int, default=None)
    ap.add_argument('--reload', action='store_true')
    ap.add_argument('--rl-weight', type=float, default=0.,
                    help='gamma in [0, 1]: self-critical training on the ROUGE-L of sampled summaries (0 = off)')
    ap.add_argument('--rl-samples', type=int, default=4, help='samples per source of a self-critical update')
    ap.add_argument('--rl-maxlen', type=int, default=100, help='longest sampled summary (<= 499)')
    ap.add_argument('--rl-seed', type=int, default=1234, help='seed of the self-critical samples')
    return ap.parse_args()


if __name__ == '__main__':
    a = _args()
    if int(os.environ.get('WORLD_SIZE', '1')) > 1:
        import torch
        torch.cuda.set_device(int(os.environ.get('LOCAL_RANK', '0')))
        torch.distributed.init_process_group('nccl')
    p = {'data-dir': [a.data_dir], 'model': [a.model], 'train': a.train, 'valid': a.valid, 'dictionary': [a.dictionary],
         'dim_word': [a.dim_word], 'dim': [a.dim], 'dim_att': [a.dim_att], 'n-words': [a.n_words],
         'patience': [a.patience], 'optimizer': [a.optimizer], 'decay-c': [a.decay_c], 'clip-c': [a.clip_c],
         'use-dropout': [False], 'learning-rate': [a.learning_rate], 'reload': [a.reload], 'batch-size': [a.batch_size],
         'rl-weight': [a.rl_weight], 'rl-samples': [a.rl_samples], 'rl-maxlen': [a.rl_maxlen], 'rl-seed': [a.rl_seed]}
    if a.finish_after is not None:
        p['finish-after'] = [a.finish_after]
    main(0, p)
