#!/usr/bin/env python
"""Command-line driver with the interface of the reference's run.py (hidasib/GRU4Rec run.py:10-133): same flags, same
parameter-file / parameter-string formats, same printed lines (paropt.py parses `PRIMARY METRIC:`).  The model class comes
in through the reference's plugin seam `-g GRFILE` (default: the root-level `gru4rec` module = the CUDA implementation)."""
import argparse
import importlib
import importlib.util
import os
import sys
import time
from collections import OrderedDict

# (flags, keyword arguments) of every command-line option; names, defaults and choices follow run.py:11-26
_TIE_MODES = ['standard', 'conservative', 'median', 'tiebreaking']
_OPTIONS = [
    (('path',), dict(metavar='PATH', type=str,
                     help='Training data (TAB separated .tsv/.txt or pickled DataFrame .pickle), or the serialized model when --load_model is given.')),
    (('-ps', '--parameter_string'), dict(metavar='PARAM_STRING', type=str,
                                         help='Training parameters as `name1=value1,name2=value2`; booleans True/False; lists use / (e.g. layers=200/200). Exclusive with -pf and -l.')),
    (('-pf', '--parameter_file'), dict(metavar='PARAM_PATH', type=str,
                                       help='Python file defining an OrderedDict named `gru4rec_params`. Exclusive with -ps and -l.')),
    (('-l', '--load_model'), dict(action='store_true', help='Load a trained model from PATH instead of training. Exclusive with -ps and -pf.')),
    (('-s', '--save_model'), dict(metavar='MODEL_PATH', type=str, help='Save the trained model to MODEL_PATH.')),
    (('--load_checkpoint',), dict(metavar='CKPT_PATH', type=str, help='Load the model, with its optimizer and training state, from a checkpoint written by --save_checkpoint. Exclusive with -ps, -pf and -l.')),
    (('--save_checkpoint',), dict(metavar='CKPT_PATH', type=str, help='Save the model with its optimizer and training state to CKPT_PATH (.npz), so that a later run can train it further.')),
    (('--fit_more',), dict(action='store_true', help='With --load_checkpoint: continue training the loaded model on the training data PATH (new items are added to the catalogue) instead of building a new model.')),
    (('--baseline',), dict(metavar='NAME', choices=['pop', 'sessionpop', 'itemknn', 'bpr', 'sknn', 'stan', 'vstan', 'sr', 'ar', 'narm', 'sasrec', 'srgnn', 'stamp', 'nextitnet', 'bert4rec'], help='Fit a session baseline (Pop, SessionPop, ItemKNN or BPR of the reference, sknn: session-based kNN, S-KNN / V-SKNN, stan: session kNN with STAN-style time and position decays, vstan: STAN with VSTAN-style vector similarity, neighbour weights and IDF, sr: sequential rules, ar: association rules, narm: the NARM neural session model, sasrec: the SASRec self-attentive model, srgnn: the SR-GNN session-graph model, stamp: the STAMP short-term attention/memory model, nextitnet: the NextItNet dilated convolutional model, bert4rec: the BERT4Rec bidirectional masked-item model) instead of GRU4Rec; -ps gives its constructor parameters (e.g. n_sims=200,lmbd=20,alpha=0.5, k=100,sample_size=500,similarity=vector, k=100,lambda_spw=1.02,lambda_snh=inf,lambda_inh=2.05, k=100,similarity=vector,lambda_ipw=inf,lambda_idf=0, steps=10,weighting=div,pruning=20 embedding=50,hidden=100,n_epochs=10, embedding=50,n_blocks=2,n_heads=1,n_epochs=10, embedding=100,step=1,n_epochs=10, embedding=100,n_epochs=10, embedding=100,dilations=1/2/1/2/1/2,n_epochs=10 or embedding=64,n_blocks=2,n_heads=2,mask_prob=0.2), each converted to the type of its default (a bool default takes True or False, a tuple default a /-separated list of integers). Exclusive with -pf, -l, -s and the checkpoint options.')),
    (('-t', '--test'), dict(metavar='TEST_PATH', type=str, nargs='+', help='Test data set(s).')),
    (('-m', '--measure'), dict(metavar='AT', type=int, nargs='+', default=[20], help='Recommendation list length(s) for recall & MRR (default: 20).')),
    (('-e', '--eval_type'), dict(metavar='EVAL_TYPE', choices=_TIE_MODES, default='standard', help='Tie handling of the ranking (see evaluate_gpu).')),
    (('--exclude_seen',), dict(action='store_true', help='Rank each test event without the items its session has already input, as recommend_next_batch(exclude_seen=True) serves (see evaluate_gpu).')),
    (('--history',), dict(metavar='HISTORY_PATH', type=str, help='Events before the test events of each test session, loaded like -t files: every test file is evaluated from its sessions\' history (see evaluate_gpu).')),
    (('--rest_of_session',), dict(action='store_true', help='Also rank every test event against all later items of its session (see evaluate_rest): after the Recall / MRR lines, one line per list length with HitRate, Precision, Recall, MAP, NDCG and MRR. Single GPU, GRU4Rec models only.')),
    (('-ss', '--sample_store_size'), dict(metavar='SS', type=int, default=10000000, help='Size of the negative-sample buffer in ids (default: 10000000).')),
    (('--sample_store_on_cpu',), dict(action='store_true', help='Legacy: draw the negative samples on the host.')),
    (('-g', '--gru4rec_model'), dict(metavar='GRFILE', type=str, default='gru4rec', help='Module that provides the GRU4Rec class (default: gru4rec).')),
    (('-ik', '--item_key'), dict(metavar='IK', type=str, default='ItemId', help='Item id column (default: ItemId).')),
    (('-sk', '--session_key'), dict(metavar='SK', type=str, default='SessionId', help='Session id column (default: SessionId).')),
    (('-tk', '--time_key'), dict(metavar='TK', type=str, default='Time', help='Timestamp column (default: Time).')),
    (('-pm', '--primary_metric'), dict(metavar='METRIC', choices=['recall', 'mrr'], default='recall', help='Primary metric for -lpm (default: recall).')),
    (('-lpm', '--log_primary_metric'), dict(action='store_true', help='Print `PRIMARY METRIC: value` at the end (one test file, one list length).')),
]


def build_parser():
    parser = argparse.ArgumentParser(description='Train or load a GRU4Rec model and measure recall / MRR on test set(s).')
    for flags, kwargs in _OPTIONS:
        parser.add_argument(*flags, **kwargs)
    return parser


def _abort(*lines):
    for line in lines:
        print(line)
    sys.exit(1)


def load_data(fname, args):
    """TSV (item ids read as str, session ids as int32) or pickled DataFrame; the three key columns must exist (run.py:45-78)."""
    import pandas as pd
    import joblib
    pickled = fname.endswith('.pickle')
    if pickled:
        print('Loading data from pickle file: {}'.format(fname))
        frame = joblib.load(fname)
        present = list(frame.columns)
    else:
        with open(fname, 'rt') as handle:
            present = handle.readline().strip().split('\t')
    required = (('session IDs', args.session_key, 'SessionId', 'session_key'),
                ('item IDs', args.item_key, 'ItemId', 'item_key'),
                ('time', args.time_key, 'Time', 'time_key'))
    for role, column, default_name, param_name in required:
        if column not in present:
            _abort('ERROR. The column specified for {} "{}" is not in the data file ({})'.format(role, column, fname),
                   'The default column name is "{}", but you can specify otherwise by setting the `{}` parameter of the model.'.format(default_name, param_name))
    if not pickled:
        print('Loading data from TAB separated file: {}'.format(fname))
        frame = pd.read_csv(fname, sep='\t', usecols=[args.session_key, args.item_key, args.time_key],
                            dtype={args.session_key: 'int32', args.item_key: 'str'})
    return frame


def _training_parameters(args):
    """OrderedDict of constructor parameters from -pf (a Python file defining `gru4rec_params`) or -ps (name=value,...)."""
    if args.parameter_file:
        location = os.path.abspath(args.parameter_file)
        module_name = os.path.split(location)[1].split('.py')[0]
        spec = importlib.util.spec_from_file_location(module_name, location)
        module = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(module)
        print('Loaded parameters from file: {}'.format(location))
        return module.gru4rec_params
    return OrderedDict(pair.split('=') for pair in args.parameter_string.split(','))


def _train(model_class, args):
    params = _training_parameters(args)
    print('Creating GRU4Rec model')
    gru = model_class()
    gru.set_params(**params)
    print('Loading training data...')
    frame = load_data(args.path, args)
    store_type = 'cpu' if args.sample_store_on_cpu else 'gpu'
    if args.sample_store_on_cpu:
        print('WARNING! The sample store is set to be on the CPU. This will make training significantly slower on the GPU.')
    print('Started training')
    started = time.time()
    gru.fit(frame, sample_store=args.sample_store_size, store_type=store_type)
    print('Total training time: {:.2f}s'.format(time.time() - started))
    _save(gru, args)
    return gru


def _save(gru, args):
    if getattr(args, 'rank', 0) != 0:
        return
    if args.save_model is not None:
        print('Saving trained model to: {}'.format(args.save_model))
        gru.savemodel(args.save_model)
    if args.save_checkpoint is not None:
        print('Saving checkpoint to: {}'.format(args.save_checkpoint))
        gru.save_checkpoint(args.save_checkpoint)


def _train_more(gru, args):
    print('Loading training data...')
    frame = load_data(args.path, args)
    print('Started training')
    started = time.time()
    gru.fit_more(frame, sample_store=args.sample_store_size, store_type='cpu' if args.sample_store_on_cpu else 'gpu')
    print('Total training time: {:.2f}s'.format(time.time() - started))
    _save(gru, args)


def _train_baseline(args):
    """a baselines.Pop / SessionPop / ItemKNN / BPR / SessionKNN / STAN / VSTAN / SR / AR / NARM / SASRec / SRGNN / STAMP / NextItNet / BERT4Rec from -ps (values converted to the type of the constructor's default; a bool
    takes True or False, a tuple a /-separated list of integers), fitted on PATH"""
    import inspect
    import baselines
    model_class = {'pop': baselines.Pop, 'sessionpop': baselines.SessionPop, 'itemknn': baselines.ItemKNN, 'bpr': baselines.BPR,
                   'sknn': baselines.SessionKNN, 'stan': baselines.STAN, 'vstan': baselines.VSTAN, 'sr': baselines.SR, 'ar': baselines.AR,
                   'narm': baselines.NARM, 'sasrec': baselines.SASRec, 'srgnn': baselines.SRGNN, 'stamp': baselines.STAMP,
                   'nextitnet': baselines.NextItNet, 'bert4rec': baselines.BERT4Rec}[args.baseline]
    defaults = {n: p.default for n, p in inspect.signature(model_class.__init__).parameters.items() if n != 'self'}
    params = {}
    for name, value in (_training_parameters(args).items() if args.parameter_string else []):
        if name not in defaults:
            _abort('ERROR. {} has no parameter "{}" (it takes: {})'.format(model_class.__name__, name, ', '.join(defaults)))
        if isinstance(defaults[name], bool):                   # bool('False') would be True
            if str(value) not in ('True', 'False'):
                _abort('ERROR. {} takes True or False, not "{}"'.format(name, value))
            params[name] = str(value) == 'True'
        elif isinstance(defaults[name], tuple):                # layers=-style lists: 1/2/1/2
            try:
                params[name] = tuple(int(v) for v in str(value).split('/'))
            except ValueError:
                _abort('ERROR. {} takes a /-separated list of integers, not "{}"'.format(name, value))
        else:
            params[name] = value if defaults[name] is None else type(defaults[name])(value)
    print('Creating {} model'.format(model_class.__name__))
    model = model_class(**params)
    print('Loading training data...')
    frame = load_data(args.path, args)
    print('Started training')
    started = time.time()
    model.fit(frame)
    print('Total training time: {:.2f}s'.format(time.time() - started))
    return model


def _evaluate(gru, evaluation, args):
    primary = ('recall', 'mrr').index(args.primary_metric.lower())
    history = None
    if args.history:
        print('Loading history data...')
        history = load_data(args.history, args)
    for test_file in args.test:
        print('Loading test data...')
        frame = load_data(test_file, args)
        print('Starting evaluation (cut-off={}, using {} mode for tiebreaking{})'.format(args.measure, args.eval_type,
                                                                                      ', seen items excluded' if args.exclude_seen else ''))
        started = time.time()
        extra = dict(exclude_seen=True) if args.exclude_seen else {}
        if history is not None:
            extra['history'] = history
        result = evaluation.evaluate_gpu(gru, frame, batch_size=512, cut_off=args.measure, mode=args.eval_type,
                                         item_key=args.item_key, session_key=args.session_key, time_key=args.time_key, **extra)
        print('Evaluation took {:.2f}s'.format(time.time() - started))
        for position, cut in enumerate(args.measure):
            print('Recall@{}: {:.6f} MRR@{}: {:.6f}'.format(cut, result[0][position], cut, result[1][position]))
        if args.rest_of_session:
            rest = evaluation.evaluate_rest(gru, frame, batch_size=512, cut_off=args.measure, mode=args.eval_type,
                                            item_key=args.item_key, session_key=args.session_key, time_key=args.time_key, **extra)
            for position, cut in enumerate(args.measure):
                print('Rest@{}: HitRate {:.6f} Precision {:.6f} Recall {:.6f} MAP {:.6f} NDCG {:.6f} MRR {:.6f}'.format(
                    cut, *(rest[m][position] for m in ('hitrate', 'precision', 'recall', 'map', 'ndcg', 'mrr'))))
        if args.log_primary_metric:
            print('PRIMARY METRIC: {}'.format(result[primary][0]))


def _join_distributed_job():
    """`torchrun --nproc-per-node N run.py ...` (one process per GPU; the reference is single-device): join the job the launcher
    described, so that fit() trains data-parallel and evaluate_gpu() scores a shard of the test sessions per rank.  Every rank
    runs the same command on the same files; only rank 0 prints and saves.  Returns (world_size, rank)."""
    if int(os.environ.get('WORLD_SIZE', '1') or 1) <= 1:
        return 1, 0
    from gru4rec_b200.parallel import init_from_env
    world, rank = init_from_env()
    if rank != 0:
        sys.stdout = open(os.devnull, 'w')
    return world, rank


def main(argv=None):
    args = build_parser().parse_args(argv)
    if args.rest_of_session and args.baseline is not None:
        _abort('ERROR. --rest_of_session does not cover the baselines yet')
    if args.rest_of_session and int(os.environ.get('WORLD_SIZE', '1') or 1) > 1:
        _abort('ERROR. --rest_of_session runs in a single process (evaluate_rest is not sharded over a torchrun job)')
    here = os.path.dirname(os.path.abspath(__file__))
    if here not in sys.path:
        sys.path.insert(0, here)
    world, rank = _join_distributed_job()
    args.rank = rank
    import evaluation
    if args.baseline is not None:
        conflicts = [flag for flag, on in (('-pf', args.parameter_file), ('-l', args.load_model), ('--load_checkpoint', args.load_checkpoint),
                                           ('--fit_more', args.fit_more), ('-s', args.save_model), ('--save_checkpoint', args.save_checkpoint)) if on]
        if conflicts:
            _abort('ERROR. --baseline cannot be combined with {}'.format(', '.join(conflicts)))
        model = _train_baseline(args)
        if args.test is not None:
            _evaluate(model, evaluation, args)
        return
    model_class = importlib.import_module(args.gru4rec_model).GRU4Rec
    chosen = [args.parameter_string is not None, args.parameter_file is not None, bool(args.load_model), args.load_checkpoint is not None]
    if sum(chosen) != 1:
        _abort('ERROR. Exactly one of the following parameters must be provided: --parameter_string, --parameter_file, --load_model'
               + (', --load_checkpoint' if args.load_checkpoint is not None or args.fit_more else ''))
    if args.fit_more and args.load_checkpoint is None:
        _abort('ERROR. --fit_more continues the model of --load_checkpoint')
    if args.load_checkpoint is not None:
        print('Loading checkpoint from file: {}'.format(args.load_checkpoint))
        gru = model_class.load_checkpoint(args.load_checkpoint)
        if args.fit_more:
            _train_more(gru, args)
    elif args.load_model:
        print('Loading trained model from file: {}'.format(args.path))
        gru = model_class.loadmodel(args.path)
    else:
        gru = _train(model_class, args)
    if args.test is not None:
        _evaluate(gru, evaluation, args)
    if world > 1:
        import torch.distributed as dist
        if dist.is_initialized():
            dist.barrier()
            dist.destroy_process_group()


if __name__ == '__main__':
    main()
