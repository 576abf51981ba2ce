"""Stand-alone argument building for when the ``pixelssl`` package itself is not importable
(e.g. the benchmark box).  Mirrors pixelssl/runner.py:12-41 + the flags of
task_template/proxy.py:20-71 and task/sseg/proxy.py:6-15 that the training step reads, including
the fields TaskProxy autosets (gpus, task, labeled_batch_size, iters_per_epoch, is_epoch_lrer)."""
import argparse

import yaml

from . import ssl_algorithm
from .nn import optimizer, lrer
from .utils import cmd, logger


def create_parser(algorithm):
    parser = argparse.ArgumentParser(description='PixelSSL-H100 Static Script Parser')
    if algorithm not in ssl_algorithm.ALL_SSL_ALGORITHMS:
        logger.log_err('Unknown semi-supervised learning algorithm: {0}\n'
                       'The support algorithms are: {1}\n'.format(algorithm, ssl_algorithm.ALL_SSL_ALGORITHMS))
    optimizer.add_parser_arguments(parser)
    lrer.add_parser_arguments(parser)
    getattr(ssl_algorithm, algorithm).add_parser_arguments(parser)
    return parser


def add_proxy_arguments(parser):
    p = parser.add_argument
    p('--exp-id', type=str, default='')
    p('--resume', type=str, default='')
    p('--validation', type=cmd.str2bool, default=False)
    p('--out-path', type=str, default='')
    p('--visualize', type=cmd.str2bool, default=False)
    p('--debug', type=cmd.str2bool, default=False)
    p('--val-freq', type=int, default=1)
    p('--log-freq', type=int, default=100)
    p('--visual-freq', type=int, default=100)
    p('--checkpoint-freq', type=int, default=1)
    p('--trainset', type=yaml.full_load, default={})
    p('--valset', type=yaml.full_load, default={})
    p('--num-workers', type=int, default=1)
    p('--im-size', type=int, default=None)
    p('--unlabeledset', type=yaml.full_load, default={})
    p('--sublabeled-path', type=str, default='')
    p('--ignore-unlabeled', type=cmd.str2bool, default=True)
    p('--ssl-algorithm', type=str, default='')
    p('--models', type=yaml.full_load, default={})
    p('--optimizers', type=yaml.full_load, default={})
    p('--lrers', type=yaml.full_load, default={})
    p('--criterions', type=yaml.full_load, default={})
    p('--epochs', type=int, default=1)
    p('--batch-size', type=int, default=16)
    p('--unlabeled-batch-size', type=int, default=0)
    p('--gpus', type=int, default=0)
    p('--task', type=str, default='')
    p('--labeled-batch-size', type=int, default=None)
    p('--checkpoint-path', type=str, default='')
    p('--visual-debug-path', type=str, default='')      # autoset by the proxy (task_template/proxy.py:67-69)
    p('--visual-train-path', type=str, default='')
    p('--visual-val-path', type=str, default='')
    p('--is-epoch-lrer', type=cmd.str2bool, default=None)
    p('--iters-per-epoch', type=int, default=None)
    # task/sseg/data.py:20-24 (used by the reference's own dataset layer)
    p('--val-rescaling', type=cmd.str2bool, default=False)
    p('--train-base-size', type=int, default=400)
    # task/sseg/proxy.py:13-14
    p('--num-classes', type=int, default=21)
    p('--ignore-index', type=int, default=255)
    from .task.sseg import model as sseg_model
    sseg_model.add_parser_arguments(parser)


def build_args(config, iters_per_epoch=100):
    """config dict (as in task/sseg/script/*.py) -> argparse.Namespace with the autoset fields."""
    parser = create_parser(config['ssl_algorithm'])
    add_proxy_arguments(parser)
    crits = config.get('criterions') or {}
    if isinstance(crits, str):
        crits = yaml.full_load(crits) or {}
    from .task.sseg import criterion as sseg_criterion
    if any(v in sseg_criterion.OHEM_CRITERIONS for v in crits.values()):
        sseg_criterion.add_ohem_parser_arguments(parser)
    from .task.sseg import evaluation as sseg_evaluation
    if any(k in config for k in sseg_evaluation.FLAGS):
        sseg_evaluation.add_val_protocol_parser_arguments(parser)
    if 'pretrained_backbone' not in config:
        config = dict(config, pretrained_backbone='none')     # programmatic builds (tests, bench): synthetic weights
    args = cmd.parse_args(parser, config)
    args.gpus = 1                     # one process drives one GPU (flags are per-GPU, proxy.py:59,260)
    args.task = 'sseg'
    args.labeled_batch_size = args.batch_size - args.unlabeled_batch_size
    args.iters_per_epoch = iters_per_epoch
    # proxy.py:239-250: per-epoch schedulers step once per epoch, 'polynomiallr' every iteration
    from .nn import lrer as _lrer
    kinds = set()
    for n in (args.lrers or {'model': 'polynomiallr'}).values():
        if n not in _lrer.VALID_LRER:
            logger.log_err('Unknown learning rate scheduler ({0}) type\n  EPOCH_LRERS\t=>\t{1}\n  ITER_LRERS\t=>\t{2}\n'
                           .format(n, _lrer.EPOCH_LRERS, _lrer.ITER_LRERS))
        kinds.add(n in _lrer.EPOCH_LRERS)
    if len(kinds) > 1:
        logger.log_err('Unmatched lr scheduler types\t=>\t{0}\nAll lrers of the task models should have the same '
                       'types (either EPOCH_LRERS or ITER_LRERS)\n'.format(args.lrers))
    args.is_epoch_lrer = kinds.pop()
    return args


def build_algorithm(args):
    """TaskProxy._build_ssl_algorithm (proxy.py:421-441) for the sseg task with by-name lookup."""
    from .task.sseg import model as sseg_model, criterion as sseg_criterion, func as sseg_func
    name = args.ssl_algorithm
    models = {k: getattr(sseg_model, v)() for k, v in (args.models or {'model': 'deeplabv2'}).items()}
    crits = {k: getattr(sseg_criterion, v)() for k, v in (args.criterions or {'model': 'sseg_criterion'}).items()}
    opts = {k: getattr(optimizer, v)(args) for k, v in (args.optimizers or {'model': 'sgd'}).items()}
    lrers = {k: getattr(lrer, v)(args) for k, v in (args.lrers or {'model': 'polynomiallr'}).items()}
    export = getattr(getattr(ssl_algorithm, name), name)
    return export(args, models, opts, lrers, crits, sseg_func.task_func()(args))


def run_script(config, proxy_file=None, proxy_class=None):
    raise NotImplementedError('the dataset/proxy layer is PixelSSL\'s own (SURVEY.md section 8f); '
                              'use pixelssl.run_script after pixelssl_b200.register_into_pixelssl()')
