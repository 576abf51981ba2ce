"""Supervised-only baseline (pixelssl/ssl_algorithm/ssl_null.py): forward, CE on the labeled
rows, backward, SGD, per-iteration LR step (ssl_null.py:78-144)."""
import torch

from ..utils import REGRESSION, CLASSIFICATION, logger, tool
from ..nn import func
from . import ssl_base


def add_parser_arguments(parser):
    ssl_base.add_parser_arguments(parser)


def ssl_null(args, model_dict, optimizer_dict, lrer_dict, criterion_dict, task_func):
    ssl_base.check_single_model_dicts('ssl_null', model_dict, optimizer_dict, lrer_dict, criterion_dict)
    algorithm = SSLNULL(args)
    algorithm.build([model_dict['model']], [optimizer_dict['model']], [lrer_dict['model']],
                    [criterion_dict['model']], task_func)
    return algorithm


class SSLNULL(ssl_base._SSLBase):
    NAME = 'ssl_null'
    SUPPORTED_TASK_TYPES = [REGRESSION, CLASSIFICATION]
    LOG_LINES = '  task-{3}\t=>\ttask-loss: {meters[task_loss]:.6f}\t'

    def __init__(self, args):
        super().__init__(args)
        self.model = self.optimizer = self.lrer = self.criterion = None

    def _build(self, model_funcs, optimizer_funcs, lrer_funcs, criterion_funcs, task_func):
        self.task_func = task_func
        self.model = func.create_model(model_funcs[0], 'model', args=self.args)
        self.models = {'model': self.model}
        self.optimizer = optimizer_funcs[0](self.model.module.param_groups)
        self.optimizers = {'optimizer': self.optimizer}
        self.lrer = lrer_funcs[0](self.optimizer)
        self.lrers = {'lrer': self.lrer}
        self.criterion = criterion_funcs[0](self.args)
        self.criterions = {'criterion': self.criterion}

    def _train(self, data_loader, epoch):
        if not (self.args.ignore_unlabeled and self.args.unlabeled_batch_size == 0):
            logger.log_err('SSL_NULL is a supervised-only algorithm\n'
                           'Please set ignore_unlabeled = True and unlabeled_batch_size = 0\n')
        super()._train(data_loader, epoch)

    def train_step(self, inp, gt, cur_step, total_steps):
        lbs = self.args.labeled_batch_size
        arena = self.model.arena
        inp, gt = ssl_base.to_device(inp), ssl_base.to_device(gt)
        arena.zero_grad()
        resulter, debugger = self.model.forward(inp)
        if 'pred' not in resulter or 'activated_pred' not in resulter:
            logger.log_err('In SSL_NULL, the \'resulter\' dict returned by the task model should '
                           'contain the keys \'pred\' and \'activated_pred\'\n')
        pred = tool.dict_value(resulter, 'pred')
        l_pred = func.split_tensor_tuple(pred, 0, lbs)
        l_gt = func.split_tensor_tuple(gt, 0, lbs)
        l_inp = func.split_tensor_tuple(inp, 0, lbs)
        task_loss = torch.mean(self.criterion.forward(l_pred, l_gt, l_inp))
        self.meters.update('task_loss', task_loss.data)
        task_loss.backward()
        arena.all_reduce_grads()
        arena.sgd_step(self.optimizer)

    def validate_step(self, inp, gt):
        inp, gt = ssl_base.to_device(inp), ssl_base.to_device(gt)
        self._validate_model(self.model, self.criterion, inp, gt, 'task_loss', 'task')
