"""pixelssl_b200: H100-native (sm_90a) engine for PixelSSL's semantic-segmentation SSL training
step, exposed behind PixelSSL's own ``ssl_algorithm`` / ``task_template`` plugin API.

    import pixelssl, pixelssl_b200
    pixelssl_b200.register_into_pixelssl(pixelssl)      # see INTEGRATION.md

Importing the package does not need a GPU; the first kernel call loads lib/libpixelssl_b200.so
(built by ``__graft_entry__.build()``) and raises if it is missing."""
from .version import __version__
from .utils import log_info, log_warn, log_err, str2bool, str2intlist, REGRESSION, CLASSIFICATION
from . import nn, ssl_algorithm
from .ssl_algorithm import (SSL_NULL, SSL_MT, SSL_ADV, SSL_S4L, SSL_GCT, SSL_CCT, SSL_CUTMIX, SSL_CPS,
                            SSL_UNIMATCH, SSL_ALGORITHMS, EXTRA_SSL_ALGORITHMS, ALL_SSL_ALGORITHMS)
from .runner import create_parser, build_args, run_script


def register_into_pixelssl(pixelssl_module=None, task_sseg_modules=None, extra_algorithms=(), extra_criterions=(),
                           val_protocol=False):
    """Drop the engine in under an unmodified ``pixelssl.runner`` / ``TaskProxy``: replaces the
    algorithm modules TaskProxy looks up by name (task_template/proxy.py:433-434), adds the ones
    PixelSSL does not have (``ssl_cps``) to ``pixelssl.ssl_algorithm.SSL_ALGORITHMS`` (the list
    ``pixelssl.runner.create_parser`` checks names against) and, if the task's ``model`` /
    ``criterion`` modules are given, replaces their export functions (proxy.py:426-427).

    ``extra_algorithms``: names from ``EXTRA_SSL_ALGORITHMS`` (``ssl_unimatch``) to install and list as well.  They
    are opt-in so that the algorithm list an existing integration sees stays the one it had.

    ``extra_criterions``: names from ``task.sseg.criterion.OHEM_CRITERIONS`` (``ohem_sseg_criterion``) to install into
    the task's criterion module (``task_sseg_modules[1]``), whose ``add_parser_arguments`` then also adds their flags
    (``--ohem-thresh``, ``--ohem-min-kept``).  Opt-in for the same reason: the default parser stays PixelSSL's.

    ``val_protocol``: the task's model module's (``task_sseg_modules[0]``) ``add_parser_arguments`` also adds the
    multi-view validation flags (``--val-protocol``, ``--val-crop-size``, ``--val-scales``, ``--val-flip``;
    task/sseg/evaluation.py).  Opt-in for the same reason."""
    from .task.sseg import criterion as b200_criterion
    unknown = [n for n in extra_algorithms if n not in EXTRA_SSL_ALGORITHMS]
    if unknown:
        raise ValueError('register_into_pixelssl: unknown extra algorithms {0}; available: {1}'.format(
            unknown, EXTRA_SSL_ALGORITHMS))
    unknown = [n for n in extra_criterions if n not in b200_criterion.OHEM_CRITERIONS]
    if unknown:
        raise ValueError('register_into_pixelssl: unknown extra criterions {0}; available: {1}'.format(
            unknown, b200_criterion.OHEM_CRITERIONS))
    if extra_criterions and task_sseg_modules is None:
        raise ValueError('register_into_pixelssl: extra_criterions are installed into the task\'s criterion module; '
                         'pass task_sseg_modules')
    if val_protocol and task_sseg_modules is None:
        raise ValueError('register_into_pixelssl: the val_protocol flags are added by the task\'s model module; '
                         'pass task_sseg_modules')
    if pixelssl_module is None:
        import pixelssl as pixelssl_module
    names = getattr(pixelssl_module.ssl_algorithm, 'SSL_ALGORITHMS', None)
    if names is None:
        names = []
        pixelssl_module.ssl_algorithm.SSL_ALGORITHMS = names
    for name in SSL_ALGORITHMS + [n for n in EXTRA_SSL_ALGORITHMS if n in extra_algorithms]:
        mod = getattr(ssl_algorithm, name)
        pixelssl_module.ssl_algorithm.__dict__[name] = mod
        setattr(pixelssl_module.ssl_algorithm, name, mod)
        if name not in names:
            names.append(name)
    # the proxy builds its sampler through ``pixelssl.nn.data`` by attribute (task_template/proxy.py:11,372):
    # the rank-aware sampler has the same constructor and, at world size 1, the same index stream
    from .nn import data as b200_data
    pixelssl_module.nn.data.TwoStreamBatchSampler = b200_data.TwoStreamBatchSampler
    if task_sseg_modules is not None:
        from .task.sseg import model as b200_model
        task_model, task_criterion = task_sseg_modules[0], task_sseg_modules[1]
        task_model.deeplabv2 = b200_model.deeplabv2
        task_model.pspnet = b200_model.pspnet
        task_model.deeplabv3plus = b200_model.deeplabv3plus
        task_criterion.sseg_criterion = b200_criterion.sseg_criterion
        for name in extra_criterions:
            setattr(task_criterion, name, getattr(b200_criterion, name))
        base = getattr(task_criterion, 'add_parser_arguments', None)
        if extra_criterions and not getattr(base, 'adds_ohem_flags', False):
            def add_parser_arguments(parser):
                if base is not None:
                    base(parser)
                b200_criterion.add_ohem_parser_arguments(parser)
            add_parser_arguments.adds_ohem_flags = True
            task_criterion.add_parser_arguments = add_parser_arguments
        model_base = getattr(task_model, 'add_parser_arguments', None)
        if val_protocol and not getattr(model_base, 'adds_val_protocol_flags', False):
            from .task.sseg import evaluation as b200_evaluation

            def add_model_parser_arguments(parser):
                if model_base is not None:
                    model_base(parser)
                b200_evaluation.add_val_protocol_parser_arguments(parser)
            add_model_parser_arguments.adds_val_protocol_flags = True
            task_model.add_parser_arguments = add_model_parser_arguments
        if len(task_sseg_modules) > 2:
            # optional third module = the task's func.py: validation metrics on the GPU (confusion matrix kernel);
            # the reference's own TaskFunc keeps working too (it moves the probability map to the host)
            from .task.sseg import func as b200_func
            task_sseg_modules[2].task_func = b200_func.task_func
    return pixelssl_module
