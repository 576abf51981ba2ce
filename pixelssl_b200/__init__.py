"""pixelssl_b200: H100-native (sm_90a) engine for PixelSSL's semantic-segmentation SSL training
step, exposed behind PixelSSL's own ``ssl_algorithm`` / ``task_template`` plugin API.

    import pixelssl, pixelssl_b200
    pixelssl_b200.register_into_pixelssl(pixelssl)      # see INTEGRATION.md

Importing the package does not need a GPU; the first kernel call loads lib/libpixelssl_b200.so
(built by ``__graft_entry__.build()``) and raises if it is missing."""
from .version import __version__
from .utils import log_info, log_warn, log_err, str2bool, str2intlist, REGRESSION, CLASSIFICATION
from . import nn, ssl_algorithm
from .ssl_algorithm import SSL_NULL, SSL_MT, SSL_ADV, SSL_S4L, SSL_GCT, SSL_CCT, SSL_CUTMIX, SSL_ALGORITHMS
from .runner import create_parser, build_args, run_script


def register_into_pixelssl(pixelssl_module=None, task_sseg_modules=None):
    """Drop the engine in under an unmodified ``pixelssl.runner`` / ``TaskProxy``: replaces the
    algorithm modules TaskProxy looks up by name (task_template/proxy.py:433-434) and, if the
    task's ``model`` / ``criterion`` modules are given, their export functions
    (proxy.py:426-427)."""
    if pixelssl_module is None:
        import pixelssl as pixelssl_module
    for name in SSL_ALGORITHMS:
        mod = getattr(ssl_algorithm, name)
        pixelssl_module.ssl_algorithm.__dict__[name] = mod
        setattr(pixelssl_module.ssl_algorithm, name, mod)
    # the proxy builds its sampler through ``pixelssl.nn.data`` by attribute (task_template/proxy.py:11,372):
    # the rank-aware sampler has the same constructor and, at world size 1, the same index stream
    from .nn import data as b200_data
    pixelssl_module.nn.data.TwoStreamBatchSampler = b200_data.TwoStreamBatchSampler
    if task_sseg_modules is not None:
        from .task.sseg import model as b200_model, criterion as b200_criterion
        task_model, task_criterion = task_sseg_modules[0], task_sseg_modules[1]
        task_model.deeplabv2 = b200_model.deeplabv2
        task_model.pspnet = b200_model.pspnet
        task_model.deeplabv3plus = b200_model.deeplabv3plus
        task_criterion.sseg_criterion = b200_criterion.sseg_criterion
        if len(task_sseg_modules) > 2:
            # optional third module = the task's func.py: validation metrics on the GPU (confusion matrix kernel);
            # the reference's own TaskFunc keeps working too (it moves the probability map to the host)
            from .task.sseg import func as b200_func
            task_sseg_modules[2].task_func = b200_func.task_func
    return pixelssl_module
