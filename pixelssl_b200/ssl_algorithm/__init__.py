"""Algorithm registry with the reference's names (pixelssl/ssl_algorithm/__init__.py:10-27), plus Cross Pseudo
Supervision (``ssl_cps``) and UniMatch (``ssl_unimatch``), which the reference does not have.

``SSL_ALGORITHMS`` is the set ``register_into_pixelssl`` installs by default (the reference's seven and ``ssl_cps``);
``EXTRA_SSL_ALGORITHMS`` are installed on request (its ``extra_algorithms``); ``ALL_SSL_ALGORITHMS`` is every
algorithm the engine's own runner accepts."""
from . import ssl_base, ssl_null, ssl_mt, ssl_cutmix, ssl_adv, ssl_gct, ssl_cct, ssl_s4l, ssl_cps, ssl_unimatch

SSL_NULL = ssl_null.SSLNULL.NAME
SSL_MT = ssl_mt.SSLMT.NAME
SSL_CUTMIX = ssl_cutmix.SSLCUTMIX.NAME
SSL_ADV = ssl_adv.SSLADV.NAME
SSL_GCT = ssl_gct.SSLGCT.NAME
SSL_CCT = ssl_cct.SSLCCT.NAME
SSL_S4L = ssl_s4l.SSLS4L.NAME
SSL_CPS = ssl_cps.SSLCPS.NAME
SSL_UNIMATCH = ssl_unimatch.SSLUNIMATCH.NAME

SSL_ALGORITHMS = [SSL_NULL, SSL_MT, SSL_ADV, SSL_S4L, SSL_GCT, SSL_CCT, SSL_CUTMIX, SSL_CPS]
EXTRA_SSL_ALGORITHMS = [SSL_UNIMATCH]
ALL_SSL_ALGORITHMS = SSL_ALGORITHMS + EXTRA_SSL_ALGORITHMS
