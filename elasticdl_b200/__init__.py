"""elasticdl_b200: H100-native parameter-server hot path behind ElasticDL's worker API.

Only what the path needs (SURVEY.md section 8): the C-ABI CUDA library
(csrc/, include/b200ps.h), the PS group wrapper (ps/), and host-side mirrors of
the reference interfaces that call into it (worker/ps_client.py, layers/embedding.py,
worker/ps_trainer.py, elasticai_api-style controller).
"""
__version__ = "0.1.0"
