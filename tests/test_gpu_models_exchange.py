"""The Wide & Deep, DCN and xDeepFM engines on the owner-computes exchange at two ranks (tests/mgpu_models_check.py
through torchrun): each rank's first-step tower outputs against the float64 reference on the rows the exchange
pulled, then the loss falls, eagerly and from the CUDA graph."""
import pytest

from tests.test_gpu_layer_trainer import _torchrun_two_ranks

pytestmark = pytest.mark.gpu


def test_wide_deep_dcn_and_xdeepfm_train_on_the_owner_exchange_via_torchrun():
    """One rank per GPU when the box has two, otherwise both ranks as processes on cuda:0 (B200_SHARED_GPU=1)."""
    out = _torchrun_two_ranks("mgpu_models_check.py", 29561)
    assert out.returncode == 0 and "mgpu_models_check ok: world=2" in out.stdout, out.stdout[-3000:] + out.stderr[-6000:]
    print(out.stdout[-2000:])
