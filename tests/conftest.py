import os, sys
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with -m gpu)")


@pytest.fixture(scope="session")
def golden():
    import numpy as np
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'golden_v1.npz'))


@pytest.fixture(scope="session")
def golden_tu():
    import numpy as np
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'golden_v2_tu.npz'))


@pytest.fixture(scope="session")
def golden_mctf_apply():
    import numpy as np
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'golden_v3_mctf_apply.npz'))


@pytest.fixture(scope="session")
def golden_frac():
    import numpy as np
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'golden_v4_frac.npz'))


@pytest.fixture(scope="session")
def golden_depquant():
    import numpy as np
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'golden_v5_depquant.npz'))


@pytest.fixture(scope="session")
def golden_rdoq():
    import numpy as np
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'golden_v6_rdoq.npz'))
