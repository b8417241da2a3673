"""The document classes the device entry point tests run on: `emu_doc` (the serial emulation build, CPU) and `gpu_doc`
(libamgpu.so, skipped without a CUDA device). A test module imports both fixtures from here."""
import os
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope='module')
def emu_doc():
    subprocess.check_call([os.path.join(HERE, '_emu', 'build.sh')])
    from automerge_classic_b200 import build
    build.build_tracegen()
    from automerge_classic_b200.engine import doc_class_for
    return doc_class_for(os.path.join(HERE, '_emu', 'libamgpu_emu.so'))


@pytest.fixture(scope='module')
def gpu_doc():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from automerge_classic_b200 import build
    build.build_all()
    from automerge_classic_b200.engine import GpuBackendDoc
    return GpuBackendDoc
