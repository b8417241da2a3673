"""GPU parity tests (run on an H100 with `-m gpu`): the CUDA engine, called through the C ABI
(libamgpu.so via automerge_classic_b200.engine), against the CPU oracle on the same inputs.

  * every reference test extracted into tests/golden/ is replayed through the Backend facade on the
    CUDA engine; a test is allowed to stop with AMG_UNSUPPORTED only if it is listed as outside the
    engine's current incremental-patch subset (EXPECTED_UNSUPPORTED) — anything else must match the
    reference's expected values exactly;
  * synthetic traces (SURVEY.md §8d C1..C4) : incremental patch, final-state patch, heads / clock /
    maxOp and the document-ordered op table with succ lists must equal the oracle's.
"""
import numpy as np
import pytest

import parity_checks
import replay
from automerge_classic_b200.backend import RangeError as FacadeRangeError

pytestmark = pytest.mark.gpu


def _cuda_ok():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.fixture(scope='module')
def gpu_doc():
    if not _cuda_ok():
        pytest.skip('no CUDA device')
    from automerge_classic_b200 import build
    build.build_all()
    from automerge_classic_b200.engine import GpuBackendDoc
    return GpuBackendDoc


def _all_cases():
    out = []
    for f in ('new_backend_test.json', 'backend_test.json'):
        out += [pytest.param(t, id=t['name'][-70:]) for t in replay.load(f) if 'skipped' not in t]
    return out


@pytest.mark.parametrize('test', _all_cases())
def test_reference_fixture(gpu_doc, test):
    from automerge_classic_b200.engine import AmgError
    r = replay.Replayer(gpu_doc, (AmgError, ValueError, TypeError, RuntimeError, FacadeRangeError), structural=False)
    fails = r.run_test(test)
    assert not fails, '\n'.join(fails[:5])


TRACES = [('C1', 0, 0), ('C2', 3000, 0), ('C2b', 5000, 0), ('C3', 20000, 10), ('C3', 3000, 3), ('C4', 4000, 4), ('C4', 20000, 100)]   # the last one: 100 new actors in one call (actor table growth)


@pytest.mark.parametrize('cfg,n,a', TRACES)
def test_trace_parity(gpu_doc, oracle_mod, cfg, n, a):
    parity_checks.check_trace_parity(gpu_doc, oracle_mod, cfg, n, a)


@pytest.mark.parametrize('n,a,chunk', [(60, 2, 1000), (300, 3, 7), (400, 4, 50), (200, 1, 3), (450, 5, 1), (1500, 4, 1000)])
def test_rich_list_parity(gpu_doc, oracle_mod, n, a, chunk):
    """C6: element updates / conflicts / deletes / re-insertions and objects nested in list elements."""
    compared = sum(parity_checks.check_rich_list(gpu_doc, oracle_mod, seed, n, a, chunk) for seed in range(1, 9))
    assert compared >= 3


@pytest.mark.parametrize('cfg,n,a', [('C1', 0, 0), ('C2', 2000, 0), ('C2b', 3000, 0), ('C3', 20000, 10), ('C4', 4000, 4), ('C6', 600, 3), ('C7', 400, 3), ('C8', 400, 3)])
def test_decoded_rows(gpu_doc, oracle_mod, cfg, n, a):
    """SURVEY.md 8c parity items 1-2: per-change hashes and decoded rows of the decode kernels vs the oracle."""
    assert parity_checks.check_decoded_rows_trace(gpu_doc, oracle_mod, cfg, n, a) > 0


def test_decoded_rows_corrupted(gpu_doc, oracle_mod):
    parity_checks.check_decode_corrupted(gpu_doc, oracle_mod)


def test_utf16_key_order(gpu_doc, oracle_mod):
    parity_checks.check_utf16_keys(gpu_doc, oracle_mod)


def test_deflate_variants(gpu_doc, oracle_mod):
    parity_checks.check_deflate_variants(gpu_doc, oracle_mod)


@pytest.mark.parametrize('n,a,chunk', [(80, 2, 1000), (300, 3, 5), (500, 4, 40), (200, 1, 1)])
def test_counters_parity(gpu_doc, oracle_mod, n, a, chunk):
    for seed in range(1, 6):
        parity_checks.check_counters(gpu_doc, oracle_mod, seed, n, a, chunk)


@pytest.mark.parametrize('cfg,n,a', [('C1', 0, 0), ('C2', 400, 0), ('C2b', 700, 0), ('C3', 3000, 10), ('C4', 2000, 4), ('C6', 400, 3), ('C7', 500, 3), ('C3', 20000, 10)])
def test_save_parity(gpu_doc, oracle_mod, cfg, n, a):
    parity_checks.check_save(gpu_doc, oracle_mod, cfg, n, a)


@pytest.mark.parametrize('cfg,n,a', [('C1', 0, 0), ('C2', 400, 0), ('C6', 300, 1), ('C7', 300, 1)])
def test_save_after_load(gpu_doc, oracle_mod, cfg, n, a):
    parity_checks.check_save_after_load(gpu_doc, oracle_mod, cfg, n, a)


@pytest.mark.parametrize('n,a,chunk', [(80, 2, 1000), (300, 3, 5), (400, 4, 40), (200, 1, 1)])
def test_list_counters_parity(gpu_doc, oracle_mod, n, a, chunk):
    compared = sum(parity_checks.check_rich_list(gpu_doc, oracle_mod, seed, n, a, chunk, cfg='C8') for seed in range(1, 9))
    assert compared >= 5


def test_full_size_properties(gpu_doc):
    parity_checks.check_full_size_properties(gpu_doc, golden=False)   # the oracle fingerprint: tests/test_zz_full_size.py


def test_pointer_array_entry(gpu_doc, oracle_mod):
    parity_checks.check_pointer_array_entry(gpu_doc, oracle_mod)


def test_incremental_calls_match_bulk(gpu_doc, oracle_mod):
    parity_checks.check_incremental_calls(gpu_doc, oracle_mod)


def test_out_of_order_delivery(gpu_doc, oracle_mod):
    parity_checks.check_out_of_order(gpu_doc, oracle_mod)


def test_errors_leave_state_untouched(gpu_doc):
    parity_checks.check_errors_atomic(gpu_doc)


def test_large_text_trace(gpu_doc, oracle_mod):
    """C3 at 100k ops: full parity against the oracle (the oracle finishes this size in seconds)."""
    parity_checks.check_large_text(gpu_doc, oracle_mod, 100000)


@pytest.mark.parametrize('cfg,n,a', [('C2', 600, 0), ('C3', 6000, 3), ('C1', 0, 0)])
def test_load_saved_document(gpu_doc, oracle_mod, cfg, n, a):
    parity_checks.check_load(gpu_doc, oracle_mod, cfg, n, a)


def test_load_without_head_indexes(gpu_doc, oracle_mod):
    parity_checks.check_load_without_head_indexes(gpu_doc, oracle_mod)


def test_load_rust_document(gpu_doc):
    parity_checks.check_rust_document(gpu_doc)


@pytest.mark.parametrize('seed', [1, 2, 3, 4])
def test_column_decoders(gpu_doc, seed):
    parity_checks.check_column_decoders(gpu_doc, seed, 150)


def test_load_parallel_columns_forced(gpu_doc, oracle_mod, monkeypatch):
    monkeypatch.setenv('AMG_PAR_DOC_MIN', '1')   # every document takes the parallel column decoders (doccols.cuh)
    parity_checks.check_load_parallel_columns(gpu_doc, oracle_mod, [('C2', 600, 0), ('C3', 6000, 3), ('C4', 3000, 4), ('C6', 500, 3), ('C7', 400, 3), ('C8', 400, 3)])
    parity_checks.check_rust_document(gpu_doc)
    parity_checks.check_save_after_load(gpu_doc, oracle_mod, 'C6', 300, 1)


@pytest.mark.parametrize('cfg,n,a', [('C3', 60000, 10), ('C2', 30000, 0), ('C4', 40000, 10)])
def test_load_long_document(gpu_doc, oracle_mod, cfg, n, a):
    parity_checks.check_load(gpu_doc, oracle_mod, cfg, n, a)   # above the default row threshold of the parallel decoders


@pytest.mark.parametrize('cfg,n,a', [('C1', 0, 0), ('C2', 300, 0), ('C2b', 400, 0), ('C3', 600, 3), ('C3', 3000, 10), ('C4', 1500, 4), ('C6', 300, 3), ('C7', 300, 3), ('C8', 300, 3), ('C3', 60000, 10), ('C4', 40000, 10)])
def test_history_after_load(gpu_doc, cfg, n, a):
    parity_checks.check_history_after_load(gpu_doc, cfg, n, a)


def test_history_after_load_late_cut(gpu_doc):
    parity_checks.check_history_after_load(gpu_doc, 'C3', 1000, 4, frac=0.9)


@pytest.mark.parametrize('cfg,n,a', [('C2', 300, 0), ('C3', 600, 3), ('C3', 2000, 4), ('C4', 1500, 4), ('C6', 300, 3), ('C7', 300, 3), ('C8', 300, 3)])
def test_history_against_oracle(gpu_doc, oracle_mod, cfg, n, a):
    parity_checks.check_history_against_oracle(gpu_doc, oracle_mod, cfg, n, a)


def test_value_validation(gpu_doc, oracle_mod):
    parity_checks.check_value_validation(gpu_doc, oracle_mod)


def test_duplicated_successor_pinned(gpu_doc, oracle_mod):
    parity_checks.check_duplicated_successor_pin(gpu_doc, oracle_mod)


def test_unknown_columns(gpu_doc, oracle_mod):
    parity_checks.check_unknown_columns(gpu_doc, oracle_mod)
