"""Host-only checks of two things the Python front relies on: `_lib.precision_mode` (and `_lib.autocast` on it)
restores the library's process-wide precision mode however its block ends, and the chunks of `chunk_bounds` keep
file order through `SpectrogramBatcher`'s length sort, which `ChunkSpectrogramParser` reads row by row."""
import pytest

from deepspeech_pytorch_b200 import _lib
from deepspeech_pytorch_b200.inference import chunk_bounds
from deepspeech_pytorch_b200.input_pipeline import SpectrogramBatcher

PRECS = (_lib.PREC_FP32, _lib.PREC_TF32, _lib.PREC_F16)


@pytest.fixture
def lib():
    lib = _lib.get_lib()
    was = lib.ds2_get_precision()
    yield lib
    lib.ds2_set_precision(was)


@pytest.mark.parametrize("start", PRECS)
def test_switches_and_restores(lib, start):
    lib.ds2_set_precision(start)
    with _lib.precision_mode(_lib.PREC_F16):
        assert lib.ds2_get_precision() == _lib.PREC_F16
    assert lib.ds2_get_precision() == start


@pytest.mark.parametrize("start", PRECS)
def test_restores_after_an_exception(lib, start):
    lib.ds2_set_precision(start)
    with pytest.raises(KeyError):
        with _lib.precision_mode(_lib.PREC_F16):
            raise KeyError("inside")
    assert lib.ds2_get_precision() == start


def test_nested_scopes_unwind(lib):
    lib.ds2_set_precision(_lib.PREC_TF32)
    with _lib.precision_mode(_lib.PREC_F16):
        with _lib.precision_mode(_lib.PREC_FP32):
            assert lib.ds2_get_precision() == _lib.PREC_FP32
            with _lib.precision_mode(None):
                assert lib.ds2_get_precision() == _lib.PREC_FP32
        assert lib.ds2_get_precision() == _lib.PREC_F16
        with pytest.raises(RuntimeError):
            with _lib.precision_mode(_lib.PREC_TF32):
                raise RuntimeError
        assert lib.ds2_get_precision() == _lib.PREC_F16
    assert lib.ds2_get_precision() == _lib.PREC_TF32


@pytest.mark.parametrize("start", PRECS)
def test_none_leaves_the_mode_alone(lib, start):
    lib.ds2_set_precision(start)
    with _lib.precision_mode(None):
        assert lib.ds2_get_precision() == start
        lib.ds2_set_precision(_lib.PREC_FP32)         # a change made inside the block is kept
    assert lib.ds2_get_precision() == _lib.PREC_FP32


@pytest.mark.parametrize("start", PRECS)
def test_autocast_is_fp16_for_precision_16_only(lib, start):
    lib.ds2_set_precision(start)
    with _lib.autocast(16):
        assert lib.ds2_get_precision() == _lib.PREC_F16
    assert lib.ds2_get_precision() == start
    with _lib.autocast(32):
        assert lib.ds2_get_precision() == start


def test_a_bad_mode_is_refused_and_nothing_changes(lib):
    lib.ds2_set_precision(_lib.PREC_TF32)
    with pytest.raises(_lib.Ds2Error, match="precision"):
        with _lib.precision_mode(7):
            pass
    assert lib.ds2_get_precision() == _lib.PREC_TF32


@pytest.mark.parametrize("sample_rate,hop", [(16000, 160), (8000, 80), (22050, 220)])
def test_chunks_keep_file_order_through_the_batcher_sort(sample_rate, hop):
    chunks = (-1, 0.01, 0.1, 0.16, 0.25, 0.33, 0.5, 0.7, 1.0, 1.3, 2.0, 2.5, 7.0)
    n_samples = (1, hop - 1, hop, hop + 1, sample_rate // 3, sample_rate - 1, sample_rate, sample_rate + 1,
                 int(1.49 * sample_rate), 5 * sample_rate + 7, 37 * sample_rate + 12345)
    for chunk in chunks:
        for n in n_samples:
            lens = [e - s for s, e in chunk_bounds(n, sample_rate, chunk)]
            order, frames = SpectrogramBatcher.order_and_frames(lens, hop)
            assert order == list(range(len(lens))), (chunk, n, lens)
            assert frames == [1 + l // hop for l in lens]
