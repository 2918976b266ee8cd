"""CPU-only: where the library places an index's f32 rows (arroy_b200_item_placement_plan, host only, no device): on the device
when the rows, the 8-bit planes, the scales, the headers and one tree's wave buffers fit in 0.7 x the free memory, else in mapped
pinned host memory, but only for the float metrics with 64 <= dim <= 8192."""
import pytest

import arroy_b200 as ab

GIB = 1 << 30
CARD = 80 * GIB   # what an 80 GB H100 reports free before anything is allocated, rounded down

FLOAT_METRICS = ["euclidean", "cosine", "dot-product", "manhattan"]
BQ_METRICS = ["binary quantized euclidean", "binary quantized cosine", "binary quantized manhattan"]


def free_after_copy(n, d):
    """The free memory of the card once a benchmark holds its own f32 copy of the items on it (and ~2 GiB of other state)."""
    return CARD - 4 * n * d - 2 * GIB


@pytest.mark.parametrize("name,metric,n,d", [
    ("C1", "euclidean", 10_000, 64),
    ("C2", "cosine", 1_000_000, 768),
    ("C3", "dot-product", 5_000_000, 768),
    ("headline", "cosine", 5_000_000, 768),
    ("C4", "cosine", 2_500_000, 1536),
    ("C5", "cosine", 100_000 + 4096, 768),
])
def test_benchmark_shapes_stay_on_the_device(name, metric, n, d):
    assert ab.item_placement_plan(metric, d, n, free_after_copy(n, d)) == "device", name


@pytest.mark.parametrize("metric", FLOAT_METRICS)
def test_small_indexes_stay_on_the_device(metric):
    for n, d in [(1, 64), (40_000, 128), (100_000, 1000), (20_000, 8192)]:
        assert ab.item_placement_plan(metric, d, n, CARD) == "device"


def test_ten_million_openai_embeddings_go_to_the_host():
    # 10M x 1536 Cosine: 61 GB of f32 rows alone
    assert ab.item_placement_plan("cosine", 1536, 10_000_000, CARD) == "host"
    assert ab.item_placement_plan("cosine", 1536, 11_000_000, CARD) == "host"


@pytest.mark.parametrize("metric", BQ_METRICS)
@pytest.mark.parametrize("n,d", [(1000, 64), (10_000_000, 1536), (4_000_000_000, 8192)])
def test_binary_quantized_is_always_device(metric, n, d):
    assert ab.item_placement_plan(metric, d, n, 0) == "device"
    assert ab.item_placement_plan(metric, d, n, CARD) == "device"


@pytest.mark.parametrize("metric", FLOAT_METRICS)
def test_dims_outside_the_planes_range_stay_on_the_device(metric):
    for d in (1, 32, 63, 8193, 16384):
        assert ab.item_placement_plan(metric, d, 100_000_000, CARD) == "device"
        assert ab.item_placement_plan(metric, d, 100_000_000, 0) == "device"


@pytest.mark.parametrize("metric", FLOAT_METRICS)
def test_range_ends_go_to_the_host_when_too_large(metric):
    assert ab.item_placement_plan(metric, 64, 4_000_000_000, CARD) == "host"
    assert ab.item_placement_plan(metric, 8192, 10_000_000, CARD) == "host"
    assert ab.item_placement_plan(metric, 64, 1000, 0) == "host"
    assert ab.item_placement_plan(metric, 8192, 1000, 0) == "host"


def test_the_rule_in_bytes():
    # 1M x 768: f32 rows 3072 MB + planes 1536 MB + scales / headers 12 MB + one tree's wave buffers
    n, d = 1_000_000, 768
    need = n * 768 * 4 + 2 * n * 768 + 12 * n
    assert ab.item_placement_plan("euclidean", d, n, int(need / 0.7)) == "host"   # the wave buffers do not fit
    assert ab.item_placement_plan("euclidean", d, n, int(need / 0.7 * 1.2)) == "device"
    # ld = dim rounded up to 32 floats: 1000 -> 1024
    n, d = 1_000_000, 1000
    need = n * 1024 * 6 + 12 * n
    assert ab.item_placement_plan("cosine", d, n, int(need / 0.7) - 1) == "host"


@pytest.mark.parametrize("metric", FLOAT_METRICS)
@pytest.mark.parametrize("n,d", [(1_000_000, 768), (10_000_000, 1536), (123_457, 100), (50_000_000, 64), (2_000_000, 8192)])
def test_monotone_in_free_bytes(metric, n, d):
    seen_device = False
    for free in [0] + [int(1.25 ** k) for k in range(1, 200) if 1.25 ** k < 2 ** 63]:
        where = ab.item_placement_plan(metric, d, n, free)
        if seen_device:
            assert where == "device", (free, where)
        seen_device = seen_device or where == "device"
    assert seen_device
