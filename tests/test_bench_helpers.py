"""CPU checks of the measurement plumbing of bench.py (no GPU): kernel-name classification and exclusive-time bookkeeping,
the roofline record of the dominant kernel (bound, algorithmic work, the committed ncu DRAM traffic only for the shape it
was captured on), and the committed bench lines under profiles/ carrying every key the contract names."""
import json
import os

import pytest

import bench

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_classify_sums_exclusive_times_per_class():
    rows = {
        'void nats::(anonymous namespace)::enc_tc_kernel<32, true>(nats::EncTc)': (3400.0, 3400.0, 1),
        'void nats::(anonymous namespace)::tma_gemm_ts_kernel<32, 8, 4, true, false>(TmaGroup)': (800.0, 1800.0, 100),
        'void nats::(anonymous namespace)::tma_gemm_ts_kernel<32, 8, 4, false, false>(TmaGroup)': (600.0, 1500.0, 82),
        'void nats::(anonymous namespace)::some_new_kernel(int)': (10.0, 12.0, 2),
    }
    cls = bench.classify(rows, steps=2)
    assert set(cls) == {'enc_tc_bwd', 'tc_gemm_3xtf32_skinny', 'other'}
    assert cls['tc_gemm_3xtf32_skinny']['launches_per_step'] == 91.0
    assert abs(cls['tc_gemm_3xtf32_skinny']['ms_per_step'] - 0.7) < 1e-12
    assert abs(cls['enc_tc_bwd']['us_per_launch'] - 3400.0) < 1e-9
    assert sum(v['ms_per_step'] for v in cls.values()) == pytest.approx((3400 + 800 + 600 + 10) / 2e3)


def test_roofline_of_names_the_dominant_kernel_and_its_bound():
    cls = {'enc_tc_bwd': {'ms_per_step': 3.49, 'us_per_launch': 3490.0},
           'att_context': {'ms_per_step': 0.66, 'us_per_launch': 22.0},
           'other': {'ms_per_step': 9.0, 'us_per_launch': 1.0}}               # 'other' never is the roofline kernel
    r = bench.roofline_of(cls, bench.WORKLOADS['c3'], 14.4)
    assert r['kernel'] == 'enc_tc_bwd' and r['bound'] == 'tensor' and r['unit'] == 'TFLOP/s'
    assert r['frac'] == pytest.approx(r['achieved'] / r['peak'])
    assert r['traffic'] is None                                                # no DRAM capture is committed
    assert bench.roofline_of(cls, bench.WORKLOADS['c2'], 5.8)['traffic'] is None
    r = bench.roofline_of({'att_context': cls['att_context']}, bench.WORKLOADS['c3'], 14.4)
    assert r['bound'] == 'hbm' and r['unit'] == 'GB/s'
    w = bench.WORKLOADS['c3']
    assert r['algo_bytes_per_launch'] == 4.0 * (w['Tx'] * w['B'] * 2 * w['dim'] + 3 * w['B'] * 2 * w['dim'] + 3 * w['B'] * w['Tx'])
