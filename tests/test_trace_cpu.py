"""The launch-trace decoder on hand-built buffers: one 16-int record of each kind (include/sdb200.h: SDB_TRACE_INTS), decoded
into the lists of the kinds an entry launches, in launch order."""
import os
import re

import numpy as np
import pytest

from stable_diffusion_burn_b200._lib import Context

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def trace(*records):
    t = np.zeros(Context.TRACE_INTS, np.int32)
    t[0] = len(records)
    for i, (kind, *fields) in enumerate(records):
        t[1 + 16 * i] = kind
        t[2 + 16 * i:2 + 16 * i + len(fields)] = fields
    return t


def test_trace_ints_match_header():
    with open(os.path.join(ROOT, "include", "sdb200.h")) as f:
        assert int(re.search(r"#define SDB_TRACE_INTS (\d+)", f.read()).group(1)) == Context.TRACE_INTS


ALL = ("gemms", "attn", "gn", "conv", "softmax", "cond_mod")


def test_decode_one_record_of_each_kind():
    t = trace((3, 4),
              (1, 2, 320, 160, 3, 4, 8, 16, 640, 6, 320, 3, 8 | 32, 0, 4),
              (2, 48, 4096, 96, 1, 1, 0),
              (4, 2, 32, 5),
              (5, 36),
              (6, 2),
              (2, 64, 77, 77, 0, 0, 1),
              (1, 0, 3072, 128, 1, 1, 1, 128, 0, 0, 0, 1, 1 | 2 | 4, 1, 5))
    assert Context._decode_trace(t, ALL) == {
        "gemms": [dict(kind=2, N=320, BN=160, split=3, TN=4, TH=8, TW=16, xk=640, gn_slots=6, a1=320, passes=3,
                       epi={"res16", "gn"}, act=0, stages=4),
                  dict(kind=0, N=3072, BN=128, split=1, TN=1, TH=1, TW=128, xk=0, gn_slots=0, a1=0, passes=1,
                       epi={"lns", "lnc", "geglu"}, act=1, stages=5)],
        "attn": [dict(dpad=48, Nq=4096, Nk=96, qk3=1, kvlen=1), dict(dpad=64, Nq=77, Nk=77, qk3=0, kvlen=0, causal=1)],
        "gn": ["sums:stats"],
        "conv": [(2, 32, 5)],
        "softmax": [36],
        "cond_mod": 2,
    }


def test_decode_every_groupnorm_path_in_order():
    t = trace(*((3, p) for p in (1, 2, 3, 4, 5, 6, 2)))
    assert Context._decode_trace(t, ("gn",)) == {"gn": ["fused", "apply", "apply+fold", "sums:stats", "sums:partials",
                                                        "sums:fold", "apply"]}


def test_decode_empty():
    assert Context._decode_trace(trace(), ("gemms", "attn")) == {"gemms": [], "attn": []}
    assert Context._decode_trace(trace(), ALL) == {"gemms": [], "attn": [], "gn": [], "conv": [], "softmax": [], "cond_mod": 0}


@pytest.mark.parametrize("records,kinds", [([(7, 1)], ALL),            # no such kind
                                           ([(3, 1)], ("gemms", "attn")),  # a kind the entry does not launch
                                           ([(6, 2), (6, 2)], ALL)])       # two conditioned conv_in launches
def test_decode_rejects(records, kinds):
    with pytest.raises(ValueError):
        Context._decode_trace(trace(*records), kinds)
