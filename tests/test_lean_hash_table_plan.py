"""The lean kernel's hash inserted-set size (dann_plan.h): 3 x the candidate bound for a search without a label key, as
far as the 21-bit slot payload of a 4-byte entry reaches; the bitmap-or-hash choice, the entry layout and keyed
searches as before (decided on 1.5 x, and 4.5 x under a key).  Host logic only: the plan runs on the CPU through the
emulator harness (tests/simt)."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "simt"))


@pytest.fixture(scope="module")
def emu():
    import emu as m
    m.lib()
    return m


def _lean(emu, **kw):
    p = emu.plan(R=64, words=24, nq=4096, allow_lean=True, **kw)
    assert p["lean"] == 1, p
    return p


def _hmin(cand_cap, keyed):
    return (cand_cap * (3 if keyed else 1) * 3 // 2 + 3) & ~3


def test_headline_plan_takes_a_table_of_three_times_the_bound(emu):
    """20M nodes, L = rescore = 600 (c_target 609): the bench's operating point."""
    p = _lean(emu, n=20_000_000, L=600, c_target=609)
    assert p["bitmap_words"] == 0 and p["entry"] == 0 and p["W"] == 16
    assert p["hash_cap"] == 2 * _hmin(p["cand_cap"], False) and p["hash_cap"] >= 3 * p["cand_cap"]


def test_keyed_searches_keep_their_table(emu):
    p = _lean(emu, n=20_000_000, L=600, c_target=609, keyed=True)
    assert p["hash_cap"] == _hmin(p["cand_cap"], True)


@pytest.mark.parametrize("L", [2000, 4000, 10000])
def test_table_stops_at_what_a_four_byte_entry_addresses(emu, L):
    """Large L: the table grows to at most 2^21 slots, never below 1.5 x the bound; the entry layout is the one the
    1.5 x table gave (4 bytes while 1.5 x fits 21 bits)."""
    p = _lean(emu, n=20_000_000, L=L, c_target=1009)
    hmin = _hmin(p["cand_cap"], False)
    assert p["hash_cap"] == max(hmin, min(2 * hmin, 1 << 21))
    assert p["entry"] == (0 if hmin <= (1 << 21) else 2)
    assert p["hash_cap"] <= (1 << 21) or p["entry"] == 2


def test_bitmap_choice_is_made_against_the_smaller_table(emu):
    """n <= 2^21: the bitmap serves whenever it is no larger than a 1.5 x table, as before."""
    p = _lean(emu, n=2_000_000, L=600, c_target=609)
    assert p["bitmap_words"] * 4 <= _hmin(p["cand_cap"], False) * 4 and p["bitmap_words"] > 0
    q = _lean(emu, n=2_000_000, L=40, c_target=49)
    bm_bytes = (2_000_000 + 127) // 128 * 16
    assert (q["bitmap_words"] > 0) == (bm_bytes <= _hmin(q["cand_cap"], False) * 4)
