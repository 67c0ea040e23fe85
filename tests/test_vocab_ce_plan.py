"""Host side of the vocabulary cross-entropy (engine.VocabCrossEntropyFn): the backward's row
windows and the label range check, on the CPU."""
import pytest
import torch

from x_clip_b200 import engine as E


def _g_bytes(rows, V):
    return 2 * rows * ((V + 7) // 8 * 8)


@pytest.mark.parametrize("n,V", [(1, 1), (7, 121), (4099, 49408), (49152, 49408), (49152, 10000),
                                 (100000, 10001), (300, 8)])
def test_windows_fit_the_budget_and_cover_the_rows(n, V):
    win = E.vocab_window_rows(n, V)
    assert 1 <= win <= n
    assert _g_bytes(win, V) <= E.VOCAB_CE_WINDOW_BYTES
    assert win == n or win % 128 == 0
    starts = list(range(0, n, win))
    assert sum(min(s + win, n) - s for s in starts) == n


def test_window_at_the_clip_vocabulary():
    """At V = 49408 one window holds 10752 rows (1.06 GB of g, under 1 GiB), against 2.4 G logits
    for the 49 k selected rows of a cfg3-shaped batch of 4096 captions."""
    assert E.vocab_window_rows(49152, 49408) == 10752
    assert E.vocab_window_rows(4099, 49408) == 4099


@pytest.mark.parametrize("budget,want", [(1, 1), (2 * 128 * 10008 - 1, 127), (2 * 128 * 10008, 128),
                                         (2 * 300 * 10008, 256)])
def test_window_rounding(budget, want):
    assert E.vocab_window_rows(100000, 10001, budget) == want


def test_labels_outside_the_vocabulary_raise():
    E.check_labels(torch.tensor([0, 5, 9]), 10)
    for bad in ([0, 10], [-1, 3]):
        with pytest.raises(RuntimeError, match="out of bounds"):
            E.check_labels(torch.tensor(bad), 10)


def test_the_loss_checks_its_labels(monkeypatch):
    """VocabCrossEntropyFn hands every call's labels and vocabulary size to check_labels before any
    kernel runs (the check itself is tested above)."""
    seen = []

    def check(labels, V):
        seen.append((labels, V))
        raise RuntimeError("checked")

    monkeypatch.setattr(E, "check_labels", check)
    labels = torch.tensor([1, 2, 3])
    with pytest.raises(RuntimeError, match="checked"):
        E.VocabCrossEntropyFn.apply(torch.zeros(3, 8, dtype=torch.bfloat16), torch.zeros(5, 8), None, labels)
    assert len(seen) == 1 and torch.equal(seen[0][0], labels) and seen[0][1] == 5
