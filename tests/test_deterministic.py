"""CPU: the deterministic-mode switch of the training operators (esr_b200.train.deterministic) follows both torch flags."""
import torch


def test_mode_follows_both_torch_flags(monkeypatch):
    from esr_b200 import _lib, train
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", False)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(False)
    try:
        assert not train.deterministic() and train._flags() == 0
        monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)      # what the reference's init_seeds sets
        assert train.deterministic() and train._flags() == _lib.DETERMINISTIC
        monkeypatch.setattr(torch.backends.cudnn, "deterministic", False)
        torch.use_deterministic_algorithms(True)
        assert train.deterministic() and train._flags() == _lib.DETERMINISTIC
        torch.use_deterministic_algorithms(False)
        assert not train.deterministic()                                     # read at every call
    finally:
        torch.use_deterministic_algorithms(prev)


def test_flag_value_matches_the_header():
    import os
    import re
    from esr_b200 import _lib
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "esr_b200.h")).read()
    assert int(re.search(r"#define ESR_DETERMINISTIC (\d+)", hdr).group(1)) == _lib.DETERMINISTIC
