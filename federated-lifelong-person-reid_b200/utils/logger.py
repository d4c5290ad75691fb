"""Console logging: one named stdlib logger per actor, the two formatted report lines the experiment log readers
expect (``tools/logger.py:23-39``; ``tests/test_reference_parity.py::test_console_line_formats_match_reference``
compares them character for character with the reference's output)."""
from __future__ import annotations

import logging
from typing import Sequence

logging.basicConfig(level=logging.INFO, format="%(asctime)s [%(name)s]: %(levelname)s - %(message)s")

# the validation report: a header line followed by an indented block, closed by an indented empty line
_INDENT = " " * 12
_RANKS = ((1, "Rank-1 :  "), (3, "Rank-3 :  "), (5, "Rank-5 :  "), (10, "Rank-10 : "))


def _percent(x: float) -> str:
    return format(x, ".2%")


class Logger:
    """Thin facade over ``logging.getLogger(name)``; ``rank`` tags the actor with its process rank."""

    def __init__(self, actuator: str = "unknown", rank: int | None = None):
        name = actuator if rank is None else f"{actuator}@r{rank}"
        self.logger = logging.getLogger(name)

    # ---- plain levels ---------------------------------------------------------------------------------------------
    def enabled_for_info(self) -> bool:
        return self.logger.isEnabledFor(logging.INFO)

    def _emit(self, level: int, msg) -> None:
        self.logger.log(level, msg)

    def debug(self, msg) -> None:
        self._emit(logging.DEBUG, msg)

    def info(self, msg) -> None:
        self._emit(logging.INFO, msg)

    def warn(self, msg) -> None:
        self._emit(logging.WARNING, msg)

    warning = warn

    def error(self, msg) -> None:
        self._emit(logging.ERROR, msg)

    # ---- formatted reports ----------------------------------------------------------------------------------------
    def info_train(self, task_name, device, train_cnt, accuracy, loss, current_epoch=0, total_epoch=0) -> None:
        parts = []
        if current_epoch and total_epoch:
            parts.append(f"[{current_epoch:0>3d}/{total_epoch:0>3d}] ")
        parts.append(f"Train '{task_name}' on {device} with {train_cnt:,} images, ")
        parts.append(f"accuracy: {_percent(accuracy)}, loss: {loss:.4f}.")
        self.info("".join(parts))

    def info_validation(self, task_name, query_cnt, gallery_cnt, cmc: Sequence[float], mAP: float,
                        label: str | None = None) -> None:
        at = lambda k: cmc[k - 1] if len(cmc) >= k else cmc[-1]  # noqa: E731  (galleries smaller than ten items)
        head = "Validation" if label is None else f"Validation ({label})"
        rows = [f"{head} '{task_name}' with {query_cnt:,} query images on {gallery_cnt:,} gallery images:"]
        rows += [f"{_INDENT}|- {label}{_percent(at(k))}" for k, label in _RANKS]
        rows.append(f"{_INDENT}|- mean AP : {_percent(mAP)}")
        rows.append(_INDENT)
        self.info("\n".join(rows))
