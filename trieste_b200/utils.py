"""Tags of local models and datasets — mirrors trieste/utils/misc.py:224-284 (``get_value_for_tag``, ``LocalizedTag``,
``ignoring_local_tags``).  A ``LocalizedTag(tag, i)`` names the local model or dataset of trust region ``i`` for the global
tag ``tag``; a plain tag is global."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Hashable, Mapping, Optional, Tuple, TypeVar, Union

from .acquisition.interface import OBJECTIVE

Tag = Hashable
T = TypeVar("T")


def get_value_for_tag(mapping: Optional[Mapping[Tag, T]], *tags: Tag) -> Tuple[Optional[Tag], Optional[T]]:
    """misc.py:224-246: the first of ``tags`` (default ``OBJECTIVE``) found in ``mapping`` and its value; (None, None) when
    the mapping is None.  Raises ``ValueError`` when none of the tags is in the mapping."""
    if not tags:
        tags = (OBJECTIVE,)
    if mapping is None:
        return None, None
    matched_tag = next((tag for tag in tags if tag in mapping), None)
    if matched_tag is None:
        raise ValueError(f"none of the tags '{tags}' found in mapping")
    return matched_tag, mapping[matched_tag]


@dataclass(frozen=True)
class LocalizedTag:
    """misc.py:249-284: a tag for a local model or dataset, a global tag and a local index (None for a global tag)."""

    global_tag: Tag
    local_index: Optional[int]

    def __post_init__(self) -> None:
        if self.local_index is not None and self.local_index < 0:
            raise ValueError(f"local index must be non-negative, got {self.local_index}")

    @property
    def is_local(self) -> bool:
        return self.local_index is not None

    @staticmethod
    def from_tag(tag: Union[Tag, "LocalizedTag"]) -> "LocalizedTag":
        if isinstance(tag, LocalizedTag):
            return tag
        return LocalizedTag(tag, None)


def ignoring_local_tags(mapping: Mapping[Tag, T]) -> Mapping[Tag, T]:
    """misc.py:287-295: the entries of ``mapping`` under global tags."""
    return {k: v for k, v in mapping.items() if not LocalizedTag.from_tag(k).is_local}
