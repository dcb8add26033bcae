"""Operator configurations: what the reference's protobuf operator configs carry
(arroyo-rpc/proto/api.proto:39-80), reduced to the supported plan subset.  Durations are int ns."""
from dataclasses import dataclass, field
from typing import List, Optional


@dataclass
class Agg:
    kind: str            # count | sum | avg | min | max
    col: Optional[str]   # input column (None for count(*))
    name: str            # output column name


@dataclass
class WindowAggConfig:
    """TumblingWindowAggregateOperator / SlidingWindowAggregateOperator.
    Input  [key cols..., value cols..., _timestamp]; output = aggregate output [keys, aggs] with the
    window struct {start, end} inserted at `window_index`, then `_timestamp = bin + width - 1 ns`
    (arroyo-planner/src/extension/aggregate.rs:292-390).  `final_projection=False` (tumbling only)
    gives [keys, aggs, _timestamp = bin].

    `width=0` is the instant window (InstantAggregatingWindowFunc): each `_timestamp` is its own bin.  Its
    `final_projection=False` form is [keys, aggs, _timestamp = instant]; with `final_projection=True` it is the nested
    form behind an upstream window of width `nested_width`: window{start = ts - nested_width + 1, end = ts + 1} at
    `window_index`, `_timestamp = instant` (extension/aggregate.rs:392-452)."""
    width: int
    slide: int = 0
    key_names: List[str] = field(default_factory=list)
    aggs: List[Agg] = field(default_factory=list)
    final_projection: bool = True
    window_index: int = 0
    # final stage of a partial -> shuffle -> final plan: name of the input column that carries how many
    # original rows each (partial-aggregate) input row stands for; None = inputs are raw rows
    partial_count_col: Optional[str] = None
    # instant window, nested form: the upstream window's width
    nested_width: int = 0


@dataclass
class SessionConfig:
    """SessionWindowAggregateOperator (planner extension/aggregate.rs:170-231)."""
    gap: int
    key_names: List[str] = field(default_factory=list)
    aggs: List[Agg] = field(default_factory=list)
    window_index: int = 0


@dataclass
class JoinConfig:
    """JoinOperator for the instant (windowed) join (arroyo-worker/src/arrow/instant_join.rs) and the join with
    expiration (join_with_expiration.rs).  `ttl` (ns) is the join with expiration's state retention, 0 meaning 24 h
    (:239-248); the instant join ignores it."""
    left_on: List[str]
    right_on: List[str]
    join_type: str = "inner"
    left_routing_keys: List[str] = field(default_factory=list)
    right_routing_keys: List[str] = field(default_factory=list)
    ttl: int = 0


@dataclass
class WindowFrame:
    """A window function's explicit frame, `{ROWS | RANGE | GROUPS} BETWEEN start AND end`: `units` is rows, range or
    groups; `start` and `end` are each "unbounded_preceding", "current_row" or "unbounded_following", or a pair
    ("preceding" | "following", n) with n >= 0 (nanoseconds for RANGE over a timestamp key)."""
    units: str
    start: object
    end: object


@dataclass
class WindowFunctionConfig:
    """WindowFunctionOperator (arroyo-worker/src/arrow/window_fn.rs): `function` (row_number | rank | dense_rank,
    the aggregate sum | count | avg | min | max of column `argument`, which count ignores, the value function lag |
    lead | first_value | last_value | nth_value of column `argument`, or percent_rank | cume_dist) OVER (PARTITION BY
    window [, `partition_by`] ORDER BY `order_by`), the function column named `name`.  `order_by` is a list of
    (column, descending); it may be empty for every function but the ranking ones, the frame then being the whole
    partition.  `top_n` > 0 fuses the `WHERE name <= top_n` that follows a ranking function; 0 lets every row through.
    `offset` is lag / lead's k (>= 0) or nth_value's n (>= 1); `default` is lag / lead's default, in the argument's
    type (None: NULL).  `frame` is the frame of an aggregate or of first_value / last_value / nth_value (None: the
    default frame)."""
    function: str
    partition_by: Optional[str]
    order_by: List[tuple]
    name: str
    top_n: int = 0
    argument: Optional[str] = None
    offset: int = 1
    default: Optional[object] = None
    frame: Optional[WindowFrame] = None
