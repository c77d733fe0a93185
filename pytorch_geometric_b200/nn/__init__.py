from .aggr import (Aggregation, FusedAggregation, MaxAggregation, MeanAggregation, MinAggregation,  # noqa: F401
                   MultiAggregation, PowerMeanAggregation, SoftmaxAggregation, StdAggregation, SumAggregation, VarAggregation,
                   aggregation_resolver)
from .conv import (CGConv, FastRGCNConv, GATConv, GATv2Conv, GCNConv, GENConv, GINConv, GINEConv, GraphConv, HeteroLinear,  # noqa: F401
                   PNAConv, ResGatedGraphConv, RGCNConv, SAGEConv, TransformerConv)
