from .aggr import (Aggregation, FusedAggregation, MaxAggregation, MeanAggregation, MedianAggregation,  # noqa: F401
                   MinAggregation, MultiAggregation, PowerMeanAggregation, QuantileAggregation, SoftmaxAggregation,
                   StdAggregation, SumAggregation, VarAggregation, aggregation_resolver)
from .conv import (CGConv, FastRGCNConv, GATConv, GATv2Conv, GCNConv, GENConv, GINConv, GINEConv, GraphConv, HeteroLinear,  # noqa: F401
                   NNConv, PNAConv, ResGatedGraphConv, RGCNConv, SAGEConv, SplineConv, TransformerConv)
from .pool import fps, graclus, knn, knn_graph, nearest, radius, radius_graph, voxel_grid  # noqa: F401
from .models import Node2Vec  # noqa: F401
