"""Attribute-style configs equal to the three in-scope reference YAML files
(config/qm8_lanczos_net.yaml, config/qm8_ada_lanczos_net.yaml, config/graph_lanczos_net.yaml);
only the fields the model constructors read (model/lanczos_net.py:18-35 etc.)."""
from types import SimpleNamespace as NS


def qm8_lanczos_net(**model_over):
  model = dict(name='LanczosNet', short_diffusion_dist=[],
               long_diffusion_dist=[1, 2, 3, 5, 7, 10, 20, 30], num_eig_vec=20,
               spectral_filter_kind='MLP', input_dim=64, hidden_dim=[128] * 7, output_dim=16,
               num_layer=7, loss='MSE', output_func='MLP')
  model.update(model_over)
  return NS(seed=1234, dataset=NS(loader_name='QM8Data', name='chemistry', num_atom=70,
                                  num_bond_type=6), model=NS(**model))


def qm8_gcn(**model_over):
  """config/qm8_gcn.yaml"""
  model = dict(name='GCN', input_dim=64, hidden_dim=[128] * 7, output_dim=16, num_layer=7,
               loss='MSE', output_func='MLP')
  model.update(model_over)
  return NS(seed=1234, dataset=NS(loader_name='QM8Data', name='chemistry', num_atom=70,
                                  num_bond_type=6), model=NS(**model))


def qm8_dcnn(**model_over):
  """config/qm8_dcnn.yaml"""
  model = dict(name='DCNN', input_dim=64, diffusion_dist=[3, 5, 7, 10, 20, 30], hidden_dim=[128] * 7,
               output_dim=16, num_layer=7, loss='MSE', output_func='MLP')
  model.update(model_over)
  return NS(seed=1234, dataset=NS(loader_name='QM8Data', name='chemistry', num_atom=70,
                                  num_bond_type=6), model=NS(**model))


def qm8_cheby_net(**model_over):
  """config/qm8_cheby_net.yaml"""
  model = dict(name='ChebyNet', input_dim=64, polynomial_order=5, hidden_dim=[128] * 7,
               output_dim=16, num_layer=7, loss='MSE', output_func='MLP')
  model.update(model_over)
  return NS(seed=1234, dataset=NS(loader_name='QM8Data', name='chemistry', num_atom=70,
                                  num_bond_type=6), model=NS(**model))


def qm8_gat(**model_over):
  """config/qm8_gat.yaml"""
  model = dict(name='GAT', input_dim=64, hidden_dim=[16] * 7, num_layer=7, num_heads=[8] * 7,
               output_dim=16, dropout=0.0, loss='MSE')
  model.update(model_over)
  return NS(seed=1234, dataset=NS(loader_name='QM8Data', name='chemistry', num_atom=70,
                                  num_bond_type=6), model=NS(**model))


def qm8_graphsage(**model_over):
  """config/qm8_graphsage.yaml"""
  model = dict(name='GraphSAGE', input_dim=64, hidden_dim=[128] * 7, output_dim=16, num_sample_neighbors=40,
               agg_func='Mean', num_layer=7, loss='MSE')
  model.update(model_over)
  return NS(seed=1234, dataset=NS(loader_name='QM8Data', name='chemistry', num_atom=70,
                                  num_bond_type=6), model=NS(**model))


def qm8_ggnn(**model_over):
  """config/qm8_ggnn.yaml"""
  model = dict(name='GGNN', num_prop=15, input_dim=64, hidden_dim=128, update_func='GRU', output_dim=16,
               msg_func='MLP', aggregate_type='avg', num_layer=1, loss='MSE')
  model.update(model_over)
  return NS(seed=1234, dataset=NS(loader_name='QM8Data', name='chemistry', num_atom=70,
                                  num_bond_type=6), model=NS(**model))


def qm8_gpnn(**model_over):
  """config/qm8_gpnn.yaml"""
  model = dict(name='GPNN', num_partition=3, num_prop=10, num_prop_cluster=1, num_prop_cut=1, input_dim=64,
               hidden_dim=128, update_func='GRU', output_dim=16, msg_func='MLP', aggregate_type='avg',
               num_layer=1, loss='MSE')
  model.update(model_over)
  return NS(seed=1234, dataset=NS(loader_name='QM8Data', name='chemistry', num_atom=70,
                                  num_bond_type=6), model=NS(**model))


def qm8_mpnn(**model_over):
  """config/qm8_mpnn.yaml"""
  model = dict(name='MPNN', num_prop=7, input_dim=64, hidden_dim=128, update_func='GRU', output_dim=16,
               msg_func='MLP', num_step_set2vec=10, aggregate_type='avg', num_layer=1, loss='MSE')
  model.update(model_over)
  return NS(seed=1234, dataset=NS(loader_name='QM8Data', name='chemistry', num_atom=70,
                                  num_bond_type=6), model=NS(**model))


def qm8_ada_lanczos_net(**model_over):
  model = dict(name='AdaLanczosNet', short_diffusion_dist=[1, 2, 3],
               long_diffusion_dist=[5, 7, 10, 20, 30], num_eig_vec=20,
               use_reorthogonalization=False, use_power_iteration_cap=False,
               spectral_filter_kind='MLP', input_dim=64, hidden_dim=[128] * 7, output_dim=16,
               num_layer=7, loss='MSE', output_func='MLP')
  model.update(model_over)
  return NS(seed=1234, dataset=NS(loader_name='QM8Data', name='chemistry', num_atom=70,
                                  num_bond_type=6), model=NS(**model))


def graph_lanczos_net(**model_over):
  model = dict(name='LanczosNetGeneral', short_diffusion_dist=[],
               long_diffusion_dist=[1, 2, 3, 5, 7, 10, 20, 30], num_eig_vec=20,
               spectral_filter_kind='MLP', input_dim=10, hidden_dim=[128] * 7, output_dim=2,
               num_layer=7, loss='MSE', output_func='MLP')
  model.update(model_over)
  return NS(seed=1234, dataset=NS(loader_name='GraphData', name='synthetic', node_emb_dim=10,
                                  graph_emb_dim=2, num_edge_type=1), model=NS(**model))
