"""Trainer: the reference's Trainer (crowd_nav/utils/trainer.py:8-71) over a memory.DeviceReplayMemory.

The reference wraps its ReplayMemory in DataLoader(memory, batch_size, shuffle=True), which collates every pair on the
host. Here the DataLoader shuffles the row indices instead: DataLoader(range(len(memory)), batch_size, shuffle=True) takes
the same draws from torch's global CPU generator as the reference's loader over a memory of the same length, so it yields
the same index batches, and the rows are gathered from the memory's device tensors. The optimiser (SGD, momentum 0.9), the
loss (MSELoss), the log lines and the errors are the reference's. The loss sums are the reference's left fold of each
batch's float32 loss widened to float64, kept on the device and read once per call.
"""
import logging

import torch
import torch.nn as nn
import torch.optim as optim
from torch.utils.data import DataLoader

from .policy import CADRLValueNetwork


class _Rows(object):
    """The row indices of a memory as a dataset whose length follows the memory's, as the reference's DataLoader sees
    len(memory) anew on every pass."""

    def __init__(self, memory):
        self.memory = memory

    def __len__(self):
        return len(self.memory)

    def __getitem__(self, i):
        return i


class Trainer(object):
    def __init__(self, model, memory, device, batch_size):
        """Train the trainable model of a policy on the pairs of a DeviceReplayMemory. A CADRL value network takes one
        joint state per pair (cadrl.py:182-185): its memory's [1][13] rows are passed as [13]."""
        self.model = model
        self.device = device
        self.criterion = nn.MSELoss().to(device)
        self.memory = memory
        self.data_loader = None
        self.batch_size = batch_size
        self.optimizer = None
        self.flat_rows = isinstance(model, CADRLValueNetwork)

    def set_learning_rate(self, learning_rate):
        logging.info('Current learning rate: %f', learning_rate)
        self.optimizer = optim.SGD(self.model.parameters(), lr=learning_rate, momentum=0.9)

    def _loader(self):
        if self.optimizer is None:
            raise ValueError('Learning rate is not set!')
        if self.data_loader is None:
            self.data_loader = DataLoader(_Rows(self.memory), self.batch_size, shuffle=True)
        return self.data_loader

    def _optimize(self, index, loss_sum):
        """One SGD step on the pairs at `index` (a CPU index batch); its loss, widened to float64, is added to loss_sum."""
        index = index.to(self.memory.states.device)
        inputs, values = self.memory.states[index], self.memory.values[index]
        if self.flat_rows:
            inputs = inputs.reshape(inputs.shape[0], -1)
        self.optimizer.zero_grad()
        outputs = self.model(inputs)
        loss = self.criterion(outputs, values)
        loss.backward()
        self.optimizer.step()
        loss_sum += loss.detach().double()

    def optimize_epoch(self, num_epochs):
        loader = self._loader()
        epoch_losses = torch.zeros(num_epochs, dtype=torch.float64, device=self.memory.states.device)
        for epoch in range(num_epochs):
            for index in loader:
                self._optimize(index, epoch_losses[epoch])
        average_epoch_loss = 0
        for epoch, epoch_loss in enumerate(epoch_losses.tolist()):
            average_epoch_loss = epoch_loss / len(self.memory)
            logging.debug('Average loss in epoch %d: %.2E', epoch, average_epoch_loss)
        return average_epoch_loss

    def optimize_batch(self, num_batches):
        loader = self._loader()
        losses = torch.zeros((), dtype=torch.float64, device=self.memory.states.device)
        for _ in range(num_batches):
            self._optimize(next(iter(loader)), losses)
        average_loss = losses.item() / num_batches
        logging.debug('Average loss : %.2E', average_loss)
        return average_loss
