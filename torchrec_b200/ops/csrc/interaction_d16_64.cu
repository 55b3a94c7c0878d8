// Dot-interaction kernel instances for D = 16, 32, 48, 64 (templates and C ABI: interaction.cuh, interaction.cu).
#include "interaction.cuh"

TRB_INTERACTION_GROUP(d16_64, 16)
