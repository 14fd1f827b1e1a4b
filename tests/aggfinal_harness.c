/* gg_aggfinal.h compiled by gcc for tests/test_aggfinal.py: the finalisation rule the device applies when it writes a group as
 * a datum row, exported for ctypes */
#include "../greengage_b200/csrc/gg_aggfinal.h"

int harness_covers(int32_t aggfnoid) { return gg_aggfinal_covers(aggfnoid); }
int harness_is_float8(int32_t aggfnoid) { return gg_aggfinal_is_float8(aggfnoid); }
uint64_t harness_aggfinal(int32_t aggfnoid, uint64_t count, uint64_t n, uint64_t acc, int *isnull)
{
	return gg_aggfinal(aggfnoid, count, n, acc, isnull);
}
