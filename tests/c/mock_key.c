/* The CPU stand-in engine of mock_chain.c with cmb200_set_file_key, TEST INFRASTRUCTURE ONLY
 * (tests/test_key_file_logic.py).  Each call is logged in the call log of mock_chain.c as "key:<hex>"
 * (the key's 32 bytes) or "key:none".  Nothing of the product links against this file. */
#include "mock_chain.c"

int cmb200_set_file_key(cmb200_engine *e, const uint8_t *key) {
	(void)e;
	char what[80] = "key:none";
	if (key)
		for (int i = 0; i < 32; i++) snprintf(what + 4 + 2 * i, sizeof(what) - 4 - 2 * i, "%02x", key[i]);
	log_call(what);
	return 0;
}
