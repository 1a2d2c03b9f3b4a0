// Device restatements of what a StatsManager CSV row prints (stats_manager.py:save_to_csv), for psd_clip_stats_csv:
//   f64_decimal / f64_len / f64_write   str() of a float64, as float and numpy.float64 print it
//   timecode_of / timecode_len / timecode_write   FrameTimecode.get_timecode() at a constant rate (common.py:421-465)
//   uint_len / uint_write               a non-negative integer (the row's frame_num + 1)
// Every *_len returns the byte count *_write writes, so a counting pass and a writing pass agree without a buffer.
// Nothing here uses local memory: digits are written from the last one back, straight to their final place.
// tests/stats_csv_twin.py restates every function in Python and pins it to str() and get_timecode().
#pragma once

#include <stdint.h>

namespace psd {

// ---- str(float): the shortest decimal that reads back as x (Schubfach's interval test), in Python's repr layout ----
// g(k) = floor(10^-k * 2^(125 - floor(-k log2 10))) + 1, a 126-bit integer split into its high and low 63 bits,
// for k = -324 .. 292 (floor(q log10 2) over the binary exponents q of finite doubles).  Printed by
// `python -m tests.stats_csv_twin`, which computes it with exact integers; a CPU test compares every entry.
constexpr int kPow10Min = -324;
__device__ const ulonglong2 kPow10G[617] = {
    {0x4f0cedc95a718dd4ull, 0x5b01e8b09aa0d1b5ull}, {0x7e7b160ef71c1621ull, 0x119ca780f767b5eeull},
    {0x652f44d8c5b011b4ull, 0x0e16ec672c52f7f2ull}, {0x50f29d7a37c00e29ull, 0x581256b8f0425ff5ull},
    {0x40c21794f96671baull, 0x79a84560c0351991ull}, {0x679cf287f570b5f7ull, 0x75da089acd21c281ull},
    {0x52e3f5399126f7f9ull, 0x44ae6d48a41b0201ull}, {0x424ff76140ebf994ull, 0x36f1f106e9af34cdull},
    {0x6a198bcece465c20ull, 0x57e981a4a918547bull}, {0x54e13ca571d1e34dull, 0x2cbace1d541376c9ull},
    {0x43e763b78e4182a4ull, 0x23c8a4e44342c56eull}, {0x6ca56c58e39c043aull, 0x060dd4a06b9e08b0ull},
    {0x56eabd13e9499cfbull, 0x1e7176e6bc7e6d59ull}, {0x458897432107b0c8ull, 0x7ec12bebc9febde1ull},
    {0x6f40f20501a5e7a7ull, 0x7e01dfdfa9979635ull}, {0x5900c19d9aeb1fb9ull, 0x4b34b319547944f7ull},
    {0x4733ce17af227fc7ull, 0x55c3c27aa9fa9d93ull}, {0x71ec7cf2b1d0cc72ull, 0x560603f7765dc8eaull},
    {0x5b2397288e40a38eull, 0x7804cff92b7e3a55ull}, {0x48e945ba0b66e93full, 0x13370cc755fe9511ull},
    {0x74a86f90123e41feull, 0x51f1ae0bbcca881bull}, {0x5d538c7341cb67feull, 0x74c1580963d539afull},
    {0x4aa93d29016f8665ull, 0x43cde0078310faf3ull}, {0x77752ea8024c0a3cull, 0x0616333f381b2b1eull},
    {0x5f90f22001d66e96ull, 0x3811c298f9af55b1ull}, {0x4c73f4e667debedeull, 0x600e35472e25de28ull},
    {0x7a532170a6313164ull, 0x3349eed849d6303full}, {0x61dc1ac084f42783ull, 0x42a18be03b11c033ull},
    {0x4e49af006a5cec69ull, 0x1bb46fe695a7ccf5ull}, {0x7d42b19a43c7e0a8ull, 0x2c53e63dbc3fae55ull},
    {0x64355ae1cfd31a20ull, 0x237651cafcffbeaaull}, {0x502aaf1b0ca8e1b3ull, 0x35f8416f30cc9888ull},
    {0x402225af3d53e7c2ull, 0x5e603458f3d6e06dull}, {0x669d0918621fd937ull, 0x4a3386f4b957cd7bull},
    {0x52173a79e8197a92ull, 0x6e8f9f2a2ddfd796ull}, {0x41ac2ec7ece12edbull, 0x720c7f54f17fdfabull},
    {0x69137e0cae3517c6ull, 0x1ce0cbbb1bffcc45ull}, {0x540f980a24f74638ull, 0x171a3c95afffd69eull},
    {0x433facd4ea5f6b60ull, 0x127b63aaf3331218ull}, {0x6b991487dd657899ull, 0x6a5f05de51eb5026ull},
    {0x5614106cb11dfa14ull, 0x5518d17ea7ef7352ull}, {0x44dcd9f08db194ddull, 0x2a7a41321ff2c2a8ull},
    {0x6e2e2980e2b5bafbull, 0x5d906850331e043full}, {0x5824ee00b55e2f2full, 0x647386a68f4b3699ull},
    {0x4683f19a2ab1bf59ull, 0x36c2d21ed908f87bull}, {0x70d31c29dde93228ull, 0x579e1cfe280e5a5dull},
    {0x5a427cee4b20f4edull, 0x2c7e7d98200b7b7eull}, {0x483530bea280c3f1ull, 0x09fecae019a2c932ull},
    {0x73884dfdd0ce064eull, 0x43314499c29e0eb6ull}, {0x5c6d0b3173d8050bull, 0x4f5a9d47cee4d891ull},
    {0x49f0d5c129799da2ull, 0x72aee4397250ad41ull}, {0x764e22cea8c295d1ull, 0x377e39f583b44868ull},
    {0x5ea4e8a553cede41ull, 0x12cb61913629d387ull}, {0x4bb72084430be500ull, 0x756f8140f8217605ull},
    {0x792500d39e796e67ull, 0x6f18cece59cf233cull}, {0x60ea670fb1fabeb9ull, 0x3f470bd847d8e8fdull},
    {0x4d885272f4c89894ull, 0x329f3cad064720caull}, {0x7c0d50b7ee0dc0edull, 0x37652de1a3a50143ull},
    {0x633dda2cbe716724ull, 0x2c50f1814fb73436ull}, {0x4f64ae8a31f45283ull, 0x3d0d8e010c92902bull},
    {0x7f077da9e986ea6bull, 0x7b48e334e0ea8045ull}, {0x659f97bb2138bb89ull, 0x49071c2a4d88669dull},
    {0x514c796280fa2fa1ull, 0x20d27ceea46d1ee4ull}, {0x4109fab533fb594dull, 0x670eca58838a7f1dull},
    {0x680ff788532bc216ull, 0x0b4add5a6c10cb62ull}, {0x533ff939dc2301abull, 0x22a24aaebcda3c4eull},
    {0x4299942e49b59aefull, 0x354ea22563e1c9d8ull}, {0x6a8f537d42bc2b18ull, 0x554a9d089fcfa95aull},
    {0x553f75fdcefcef46ull, 0x776ee406e63fbaaeull}, {0x4432c4cb0bfd8c38ull, 0x5f8be99f1e996225ull},
    {0x6d1e07ab466279f4ull, 0x327975cb64289d08ull}, {0x574b3955d1e86190ull, 0x28612b091ced4a6dull},
    {0x45d5c777db204e0dull, 0x06b4226db0bdd524ull}, {0x6fbc72595e9a167bull, 0x24536a491ac95506ull},
    {0x59638eade54811fcull, 0x1d0f883a7bd44405ull}, {0x4782d88b1dd34196ull, 0x4a72d361fca9d004ull},
    {0x726af411c952028aull, 0x43eaebcffaa94cd3ull}, {0x5b88c3416ddb353bull, 0x4fef230cc88770a9ull},
    {0x493a35cdf17c2a96ull, 0x0cbf4f3d6d3926eeull}, {0x7529efafe8c6aa89ull, 0x61321862485b717cull},
    {0x5dbb262653d22207ull, 0x675b46b506af8dfdull}, {0x4afc1e850fdb4e6cull, 0x52af6bc405593e64ull},
    {0x77f9ca6e7fc54a47ull, 0x377f12d33bc1fd6dull}, {0x5ffb085866376e9full, 0x45ff42429634cabdull},
    {0x4cc8d379eb5f8bb2ull, 0x6b329b68782a3bcbull}, {0x7adaebf64565ac51ull, 0x2b842bda59dd2c77ull},
    {0x6248bcc5045156a7ull, 0x3c69bcaeae4a89f9ull}, {0x4ea0970403744552ull, 0x6387ca25583ba194ull},
    {0x7dcdbe6cd253a21eull, 0x05a6103bc05f68edull}, {0x64a498570ea94e7eull, 0x37b80cfc99e5ed8aull},
    {0x5083ad1272210b98ull, 0x2c933d96e184be08ull}, {0x40695741f4e73c79ull, 0x7075cadf1ad09807ull},
    {0x670ef2032171fa5cull, 0x4d8944982ae759a4ull}, {0x52725b35b45b2eb0ull, 0x3e076a135585e150ull},
    {0x41f515c49048f226ull, 0x64d2bb42aad1810dull}, {0x698822d41a0e503eull, 0x07b7920444826815ull},
    {0x546ce8a9ae71d9cbull, 0x1fc60e69d0685344ull}, {0x438a53baf1f4ae3cull, 0x196b3ebb0d20429dull},
    {0x6c1085f7e9877d2dull, 0x0f11fdf815006a94ull}, {0x56739e5fee05fdbdull, 0x58db319344005543ull},
    {0x45294b7ff19e6497ull, 0x60af5adc3666aa9cull}, {0x6ea878ccb5ca3a8cull, 0x344bc4938a3dddc7ull},
    {0x5886c70a2b082ed6ull, 0x5d096a0fa1cb17d2ull}, {0x46d238d4ef39bf12ull, 0x173abb3fb4a27975ull},
    {0x71505aee4b8f981dull, 0x0b912b992103f588ull}, {0x5aa6af25093face4ull, 0x0940efadb4032ad3ull},
    {0x488558ea6dcc8a50ull, 0x07672624900288a9ull}, {0x74088e43e2e0dd4cull, 0x723ea36db337410eull},
    {0x5cd3a5031be71770ull, 0x5b654f8af5c5cda5ull}, {0x4a42ea68e31f45f3ull, 0x62b772d5916b0aebull},
    {0x76d1770e38320986ull, 0x0458b7bc1bde77ddull}, {0x5f0df8d82cf4d46bull, 0x1d13c630164b9318ull},
    {0x4c0b2d79bd90a9efull, 0x30dc9e8cdea2dc13ull}, {0x79ab7bf5fc1aa97full, 0x0160fdae31049351ull},
    {0x6155fcc4c9aeedffull, 0x1ab3fe24f403a90eull}, {0x4dde63d0a158be65ull, 0x6229981d9002eda5ull},
    {0x7c97061a9bc130a2ull, 0x69dc2695b337e2a1ull}, {0x63ac04e2163426e8ull, 0x54b01ede28f9821bull},
    {0x4fbcd0b4de901f20ull, 0x43c018b1ba6134e2ull}, {0x7f9481216419cb67ull, 0x1f99c11c5d68549dull},
    {0x6610674de9ae3c52ull, 0x4c7b00e37ded107eull}, {0x51a6b90b21583042ull, 0x09fc00b5fe574065ull},
    {0x41522da2811359ceull, 0x3b3000919845cd1dull}, {0x68837c3734ebc2e3ull, 0x784ccdb5c06fae95ull},
    {0x539c635f5d8968b6ull, 0x2d0a3e2b00595877ull}, {0x42e382b2b13aba2bull, 0x3da1cb5599e11393ull},
    {0x6b059deab52ac378ull, 0x629c7888f634ec1eull}, {0x559e17eef755692dull, 0x3549fa072b5d89b1ull},
    {0x447e798bf91120f1ull, 0x1107fb38ef7e07c1ull}, {0x6d9728dff4e834b5ull, 0x01a65ec17f300c68ull},
    {0x57ac20b32a535d5dull, 0x4e1eb23465c009edull}, {0x46234d5c21dc4ab1ull, 0x24e55b5d1e333b24ull},
    {0x70387bc69c93aab5ull, 0x216ef894fd1ec506ull}, {0x59c6c96bb076222aull, 0x4df2607730e56a6cull},
    {0x47d23abc8d2b4e88ull, 0x3e5b805f5a5121f0ull}, {0x72e9f79415121740ull, 0x63c59a322a1b697full},
    {0x5bee5fa9aa74df67ull, 0x03047b5b54e2baccull}, {0x498b7fbaeec3e5ecull, 0x0269fc4910b5623dull},
    {0x75abff917e063cacull, 0x6a432d41b45569fbull}, {0x5e2332dacb38308aull, 0x21cf5767c37787fcull},
    {0x4b4f5be23c2cf3a1ull, 0x67d912b9692c6ccaull}, {0x787ef969f9e185cfull, 0x595b5128a8471476ull},
    {0x60659454c7e79e3full, 0x6115da86ed05a9f8ull}, {0x4d1e1043d31fb1ccull, 0x4dab1538bd9e2193ull},
    {0x7b634d3951cc4fadull, 0x62ab552795c9cf52ull}, {0x62b5d7610e3d0c8bull, 0x0222aa86116e3f75ull},
    {0x4ef7df80d830d6d5ull, 0x4e822204dabe992aull}, {0x7e59659af38157bcull, 0x17369cd49130f510ull},
    {0x65145148c2cddfc9ull, 0x5f5ee3dd40f3f740ull}, {0x50dd0dd3cf0b196eull, 0x1918b64a9a5cc5cdull},
    {0x40b0d7dca5a27abeull, 0x4746f83baeb09e3eull}, {0x678159610903f797ull, 0x253e59f91780fd2full},
    {0x52cde11a6d9cc612ull, 0x50feae60df9a6426ull}, {0x423e4daebe1704dbull, 0x5a65584d7faeb685ull},
    {0x69fd4917968b3af9ull, 0x10a226e265e4573bull}, {0x54caa0dfaba29594ull, 0x0d4e8581eb1d1295ull},
    {0x43d54d7fbc821143ull, 0x243ed134bc174211ull}, {0x6c887bff94034ed2ull, 0x06cae85460253682ull},
    {0x56d396661002a574ull, 0x6bd586a9e6842b9bull}, {0x457611eb40021df7ull, 0x09779eee52035616ull},
    {0x6f234fdeccd02ff1ull, 0x5bf297e3b66bbcefull}, {0x58e90cb23d73598eull, 0x165bacb62b8963f3ull},
    {0x4720d6f4fdf5e13eull, 0x451623c4efa11cc2ull}, {0x71ce24bb2fefcecaull, 0x3b569fa17f682e03ull},
    {0x5b0b5095bff30bd5ull, 0x15dee61acc535803ull}, {0x48d5da11665c0977ull, 0x2b18b8157042accfull},
    {0x74895ce8a3c6758bull, 0x5e8df355806aae18ull}, {0x5d3ab0ba1c9ec46full, 0x653e5c4466bbbe7aull},
    {0x4a955a2e7d4bd059ull, 0x3765169d1efc9861ull}, {0x77555d172edfb3c2ull, 0x256e8a94fe60f3cfull},
    {0x5f777dac257fc301ull, 0x6abed543feb3f63full}, {0x4c5f97bceacc9c01ull, 0x3bcbddcffef65e99ull},
    {0x7a328c6177adc668ull, 0x5fac961997f0975bull}, {0x61c209e792f16b86ull, 0x7fbd44e1465a12afull},
    {0x4e34d4b9425abc6bull, 0x7fca9d810514dbbfull}, {0x7d21545b9d5dfa46ull, 0x32ddc8ce6e87c5ffull},
    {0x641aa9e2e44b2e9eull, 0x5be4a0a525396b32ull}, {0x501554b5836f587eull, 0x7cb6e6ea842def5cull},
    {0x4011109135f2ad32ull, 0x30925255368b25e3ull}, {0x6681b41b89844850ull, 0x4db6ea21f0dea304ull},
    {0x52015ce2d469d373ull, 0x57c5881b2718826aull}, {0x419ab0b576bb0f8full, 0x5fd139af527a01efull},
    {0x68f781225791b27full, 0x4c81f5e550c3364aull}, {0x53f9341b79415b99ull, 0x239b2b1dda35c508ull},
    {0x432dc3492dcde2e1ull, 0x02e288e4ae916a6dull}, {0x6b7c6ba849496b01ull, 0x516a74a1174f10aeull},
    {0x55fd22ed076def34ull, 0x4121f6e745d8da25ull}, {0x44ca82573924bf5dull, 0x1a8192529e4714ebull},
    {0x6e10d08b8ea1322eull, 0x5d9c1d50fd3e87ddull}, {0x580d73a2d880f4f2ull, 0x17b01773fdcb9fe4ull},
    {0x4671294f139a5d8eull, 0x4626792997d61984ull}, {0x70b50ee4ec2a2f4aull, 0x3d0a5b75bfbcf59full},
    {0x5a2a7250bcee8c3bull, 0x4a6eaf916630c47full}, {0x4821f50d63f209c9ull, 0x21f2260deb5a36ccull},
    {0x736988156cb6760eull, 0x69837016455d247aull}, {0x5c546cddf091f80bull, 0x6e02c011d1175062ull},
    {0x49dd23e4c074c66full, 0x719bccdb0dac404eull}, {0x762e9fd467213d7full, 0x68f947c4e2ad33b0ull},
    {0x5e8bb3105280fdffull, 0x6d94396a4ef0f627ull}, {0x4ba2f5a6a8673199ull, 0x3e102deea58d91b9ull},
    {0x7904bc3dda3eb5c2ull, 0x3019e3176f48e927ull}, {0x60d09697e1cbc49bull, 0x4014b5ac590720ecull},
    {0x4d73abacb4a303afull, 0x4cdd5e237a6c1a57ull}, {0x7bec45e12104d2b2ull, 0x47c8969f2a46908aull},
    {0x63236b1a80d0a88eull, 0x6ca0787f5505406full}, {0x4f4f88e200a6ed3full, 0x0a19f9ff773766bfull},
    {0x7ee5a7d0010b1531ull, 0x5cf65ccbf1f23dfeull}, {0x6584864000d5aa8eull, 0x172b7d6ff4c1cb32ull},
    {0x5136d1cccd77bba4ull, 0x78ef978cc3ce3c28ull}, {0x40f8a7d70ac62fb7ull, 0x13f2dfa3cfd83020ull},
    {0x67f43fbe77a37f8bull, 0x398499061959e699ull}, {0x5329cc985fb5ffa2ull, 0x6136e0d1ade18548ull},
    {0x4287d6e04c91994full, 0x00f8b3daf181376dull}, {0x6a72f166e0e8f54bull, 0x1b27862b1c01f247ull},
    {0x5528c11f1a53f76full, 0x2f52d1bc1667f506ull}, {0x44209a7f48432c59ull, 0x0c424163451ff738ull},
    {0x6d00f7320d3846f4ull, 0x7a039bd208332526ull}, {0x5733f8f4d76038c3ull, 0x7b361641a028ea85ull},
    {0x45c32d90ac4cfa36ull, 0x2f5e78348020bb9eull}, {0x6f9eaf4de07b29f0ull, 0x4bca59ed99cdf8fcull},
    {0x594bbf71806287f3ull, 0x563b7b247b0b2d96ull}, {0x476fcc5acd1b9ff6ull, 0x11c92f50626f57acull},
    {0x724c7a2ae1c5ccbdull, 0x02db7ee703e55912ull}, {0x5b7061bbe7d17097ull, 0x1be2cbec031de0dcull},
    {0x4926b496530df3acull, 0x164f09899c17e716ull}, {0x750aba8a1e7cb913ull, 0x3d4b4275c68ca4f0ull},
    {0x5da22ed4e530940full, 0x4aa29b916ba3b726ull}, {0x4ae825771dc07672ull, 0x6ee87c74561c9285ull},
    {0x77d9d58b62cd8a51ull, 0x3173fa53bcfa8408ull}, {0x5fe177a2b5713b74ull, 0x278ffb7630c869a0ull},
    {0x4cb45fb55df42f90ull, 0x1fa662c4f3d387b3ull}, {0x7aba32bbc986b280ull, 0x32a3d13b1fb8d91full},
    {0x622e8efca1388ecdull, 0x0ee9742f4c93e0e6ull}, {0x4e8ba596e760723dull, 0x58bac3590a0fe71eull},
    {0x7dac3c24a5671d2full, 0x412ad228101971c9ull}, {0x6489c9b6eab8e426ull, 0x00ef0e8673478e3bull},
    {0x506e3af8bbc71cebull, 0x1a58d86b8f6c71c9ull}, {0x40582f2d6305b0bcull, 0x1513e0560c56c16eull},
    {0x66f37eaf04d5e793ull, 0x3b530089ad579be2ull}, {0x525c6558d0ab1fa9ull, 0x15dc006e2446164full},
    {0x41e384470d55b2edull, 0x5e4999f1b69e783full}, {0x696c06d81555eb15ull, 0x7d428fe92430c065ull},
    {0x54566be0111188deull, 0x31020cba835a3384ull}, {0x4378564cda746d7eull, 0x5a680a2ecf7b5c69ull},
    {0x6bf3bd47c3ed7bfdull, 0x770cdd17b25efa42ull}, {0x565c976c9cbdfccbull, 0x1270b0dfc1e59502ull},
    {0x4516df8a16fe63d5ull, 0x5b8d5a4c9b1e10ceull}, {0x6e8aff4357fd6c89ull, 0x127bc3adc4fce7b0ull},
    {0x586f329c466456d4ull, 0x0ec96957d0ca52f3ull}, {0x46bf5bb038504576ull, 0x3f07877973d50f29ull},
    {0x71322c4d26e6d58aull, 0x31a5a58f1fbb4b75ull}, {0x5a8e89d75252446eull, 0x5aeaead8e62f6f91ull},
    {0x487207df750e9d25ull, 0x2f22557a51bf8c74ull}, {0x73e9a63254e42ea2ull, 0x1836ef2a1c65ad86ull},
    {0x5cbaeb5b771cf21bull, 0x2cf8bf54e3848ad2ull}, {0x4a2f22af927d8e7cull, 0x23fa32aa4f9d3bdbull},
    {0x76b1d118ea627d93ull, 0x5329eaaa18fb92f8ull}, {0x5ef4a74721e86476ull, 0x0f54bbbb472fa8c6ull},
    {0x4bf6ec38e7ed1d2bull, 0x25dd62fc38f2ed6cull}, {0x798b138e3fe1c845ull, 0x22fbd1938e517bdfull},
    {0x613c0fa4ffe7d36aull, 0x4f2fdadc71dac97full}, {0x4dc9a61d998642bbull, 0x58f3157d27e23accull},
    {0x7c75d695c2706ac5ull, 0x74b82261d969f7adull}, {0x63917877cec0556bull, 0x10934eb4adee5fbeull},
    {0x4fa793930bcd1122ull, 0x4075d8908b251965ull}, {0x7f7285b812e1b504ull, 0x00bc8db411d4f56eull},
    {0x65f537c675815d9cull, 0x66fd3e29a7dd9125ull}, {0x5190f96b91344ae3ull, 0x6bfdcb54864ada84ull},
    {0x4140c78940f6a24full, 0x6ffe3c439ea2486aull}, {0x6867a5a867f103b2ull, 0x7ffd2d38fdd073dcull},
    {0x53861e2053273628ull, 0x6664242d97d9f64aull}, {0x42d1b1b375b8f820ull, 0x51e9b68adfe191d5ull},
    {0x6ae91c5255f4c034ull, 0x1ca924116635b621ull}, {0x558749db77f70029ull, 0x63ba83411e915e81ull},
    {0x446c3b15f9926687ull, 0x6962029a7edab201ull}, {0x6d79f82328ea3da6ull, 0x0f03375d97c45001ull},
    {0x5794c6828721caebull, 0x259c2c4adfd04001ull}, {0x46109eced2816f22ull, 0x5149bd08b30d0001ull},
    {0x701a97b150cf1837ull, 0x3542c80deb480001ull}, {0x59aedfc10d7279c5ull, 0x7768a00b22a00001ull},
    {0x47bf19673df52e37ull, 0x79208008e8800001ull}, {0x72cb5bd86321e38cull, 0x5b67334174000001ull},
    {0x5bd5e313828182d6ull, 0x7c528f6790000001ull}, {0x4977e8dc68679bdfull, 0x16a872b940000001ull},
    {0x758ca7c70d7292feull, 0x5773eac200000001ull}, {0x5e0a1fd271287598ull, 0x45f6556800000001ull},
    {0x4b3b4ca85a86c47aull, 0x04c5112000000001ull}, {0x785ee10d5da46d90ull, 0x07a1b50000000001ull},
    {0x604be73de4838ad9ull, 0x52e7c40000000001ull}, {0x4d0985cb1d3608aeull, 0x0f1fd00000000001ull},
    {0x7b426fab61f00de3ull, 0x31cc800000000001ull}, {0x629b8c891b267182ull, 0x5b0a000000000001ull},
    {0x4ee2d6d415b85aceull, 0x7c08000000000001ull}, {0x7e37be2022c0914bull, 0x1340000000000001ull},
    {0x64f964e68233a76full, 0x2900000000000001ull}, {0x50c783eb9b5c85f2ull, 0x5400000000000001ull},
    {0x409f9cbc7c4a04c2ull, 0x1000000000000001ull}, {0x6765c793fa10079dull, 0x0000000000000001ull},
    {0x52b7d2dcc80cd2e4ull, 0x0000000000000001ull}, {0x422ca8b0a00a4250ull, 0x0000000000000001ull},
    {0x69e10de76676d080ull, 0x0000000000000001ull}, {0x54b40b1f852bda00ull, 0x0000000000000001ull},
    {0x43c33c1937564800ull, 0x0000000000000001ull}, {0x6c6b935b8bbd4000ull, 0x0000000000000001ull},
    {0x56bc75e2d6310000ull, 0x0000000000000001ull}, {0x4563918244f40000ull, 0x0000000000000001ull},
    {0x6f05b59d3b200000ull, 0x0000000000000001ull}, {0x58d15e1762800000ull, 0x0000000000000001ull},
    {0x470de4df82000000ull, 0x0000000000000001ull}, {0x71afd498d0000000ull, 0x0000000000000001ull},
    {0x5af3107a40000000ull, 0x0000000000000001ull}, {0x48c2739500000000ull, 0x0000000000000001ull},
    {0x746a528800000000ull, 0x0000000000000001ull}, {0x5d21dba000000000ull, 0x0000000000000001ull},
    {0x4a817c8000000000ull, 0x0000000000000001ull}, {0x7735940000000000ull, 0x0000000000000001ull},
    {0x5f5e100000000000ull, 0x0000000000000001ull}, {0x4c4b400000000000ull, 0x0000000000000001ull},
    {0x7a12000000000000ull, 0x0000000000000001ull}, {0x61a8000000000000ull, 0x0000000000000001ull},
    {0x4e20000000000000ull, 0x0000000000000001ull}, {0x7d00000000000000ull, 0x0000000000000001ull},
    {0x6400000000000000ull, 0x0000000000000001ull}, {0x5000000000000000ull, 0x0000000000000001ull},
    {0x4000000000000000ull, 0x0000000000000001ull}, {0x6666666666666666ull, 0x3333333333333334ull},
    {0x51eb851eb851eb85ull, 0x0f5c28f5c28f5c29ull}, {0x4189374bc6a7ef9dull, 0x5916872b020c49bbull},
    {0x68db8bac710cb295ull, 0x74f0d844d013a92bull}, {0x53e2d6238da3c211ull, 0x43f3e0370cdc8755ull},
    {0x431bde82d7b634daull, 0x698fe69270b06c44ull}, {0x6b5fca6af2bd215eull, 0x0f4ca41d811a46d4ull},
    {0x55e63b88c230e77eull, 0x3f70834acdae9f10ull}, {0x44b82fa09b5a52cbull, 0x4c5a02a23e254c0dull},
    {0x6df37f675ef6eadfull, 0x2d5cd10396a21347ull}, {0x57f5ff85e592557full, 0x3de3da69454e75d3ull},
    {0x465e6604b7a84465ull, 0x7e4fe1edd10b9175ull}, {0x709709a125da0709ull, 0x4a19697c81ac1befull},
    {0x5a126e1a84ae6c07ull, 0x54e1213067bce326ull}, {0x480ebe7b9d58566cull, 0x43e74dc052fd8285ull},
    {0x734aca5f6226f0adull, 0x530baf9a1e626a6dull}, {0x5c3bd5191b525a24ull, 0x426fbfae7eb521f1ull},
    {0x49c97747490eae83ull, 0x4ebfcc8b9890e7f4ull}, {0x760f253edb4ab0d2ull, 0x4acc7a78f41b0cbaull},
    {0x5e72843249088d75ull, 0x223d2ec729af3d62ull}, {0x4b8ed0283a6d3df7ull, 0x34fdbf05baf29781ull},
    {0x78e480405d7b9658ull, 0x54c931a2c4b758cfull}, {0x60b6cd004ac94513ull, 0x5d6dc14f03c5e0a5ull},
    {0x4d5f0a66a23a9da9ull, 0x31249aa59c9e4d51ull}, {0x7bcb43d769f762a8ull, 0x4ea0f76f60fd4882ull},
    {0x63090312bb2c4eedull, 0x254d92bf80caa068ull}, {0x4f3a68dbc8f03f24ull, 0x1dd7a89933d54d20ull},
    {0x7ec3daf941806506ull, 0x62f2a75b86221500ull}, {0x65697bfa9acd1d9full, 0x025bb91604e810cdull},
    {0x51212ffbaf0a7e18ull, 0x684960de6a5340a4ull}, {0x40e7599625a1fe7aull, 0x203ab3e521dc33b6ull},
    {0x67d88f56a29cca5dull, 0x19f7863b696052bdull}, {0x5313a5dee87d6eb0ull, 0x7b2c6b62bab37564ull},
    {0x42761e4bed31255aull, 0x2f56bc4efbc2c450ull}, {0x6a5696dfe1e83bc3ull, 0x655793b192d13a1aull},
    {0x5512124cb4b9c969ull, 0x377942f475742e7bull}, {0x440e750a2a2e3abaull, 0x5f9435905df68b96ull},
    {0x6ce3ee76a9e3912aull, 0x65b9ef4d63241289ull}, {0x571cbec554b60dbbull, 0x6afb25d782834207ull},
    {0x45b0989ddd5e7163ull, 0x08c8eb12cecf6806ull}, {0x6f80f42fc8971bd1ull, 0x5adb11b7b14bd9a3ull},
    {0x5933f68ca078e30eull, 0x157c0e2c8dd647b5ull}, {0x475cc53d4d2d8271ull, 0x5dfcd823a4ab6c91ull},
    {0x722e086215159d82ull, 0x632e269f6ddf141bull}, {0x5b5806b4ddaae468ull, 0x4f581ee5f17f4349ull},
    {0x49133890b1558386ull, 0x72ace584c1329c3bull}, {0x74eb8db44eef38d7ull, 0x6aae3c079b842d2aull},
    {0x5d893e29d8bf60acull, 0x5558300616035755ull}, {0x4ad431bb13cc4d56ull, 0x7779c004de6912abull},
    {0x77b9e92b52e07bbeull, 0x258f99a163db5111ull}, {0x5fc7edbc424d2fcbull, 0x37a614811caf740dull},
    {0x4c9ff163683dbfd5ull, 0x7951aa00e3bf900bull}, {0x7a998238a6c932efull, 0x754f7667d2cc19abull},
    {0x6214682d523a8f26ull, 0x2aa5f8530f09ae22ull}, {0x4e76b9bddb620c1eull, 0x55519375a5a1581bull},
    {0x7d8ac2c95f034697ull, 0x3bb5b8bc3c3559c5ull}, {0x646f023ab2690545ull, 0x7c9160969691149eull},
    {0x5058ce955b87376bull, 0x16dab3ababa743b2ull}, {0x40470baaaf9f5f88ull, 0x78aef622efb902f5ull},
    {0x66d812aab29898dbull, 0x0de4bd04b2c19e54ull}, {0x524675555bad4715ull, 0x57ea30d08f014b76ull},
    {0x41d1f7777c8a9f44ull, 0x4654f3da0c01092cull}, {0x694ff258c7443207ull, 0x23bb1fc346680eacull},
    {0x543ff513d29cf4d2ull, 0x4fc8e635d1ecd88aull}, {0x43665da9754a5d75ull, 0x263a51c4a7f0ad3bull},
    {0x6bd6fc425543c8bbull, 0x56c3b607731aaec4ull}, {0x5645969b77696d62ull, 0x789c919f8f488bd0ull},
    {0x4504787c5f878ab5ull, 0x46e3a7b2d906d640ull}, {0x6e6d8d93cc0c1122ull, 0x3e390c515b3e239aull},
    {0x5857a4763cd6741bull, 0x4b60d6a77c31b615ull}, {0x46ac8391ca4529afull, 0x55e7121f968e2b44ull},
    {0x711405b6106ea919ull, 0x0971b698f0e3786dull}, {0x5a766af80d255414ull, 0x078e2bad8d82c6bdull},
    {0x485ebbf9a41ddcdcull, 0x6c71bc8ad79bd231ull}, {0x73cac65c39c96161ull, 0x2d82c7448c2c8382ull},
    {0x5ca23849c7d44de7ull, 0x3e023903a356cf9bull}, {0x4a1b603b06437185ull, 0x7e682d9c82abd949ull},
    {0x76923391a39f1c09ull, 0x4a4048fa6aac8edbull}, {0x5edb5c7482e5b007ull, 0x55003a61eef07249ull},
    {0x4be2b05d35848cd2ull, 0x773361e7f259f507ull}, {0x796ab3c855a0e151ull, 0x3eb89ca6508fee71ull},
    {0x6122296d114d810dull, 0x7efa16eb73a6585bull}, {0x4db4edf0daa4673eull, 0x3261abef8fb846afull},
    {0x7c54afe7c43a3ecaull, 0x1d691318e5f3a44bull}, {0x6376f31fd02e98a1ull, 0x64540f471e5c836full},
    {0x4f925c1973587a1bull, 0x0376729f4b7d35f3ull}, {0x7f50935bebc0c35eull, 0x38bd84321261efebull},
    {0x65da0f7cbc9a35e5ull, 0x13cad0280eb4bfefull}, {0x517b3f96fd482b1dull, 0x5ca240200bc3ccbfull},
    {0x412f66126439bc17ull, 0x63b50019a3030a33ull}, {0x684bd683d38f9359ull, 0x1f88002904d1a9eaull},
    {0x536fdecfdc72dc47ull, 0x32d3335403daee55ull}, {0x42bfe57316c249d2ull, 0x5bdc291003158b77ull},
    {0x6acca251be03a951ull, 0x12f9db4cd1bc1258ull}, {0x557081dafe695440ull, 0x7594af70a7c9a847ull},
    {0x445a017bfebaa9cdull, 0x4476f2c0863aed06ull}, {0x6d5ccf2ccac442e2ull, 0x3a57eacda3917b3cull},
    {0x577d728a3bd03581ull, 0x7b7988a482dac8fdull}, {0x45fdf53b630cf79bull, 0x15fad3b6cf156d97ull},
    {0x6ffcbb923814bf5eull, 0x565e1f8ae4ef15beull}, {0x5996fc74f9aa32b2ull, 0x11e4e608b725aaffull},
    {0x47abfd2a6154f55bull, 0x27ea51a0928488ccull}, {0x72acc843ceee555eull, 0x7310829a84074146ull},
    {0x5bbd6d030bf1dde5ull, 0x42739baed005cdd2ull}, {0x49645735a327e4b7ull, 0x4ec2e2f24004a4a8ull},
    {0x756d5855d1d96df2ull, 0x4ad16b1d333aa10cull}, {0x5df11377db1457f5ull, 0x2241227dc2954da3ull},
    {0x4b2742c648dd132aull, 0x4e9a81fe35443e1cull}, {0x783ed13d4161b844ull, 0x175d9cc9eed39694ull},
    {0x603240fdcde7c69cull, 0x7917b0a18bdc7876ull}, {0x4cf500cb0b1fd217ull, 0x1412f3b46fe39392ull},
    {0x7b219ade7832e9beull, 0x535185ed7fd285b6ull}, {0x628148b1f9c25498ull, 0x42a79e57997537c5ull},
    {0x4ecdd3c1949b76e0ull, 0x3552e512e12a9304ull}, {0x7e161f9c20f8be33ull, 0x6eeb081e3510eb39ull},
    {0x64de7fb01a609829ull, 0x3f226ce4f740bc2eull}, {0x50b1ffc0151a1354ull, 0x3281f0b72c33c9beull},
    {0x408e66334414dc43ull, 0x42018d5f568fd498ull}, {0x674a3d1ed354939full, 0x1ccf48988a7fba8dull},
    {0x52a1ca7f0f76dc7full, 0x30a5d3ad3b99620bull}, {0x421b0865a5f8b065ull, 0x73b7dc8a96144e6full},
    {0x69c4da3c3cc11a3cull, 0x52bfc7442353b0b1ull}, {0x549d7b6363cdae96ull, 0x756639034f7626f4ull},
    {0x43b12f82b63e2545ull, 0x4451c735d92b525dull}, {0x6c4eb26abd303ba2ull, 0x3a1c71efc1deea2eull},
    {0x56a55b889759c94eull, 0x61b05b2634b254f2ull}, {0x45511606df7b0772ull, 0x1af37c1e908eaa5bull},
    {0x6ee8233e325e7250ull, 0x2b1f2cfdb41776f8ull}, {0x58b9b5cb5b7ec1d9ull, 0x6f4c23fe29ac5f2dull},
    {0x46faf7d5e2cbce47ull, 0x72a34ffe87bd18f1ull}, {0x71918c896adfb073ull, 0x04387ffda5fb5b1bull},
    {0x5adad6d4557fc05cull, 0x0360666484c915afull}, {0x48af1243779966b0ull, 0x02b3851d3707448cull},
    {0x744b506bf28f0ab3ull, 0x1dec082ebe720746ull}, {0x5d090d2328726ef5ull, 0x64bcd358985b3905ull},
    {0x4a6da41c205b8bf7ull, 0x6a30a913ad15c738ull}, {0x7715d36033c5acbfull, 0x5d1aa81f7b560b8cull},
    {0x5f44a919c3048a32ull, 0x7daeece5fc44d609ull}, {0x4c36edae359d3b5bull, 0x7e258a51969d7808ull},
    {0x79f17c49ef61f893ull, 0x16a276e8f0fbf33full}, {0x618dfd07f2b4c6dcull, 0x121b9253f3fcc299ull},
    {0x4e0b30d328909f16ull, 0x41afa84329970214ull}, {0x7cdeb4850db431bdull, 0x4f7f739ea8f19cedull},
    {0x63e55d373e29c164ull, 0x3f99294bba5ae3f1ull}, {0x4feab0f8fe87cde9ull, 0x7fadbaa2fb7be98dull},
    {0x7fdde7f4ca72e30full, 0x7f7c5dd1925fdc15ull}, {0x664b1ff7085be8d9ull, 0x4c637e4141e649abull},
    {0x51d5b32c06afed7aull, 0x704f983434b83aefull}, {0x4177c2899ef32462ull, 0x26a6135cf6f9c8bfull},
    {0x68bf9da8fe51d3d0ull, 0x3dd685618b294132ull}, {0x53cc7e20cb74a973ull, 0x4b12044e08edcdc2ull},
    {0x4309fe80a2c3bac2ull, 0x6f419d0b3a57d7ceull}, {0x6b4330cdd1392ad1ull, 0x320294dec3bfbfb0ull},
    {0x55cf5a3e40fa88a7ull, 0x419baa4bcfcc995aull}, {0x44a5e1cb672ed3b9ull, 0x1ae2eea30ca3ade1ull},
    {0x6dd636123eb152c1ull, 0x77d17dd1add2afcfull}, {0x57de91a832277567ull, 0x797464a7be42263full},
    {0x464ba7b9c1b92ab9ull, 0x4790508631ce84ffull}, {0x70790c5c6928445cull, 0x0c1a1a704fb0d4ccull},
    {0x59fa7049edb9d049ull, 0x567b4859d95a43d6ull}, {0x47fb8d07f161736eull, 0x11fc39e17aae9cabull},
    {0x732c14d98235857dull, 0x032d2968c44a9445ull}, {0x5c2343e134f79dfdull, 0x4f575453d03ba9d1ull},
    {0x49b5cfe75d92e4caull, 0x72ac4376402fbb0eull}, {0x75efb30bc8eb07abull, 0x0446d256cd192b49ull},
    {0x5e595c096d88d2efull, 0x1d0575123dadbc3aull}, {0x4b7ab0078ad3dbf2ull, 0x4a6ac40e97be302full},
    {0x78c44cd8de1fc650ull, 0x771139b0f2c9e6b1ull}, {0x609d0a4718196b73ull, 0x78da948d8f07ebc1ull},
    {0x4d4a6e9f467abc5cull, 0x60aedd3e0c065634ull}, {0x7baa4a9870c46094ull, 0x344afb9679a3bd20ull},
    {0x62eea2138d69e6ddull, 0x103bfc78614fca80ull}, {0x4f254e760abb1f17ull, 0x26966393810ca200ull},
    {0x7ea21723445e9825ull, 0x2423d2859b476999ull}, {0x654e78e9037ee01dull, 0x69b642047c392148ull},
    {0x510b93ed9c658017ull, 0x6e2b680396941aa0ull}, {0x40d60ff149eaccdfull, 0x71bc53361210154dull},
    {0x67bce64edcaae166ull, 0x1c6085235019bbaeull}, {0x52fd850be3bbe784ull, 0x7d1a041c40149625ull},
    {0x42646a6fe9631f9dull, 0x4a7b367d0010781dull}, {0x6a3a43e642383295ull, 0x5d91f0c8001a59c8ull},
    {0x54fb698501c68edeull, 0x17a7f3d3334847d4ull}, {0x43fc546a67d20be4ull, 0x79532975c2a03976ull},
    {0x6cc6ed770c83463bull, 0x0eeb75893766c256ull}, {0x57058ac5a39c382full, 0x25892ad42c523512ull},
    {0x459e089e1c7cf9bfull, 0x37a0ef102374f742ull}, {0x6f6340fcfa618f98ull, 0x59017e8038bb2536ull},
    {0x591c33fd951ad946ull, 0x7a67986693c8ea91ull}, {0x4749c33144157a9full, 0x151fad1edca0bba8ull},
    {0x720f9eb539bbf765ull, 0x0832ae97c76792a5ull}, {0x5b3fb22a94965f84ull, 0x068ef21305ec7551ull},
    {0x48ffc1bbaa11e603ull, 0x1ed8c1a8d189f774ull}, {0x74cc692c434fd66bull, 0x4af4690e1c0ff253ull},
    {0x5d705423690cab89ull, 0x225d20d816732843ull}, {0x4ac0434f873d5607ull, 0x35174d79ab8f5369ull},
    {0x779a054c0b955672ull, 0x21bee25c45b21f0eull}, {0x5fae6aa33c77785bull, 0x3498b5169e2818d8ull},
    {0x4c8b888296c5f9e2ull, 0x5d46f7454b534713ull}, {0x7a78da6a8ad65c9dull, 0x7ba4bed545520b52ull},
    {0x61fa48553bdeb07eull, 0x2fb6ff110441a2a8ull}, {0x4e61d37763188d31ull, 0x72f8cc0d9d014eedull},
    {0x7d6952589e8daeb6ull, 0x1e5ae015c80217e1ull}, {0x645441e07ed7bef8ull, 0x1848b344a001acb4ull},
    {0x504367e6cbdfcbf9ull, 0x603a2903b3348a2aull}, {0x4035ecb8a3196ffbull, 0x002e873628f6d4eeull},
    {0x66bcadf43828b32bull, 0x19e40b89db2487e3ull}, {0x52308b29c686f5bcull, 0x14b66fa17c1d3983ull},
    {0x41c06f549ed25e30ull, 0x1091f2e7967dc79cull}, {0x6933e554315096b3ull, 0x341cb7d8f0c93f5full},
    {0x542984435aa6def5ull, 0x767d5fe0c0a0ff80ull}, {0x435469cf7bb8b25eull, 0x2b977fe70080cc66ull},
    {0x6bba42e592c11d63ull, 0x5f58cca4cd9ae0a3ull}, {0x562e9beadbcdb11cull, 0x4c470a1d7148b3b6ull},
    {0x44f216557ca48db0ull, 0x3d05a1b1276d5c92ull}, {0x6e5023bbfaa0e2b3ull, 0x7b3c35e83f1560e9ull},
    {0x58401c96621a4ef6ull, 0x2f635e5365aab3edull}, {0x4699b0784e7b725eull, 0x591c4b75eaeef658ull},
    {0x70f5e726e3f8b6fdull, 0x74fa125644b18a26ull}, {0x5a5e5285832d5f31ull, 0x43fb41de9d5ad4ebull},
    {0x484b75379c244c27ull, 0x4ffc34b2177bdd89ull}, {0x73abeebf603a1372ull, 0x4cc6bab68bf96274ull},
    {0x5c898bcc4cfb42c2ull, 0x0a38955ed6611b90ull}, {0x4a07a309d72f689bull, 0x21c6dde5784dafa7ull},
    {0x76729e762518a75eull, 0x693e2fd58d49190bull}, {0x5ec2185e8413b918ull, 0x5431bfde0aa0e0d5ull},
    {0x4bce79e536762dadull, 0x29c1664b3bb3e711ull}, {0x794a5ca1f0bd15e2ull, 0x0f9bd6dec5eca4e8ull},
    {0x61084a1b26fdab1bull, 0x2616457f04bd50baull}, {0x4da03b48ebfe227cull, 0x1e783798d09773c8ull},
    {0x7c33920e46636a60ull, 0x30c058f480f252d9ull}, {0x635c74d8384f884dull, 0x0d66ad9067284247ull},
    {0x4f7d2a469372d370ull, 0x711ef14052869b6cull}, {0x7f2eaa0a85848581ull, 0x34fe4ecd50d75f14ull},
    {0x65beee6ed136d134ull, 0x2a650bd773df7f43ull}, {0x51658b8bda9240f6ull, 0x551da312c319329cull},
    {0x411e093caedb672bull, 0x5db14f4235adc217ull}, {0x68300ec77e2bd845ull, 0x7c4ee536bc49368aull},
    {0x5359a56c64efe037ull, 0x7d0bea92303a9208ull}, {0x42ae1df050bfe693ull, 0x173cbba8269541a0ull},
    {0x6ab02fe6e79970ebull, 0x3ec792a6a422029aull}, {0x5559bfebec7ac0bcull, 0x3239421ee9b4cee1ull},
    {0x4447ccbcbd2f0096ull, 0x5b6101b25490a581ull}, {0x6d3fadfac84b3424ull, 0x2bce691d541aa268ull},
    {0x576624c8a03c29b6ull, 0x563eba7ddce21b87ull}, {0x45eb50a08030215eull, 0x78322ecb171b4939ull},
    {0x6fdee76733803564ull, 0x59e9e47824f87527ull}, {0x597f1f85c2ccf783ull, 0x6187e9f9b72d2a86ull},
    {0x4798e6049bd72c69ull, 0x346cbb2e2c242205ull}, {0x728e3cd42c8b7a42ull, 0x20adf849e039d007ull},
    {0x5ba4fd768a092e9bull, 0x33be603b19c7d99full}, {0x4950cac53b3a8bafull, 0x42feb3627b0647b3ull},
    {0x754e113b91f745e5ull, 0x5197856a5e7072b8ull}, {0x5dd80dc941929e51ull, 0x27ac6abb7ec05bc6ull},
    {0x4b133e3a9adbb1daull, 0x52f05562cbcd1638ull}, {0x781ec9f75e2c4fc4ull, 0x1e4d556adfae89f3ull},
    {0x6018a192b1bd0c9cull, 0x7ea444557fbed4c3ull}, {0x4ce0814227ca707dull, 0x4bb69d1132ff109cull},
    {0x7b00ced03faa4d95ull, 0x5f8a94e851981a93ull}, {0x62670bd9cc883e11ull, 0x32d543ed0e134875ull},
    {0x4eb8d647d6d364daull, 0x5bddcff0d80f6d2bull}, {0x7df48a0c8aebd491ull, 0x12fc7fe7c018aeabull},
    {0x64c3a1a3a25643a7ull, 0x28c9ffec99ad5889ull}, {0x509c814fb511cfb9ull, 0x0707fff07af113a1ull},
    {0x407d343fc40e3fc7ull, 0x1f39998d2f2742e7ull}, {0x672eb9ffa016cc71ull, 0x7ec28f484b7204a4ull},
    {0x528bc7ffb345705bull, 0x189ba5d36f8e6a1dull}, {0x42096ccc8f6ac048ull, 0x7a161e42bfa521b1ull},
    {0x69a8ae1418aacd41ull, 0x435696d132a1cf81ull}, {0x5486f1a9ad557101ull, 0x1c454574288172ceull},
    {0x439f27baf1112734ull, 0x169dd129ba0128a5ull}, {0x6c31d92b1b4ea520ull, 0x242fb50f9001daa1ull},
    {0x568e4755af721db3ull, 0x368c90d940017bb4ull}, {0x453e9f77bf8e7e29ull, 0x120a0d7a999ac95dull},
    {0x6eca98bf98e3fd0eull, 0x50101590f5c47561ull}, {0x58a213cc7a4ffda5ull, 0x26734473f7d05de8ull},
    {0x46e80fd6c83ffe1dull, 0x6b8f69f65fd9e4b9ull}, {0x71734c8ad9fffcfcull, 0x45b24323cc8fd45cull},
    {0x5ac2a3a247fffd96ull, 0x6af502830a0ca9e3ull}, {0x489bb61b6ccccadfull, 0x08c402026e7087e9ull},
    {0x742c569247ae1164ull, 0x746cd003e3e73fdbull}, {0x5cf04541d2f1a783ull, 0x76bd73364fec3315ull},
    {0x4a59d101758e1f9cull, 0x5efdf5c50cbcf5abull}, {0x76f61b3588e365c7ull, 0x4b2fefa1adfb22abull},
    {0x5f2b48f7a0b5eb06ull, 0x08f3261af195b555ull}, {0x4c22a0c61a2b226bull, 0x20c284e25ade2aabull},
    {0x79d1013cf6ab6a45ull, 0x1ad0d49d5e304444ull}, {0x617400fd9222bb6aull, 0x48a7107de4f369d0ull},
    {0x4df6673141b562bbull, 0x53b8d9fe50c2bb0dull}, {0x7cbd71e869223792ull, 0x52c15cca1ad12b48ull},
    {0x63cac186ba81c60eull, 0x75677d6e7bda8906ull}, {0x4fd5679efb9b04d8ull, 0x5dec645863153a6cull},
    {0x7fbbd8fe5f5e6e27ull, 0x497a3a2704eec3dfull},
};

__device__ __forceinline__ int flog10pow2(int e) { return (int)(((int64_t)e * 661971961083LL) >> 41); }
__device__ __forceinline__ int flog10three_quarters_pow2(int e) {
    return (int)(((int64_t)e * 661971961083LL - 274743187321LL) >> 41);
}
__device__ __forceinline__ int flog2pow10(int e) { return (int)(((int64_t)e * 913124641741LL) >> 38); }

// floor(g * cp / 2^127) with a sticky low bit: 1 when bits below were dropped (round to odd)
__device__ __forceinline__ uint64_t round_odd(uint64_t g1, uint64_t g0, uint64_t cp) {
    const uint64_t x1 = __umul64hi(g0, cp);
    const uint64_t y0 = g1 * cp;
    const uint64_t y1 = __umul64hi(g1, cp);
    const uint64_t z = (y0 >> 1) + x1;
    const uint64_t vbp = y1 + (z >> 63);
    return vbp | (((z & 0x7FFFFFFFFFFFFFFFull) + 0x7FFFFFFFFFFFFFFFull) >> 63);
}

struct Decimal {
    uint64_t f;    // significant digits, no trailing zero (finite nonzero x)
    int32_t e10;   // decimal exponent of the first digit
    int32_t n;     // number of digits of f
    int32_t kind;  // 0 finite nonzero, 1 zero, 2 infinity, 3 NaN
    bool neg;      // sign bit (NaN prints without it, as Python prints it)
};

__device__ __forceinline__ int uint_len(uint64_t v) {
    int n = 1;
    for (uint64_t p = 10; n < 20 && v >= p; p *= 10) ++n;
    return n;
}

// the shortest f * 10^e in the rounding interval of c * 2^q (c >= 3), the nearest when there are two; ties to even
__device__ __forceinline__ void schubfach(int q, uint64_t c, uint64_t& f, int& e) {
    const uint64_t out = c & 1;  // an even significand's interval includes its ends (round half to even reads back)
    const uint64_t cb = c << 2, cbr = cb + 2;
    uint64_t cbl;
    int k;
    if (c != (1ull << 52) || q == -1074) {
        cbl = cb - 2;
        k = flog10pow2(q);
    } else {  // the lower neighbour is half as far: the interval is asymmetric
        cbl = cb - 1;
        k = flog10three_quarters_pow2(q);
    }
    const int h = q + flog2pow10(-k) + 2;
    const ulonglong2 g = kPow10G[k - kPow10Min];
    const uint64_t vb = round_odd(g.x, g.y, cb << h);
    const uint64_t vbl = round_odd(g.x, g.y, cbl << h);
    const uint64_t vbr = round_odd(g.x, g.y, cbr << h);
    const uint64_t s = vb >> 2;
    e = k;
    if (s >= 10) {  // one digit fewer, if a multiple of ten lies in the interval
        const uint64_t sp10 = 10 * __umul64hi(s, 115292150460684698ull << 4), tp10 = sp10 + 10;
        const bool upin = vbl + out <= sp10 << 2;
        const bool wpin = (tp10 << 2) + out <= vbr;
        if (upin != wpin) {
            f = upin ? sp10 : tp10;
            return;
        }
    }
    const uint64_t t = s + 1;
    const bool uin = vbl + out <= s << 2;
    const bool win = (t << 2) + out <= vbr;
    if (uin != win) {
        f = uin ? s : t;
        return;
    }
    const int64_t cmp = (int64_t)(vb - ((s + t) << 1));
    f = (cmp < 0 || (cmp == 0 && (s & 1) == 0)) ? s : t;
}

__device__ __forceinline__ Decimal f64_decimal(double x) {
    const uint64_t bits = (uint64_t)__double_as_longlong(x);
    const int bq = (int)((bits >> 52) & 0x7FF);
    const uint64_t t = bits & ((1ull << 52) - 1);
    Decimal d{0, 0, 0, 0, (bits >> 63) != 0};
    if (bq == 0x7FF) {
        d.kind = t ? 3 : 2;
        return d;
    }
    if (bq == 0 && t == 0) {
        d.kind = 1;
        return d;
    }
    uint64_t f;
    int e;
    if (bq) {
        const int mq = 1075 - bq;  // x = c * 2^-mq
        const uint64_t c = (1ull << 52) | t;
        if (mq > 0 && mq < 53 && ((c >> mq) << mq) == c) {  // an integer below 2^53 prints exactly
            f = c >> mq;
            e = 0;
        } else {
            schubfach(-mq, c, f, e);
        }
    } else if (t < 3) {  // 2^-1074 and 2^-1073: their intervals are too narrow for the table's precision
        f = t == 1 ? 5 : 1;
        e = t == 1 ? -324 : -323;
    } else {
        schubfach(-1074, t, f, e);
    }
    while (f % 10 == 0) {
        f /= 10;
        ++e;
    }
    d.f = f;
    d.n = uint_len(f);
    d.e10 = e + d.n - 1;
    return d;
}

// repr layout: fixed notation for decimal exponents -4 .. 15 ("0.0001", "27.0"), else "1e-05", "1.5e+16"
__device__ __forceinline__ int f64_len(const Decimal& d) {
    if (d.kind == 3) return 3;                  // nan
    const int sign = d.neg ? 1 : 0;
    if (d.kind == 2) return sign + 3;           // inf
    if (d.kind == 1) return sign + 3;           // 0.0
    if (d.e10 >= -4 && d.e10 <= 15) {
        if (d.e10 < 0) return sign + 1 - d.e10 + d.n;          // 0.000ddd
        if (d.e10 + 1 < d.n) return sign + d.n + 1;            // dd.ddd
        return sign + d.e10 + 1 + 2;                           // dd000.0
    }
    const int ae = d.e10 < 0 ? -d.e10 : d.e10;
    return sign + d.n + (d.n > 1 ? 1 : 0) + 2 + (ae >= 100 ? 3 : 2);  // d.ddde+XX
}

// the digits of v, n of them (zero-padded on the left), digit j at out[j] or out[j + 1] from j = point on
__device__ __forceinline__ void put_digits(uint64_t v, int n, char* out, int point) {
    for (int j = n - 1; j >= 0; --j) {
        out[j + (j >= point ? 1 : 0)] = (char)('0' + v % 10);
        v /= 10;
    }
}

__device__ __forceinline__ void put3(char* out, char a, char b, char c) {
    out[0] = a;
    out[1] = b;
    out[2] = c;
}

__device__ __forceinline__ char* f64_write(const Decimal& d, char* out) {
    if (d.kind == 3) {
        put3(out, 'n', 'a', 'n');
        return out + 3;
    }
    if (d.neg) *out++ = '-';
    if (d.kind == 2) {
        put3(out, 'i', 'n', 'f');
        return out + 3;
    }
    if (d.kind == 1) {
        put3(out, '0', '.', '0');
        return out + 3;
    }
    if (d.e10 >= -4 && d.e10 <= 15) {
        if (d.e10 < 0) {
            out[0] = '0';
            out[1] = '.';
            for (int z = 0; z < -d.e10 - 1; ++z) out[2 + z] = '0';
            put_digits(d.f, d.n, out + 1 - d.e10, d.n);
            return out + 1 - d.e10 + d.n;
        }
        if (d.e10 + 1 < d.n) {
            put_digits(d.f, d.n, out, d.e10 + 1);
            out[d.e10 + 1] = '.';
            return out + d.n + 1;
        }
        put_digits(d.f, d.n, out, d.n);
        for (int z = d.n; z <= d.e10; ++z) out[z] = '0';
        out[d.e10 + 1] = '.';
        out[d.e10 + 2] = '0';
        return out + d.e10 + 3;
    }
    put_digits(d.f, d.n, out, 1);
    char* p = out + d.n;
    if (d.n > 1) {
        out[1] = '.';
        ++p;
    }
    *p++ = 'e';
    *p++ = d.e10 < 0 ? '-' : '+';
    const int ae = d.e10 < 0 ? -d.e10 : d.e10;
    const int ne = ae >= 100 ? 3 : 2;
    put_digits((uint64_t)ae, ne, p, ne);
    return p + ne;
}

// ---- FrameTimecode.get_timecode(): HH:MM:SS.nnn ----
struct Timecode {
    int64_t hrs;
    int32_t mins;
    int32_t ms;  // seconds in the minute, in milliseconds: round(secs, 3) * 1000
};

// round(secs * 1000), half to even, on the exact value of 0 <= secs < 2^10: what round(secs, 3) prints
__device__ __forceinline__ int32_t round_millis(double secs) {
    const uint64_t bits = (uint64_t)__double_as_longlong(secs);
    const int bq = (int)((bits >> 52) & 0x7FF);
    const uint64_t t = bits & ((1ull << 52) - 1);
    if (bq == 0 && t == 0) return 0;
    const uint64_t m = bq ? ((1ull << 52) | t) : t;
    const int sh = bq ? 1075 - bq : 1074;  // secs = m * 2^-sh
    const uint64_t n = m * 1000;            // < 2^63
    if (sh <= 0) return (int32_t)(n << -sh);
    if (sh >= 64) return 0;                 // below one half
    uint64_t q = n >> sh;
    const uint64_t rem = n & ((1ull << sh) - 1), half = 1ull << (sh - 1);
    if (rem > half || (rem == half && (q & 1))) ++q;
    return (int32_t)q;
}

// frame / float(rate), then common.py:441-455 in IEEE double, operation by operation (no contraction)
__device__ __forceinline__ Timecode timecode_of(int64_t frame, double rate) {
    double secs = __ddiv_rn((double)frame, rate);
    Timecode tc;
    tc.hrs = (int64_t)__ddiv_rn(secs, 3600.0);
    secs = __dsub_rn(secs, __dmul_rn((double)tc.hrs, 3600.0));
    int64_t mins = (int64_t)__ddiv_rn(secs, 60.0);
    secs = fmax(0.0, __dsub_rn(secs, __dmul_rn((double)mins, 60.0)));
    tc.ms = round_millis(secs);
    if (tc.ms >= 60000) {  // min(60.0, secs) and the carry of int(secs) == 60
        tc.ms = 0;
        if (++mins >= 60) {
            mins = 0;
            ++tc.hrs;
        }
    }
    tc.mins = (int32_t)mins;
    return tc;
}

__device__ __forceinline__ int timecode_len(const Timecode& tc) {
    const int h = uint_len((uint64_t)tc.hrs);
    return (h < 2 ? 2 : h) + 10;
}

__device__ __forceinline__ char* timecode_write(const Timecode& tc, char* out) {
    int h = uint_len((uint64_t)tc.hrs);
    h = h < 2 ? 2 : h;
    put_digits((uint64_t)tc.hrs, h, out, h);
    out += h;
    out[0] = ':';
    put_digits((uint64_t)tc.mins, 2, out + 1, 2);
    out[3] = ':';
    put_digits((uint64_t)tc.ms, 5, out + 4, 2);  // SS.nnn
    out[6] = '.';
    return out + 10;
}

__device__ __forceinline__ char* uint_write(uint64_t v, char* out) {
    const int n = uint_len(v);
    put_digits(v, n, out, n);
    return out + n;
}

}  // namespace psd
