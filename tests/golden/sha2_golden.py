"""Golden SHA-2 vectors (DATA) for Hash.sha{224,256,384,512}NullsPreserved.

NIST: the FIPS 180-4 example messages (NIST CSRC "Examples with Intermediate Values" for SHA-224/256/384/512).
JAVA: the 11 inputs of src/test/java/com/nvidia/spark/rapids/jni/HashTest.java:888-901 of the reference (paths relative
      to its root), whose expected values come from java.security.MessageDigest; a None input is a null row and gives a
      null output row.  Strings are python str, UTF-8 encoded by the loader.
DIGESTS maps digest bits -> lowercase hex, per input.
"""

NIST = [
    dict(name='nist_abc', input='abc',  # FIPS 180-4 examples (NIST CSRC 'Examples with Intermediate Values'): one-block message
         digests={
             224: '23097d223405d8228642a477bda255b32aadbce4bda0b3f7e36c9da7',
             256: 'ba7816bf8f01cfea414140de5dae2223b00361a396177a9cb410ff61f20015ad',
             384: 'cb00753f45a35e8bb5a03d699ac65007272c32ab0eded1631a8b605a43ff5bed8086072ba1e7cc2358baeca134c825a7',
             512: 'ddaf35a193617abacc417349ae20413112e6fa4e89a97ea20a9eeee64b55d39a2192992a274fc1a836ba3c23a3feebbd454d4423643ce80e2a9ac94fa54ca49f',
         }),
    dict(name='nist_empty', input='',  # the empty message
         digests={
             224: 'd14a028c2a3a2bc9476102bb288234c415a2b01f828ea62ac5b3e42f',
             256: 'e3b0c44298fc1c149afbf4c8996fb92427ae41e4649b934ca495991b7852b855',
             384: '38b060a751ac96384cd9327eb1b1e36a21fdb71114be07434c0cc7bf63f6e1da274edebfe76f65fbd51ad2f14898b95b',
             512: 'cf83e1357eefb8bdf1542850d66d8007d620e4050b5715dc83f4a921d36ce9ce47d0d13c5d85f2b0ff8318d2877eec2f63b931bd47417a81a538327af927da3e',
         }),
    dict(name='nist_448', input='abcdbcdecdefdefgefghfghighijhijkijkljklmklmnlmnomnopnopq',  # 448-bit two-block message (SHA-224/256)
         digests={
             224: '75388b16512776cc5dba5da1fd890150b0c6455cb4f58b1952522525',
             256: '248d6a61d20638b8e5c026930c3e6039a33ce45964ff2167f6ecedd419db06c1',
             384: '3391fdddfc8dc7393707a65b1b4709397cf8b1d162af05abfe8f450de5f36bc6b0455a8520bc4e6f5fe95b1fe3c8452b',
             512: '204a8fc6dda82f0a0ced7beb8e08a41657c16ef468b228a8279be331a703c33596fd15c13b1b07f9aa1d3bea57789ca031ad85c7a71dd70354ec631238ca3445',
         }),
    dict(name='nist_896', input='abcdefghbcdefghicdefghijdefghijkefghijklfghijklmghijklmnhijklmnoijklmnopjklmnopqklmnopqrlmnopqrsmnopqrstnopqrstu',  # 896-bit two-block message (SHA-384/512)
         digests={
             224: 'c97ca9a559850ce97a04a96def6d99a9e0e0e2ab14e6b8df265fc0b3',
             256: 'cf5b16a778af8380036ce59e7b0492370b249b11e8f07a51afac45037afee9d1',
             384: '09330c33f71147e83d192fc782cd1b4753111b173b3b05d22fa08086e3b0f712fcc7c71a557e2db966c3e9fa91746039',
             512: '8e959b75dae313da8cf4f72814fc143f8f7779c6eb9f7fa17299aeadb6889018501d289e4900f7e4331b99dec4b5433ac7d329eeb6dd26545e96e55b874be909',
         }),
]

# HashTest.java:888-901, in order
JAVA_INPUTS = [
    None,
    '',
    '0',
    'A 56 character string to test message padding algorithm.',
    'A 63 character string to test message padding algorithm, again.',
    'A 64 character string to test message padding algorithm, again!!',
    'A very long (greater than 128 bytes/char string) to execute a multi hash-step data point in the hash function being tested. This string needed to be longer.',
    'All work and no play makes Jack a dull boy',
    '',
    'Multi-byte characters: é¼³⅝',
    '(!"#$%&\'()*+,-./0123456789:;<=>?@[\\]^_`{|}~)',
]

JAVA_DIGESTS = {
    224: [
        None,
        'd14a028c2a3a2bc9476102bb288234c415a2b01f828ea62ac5b3e42f',
        'dfd5f9139a820075df69d7895015360b76d0360f3d4b77a845689614',
        '5d1ed8373987e403482cefe1662a63fa3076c0a5331d141f41654bbe',
        '0662c91000b99de7a20c89097dd62f59120398d52499497489ccff95',
        'f9ea303770699483f3e53263b32a3b3c876d1b8808ce84df4b8ca1c4',
        '2da6cd4bdaa0a99fd7236cd5507c52e12328e71192e83b32d2f110f9',
        'e7d0adb165079efc6c6343112f8b154aa3644ca6326f658aaa0f8e4a',
        'd14a028c2a3a2bc9476102bb288234c415a2b01f828ea62ac5b3e42f',
        '6c728722ae8eafd058672bd92958199ff3a5a129e8c076752f7650f8',
        'c8d920ee451f1bdf35deb72dae3adbc3d72a848697d164857b928c57',
    ],
    256: [
        None,
        'e3b0c44298fc1c149afbf4c8996fb92427ae41e4649b934ca495991b7852b855',
        '5feceb66ffc86f38d952786c6d696c79c2dbc239dd4e91b46729d73a27fb57e9',
        'd16883c666112142c1d72c9080b41161be7563250539e3f6ab6e2fdf2210074b',
        '11174fa180460f5d683c2e63fcdd897dcbf10c28a9225d3ced9a8bbc3774415d',
        '10a7d211e692c6f71bb9f7524ba1437588c2797356f05fc585340f002fe7015e',
        '339d610dcb030bb4222bcf18c8ab82d911bfe7fb95b2cd9f6785fd4562b02401',
        '2ce9936a4a2234bf8a76c37d92e01d549d03949792242e7f8a1ad68575e4e4a8',
        'e3b0c44298fc1c149afbf4c8996fb92427ae41e4649b934ca495991b7852b855',
        '9f9a89d448937f853c0067a3e2cb732d703eca971e3fb0f88fc73a730b7a85f4',
        '9304b2ae7baac2cf11b4cd6c8fb50f53f7f15d5a18f5125f541fda78f7aa3dbd',
    ],
    384: [
        None,
        '38b060a751ac96384cd9327eb1b1e36a21fdb71114be07434c0cc7bf63f6e1da274edebfe76f65fbd51ad2f14898b95b',
        '5f91550edb03f0bb8917da57f0f8818976f5da971307b7ee4886bb951c4891a1f16f840dae8f655aa5df718884ebc15b',
        '982000cce895dc439edbcb7ba5b908cb5b7e939fe913d58506a486735a914b0dfbcebb02c33c428287baa0bfc7fe0948',
        'c3ea54e4d6d97c2a84dac9ac48ed9dd1a49118be880d8466044720cfdcd23427bf556f12204bb34ede29dbf20703378c',
        '5d7a853a18138fa90feac07c896dfca65a0f1eb2ed40f1fd7be6238dd7ef429bb1aeb0236735500eb954c9b4ba923254',
        'c72bcaf3a4b01986711cd5d2614aa8f9d7fad61455613eac4561b1468f9a25dd26566c8ad1190dec7567be4f6fc1db29',
        '281826f23bebb3f835d2f15edcb0cdb3078ae2d7dc516f3a366af172dff4db6dd5833bc1e5ee411d52c598773e9397b6',
        '38b060a751ac96384cd9327eb1b1e36a21fdb71114be07434c0cc7bf63f6e1da274edebfe76f65fbd51ad2f14898b95b',
        'f6d9687e48ef1f69f7523c2a06c338e2b2e6cb251823d46bfa7f9ba65a071693919726b85f6dd77726a73c57a0e3a4a5',
        '29f47878686ef0b716d15167f4dd52603196f24371f3f5d21437a2d4738a2a14e463ec7382e055e8a1c22640a6e5070a',
    ],
    512: [
        None,
        'cf83e1357eefb8bdf1542850d66d8007d620e4050b5715dc83f4a921d36ce9ce47d0d13c5d85f2b0ff8318d2877eec2f63b931bd47417a81a538327af927da3e',
        '31bca02094eb78126a517b206a88c73cfa9ec6f704c7030d18212cace820f025f00bf0ea68dbf3f3a5436ca63b53bf7bf80ad8d5de7d8359d0b7fed9dbc3ab99',
        '1d8b355dbe0c4ad81c9815a1490f0b6a6fa710e42ca60767ffd6d845acd116defe307c9496a80c4a67653873af6ed83e2e04c2102f55f9cd402677b246832e4c',
        '8ac8ae9de5597aa630f071f81fcb94dc93b6a8f92d8f2cdd5a469764a5daf6ef387b6465ae097dcd6e0c64286260dcc3d2c789d2cf5960df648c78a765e6c27c',
        '9c436e24be60e17425a1a829642d97e7180b57485cf95db007cf5b32bbae1f2325b6874b3377e37806b15b739bffa412ea6d095b726487d70e7b50e92d56c750',
        '6a25ca1f20f6e79faea2a0770075e4262beb66b40f59c22d3e8abdb6188ef8d8914faf5dbf6df76165bb61b81dfda46643f0d6366a39f7bd3d270312f9d3cf87',
        'bae9eb4b5c05a4c5f85750b70b2f0ce78e387f992f0927a017eb40bd180a13004f6252a6bbf9816f195fb7d86668c393dc0985aaf7168f48e8b905f3b9b02df2',
        'cf83e1357eefb8bdf1542850d66d8007d620e4050b5715dc83f4a921d36ce9ce47d0d13c5d85f2b0ff8318d2877eec2f63b931bd47417a81a538327af927da3e',
        '1a15d73f16820b25f2af1c824a00a6ab18fe3eb91adaae31f441f4eca7ca11baf56d2f56e4f600781bf3637a49a4fbdbd5d7e0d8e894c51144e28eed59b3721a',
        '1a9f0f04ddc4112e6c0ce97dbcd85a37e130f6735400e86bfa6ac447b6cfbc372982e907b1f2cd74c6f6364bea9cdcdeff31d633fa930fe7e82dfbe14906e901',
    ],
}
